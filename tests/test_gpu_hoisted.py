"""Hoisted rotations (fhe_b200_galois_many_hoisted) and their Python / C++ mirrors.

Output j must be, word for word, output j of fhe_b200_galois_many with the same arguments (pinned to the single calls
by test_gpu_rotations.py), and on a subset the oracle's GaloisKey.relinearize.  n_hoisted must equal the count the CPU
predicate of tests/hoisting_reference.py gives: every output of a multi-output source for random input, fewer for
crafted zeros.  The word checks are rerun in subprocesses under the kernel-selection and chunking switches.  Run with
`-m gpu`."""
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
TESTS = os.path.join(ROOT, "tests")
if TESTS not in sys.path:
    sys.path.insert(0, TESTS)
if os.path.join(ROOT, "oracle") not in sys.path:
    sys.path.insert(0, os.path.join(ROOT, "oracle"))

import edge_inputs   # noqa: E402
import hoisting_reference as H   # noqa: E402
from test_gpu_rotations import CASES, Setup, _exponents, _index, _source, rand_rows   # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def F():
    from conftest import has_gpu
    if not has_gpu():
        pytest.skip("no CUDA device")
    import fhe_rs_b200
    return fhe_rs_b200


def c1_power(S):
    """the power-basis c1 rows [count][L][N] of the batch"""
    return S.A.clone().into_power_basis().to_host()[:, 1]


def check_hoisted(S, index, source=None, expect_all=False):
    """hoisted == galois_many word for word, and n_hoisted == the CPU predicate's count"""
    F = S.F
    got, nh = F.galois_many_hoisted(S.A, S.gks, index, source)
    got = got.to_host()
    want = S.many(index, source)
    bad = [j for j in range(want.shape[0]) if not (got[j] == want[j]).all()]
    assert not bad, (S.degree, S.count, bad[:8])
    src = list(range(S.count)) if source is None else list(source)
    exps = [S.gks[k].exponent % (2 * S.degree) for k in index]
    if len(S.moduli) - S.key_level == 1:
        expected = 0   # a single-modulus key level: base-2^b digits are never hoisted
    else:
        expected = H.hoisted_count(c1_power(S), exps, src)
    assert nh == expected, (nh, expected)
    if expect_all:
        uses = np.bincount(np.asarray(src), minlength=S.count)
        assert nh == sum(1 for s in src if uses[s] >= 2)
    return nh


# (shape, count, index pattern, source pattern): the work-split shapes plus n16, n64, c_l1 (level-1 batch, level-0
# keys) and single_mod (base-2^b keys, nothing hoisted)
HOIST_RUNS = [("n13_2x62", 7, "alt", "repeat"), ("n13_62_40_30", 33, "runs5", "zero"), ("n14_8x62", 33, "alt", "repeat"),
              ("n15_14x62", 3, "distinct", "zero"), ("n16", 5, "alt", "repeat"), ("n64", 7, "runs2", "zero"),
              ("c_l1", 3, "alt", "zero"), ("single_mod", 5, "distinct", "repeat")]


def word_checks(F, quick=False):
    """the sweep the switch reruns repeat"""
    for name, count, pattern, src in HOIST_RUNS:
        if quick and name in ("n15_14x62", "c_l1"):
            continue
        degree, t, sizes, level, key_level = CASES[name]
        n_keys = 4 if pattern != "distinct" else count
        S = Setup(F, degree, t, sizes, level, key_level, _exponents(degree, n_keys), count, hash(name) & 0xffff)
        check_hoisted(S, _index(pattern, count, n_keys), _source(src, count, count),
                      expect_all=name != "single_mod")
    # 130 keys, one source; and 33 sources x 5 steps interleaved, with single-output sources, at counts that cut chunks
    S = Setup(F, 1 << 13, 786433, [62, 62], 0, 0, _exponents(1 << 13, 130), 40, 5)
    check_hoisted(S, list(range(130)) + [129 - j for j in range(130)], [7] * 130 + [j % 40 for j in range(130)],
                  expect_all=True)
    check_hoisted(S, [j // 33 for j in range(165)] + [100, 101], [j % 33 for j in range(165)] + [35, 36],
                  expect_all=True)


@pytest.mark.parametrize("name,count,pattern,src", HOIST_RUNS)
def test_hoisted_equals_galois_many(F, name, count, pattern, src):
    degree, t, sizes, level, key_level = CASES[name]
    n_keys = 4 if pattern != "distinct" else count
    S = Setup(F, degree, t, sizes, level, key_level, _exponents(degree, n_keys), count, 11)
    nh = check_hoisted(S, _index(pattern, count, n_keys), _source(src, count, count), expect_all=name != "single_mod")
    assert (nh == 0) == (name == "single_mod"), nh
    assert check_hoisted(S, [count % n_keys] * count) == 0   # every source used once: nothing hoisted


def test_source_patterns(F):
    """one ciphertext by 16 steps at set C and by 64 at N = 2^13; 33 ciphertexts x 5 steps; sources repeated,
    permuted and interleaved; single- and multi-output sources mixed; 130 keys"""
    S = Setup(F, 1 << 15, 786433, [62] * 14, 0, 0, _exponents(1 << 15, 16), 2, 21)
    assert check_hoisted(S, list(range(16)), [1] * 16) == 16
    degree, t, sizes = 1 << 13, 786433, [62, 62]
    S = Setup(F, degree, t, sizes, 0, 0, _exponents(degree, 130), 33, 5)
    assert check_hoisted(S, list(range(64)), [0] * 64) == 64
    assert check_hoisted(S, [j // 33 for j in range(165)], [j % 33 for j in range(165)]) == 165   # step-major
    assert check_hoisted(S, [j % 5 for j in range(165)], [j // 5 for j in range(165)]) == 165     # source-major
    perm = list(np.random.default_rng(3).permutation(165))
    assert check_hoisted(S, [perm[j] % 5 for j in range(165)], [perm[j] // 5 for j in range(165)]) == 165
    assert check_hoisted(S, [j % 130 for j in range(300)], [(j * 7) % 11 for j in range(300)]) == 300
    mixed_src = [0, 1, 0, 2, 3, 3, 4, 0, 5, 6, 6, 6]
    assert check_hoisted(S, [j % 130 for j in range(12)], mixed_src) == 8
    assert check_hoisted(S, list(range(130)), [32] * 130) == 130
    assert check_hoisted(S, [0, 1, 0], [2, 2, 2]) == 3                           # one key twice for one source
    for count in (1, 2, 3, 17):
        Sc = Setup(F, degree, t, sizes, 0, 0, _exponents(degree, 6), count, count)
        check_hoisted(Sc, [(j // 3) % 6 for j in range(2 * count)], [j // 2 for j in range(2 * count)],
                      expect_all=True)


def _with_c1(F, S, rows):
    """S with its ciphertexts' c1 replaced by the power-basis rows [count][L][N]"""
    words = S.A.clone().into_power_basis().to_host()
    words[:, 1] = rows
    S.A = F.Ciphertext.from_host(S.par, words, level=S.level, repr=F.POWER_BASIS).into_ntt()
    return S


def test_crafted_zeros(F):
    """zeros at s = 0 (all outputs hoisted), zeros at positions some exponents negate, c1 = 0 from ct - ct, and the
    boundary primes' residue rows: fewer outputs hoisted, every output word-equal"""
    degree, t = 1 << 12, 786433
    moduli = [edge_inputs.gen62(degree, 0)] + list(edge_inputs.BOUNDARY_PRIMES.values())
    sizes = None
    S = Setup(F, degree, t, sizes, 0, 0, _exponents(degree, 8), 4, 31, moduli=moduli)
    index, source = [j % 8 for j in range(16)], [j // 4 for j in range(16)]
    rows = c1_power(S)
    rows[:, :, 0] = 0
    assert check_hoisted(_with_c1(F, S, rows), index, source) == 16
    rows = c1_power(S)
    rows[1, 0, 5] = 0                 # position 5 of ciphertext 1, limb 0
    rows[2, 2, degree - 1] = 0
    rows[2, 1, 3] = 0
    nh = check_hoisted(_with_c1(F, S, rows), index, source)
    assert 8 <= nh < 16, nh
    D = Setup(F, degree, t, sizes, 0, 0, _exponents(degree, 8), 4, 31, moduli=moduli)
    D.A = D.A - D.A                    # c1 = 0: only exponent 1 could hoist, and none of these is 1
    assert check_hoisted(D, index, source) == 0
    ids = F.GaloisKey(1, D.gks[0].ksk)
    D.gks = D.gks + [ids]
    assert check_hoisted(D, [8, 8, 0, 1], [0, 0, 1, 1]) == 2   # the identity substitution negates nothing
    ed = edge_inputs.residue_rows(S.moduli, degree)
    rows = np.stack([ed[k] for k in ("zero", "max", "alternating", "one_first")])
    nh = check_hoisted(_with_c1(F, S, rows), index, source)
    assert 4 <= nh < 16, nh   # the all-(q - 1) rows have no zero; the others fall back for most exponents


def test_against_the_oracle(oracle, F):
    """samples of the hoisted call against the oracle's GaloisKey.relinearize, a leveled key at N = 64"""
    for degree, t, sizes, level, key_level in ((16, 1153, [62] * 3, 0, 0), (64, 1153, [62] * 3, 1, 0),
                                               (1 << 12, 786433, [62, 40, 30], 0, 0)):
        opar = oracle.BfvParameters(degree, t, moduli_sizes=sizes)
        S = Setup(F, degree, t, sizes, level, key_level, _exponents(degree, 5), 2, degree, moduli=opar.moduli)
        index, source = [0, 1, 2, 3, 4, 0], [0, 0, 0, 1, 1, 1]
        got, nh = F.galois_many_hoisted(S.A, S.gks, index, source)
        assert nh == 6
        got, a = got.to_host(), S.A.to_host()
        for j, (k, s) in enumerate(zip(index, source)):
            g = S.gks[k]
            o = oracle.GaloisKey.__new__(oracle.GaloisKey)
            o.exponent = g.exponent % (2 * degree)
            o.ksk = oracle.KeySwitchingKey.from_arrays(opar, *g.ksk.arrays(), level, key_level)
            want = o.relinearize(oracle.Ciphertext.from_array(opar, a[s], level))
            assert (want.to_array() == got[j]).all(), (degree, j)


def test_real_keys_decrypt_to_the_rotations(F):
    """device-generated keys: every hoisted rotation of two ciphertexts decrypts to the rotated plaintext"""
    degree, t, half = 64, 1153, 32
    par = F.BfvParameters(degree, t, moduli_sizes=[62, 62], device=0)
    sk = F.SecretKey.random_vec(par, 1, seed=bytes([15]) * 32)[0]
    b = F.EvaluationKeyBuilder.new(sk)
    steps = [1, 2, 3, 5, 8, 13, 21, 31]
    for i in steps:
        b.enable_column_rotation(i)
    ek = b.build(seed=bytes([16]) * 32)
    rng = np.random.default_rng(17)
    rows = rng.integers(0, t, (2, 2, half)).astype(np.uint64)
    enc = F.Encoding.simd()
    ct = sk.try_encrypt(F.PlaintextVec.try_encode(rows.reshape(-1), enc, par), seed=bytes([18]) * 32)
    rot = ek.rotates_columns_by_many_hoisted(ct, steps)
    assert (rot.to_host() == ek.rotates_columns_by_many(ct, steps).to_host()).all()
    for i, st in enumerate(steps):
        for q in range(2):
            dec = sk.try_decrypt(rot.take(i * 2 + q, 1)).try_decode(enc).reshape(2, half)
            assert (dec == np.roll(rows[q], -st, axis=1)).all(), (st, q)


def test_baby_step_giant_step_matrix_times_vector(F):
    """M v at N = 64 by baby-step/giant-step diagonals: the 8 baby-step rotations of v in one hoisted call, each
    giant step the dot product of the baby steps with the giant step's pre-rotated diagonals, rotated by its giant
    step; both rows of the sum decrypt to M v mod t"""
    degree, t, half, n1 = 64, 1153, 32, 8
    n2 = half // n1
    par = F.BfvParameters(degree, t, moduli_sizes=[62, 62], device=0)
    sk = F.SecretKey.random_vec(par, 1, seed=bytes([25]) * 32)[0]
    b = F.EvaluationKeyBuilder.new(sk)
    for i in list(range(1, n1)) + [n1 * g for g in range(1, n2)]:
        b.enable_column_rotation(i)
    ek = b.build(seed=bytes([26]) * 32)
    ek.add_galois_key(F.GaloisKey.new(sk, 1, seed=bytes([27]) * 32))   # step 0
    rng = np.random.default_rng(28)
    M = rng.integers(0, t, (half, half)).astype(np.int64)
    rows = rng.integers(0, t, (2, half)).astype(np.int64)
    enc = F.Encoding.simd()
    ct = sk.try_encrypt(F.PlaintextVec.try_encode(rows.reshape(-1).astype(np.uint64), enc, par), seed=bytes([29]) * 32)
    baby, nh = F.galois_many_hoisted(ct, *ek._many_args(ct, list(range(n1))))
    assert nh == n1
    acc = None
    for g in range(n2):
        # diagonal i = g n1 + j, rotated right by g n1 so that rot_{g n1}(sum_j diag' * rot_j(v)) = sum_j diag * rot_i(v)
        diags = np.zeros((n1, degree), np.uint64)
        for j in range(n1):
            i = g * n1 + j
            d = np.array([M[r][(r + i) % half] for r in range(half)], np.int64)
            d = np.roll(d, g * n1).astype(np.uint64)
            diags[j] = np.concatenate([d, d])
        inner = F.dot_product_scalar(baby, F.PlaintextVec.try_encode(diags.reshape(-1), enc, par))
        part = ek.rotates_columns_by(inner, g * n1) if g else inner
        acc = part if acc is None else acc + part
    res = sk.try_decrypt(acc).try_decode(enc).reshape(2, half)
    want = np.stack([(M @ r) % t for r in rows]).astype(np.uint64)
    assert (res == want).all()


def test_no_state_outlives_the_call(F):
    """hoisting 64 exponents the parameter set has not seen leaves the device memory in use unchanged"""
    import torch
    degree = 1 << 15
    S = Setup(F, degree, 786433, [62, 62], 0, 0, [3], 2, 6)
    ksk = S.gks[0].ksk
    S.gks = [F.GaloisKey(e, ksk) for e in _exponents(degree, 128)]
    F.galois_many_hoisted(S.A, S.gks, list(range(64)), [0] * 64)   # the scratch pool at this shape
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    out, nh = F.galois_many_hoisted(S.A, S.gks, list(range(64, 128)), [0] * 64)
    assert nh == 64
    del out
    torch.cuda.synchronize()
    assert abs(torch.cuda.mem_get_info()[0] - free0) < 2 << 20


def test_refusals_write_nothing_and_keep_no_memory(F):
    """every error of fhe_b200_galois_many, from the hoisted call: the output words, device memory and n_hoisted are
    unchanged by each refusal"""
    import ctypes as C
    import torch
    from fhe_rs_b200 import _capi
    lib = _capi.lib()
    degree, t, sizes = 1 << 13, 786433, [62, 62]
    S = Setup(F, degree, t, sizes, 0, 0, [3, 5, 2 * degree - 1], 4, 1)
    other = Setup(F, degree, t, sizes, 0, 0, [3], 4, 2)
    rng = np.random.default_rng(4)
    l1k0 = F.KeySwitchingKey.from_arrays(S.par, *rand_rows(rng, S.moduli, (2, 1), degree), 1, 0)
    l1k1 = F.KeySwitchingKey.from_arrays(S.par, *rand_rows(rng, S.moduli[:1], (2, 2), degree), 1, 1)
    a_l1 = F.Ciphertext.from_host(S.par, rand_rows(rng, S.moduli[:1], (4, 2), degree), level=1)
    out = F.Ciphertext(S.par, 4, 2)
    out_l1 = F.Ciphertext(S.par, 4, 2, 1)
    out3 = F.Ciphertext(S.par, 3, 2)
    sentinels = [(b, b.to_host()) for b in (out, out_l1, out3, S.A)]
    P = S.A.clone().into_power_basis()

    def arr(hs):
        a = (C.c_void_p * max(1, len(hs)))(*[getattr(h, "value", h) for h in hs])
        return C.cast(a, C.POINTER(C.c_void_p))

    def u(v):
        return (C.c_uint32 * max(1, len(v)))(*v)
    k = [g.ksk._h for g in S.gks]
    ex = u([3, 5, 2 * degree - 1])
    good = u([0, 1, 2, 0])
    same = u([0, 0, 0])   # every output from ciphertext 0: a hoisting call
    n_h = C.c_uint32(77)
    nh = C.byref(n_h)

    def many(a, src, keys, exps, n, ix, o):
        return lib.fhe_b200_galois_many_hoisted(a, src, keys, exps, n, ix, o, nh, None)
    bad_arg = _capi.INVALID_ARGUMENT
    cases = [
        ("null list", lambda: many(S.A._h, same, None, ex, 3, good, out3._h), bad_arg),
        ("null exponents", lambda: many(S.A._h, same, arr(k), None, 3, good, out3._h), bad_arg),
        ("null index", lambda: many(S.A._h, same, arr(k), ex, 3, None, out3._h), bad_arg),
        ("no keys", lambda: many(S.A._h, same, arr(k), ex, 0, good, out3._h), bad_arg),
        ("null key", lambda: many(S.A._h, same, arr([k[0], None, k[2]]), ex, 3, good, out3._h), bad_arg),
        ("index beyond", lambda: many(S.A._h, same, arr(k), ex, 3, u([0, 3, 0]), out3._h), bad_arg),
        ("source beyond", lambda: many(S.A._h, u([0, 4, 0]), arr(k), ex, 3, good, out3._h), bad_arg),
        ("counts differ", lambda: many(S.A._h, None, arr(k), ex, 3, good, out3._h), bad_arg),
        ("aliased", lambda: many(S.A._h, None, arr(k), ex, 3, good, S.A._h), bad_arg),
        ("even exponent", lambda: many(S.A._h, same, arr(k), u([3, 6, 5]), 3, good, out3._h), _capi.INVALID_EXPONENT),
        ("key levels differ", lambda: many(a_l1._h, None, arr([l1k0._h, l1k1._h]), u([3, 5]), 2, u([0, 1, 0, 1]),
                                           out_l1._h), bad_arg),
        ("other parameters", lambda: many(S.A._h, same, arr(k + [other.gks[0].ksk._h]), u([3, 5, 7, 3]), 4, good,
                                          out3._h), _capi.CONTEXT_MISMATCH),
        ("other level", lambda: many(S.A._h, None, arr([l1k0._h]), ex, 1, u([0] * 4), out._h), _capi.INVALID_LEVEL),
        ("representation", lambda: many(P._h, same, arr(k), ex, 3, good, out3._h), _capi.INVALID_REPRESENTATION),
    ]
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    for what, call, code in cases:
        got = call()
        assert got == code, (what, got, lib.fhe_b200_last_error())
    torch.cuda.synchronize()
    assert abs(torch.cuda.mem_get_info()[0] - free0) < 4 << 20
    assert n_h.value == 77
    for b, words in sentinels:
        assert (b.to_host() == words).all()


def test_cpp_mirror(F, tmp_path):
    """the C++ mirror's galois_many_hoisted (with n_hoisted) and rotates_columns_by_many_hoisted give the Python
    mirror's words"""
    degree, t, sizes = 64, 1153, [62, 62, 62]
    exps = [pow(3, i, 2 * degree) for i in (1, 2, 4)] + [2 * degree - 1]
    S = Setup(F, degree, t, sizes, 0, 0, exps, 5, 12)
    count = 9
    index = [(j * 5) % len(exps) for j in range(count)]
    source = [(j * 3) % 5 for j in range(count)]
    lines = ["%d %d %d %d %d %d" % (degree, t, len(S.moduli), 5, count, len(exps)), " ".join(map(str, S.moduli)),
             " ".join(map(str, exps)), " ".join(map(str, index)), " ".join(map(str, source))]
    for k, g in enumerate(S.gks):
        c0, c1 = g.ksk.arrays()
        c0.tofile(str(tmp_path / ("k%d_c0.bin" % k)))
        c1.tofile(str(tmp_path / ("k%d_c1.bin" % k)))
    (tmp_path / "args.txt").write_text("\n".join(lines) + "\n")
    S.A.to_host().tofile(str(tmp_path / "a.bin"))
    exe = str(tmp_path / "hoisted_test")
    lib_dir = os.path.join(ROOT, "fhe_rs_b200")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "cpp", "hoisted_test.cpp"), "-o", exe,
                           "-L", lib_dir, "-lfhe_b200", "-Wl,-rpath," + lib_dir])
    out = subprocess.run([exe, str(tmp_path)], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0 and out.stdout.startswith("OK"), out.stdout + out.stderr
    many, nh = F.galois_many_hoisted(S.A, S.gks, index, source)
    assert "n_hoisted %d" % nh in out.stdout, out.stdout
    ek = F.EvaluationKey(S.par)
    for g in S.gks:
        ek.add_galois_key(g)
    want = {"many": many.to_host(), "rot": ek.rotates_columns_by_many_hoisted(S.A, [1, 2, 4]).to_host()}
    for name, w in want.items():
        assert (np.fromfile(str(tmp_path / ("out_%s.bin" % name)), np.uint64) == w.ravel()).all(), name


SWITCHES = {"fast": {"FHE_B200_NTT": "fast"}, "tma_ntt": {"FHE_B200_NTT": "tma"},
            "tma": {"FHE_B200_KSMAC": "tma"}, "classic": {"FHE_B200_KSMAC": "classic"},
            "stages3": {"FHE_B200_KS_STAGES": "3"}, "chunk1": {"FHE_B200_CHUNK": "1"},
            "chunk5": {"FHE_B200_CHUNK": "5", "FHE_B200_STREAMS": "3"},
            "streams1": {"FHE_B200_STREAMS": "1"}, "streams4": {"FHE_B200_STREAMS": "4", "FHE_B200_CHUNK": "16"}}


def test_switch_reruns():
    """the word checks under each transform, key-switch path and chunking switch, one process per switch (read once
    per process), side by side"""
    procs = {}
    for name, env in SWITCHES.items():
        e = dict(os.environ, **env)
        procs[name] = subprocess.Popen([sys.executable, os.path.abspath(__file__), "--word-checks"], cwd=ROOT, env=e,
                                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    fails = {}
    for name, p in procs.items():
        out, _ = p.communicate(timeout=1800)
        if p.returncode != 0 or "WORD CHECKS OK" not in out:
            fails[name] = out[-3000:]
    assert not fails, fails


if __name__ == "__main__" and "--word-checks" in sys.argv:
    import fhe_rs_b200
    word_checks(fhe_rs_b200, quick=os.environ.get("FHE_B200_CHUNK") == "1")
    print("WORD CHECKS OK")
