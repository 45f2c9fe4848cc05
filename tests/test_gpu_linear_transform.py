"""Linear transforms (fhe_b200_linear_transform) and their Python / C++ mirrors.

The call must return, word for word, the composition of tests/linear_transform_reference.py run from existing device
calls: GaloisKey.relinearize (fhe_b200_galois) for each baby and giant step, Ciphertext.mul_plain with the diagonals
(fhe_b200_mul_plain_batch) and +.  n_fallback must equal the CPU zero predicate's count (tests/hoisting_reference.py)
on the fused path and count * (b - 1) on the unfused one.  The word checks are rerun in subprocesses under the
kernel-selection and chunking switches.  Run with `-m gpu`."""
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
import linear_transform_reference as R   # noqa: E402
from test_gpu_rotations import CASES, Setup, rand_rows   # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def F():
    from conftest import has_gpu
    if not has_gpu():
        pytest.skip("no CUDA device")
    import fhe_rs_b200
    return fhe_rs_b200


def setup(F, degree, t, sizes, level, key_level, n, baby, count, seed, moduli=None):
    """random ciphertexts and one random key per step the transform needs (step 1 at least)"""
    steps = R.steps(n, baby) or [1]
    S = Setup(F, degree, t, sizes, level, key_level, [pow(3, s, 2 * degree) for s in steps], count, seed,
              moduli=moduli)
    S.step_key = dict(zip(steps, S.gks))
    return S


def random_diags(F, S, m, seed):
    rng = np.random.default_rng(seed)
    ct_mod = S.moduli[:len(S.moduli) - S.level]
    return F.Ciphertext.from_host(S.par, rand_rows(rng, ct_mod, (m, 1), S.degree), level=S.level)


def composition(F, A, diags, n, baby, step_key, per_ct):
    """the definition from existing calls: rotations, mul_plain and +"""
    count = A.count
    enc = F.Encoding.simd_at_level(A.level)
    acc = None
    for g in range(-(-n // baby)):
        part = None
        for i in range(min(baby, n - g * baby)):
            k = g * baby + i
            x = A.clone() if i == 0 else step_key[i].relinearize(A)
            x.mul_plain(F.PlaintextVec(diags.take(k, count, n) if per_ct else diags.take(k, 1), enc))
            part = x if part is None else part + x
        if g:
            part = step_key[g * baby].relinearize(part)
        acc = part if acc is None else acc + part
    return acc.to_host()


def c1_power(A):
    return A.clone().into_power_basis().to_host()[:, 1]


def expected_fallback(S, A, baby, fused):
    if not fused:
        return A.count * (baby - 1)
    c1 = c1_power(A)
    return sum(1 for c in range(A.count) for i in range(1, baby)
               if H.needs_fallback(c1[c], pow(3, i, 2 * S.degree)))


def check(F, S, n, baby, per_ct, seed=7, A=None, fused=None):
    A = S.A if A is None else A
    diags = random_diags(F, S, n * (A.count if per_ct else 1), seed)
    got, nf = F.linear_transform(A, diags, baby, S.gks, n)
    want = composition(F, A, diags, n, baby, S.step_key, per_ct)
    got = got.to_host()
    bad = [c for c in range(A.count) if not (got[c] == want[c]).all()]
    assert not bad, (S.degree, n, baby, per_ct, bad[:8])
    if fused is None:
        fused = S.key_level == S.level and len(S.moduli) - S.key_level > 1
    assert nf == expected_fallback(S, A, baby, fused), (nf, n, baby)
    return nf


def _babies(n):
    return sorted({1, max(1, int(np.sqrt(n))), n})


# (case, count, [(n, baby, per_ct)])
RUNS = [("n16", 3, [(n, b, p) for n in (1, 7, 8) for b in _babies(n) for p in (False, True)]),
        ("n64", 5, [(n, b, p) for n in (1, 7, 16, 32) for b in _babies(n) for p in (False, True)]),
        ("n13_62_40_30", 5, [(7, 2, False), (16, 4, True)]),
        ("n13_2x62", 9, [(16, 4, False), (5, 5, True)]),
        ("n14_8x62", 3, [(8, 3, False)]),
        ("n15_14x62", 2, [(8, 3, False), (4, 2, True)]),
        ("c_l1", 2, [(5, 2, False)]),              # level-1 batch, level-0 keys: the unfused route
        ("single_mod", 3, [(7, 3, True)])]         # base-2^b keys: the unfused route


def word_checks(F, quick=False):
    for name, count, shapes in RUNS:
        if quick and name in ("n15_14x62", "c_l1", "n14_8x62"):
            continue
        degree, t, sizes, level, key_level = CASES[name]
        for n, b, per_ct in shapes:
            S = setup(F, degree, t, sizes, level, key_level, n, b, count, hash((name, n, b)) & 0xffff)
            check(F, S, n, b, per_ct)
    # a level-1 batch with level-1 keys (fused), and counts that cut chunks
    S = setup(F, 64, 1153, [62] * 3, 1, 1, 16, 4, 9, 3)
    check(F, S, 16, 4, True)
    S = setup(F, 1 << 12, 786433, [62, 62], 0, 0, 9, 3, 37, 4)
    check(F, S, 9, 3, False)
    check(F, S, 9, 3, True)


@pytest.mark.parametrize("name,count,shapes", RUNS)
def test_equals_the_composition(F, name, count, shapes):
    degree, t, sizes, level, key_level = CASES[name]
    for n, b, per_ct in shapes:
        S = setup(F, degree, t, sizes, level, key_level, n, b, count, 11 + n + b)
        check(F, S, n, b, per_ct)


def test_levels_and_counts(F):
    """level 1 with level-1 keys (fused), level 2 of four moduli, and counts 1, 17 and 37 at N = 2^12"""
    S = setup(F, 64, 1153, [62] * 3, 1, 1, 16, 4, 9, 3)
    assert check(F, S, 16, 4, True) == 0
    S = setup(F, 1 << 12, 786433, [62] * 4, 2, 2, 12, 4, 3, 5)
    check(F, S, 12, 4, False)
    for count in (1, 17, 37):
        S = setup(F, 1 << 12, 786433, [62, 62], 0, 0, 9, 3, count, count)
        check(F, S, 9, 3, False)
        check(F, S, 9, 3, True)


def _with_c1(F, S, rows):
    words = S.A.clone().into_power_basis().to_host()
    words[:, 1] = rows
    return F.Ciphertext.from_host(S.par, words, level=S.level, repr=F.POWER_BASIS).into_ntt()


def test_fallback_terms(F):
    """crafted zero residues, c1 = 0 and the boundary primes' residue rows: the terms the zero check flags take the
    unhoisted rotation, n_fallback is the CPU predicate's count, and every word equals the composition"""
    degree, t = 1 << 12, 786433
    moduli = [edge_inputs.gen62(degree, 0)] + list(edge_inputs.BOUNDARY_PRIMES.values())
    S = setup(F, degree, t, None, 0, 0, 16, 4, 4, 31, moduli=moduli)
    assert check(F, S, 16, 4, False) == 0
    rows = c1_power(S.A)
    rows[:, :, 0] = 0                 # s = 0 is never negated: nothing falls back
    assert check(F, S, 16, 4, False, A=_with_c1(F, S, rows)) == 0
    rows = c1_power(S.A)
    rows[1, 0, 2000] = 0              # negated by the exponents 3 and 27 of steps 1 and 3
    rows[2, 2, 500] = 0               # negated by 9 and 27 (steps 2 and 3)
    rows[3, 1, 3] = 0                 # negated by none of them
    assert check(F, S, 16, 4, True, A=_with_c1(F, S, rows)) == 4
    assert check(F, S, 16, 4, False, A=S.A - S.A) == 12   # c1 = 0: every baby step falls back
    ed = edge_inputs.residue_rows(S.moduli, degree)
    rows = np.stack([ed[k] for k in ("zero", "max", "alternating", "one_first")])
    nf = check(F, S, 16, 4, False, A=_with_c1(F, S, rows))
    assert 3 <= nf <= 9, nf   # the all-(q - 1) rows have no zero, the zero rows fall back for every step


def test_real_keys_decrypt_to_matrix_times_vector(F):
    """device-generated keys and encode_diagonals: both rows decrypt to M v mod t, for a random matrix (n = N/2), a
    banded one (n < N/2), a pair of matrices (one per row) and one matrix per ciphertext"""
    degree, t, half = 64, 1153, 32
    par = F.BfvParameters(degree, t, moduli_sizes=[62, 62], device=0)
    sk = F.SecretKey.random_vec(par, 1, seed=bytes([35]) * 32)[0]
    rng = np.random.default_rng(36)
    enc = F.Encoding.simd()
    v = rng.integers(0, t, (3, 2, half)).astype(np.int64)
    ct = sk.try_encrypt(F.PlaintextVec.try_encode(v.reshape(-1).astype(np.uint64), enc, par), seed=bytes([37]) * 32)
    band = rng.integers(0, t, (half, half)).astype(np.int64)
    band *= ((np.arange(half)[None, :] - np.arange(half)[:, None]) % half) < 5
    cases = [(rng.integers(0, t, (half, half)), half, 6), (band, 5, 2), (band, 5, 5),
             (rng.integers(0, t, (2, half, half)), half, 8), (rng.integers(0, t, (3, 2, half, half)), half, 4)]
    for M, n, baby in cases:
        b = F.EvaluationKeyBuilder.new(sk)
        for s in F.linear_transform_steps(n, baby):
            b.enable_column_rotation(s)
        ek = b.build(seed=bytes([38]) * 32)
        diags = F.encode_diagonals(par, M, baby, n_diags=n)
        out = ek.linear_transform(ct, diags, baby)
        Ms = np.asarray(M, np.int64)
        if Ms.ndim == 2:
            Ms = np.stack([Ms, Ms])
        if Ms.ndim == 3:
            Ms = Ms[None]
        Ms = np.broadcast_to(Ms, (3, 2, half, half))
        for c in range(3):
            dec = sk.try_decrypt(out.take(c, 1)).try_decode(enc).reshape(2, half)
            want = np.stack([(Ms[c, q] @ v[c, q]) % t for q in range(2)]).astype(np.uint64)
            assert (dec == want).all(), (n, baby, c)


def test_matches_the_hand_built_product(F):
    """the seeds of test_baby_step_giant_step_matrix_times_vector: the call decrypts to the slots of the hand-built
    composition (its words differ: there step 0 is a key switch by exponent 1)"""
    degree, t, half, n1 = 64, 1153, 32, 8
    n2 = half // n1
    par = F.BfvParameters(degree, t, moduli_sizes=[62, 62], device=0)
    sk = F.SecretKey.random_vec(par, 1, seed=bytes([25]) * 32)[0]
    b = F.EvaluationKeyBuilder.new(sk)
    for i in list(range(1, n1)) + [n1 * g for g in range(1, n2)]:
        b.enable_column_rotation(i)
    ek = b.build(seed=bytes([26]) * 32)
    ek.add_galois_key(F.GaloisKey.new(sk, 1, seed=bytes([27]) * 32))
    rng = np.random.default_rng(28)
    M = rng.integers(0, t, (half, half)).astype(np.int64)
    rows = rng.integers(0, t, (2, half)).astype(np.int64)
    enc = F.Encoding.simd()
    ct = sk.try_encrypt(F.PlaintextVec.try_encode(rows.reshape(-1).astype(np.uint64), enc, par), seed=bytes([29]) * 32)
    baby, _ = F.galois_many_hoisted(ct, *ek._many_args(ct, list(range(n1))))
    acc = None
    d = F.bfv.diagonals(M, half, half, n1)[0]
    for g in range(n2):
        inner = F.dot_product_scalar(baby, F.PlaintextVec.try_encode(d[g * n1:(g + 1) * n1].reshape(-1), enc, par))
        part = ek.rotates_columns_by(inner, g * n1) if g else inner
        acc = part if acc is None else acc + part
    hand = sk.try_decrypt(acc).try_decode(enc)
    out = ek.linear_transform(ct, F.encode_diagonals(par, M, n1), n1)
    assert (sk.try_decrypt(out).try_decode(enc) == hand).all()
    assert (hand.reshape(2, half) == np.stack([(M @ r) % t for r in rows]).astype(np.uint64)).all()


def test_no_state_outlives_the_call(F):
    import torch
    S = setup(F, 1 << 13, 786433, [62, 62], 0, 0, 16, 4, 4, 6)
    diags = random_diags(F, S, 16, 1)
    F.linear_transform(S.A, diags, 4, S.gks, 16)
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    for _ in range(3):
        out, _ = F.linear_transform(S.A, diags, 4, S.gks, 16)
        del out
    torch.cuda.synchronize()
    assert abs(torch.cuda.mem_get_info()[0] - free0) < 2 << 20


def test_refusals_write_nothing_and_keep_no_memory(F):
    import ctypes as C
    import torch
    from fhe_rs_b200 import _capi
    lib = _capi.lib()
    degree = 1 << 12
    S = setup(F, degree, 786433, [62, 62], 0, 0, 8, 3, 3, 1)    # steps 1, 2, 3, 6
    other = setup(F, degree, 786433, [62, 62], 0, 0, 8, 3, 3, 2)
    d = random_diags(F, S, 8, 3)
    d_l1 = F.Ciphertext.from_host(S.par, rand_rows(np.random.default_rng(5), S.moduli[:1], (8, 1), degree), level=1)
    P = S.A.clone().into_power_basis()
    dP = d.clone().into_power_basis()
    out = F.Ciphertext(S.par, 3, 2)
    out2 = F.Ciphertext(S.par, 2, 2)
    sentinels = [(b, b.to_host()) for b in (out, out2, S.A, d)]

    def arr(hs):
        a = (C.c_void_p * max(1, len(hs)))(*[getattr(h, "value", h) for h in hs])
        return C.cast(a, C.POINTER(C.c_void_p))

    def u(v):
        return (C.c_uint32 * max(1, len(v)))(*v)
    k = [g.ksk._h for g in S.gks]
    ex = u([g.exponent for g in S.gks])
    nfv = C.c_uint32(77)
    nf = C.byref(nfv)

    def lt(a, dg, n, b, keys, exps, nk, o):
        return lib.fhe_b200_linear_transform(a, dg, n, b, keys, exps, nk, o, nf, None)
    bad = _capi.INVALID_ARGUMENT
    cases = [
        ("missing step", lambda: lt(S.A._h, d._h, 8, 3, arr(k[:3]), ex, 3, out._h), bad, b"by 6"),
        ("missing baby", lambda: lt(S.A._h, d._h, 8, 3, arr(k[1:]), u([g.exponent for g in S.gks[1:]]), 3, out._h),
         bad, b"by 1"),
        ("no keys", lambda: lt(S.A._h, d._h, 8, 3, None, None, 0, out._h), bad, None),
        ("baby 0", lambda: lt(S.A._h, d._h, 8, 0, arr(k), ex, 4, out._h), bad, None),
        ("baby beyond", lambda: lt(S.A._h, d._h, 8, 9, arr(k), ex, 4, out._h), bad, None),
        ("no diagonals", lambda: lt(S.A._h, d._h, 0, 1, arr(k), ex, 4, out._h), bad, None),
        ("beyond N/2", lambda: lt(S.A._h, d._h, degree // 2 + 1, 3, arr(k), ex, 4, out._h), bad, None),
        ("diag count", lambda: lt(S.A._h, d._h, 7, 3, arr(k), ex, 4, out._h), bad, None),
        ("out shape", lambda: lt(S.A._h, d._h, 8, 3, arr(k), ex, 4, out2._h), bad, None),
        ("aliased", lambda: lt(S.A._h, d._h, 8, 3, arr(k), ex, 4, S.A._h), bad, None),
        ("null key", lambda: lt(S.A._h, d._h, 8, 3, arr([k[0], None, k[2], k[3]]), ex, 4, out._h), bad, None),
        ("even exponent", lambda: lt(S.A._h, d._h, 8, 3, arr(k), u([3, 6, 5, 7]), 4, out._h),
         _capi.INVALID_EXPONENT, None),
        ("other parameters", lambda: lt(S.A._h, d._h, 8, 3, arr(k[:3] + [other.gks[3].ksk._h]), ex, 4, out._h),
         _capi.CONTEXT_MISMATCH, None),
        ("level", lambda: lt(S.A._h, d_l1._h, 8, 3, arr(k), ex, 4, out._h), _capi.INVALID_LEVEL, None),
        ("representation", lambda: lt(P._h, d._h, 8, 3, arr(k), ex, 4, out._h), _capi.INVALID_REPRESENTATION, None),
        ("diag representation", lambda: lt(S.A._h, dP._h, 8, 3, arr(k), ex, 4, out._h),
         _capi.INVALID_REPRESENTATION, None),
    ]
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    for _ in range(2):
        for what, call, code, msg in cases:
            got = call()
            assert got == code, (what, got, lib.fhe_b200_last_error())
            if msg:
                assert msg in lib.fhe_b200_last_error(), (what, lib.fhe_b200_last_error())
    torch.cuda.synchronize()
    assert abs(torch.cuda.mem_get_info()[0] - free0) < 4 << 20
    assert nfv.value == 77
    for b, words in sentinels:
        assert (b.to_host() == words).all()
    with pytest.raises(F.FheError) as e:   # the mirror names the missing step
        ek = F.EvaluationKey(S.par)
        ek.add_galois_key(S.gks[0])
        ek.linear_transform(S.A, d, 3, 8)
    assert e.value.code == bad and "by 2" in str(e.value)


def test_cpp_mirror(F, tmp_path):
    """the C++ mirror's linear_transform (with n_fallback) and EvaluationKey::linear_transform give the Python
    mirror's words"""
    degree, t, sizes, n, baby, count = 64, 1153, [62, 62, 62], 10, 3, 4
    S = setup(F, degree, t, sizes, 0, 0, n, baby, count, 12)
    d = random_diags(F, S, n * count, 13)
    steps = R.steps(n, baby)
    exps = [g.exponent for g in S.gks]
    lines = ["%d %d %d %d %d %d %d" % (degree, t, len(S.moduli), count, n, baby, len(exps)),
             " ".join(map(str, S.moduli)), " ".join(map(str, exps))]
    for kk, g in enumerate(S.gks):
        c0, c1 = g.ksk.arrays()
        c0.tofile(str(tmp_path / ("k%d_c0.bin" % kk)))
        c1.tofile(str(tmp_path / ("k%d_c1.bin" % kk)))
    (tmp_path / "args.txt").write_text("\n".join(lines) + "\n")
    S.A.to_host().tofile(str(tmp_path / "a.bin"))
    d.to_host().tofile(str(tmp_path / "d.bin"))
    exe = str(tmp_path / "linear_transform_test")
    lib_dir = os.path.join(ROOT, "fhe_rs_b200")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "cpp", "linear_transform_test.cpp"), "-o", exe,
                           "-L", lib_dir, "-lfhe_b200", "-Wl,-rpath," + lib_dir])
    out = subprocess.run([exe, str(tmp_path)], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0 and out.stdout.startswith("OK"), out.stdout + out.stderr
    got, nf = F.linear_transform(S.A, d, baby, S.gks, n)
    assert "n_fallback %d" % nf in out.stdout, out.stdout
    ek = F.EvaluationKey(S.par)
    for g in S.gks:
        ek.add_galois_key(g)
    assert len(steps) == len(S.gks)
    want = {"call": got.to_host(), "ek": ek.linear_transform(S.A, d, baby, n).to_host()}
    for name, w in want.items():
        assert (np.fromfile(str(tmp_path / ("out_%s.bin" % name)), np.uint64) == w.ravel()).all(), name


SWITCHES = {"fast": {"FHE_B200_NTT": "fast"}, "tma_ntt": {"FHE_B200_NTT": "tma"},
            "tma": {"FHE_B200_KSMAC": "tma"}, "classic": {"FHE_B200_KSMAC": "classic"},
            "no_solinas": {"FHE_B200_NO_SOLINAS": "1"}, "chunk1": {"FHE_B200_CHUNK": "1"},
            "chunk2_streams2": {"FHE_B200_CHUNK": "2", "FHE_B200_STREAMS": "2"},
            "streams1": {"FHE_B200_STREAMS": "1"}, "streams4": {"FHE_B200_STREAMS": "4", "FHE_B200_CHUNK": "16"}}


def test_switch_reruns():
    """the word checks under each transform, key-switch, arithmetic and chunking switch, one process per switch (read
    once per process), side by side"""
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
    word_checks(fhe_rs_b200, quick=os.environ.get("FHE_B200_CHUNK") in ("1", "2"))
    print("WORD CHECKS OK")
