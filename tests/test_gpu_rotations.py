"""Per-ciphertext Galois exponents (fhe_b200_galois_many) and the batched inner sum (fhe_b200_inner_sum, _keyed), and
their Python / C++ mirrors.

Output j of galois_many must be, word for word, the single fhe_b200_galois call on ciphertext source[j] with the
exponent and key of index[j]; the single call is pinned to the oracle by test_gpu_parity.py and test_gpu_keyed.py.  The
inner sum must equal the loop of fhe_b200_galois + fhe_b200_add that the mirrors ran before, and the oracle's
computes_inner_sum.  The shapes are those of tests/work_split_cases.SHAPES plus N = 16 and 64, a set C level-1 batch
with level-0 keys and a single-modulus key level (base-2^b digits).  The word checks are rerun in subprocesses under
the kernel-selection and chunking switches.  Run with `-m gpu`."""
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

from work_split_cases import SHAPES   # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def F():
    from conftest import has_gpu
    if not has_gpu():
        pytest.skip("no CUDA device")
    import fhe_rs_b200
    return fhe_rs_b200


def rand_rows(rng, moduli, prefix, n):
    a = np.zeros(tuple(prefix) + (len(moduli), n), np.uint64)
    for i, q in enumerate(moduli):
        a[..., i, :] = rng.integers(0, q, size=tuple(prefix) + (n,), dtype=np.uint64)
    return a


def inner_sum_exponents(degree):
    """the exponents of the inner sum's steps: 3^i mod 2N for i = 1, 2, 4, ..., N/4, then 2N - 1"""
    return [pow(3, 1 << l, 2 * degree) for l in range(degree.bit_length() - 2)] + [2 * degree - 1]


class Setup:
    """a parameter set, `count` random ciphertexts at `level` and one random key per exponent (bit-exactness needs no
    real keys)"""

    def __init__(self, F, degree, t, sizes, level, key_level, exponents, count, seed, moduli=None):
        self.F = F
        self.par = F.BfvParameters(degree, t, moduli=moduli, moduli_sizes=None if moduli else sizes, device=0)
        self.moduli = [int(q) for q in self.par.moduli()]
        self.level, self.key_level, self.count, self.degree = level, key_level, count, degree
        rng = np.random.default_rng(seed)
        ct_mod = self.moduli[:len(self.moduli) - level]
        key_mod = self.moduli[:len(self.moduli) - key_level]
        if len(key_mod) == 1:   # key_switching_key.rs:92-126: base 2^(log q / 2)
            lq = (self.moduli[0] - 1).bit_length()
            n_dig = -(-lq // (lq // 2))
        else:
            n_dig = len(ct_mod)
        self.gks = []
        for e in exponents:
            c = rand_rows(rng, key_mod, (2, n_dig), degree)
            self.gks.append(F.GaloisKey(e, F.KeySwitchingKey.from_arrays(self.par, c[0], c[1], level, key_level)))
        self.A = F.Ciphertext.from_host(self.par, rand_rows(rng, ct_mod, (count, 2), degree), level=level)

    def many(self, index, source=None):
        return self.F.galois_many(self.A, self.gks, index, source).to_host()

    def expected(self, index, source=None):
        """output j from single fhe_b200_galois calls: one call on the whole batch per key when few keys are used,
        else one call per output"""
        src = list(range(self.count)) if source is None else list(source)
        distinct = sorted(set(index))
        if len(distinct) <= 4:
            whole = {k: self.gks[k].relinearize(self.A).to_host() for k in distinct}
            return np.stack([whole[k][s] for k, s in zip(index, src)])
        return np.stack([self.gks[k].relinearize(self.A.take(s, 1)).to_host()[0] for k, s in zip(index, src)])

    def check(self, index, source=None):
        got = self.many(index, source)
        exp = self.expected(index, source)
        bad = [j for j in range(got.shape[0]) if not (got[j] == exp[j]).all()]
        assert not bad, (self.degree, self.count, bad[:8])


# name -> (degree, t, sizes, level, key level)
def _cases():
    c = {}
    for name, s in SHAPES.items():
        c[name] = (1 << s["logn"], s["t"], s["sizes"], 0, 0)
    c["n16"] = (16, 1153, [62] * 3, 0, 0)
    c["n64"] = (64, 1153, [62] * 3, 0, 0)
    c["c_l1"] = (1 << 15, 786433, [62] * 14, 1, 0)
    c["single_mod"] = (1 << 13, 65537, [62, 62], 1, 1)
    return c


CASES = _cases()
# (shape, count, index pattern, source pattern)
SHAPE_RUNS = [("n13_2x62", 7, "alt", None), ("n13_62_40_30", 33, "runs5", "perm"), ("n14_8x62", 33, "alt", "zero"),
              ("n15_14x62", 3, "distinct", "repeat"), ("n16", 5, "alt", "perm"), ("n64", 7, "runs2", None),
              ("c_l1", 3, "alt", "zero"), ("single_mod", 5, "distinct", "repeat")]


def _exponents(degree, n):
    """n distinct Galois exponents: 2N - 1, the column rotations 3^i, the expansion elements (N >> l) + 1, then two
    at or above 2N (reduced by the call), then further odd exponents"""
    m = 2 * degree
    out = [m - 1]
    for i in range(1, degree // 2):
        e = pow(3, i, m)
        if e not in out:
            out.append(e)
    out += [(degree >> l) + 1 for l in range(degree.bit_length() - 1) if (degree >> l) + 1 not in out]
    big = [3 + m, m - 1 + 4 * m]
    out = out[:max(0, n - 2)] + big
    e = 5
    while len(out) < n:
        if e not in out and e + m not in out and e + 5 * m not in out:
            out.append(e)
        e += 2
    return out[:n]


def _index(pattern, count, n_keys):
    if pattern == "alt":
        return [j % 2 for j in range(count)]
    if pattern == "distinct":
        return [j % n_keys for j in range(count)]
    if pattern.startswith("runs"):
        run = int(pattern[4:])
        return [min(j // run, n_keys - 1) for j in range(count)]
    raise ValueError(pattern)


def _source(pattern, count, n_in):
    if pattern is None:
        return None
    if pattern == "zero":
        return [0] * count
    if pattern == "perm":
        return list(np.random.default_rng(count).permutation(n_in))[:count]
    if pattern == "repeat":
        return [(j // 2) % n_in for j in range(count)]
    raise ValueError(pattern)


def word_checks(F, quick=False):
    """the bit-exactness sweep the switch reruns repeat"""
    for name, count, pattern, src in SHAPE_RUNS:
        if quick and name in ("n15_14x62", "c_l1"):
            continue
        degree, t, sizes, level, key_level = CASES[name]
        n_keys = 4 if pattern != "distinct" else count
        S = Setup(F, degree, t, sizes, level, key_level, _exponents(degree, n_keys), count, hash(name) & 0xffff)
        S.check(_index(pattern, count, n_keys), _source(src, count, count))
    # 130 keys (more than one substitution and inner-product launch per chunk), runs cutting chunks
    S = Setup(F, 1 << 13, 786433, [62, 62], 0, 0, _exponents(1 << 13, 130), 259, 5)
    S.check(list(range(130)) + [129 - j % 130 for j in range(129)])
    S.check([j // 22 for j in range(259)], [258 - j for j in range(259)])
    # inner sums
    for name in ("n16", "n64", "n13_62_40_30"):
        degree, t, sizes, level, key_level = CASES[name]
        S = Setup(F, degree, t, sizes, level, key_level, inner_sum_exponents(degree), 5, 3)
        _check_inner_sum(F, S)


@pytest.mark.parametrize("name,count,pattern,src", SHAPE_RUNS)
def test_many_equals_single_calls(F, name, count, pattern, src):
    degree, t, sizes, level, key_level = CASES[name]
    n_keys = 4 if pattern != "distinct" else count
    S = Setup(F, degree, t, sizes, level, key_level, _exponents(degree, n_keys), count, 11)
    S.check(_index(pattern, count, n_keys), _source(src, count, count))
    S.check([count % n_keys] * count)


def test_exponent_and_source_patterns(F):
    """all exponents distinct, alternating, runs at counts that cut chunks, 65 and 130 keys; source NULL, all zero, a
    permutation and repeated entries; one ciphertext rotated by every exponent"""
    degree, t, sizes = 1 << 13, 786433, [62, 62]
    S = Setup(F, degree, t, sizes, 0, 0, _exponents(degree, 130), 259, 5)
    S.check(list(range(130)) + [129 - j % 130 for j in range(129)])
    S.check([j % 65 for j in range(259)])
    S.check([j % 2 for j in range(259)])
    S.check([j // 22 for j in range(259)])
    S.check([j % 130 for j in range(300)], [0] * 300)                                # one source, 300 outputs
    S.check([j % 7 for j in range(259)], list(np.random.default_rng(1).permutation(259)))
    S.check([j % 3 for j in range(100)], [(j * 7) % 11 for j in range(100)])         # repeated sources
    S.check(list(range(130)), [42] * 130)                                            # one ciphertext, 130 exponents
    for count in list(range(1, 15)) + [17, 33]:
        Sc = Setup(F, degree, t, sizes, 0, 0, _exponents(degree, 6), count, count)
        Sc.check([(j // 3) % 6 for j in range(count)])


def test_one_exponent_equals_galois_keyed(F):
    """a single exponent: galois_keyed's words and launch count"""
    lib = F._capi.lib()
    degree, t, sizes = 1 << 13, 786433, [62, 62]
    for count in (33, 259):
        S = Setup(F, degree, t, sizes, 0, 0, [3] * 5, count, count)
        index = [j % 5 for j in range(count)]
        n0 = lib.fhe_b200_launch_count()
        w = F.galois_keyed(S.A, S.gks, index).to_host()
        n1 = lib.fhe_b200_launch_count()
        g = S.many(index)
        n2 = lib.fhe_b200_launch_count()
        assert (g == w).all(), count
        assert n2 - n1 == n1 - n0, (count, n1 - n0, n2 - n1)


def _loop_inner_sum(F, ct, gks):
    """the mirrors' previous inner sum: log2 N fhe_b200_galois calls, each followed by fhe_b200_add"""
    out = ct.clone()
    for g in gks:
        out += g.relinearize(out)
    return out


def _check_inner_sum(F, S):
    lib = F._capi.lib()
    ek = F.EvaluationKey(S.par, S.level, S.key_level)
    for g in S.gks:
        ek.add_galois_key(g)
    before = S.A.to_host()
    n0 = lib.fhe_b200_launch_count()
    got = ek.computes_inner_sum(S.A).to_host()
    n1 = lib.fhe_b200_launch_count()
    want = _loop_inner_sum(F, S.A, ek.inner_sum_keys()).to_host()
    n2 = lib.fhe_b200_launch_count()
    assert (got == want).all(), S.degree
    assert (S.A.to_host() == before).all()
    return n1 - n0, n2 - n1


def test_inner_sum_equals_the_loop(F):
    """fhe_b200_inner_sum against the loop of fhe_b200_galois + fhe_b200_add, with fewer launches (no add kernels)"""
    for name, count in (("n16", 5), ("n64", 7), ("n13_2x62", 259), ("n13_62_40_30", 33), ("c_l1", 3),
                        ("single_mod", 4)):
        degree, t, sizes, level, key_level = CASES[name]
        S = Setup(F, degree, t, sizes, level, key_level, inner_sum_exponents(degree), count, 7)
        fused, loop = _check_inner_sum(F, S)
        assert fused < loop, (name, fused, loop)


def test_inner_sum_against_the_oracle(oracle, F):
    """samples of fhe_b200_inner_sum against the oracle's computes_inner_sum, leveled keys at set C"""
    for degree, t, sizes, level, key_level in ((16, 1153, [62] * 3, 0, 0), (64, 1153, [62] * 3, 1, 0),
                                               (1 << 15, 786433, [62] * 14, 1, 0)):
        opar = oracle.BfvParameters(degree, t, moduli_sizes=sizes)
        S = Setup(F, degree, t, sizes, level, key_level, inner_sum_exponents(degree), 3, degree, moduli=opar.moduli)
        ek = F.EvaluationKey(S.par, level, key_level)
        for g in S.gks:
            ek.add_galois_key(g)
        got = ek.computes_inner_sum(S.A).to_host()
        a = S.A.to_host()
        ogks = {}
        for g in S.gks:
            o = oracle.GaloisKey.__new__(oracle.GaloisKey)
            o.exponent, o.ksk = g.exponent % (2 * degree), oracle.KeySwitchingKey.from_arrays(opar, *g.ksk.arrays(),
                                                                                            level, key_level)
            ogks[o.exponent] = o
        for j in (0, 2):
            want = oracle.computes_inner_sum(opar, ogks, oracle.Ciphertext.from_array(opar, a[j], level))
            assert (want.to_array() == got[j]).all(), (degree, j)


def test_inner_sum_keyed_equals_single(F):
    """each ciphertext of the keyed inner sum equals the single inner sum with its own key set"""
    degree, t, sizes = 1 << 13, 786433, [62, 62]
    exps = inner_sum_exponents(degree)
    sets = [Setup(F, degree, t, sizes, 0, 0, exps, 1, 100 + s) for s in range(3)]
    base = sets[0]
    for s in sets[1:]:   # the keys of every set on the first set's parameters
        s.gks = [F.GaloisKey(g.exponent, F.KeySwitchingKey.from_arrays(base.par, *g.ksk.arrays())) for g in s.gks]
    eks = []
    for s in sets:
        ek = F.EvaluationKey(base.par)
        for g in s.gks:
            ek.add_galois_key(g)
        eks.append(ek)
    A = F.Ciphertext.from_host(base.par, rand_rows(np.random.default_rng(9), base.moduli, (67, 2), degree))
    index = [(j * 5) % 3 for j in range(67)]
    got = F.computes_inner_sum_keyed(A, eks, index).to_host()
    single = [ek.computes_inner_sum(A).to_host() for ek in eks]
    bad = [j for j in range(67) if not (got[j] == single[index[j]][j]).all()]
    assert not bad, bad[:8]


def test_clients_inner_sums_decrypt_under_their_own_keys(F):
    """eight clients with device-generated keys: each SIMD inner sum decrypts under its own key to the sum of the
    slots in every slot, and not under a neighbour's key"""
    degree, t, n = 64, 1153, 8
    par = F.BfvParameters(degree, t, moduli_sizes=[62, 62], device=0)
    sks = F.SecretKey.random_vec(par, n, seed=bytes(range(32)))
    eks = [F.EvaluationKeyBuilder.new(sk).enable_inner_sum().build(seed=bytes([c + 1]) * 32)
           for c, sk in enumerate(sks)]
    rng = np.random.default_rng(4)
    vals = [rng.integers(0, t, degree).astype(np.uint64) for _ in range(n)]
    enc = F.Encoding.simd()
    cts = [sk.try_encrypt(F.PlaintextVec.try_encode(vals[c], enc, par), seed=bytes([c + 41]) * 32)
           for c, sk in enumerate(sks)]
    words = np.concatenate([c.to_host() for c in cts])
    A = F.Ciphertext.from_host(par, words)
    out = F.computes_inner_sum_keyed(A, eks, list(range(n)))
    for c in range(n):
        dec = sks[c].try_decrypt(out.take(c, 1)).try_decode(enc)
        assert (dec == int(vals[c].astype(object).sum()) % t).all(), c
        wrong = sks[(c + 1) % n].try_decrypt(out.take(c, 1)).try_decode(enc)
        assert not (wrong == int(vals[c].astype(object).sum()) % t).all(), c


def test_diagonal_matrix_times_encrypted_vector(F):
    """M v at N = 64 by the diagonal method: one rotates_columns_by_many call for steps 0..31, then dot_product_scalar
    with the SIMD-encoded diagonals; both rows of the result decrypt to M v mod t"""
    degree, t, half = 64, 1153, 32
    par = F.BfvParameters(degree, t, moduli_sizes=[62, 62], device=0)
    sk = F.SecretKey.random_vec(par, 1, seed=bytes([5]) * 32)[0]
    b = F.EvaluationKeyBuilder.new(sk)
    for i in range(1, half):
        b.enable_column_rotation(i)
    ek = b.build(seed=bytes([6]) * 32)
    ek.add_galois_key(F.GaloisKey.new(sk, 1, seed=bytes([7]) * 32))   # step 0: the identity substitution
    rng = np.random.default_rng(8)
    M = rng.integers(0, t, (half, half)).astype(np.int64)
    rows = rng.integers(0, t, (2, half)).astype(np.int64)   # one vector per SIMD row
    enc = F.Encoding.simd()
    ct = sk.try_encrypt(F.PlaintextVec.try_encode(rows.reshape(-1).astype(np.uint64), enc, par), seed=bytes([9]) * 32)
    rot = ek.rotates_columns_by_many(ct, list(range(half)))
    assert rot.count == half
    one = sk.try_decrypt(rot.take(1, 1)).try_decode(enc).reshape(2, half)
    assert (one == np.roll(rows, -1, axis=1)).all(), "rotation by one moves slot j + 1 to slot j"
    # diagonal i: slot j of each row holds M[j][(j + i) mod 32]
    diags = np.zeros((half, degree), np.uint64)
    for i in range(half):
        d = np.array([M[j][(j + i) % half] for j in range(half)], np.uint64)
        diags[i] = np.concatenate([d, d])
    pts = F.PlaintextVec.try_encode(diags.reshape(-1), enc, par)
    res = sk.try_decrypt(F.dot_product_scalar(rot, pts)).try_decode(enc).reshape(2, half)
    want = np.stack([(M @ r) % t for r in rows]).astype(np.uint64)
    assert (res == want).all()


def test_refusals_write_nothing_and_keep_no_memory(F):
    """every error of the new calls; the output words and device memory are unchanged by each refusal"""
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
    isum_keys = Setup(F, degree, t, sizes, 0, 0, inner_sum_exponents(degree), 1, 5)
    ik = [F.KeySwitchingKey.from_arrays(S.par, *g.ksk.arrays()) for g in isum_keys.gks]

    def arr(hs):
        a = (C.c_void_p * max(1, len(hs)))(*[getattr(h, "value", h) for h in hs])
        return C.cast(a, C.POINTER(C.c_void_p))

    def u(v):
        return (C.c_uint32 * max(1, len(v)))(*v)
    k = [g.ksk._h for g in S.gks]
    ex = u([3, 5, 2 * degree - 1])
    good = u([0, 1, 2, 0])
    bad_arg, many = _capi.INVALID_ARGUMENT, lib.fhe_b200_galois_many
    cases = [
        ("null list", lambda: many(S.A._h, None, None, ex, 3, good, out._h, None), bad_arg),
        ("null exponents", lambda: many(S.A._h, None, arr(k), None, 3, good, out._h, None), bad_arg),
        ("null index", lambda: many(S.A._h, None, arr(k), ex, 3, None, out._h, None), bad_arg),
        ("no keys", lambda: many(S.A._h, None, arr(k), ex, 0, good, out._h, None), bad_arg),
        ("null key", lambda: many(S.A._h, None, arr([k[0], None, k[2]]), ex, 3, good, out._h, None), bad_arg),
        ("index beyond", lambda: many(S.A._h, None, arr(k), ex, 3, u([0, 3, 0, 0]), out._h, None), bad_arg),
        ("source beyond", lambda: many(S.A._h, u([0, 4, 0]), arr(k), ex, 3, good, out3._h, None), bad_arg),
        ("counts differ", lambda: many(S.A._h, None, arr(k), ex, 3, good, out3._h, None), bad_arg),
        ("aliased", lambda: many(S.A._h, None, arr(k), ex, 3, good, S.A._h, None), bad_arg),
        ("even exponent", lambda: many(S.A._h, None, arr(k), u([3, 6, 5]), 3, good, out._h, None),
         _capi.INVALID_EXPONENT),
        ("key levels differ", lambda: many(a_l1._h, None, arr([l1k0._h, l1k1._h]), u([3, 5]), 2, u([0, 1, 0, 1]),
                                           out_l1._h, None), bad_arg),
        ("other parameters", lambda: many(S.A._h, None, arr(k + [other.gks[0].ksk._h]), u([3, 5, 7, 3]), 4, good,
                                          out._h, None), _capi.CONTEXT_MISMATCH),
        ("other level", lambda: many(S.A._h, None, arr([l1k0._h]), ex, 1, u([0] * 4), out._h, None),
         _capi.INVALID_LEVEL),
        ("representation", lambda: many(P._h, None, arr(k), ex, 3, good, out._h, None),
         _capi.INVALID_REPRESENTATION),
        ("inner sum n_gks", lambda: lib.fhe_b200_inner_sum(S.A._h, arr([x._h for x in ik]), len(ik) - 1, out._h, None), bad_arg),
        ("inner sum null key", lambda: lib.fhe_b200_inner_sum(S.A._h, arr([x._h for x in ik[:-1]] + [None]), len(ik), out._h, None),
         bad_arg),
        ("inner sum aliased", lambda: lib.fhe_b200_inner_sum(S.A._h, arr([x._h for x in ik]), len(ik), S.A._h, None), bad_arg),
        ("inner sum shape", lambda: lib.fhe_b200_inner_sum(S.A._h, arr([x._h for x in ik]), len(ik), out3._h, None), bad_arg),
        ("inner sum level", lambda: lib.fhe_b200_inner_sum(a_l1._h, arr([x._h for x in ik]), len(ik), out_l1._h, None),
         _capi.INVALID_LEVEL),
        ("keyed no sets", lambda: lib.fhe_b200_inner_sum_keyed(S.A._h, arr([x._h for x in ik]), len(ik), 0, good, out._h, None),
         bad_arg),
        ("keyed null index", lambda: lib.fhe_b200_inner_sum_keyed(S.A._h, arr([x._h for x in ik]), len(ik), 1, None, out._h, None),
         bad_arg),
        ("keyed set beyond", lambda: lib.fhe_b200_inner_sum_keyed(S.A._h, arr([x._h for x in ik]), len(ik), 1, u([0, 1, 0, 0]),
                                                                  out._h, None), bad_arg),
    ]
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    for what, call, code in cases:
        got = call()
        assert got == code, (what, got, lib.fhe_b200_last_error())
    torch.cuda.synchronize()
    assert abs(torch.cuda.mem_get_info()[0] - free0) < 4 << 20
    for b, words in sentinels:
        assert (b.to_host() == words).all()


def test_new_exponents_build_no_tables(F):
    """rotating by 64 exponents the parameter set has not seen leaves the device memory in use unchanged"""
    import torch
    degree = 1 << 15
    S = Setup(F, degree, 786433, [62, 62], 0, 0, [3], 64, 6)
    ksk = S.gks[0].ksk
    S.gks = [F.GaloisKey(3, ksk)]
    S.many([0] * 64)   # the scratch pool at this shape
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    S.gks = [F.GaloisKey(e, ksk) for e in _exponents(degree, 64)]
    S.many(list(range(64)))
    torch.cuda.synchronize()
    assert abs(torch.cuda.mem_get_info()[0] - free0) < 2 << 20


def test_cpp_mirror(F, tmp_path):
    """the C++ mirror's galois_many, rotates_columns_by_many, computes_inner_sum and computes_inner_sum_keyed give the
    Python mirror's words"""
    degree, t, sizes = 64, 1153, [62, 62, 62]
    exps = inner_sum_exponents(degree)
    S = Setup(F, degree, t, sizes, 0, 0, exps, 5, 12)
    count = 9
    index = [(j * 5) % len(exps) for j in range(count)]
    source = [(j * 3) % 5 for j in range(count)]
    sets = [j % 2 for j in range(5)]
    lines = ["%d %d %d %d %d %d" % (degree, t, len(S.moduli), 5, count, len(exps)), " ".join(map(str, S.moduli)),
             " ".join(map(str, exps)), " ".join(map(str, index)), " ".join(map(str, source)), " ".join(map(str, sets))]
    for k, g in enumerate(S.gks):
        c0, c1 = g.ksk.arrays()
        c0.tofile(str(tmp_path / ("k%d_c0.bin" % k)))
        c1.tofile(str(tmp_path / ("k%d_c1.bin" % k)))
    (tmp_path / "args.txt").write_text("\n".join(lines) + "\n")
    S.A.to_host().tofile(str(tmp_path / "a.bin"))
    exe = str(tmp_path / "rotations_test")
    lib_dir = os.path.join(ROOT, "fhe_rs_b200")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "cpp", "rotations_test.cpp"), "-o", exe,
                           "-L", lib_dir, "-lfhe_b200", "-Wl,-rpath," + lib_dir])
    out = subprocess.run([exe, str(tmp_path)], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0 and out.stdout.startswith("OK"), out.stdout + out.stderr
    ek0, ek1 = F.EvaluationKey(S.par), F.EvaluationKey(S.par)
    for k, g in enumerate(S.gks):
        ek0.add_galois_key(g)
        ek1.add_galois_key(F.GaloisKey(g.exponent, S.gks[(k + 1) % len(exps)].ksk))
    want = {"many": S.many(index, source), "rot": ek0.rotates_columns_by_many(S.A, [1, 2, 4]).to_host(),
            "isum": ek0.computes_inner_sum(S.A).to_host(),
            "isum_keyed": F.computes_inner_sum_keyed(S.A, [ek0, ek1], sets).to_host()}
    for name, w in want.items():
        assert (np.fromfile(str(tmp_path / ("out_%s.bin" % name)), np.uint64) == w.ravel()).all(), name


SWITCHES = {"tma": {"FHE_B200_KSMAC": "tma"}, "classic": {"FHE_B200_KSMAC": "classic"},
            "stages3": {"FHE_B200_KS_STAGES": "3"}, "chunk1": {"FHE_B200_CHUNK": "1"},
            "streams1": {"FHE_B200_STREAMS": "1"}, "streams4": {"FHE_B200_STREAMS": "4"}}


def test_switch_reruns():
    """the word checks under each key-switch path and chunking switch, one process per switch (read once per process),
    side by side"""
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
