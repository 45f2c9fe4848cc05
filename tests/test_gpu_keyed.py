"""Per-ciphertext keys in the batched key switch (the fhe_b200_*_keyed entry points and their Python / C++ mirrors):
output j of a keyed call must be, word for word, the single-key call's output on ciphertext j with key index[j].

Every output word of each keyed call is compared with the single-key device call (itself pinned to the oracle by
test_gpu_parity.py / test_gpu_expand.py); samples are compared with the oracle directly.  The shapes are those of
tests/work_split_cases.SHAPES plus N = 16 and 64 (the per-thread inner product), a set C level-1 batch with level-0 keys
(13 digits against 14 key limbs, switched down after) and a single-modulus key level (base-2^b digits).  The index
patterns: one key, all distinct, alternating, sorted runs at counts that cut CTA ranges and chunks, 65 and 130
distinct keys (more than one inner-product launch per chunk), unused keys and a repeated handle.  The word checks are
rerun in subprocesses under the kernel-selection and chunking switches.  Run with `-m gpu`."""
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
MULPIR_T = (1 << 20) + (1 << 19) + (1 << 17) + (1 << 16) + (1 << 14) + 1   # examples/mulpir.rs:36
OPS = ("mul", "mul_ms", "relin", "galois", "ks", "expand")
SIZE = 4   # expansion size: two levels, keys for N + 1 and N/2 + 1


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


class Setup:
    """a parameter set, operands at `level` and `n_keys` random keys (bit-exactness needs no real keys).  Key k serves
    as relinearization key, Galois key for 3, expansion keys (N + 1, N/2 + 1) and both halves of an RGSW ciphertext."""

    def __init__(self, F, degree, t, sizes, level, key_level, n_keys, count, seed, moduli=None):
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
        self.ksks = []
        for _ in range(n_keys):
            c = rand_rows(rng, key_mod, (2, n_dig), degree)
            self.ksks.append(F.KeySwitchingKey.from_arrays(self.par, c[0], c[1], level, key_level))
        self.rks = [F.RelinearizationKey(k) for k in self.ksks]
        self.gks = [F.GaloisKey(3, k) for k in self.ksks]
        self.eks = []
        for k in self.ksks:
            ek = F.EvaluationKey(self.par, level, key_level)
            ek.add_galois_key(F.GaloisKey(degree + 1, k))
            ek.add_galois_key(F.GaloisKey(degree // 2 + 1, k))
            self.eks.append(ek)
        self.A = F.Ciphertext.from_host(self.par, rand_rows(rng, ct_mod, (count, 2), degree), level=level)
        self.B = F.Ciphertext.from_host(self.par, rand_rows(rng, ct_mod, (count, 2), degree), level=level)
        self.C3 = self.A * self.B
        self.P = self.A.clone().into_power_basis()

    def ops(self):
        return [op for op in OPS if op != "mul_ms" or self.level < len(self.moduli) - 1]

    def keyed(self, op, index, keys=None):
        F, ks = self.F, (keys if keys is not None else list(range(len(self.ksks))))
        if op in ("mul", "mul_ms"):
            return F.multiply_keyed(self.A, self.B, [self.rks[k] for k in ks], index, mod_switch=op == "mul_ms")
        if op == "relin":
            return F.relinearizes_keyed(self.C3, [self.rks[k] for k in ks], index)
        if op == "galois":
            return F.galois_keyed(self.A, [self.gks[k] for k in ks], index)
        if op == "ks":
            return F.key_switch_keyed(self.P, 1, [self.ksks[k] for k in ks], index)
        return F.expands_batch_keyed(self.A, [self.eks[k] for k in ks], index, SIZE)

    def single(self, op, k, a=None, b=None):
        """the single-key call with key k on the whole batch, or on the batches a (and b)"""
        F = self.F
        a = a if a is not None else self.A
        b = b if b is not None else self.B
        if op in ("mul", "mul_ms"):
            m = F.Multiplicator.default(self.rks[k])
            if op == "mul_ms":
                m.enable_mod_switching()
            return m.multiply(a, b)
        if op == "relin":
            return self.rks[k].relinearizes(self.C3 if a is self.A else a * b)
        if op == "galois":
            return self.gks[k].relinearize(a)
        if op == "ks":
            return self.ksks[k].key_switch(self.P if a is self.A else a.clone().into_power_basis(), 1)
        return self.eks[k].expands_batch(a, SIZE)

    def expected(self, op, key_of):
        """output words of every ciphertext j with key key_of[j] (handle positions), from single-key calls: one call
        on the whole batch per key when there are few keys, else one call per ciphertext"""
        Q = self.count
        distinct = sorted(set(key_of))
        rows = SIZE * Q if op == "expand" else Q
        out = None
        if len(distinct) <= 4:
            for k in distinct:
                w = self.single(op, k).to_host()
                if out is None:
                    out = np.zeros_like(w)
                for j in range(rows):
                    if key_of[j % Q] == k:
                        out[j] = w[j]
            return out
        for j in range(Q):
            a, b = self.A.take(j, 1), self.B.take(j, 1)
            w = self.single(op, key_of[j], a, b).to_host()
            if out is None:
                out = np.zeros((rows,) + w.shape[1:], np.uint64)
            if op == "expand":
                for i in range(SIZE):
                    out[i * Q + j] = w[i]
            else:
                out[j] = w[0]
        return out

    def check(self, op, index, keys=None):
        got = self.keyed(op, index, keys)
        got = got if isinstance(got, np.ndarray) else got.to_host()
        ks = keys if keys is not None else list(range(len(self.ksks)))
        exp = self.expected(op, [ks[i] for i in index])
        bad = [j for j in range(got.shape[0]) if not (got[j] == exp[j]).all()]
        assert not bad, (op, self.degree, self.count, bad[:8])


def _runs(count, run):
    return [j // run for j in range(count)]


# name -> (degree, t, sizes, level, key level, [(count, index pattern)])
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
# (shape, count, n_keys, index): the shapes with the patterns that cut each kernel's work split
SHAPE_RUNS = [("n13_2x62", 7, 3, "alt"), ("n13_62_40_30", 33, 4, "runs5"), ("n14_8x62", 33, 4, "alt"),
              ("n15_14x62", 3, 3, "distinct"), ("n16", 5, 3, "alt"), ("n64", 7, 4, "runs2"),
              ("c_l1", 3, 2, "alt"), ("single_mod", 5, 3, "alt")]


def _index(pattern, count, n_keys):
    if pattern == "alt":
        return [j % 2 for j in range(count)]
    if pattern == "distinct":
        return list(range(count))
    if pattern.startswith("runs"):
        run = int(pattern[4:])
        return [min(j // run, n_keys - 1) for j in range(count)]
    raise ValueError(pattern)


def word_checks(F, quick=False):
    """the bit-exactness sweep the switch reruns repeat"""
    for name, count, n_keys, pattern in SHAPE_RUNS:
        if quick and name in ("n15_14x62", "c_l1"):
            continue
        degree, t, sizes, level, key_level = CASES[name]
        S = Setup(F, degree, t, sizes, level, key_level, n_keys, count, hash(name) & 0xffff)
        for op in S.ops():
            S.check(op, _index(pattern, count, n_keys))
    # the split at 64 keys and runs cutting CTA ranges and chunks, on the cheapest TMA shape
    degree, t, sizes, _, _ = CASES["n13_2x62"]
    S = Setup(F, degree, t, sizes, 0, 0, 130, 259, 5)
    for op in ("mul", "galois", "ks"):
        S.check(op, list(range(130)) + [129 - j % 130 for j in range(129)])
    S.check("relin", [j % 65 for j in range(130)] + [0] * 129)
    S.check("mul", _runs(259, 5))
    S.check("expand", [j % 65 for j in range(130)] + [7] * 129)


@pytest.mark.parametrize("name,count,n_keys,pattern", SHAPE_RUNS)
def test_keyed_equals_single_key(F, name, count, n_keys, pattern):
    degree, t, sizes, level, key_level = CASES[name]
    S = Setup(F, degree, t, sizes, level, key_level, n_keys, count, 11)
    for op in S.ops():
        S.check(op, _index(pattern, count, n_keys))
        S.check(op, list(range(count)) if count <= n_keys else [count % n_keys] * count)


def test_index_patterns_and_the_split_at_64(F):
    """one key, all distinct, alternating, sorted runs at counts 1-14, 17, 33, 259 (chunks of 128, 128, 3), 65 and
    130 distinct keys, unused keys and a repeated handle"""
    degree, t, sizes, _, _ = CASES["n13_2x62"]
    S = Setup(F, degree, t, sizes, 0, 0, 130, 259, 5)
    for op in ("mul", "galois", "ks", "relin", "expand"):
        S.check(op, list(range(130)) + [129 - j % 130 for j in range(129)])   # 130 keys in every chunk
        S.check(op, [j % 65 for j in range(259)])                              # 65 keys: one key past the split
        S.check(op, [j % 2 for j in range(259)])                               # runs of length 1
    for count in list(range(1, 15)) + [17, 33, 259]:
        Sc = Setup(F, degree, t, sizes, 0, 0, 12, count, count)
        for op in ("mul", "ks"):
            Sc.check(op, _runs(count, 3 if count < 15 else 22))
    # unused keys, a handle listed twice (positions 1 and 3 are one key)
    S6 = Setup(F, degree, t, sizes, 0, 0, 4, 9, 9)
    for op in S6.ops():
        S6.check(op, [1, 3, 1, 3, 3, 1, 0, 0, 1], keys=[2, 0, 2, 1, 0])


def test_one_key_and_launch_counts(F):
    """one key: the words and launch count of the single-key call; up to 64 distinct keys per chunk: the launch count of
    the single-key call on the same batch"""
    lib = F._capi.lib()
    degree, t, sizes, _, _ = CASES["n13_2x62"]
    wrong = []
    for count, n_keys in ((33, 33), (259, 52)):
        S = Setup(F, degree, t, sizes, 0, 0, n_keys, count, count)
        for op in S.ops():
            n0 = lib.fhe_b200_launch_count()
            w1 = S.single(op, 0)
            w1 = w1.to_host()
            n1 = lib.fhe_b200_launch_count()
            g = S.keyed(op, [0] * count, keys=[0])
            g = g if isinstance(g, np.ndarray) else g.to_host()
            n2 = lib.fhe_b200_launch_count()
            assert (g == w1).all(), op
            if n2 - n1 != n1 - n0:
                wrong.append(("one key", op, count, n1 - n0, n2 - n1))
            idx = _runs(count, 5)
            assert max(idx) < n_keys
            n3 = lib.fhe_b200_launch_count()
            g = S.keyed(op, idx)
            n4 = lib.fhe_b200_launch_count()
            if n4 - n3 != n1 - n0:
                wrong.append(("runs of 5", op, count, n1 - n0, n4 - n3))
    assert not wrong, wrong


def test_against_the_oracle(oracle, F):
    """samples of each keyed call against the oracle's restatement of the reference, key index[j] per ciphertext"""
    for degree, sizes in ((64, [62] * 3), (1 << 13, [62, 62])):
        t = 1153
        opar = oracle.BfvParameters(degree, t, moduli_sizes=sizes)
        S = Setup(F, degree, t, sizes, 0, 0, 3, 4, degree, moduli=opar.moduli)
        index = [2, 0, 1, 2]
        a, b, c3 = S.A.to_host(), S.B.to_host(), S.C3.to_host()
        oks = [oracle.KeySwitchingKey.from_arrays(opar, *k.arrays(), 0, 0) for k in S.ksks]
        orks = [oracle.RelinearizationKey.from_ksk(k) for k in oks]

        def ogk(k, e):
            g = oracle.GaloisKey.__new__(oracle.GaloisKey)
            g.exponent, g.ksk = e % (2 * degree), oks[k]
            return g
        got = {op: S.keyed(op, index) for op in ("mul", "relin", "galois", "expand")}
        got = {op: (g if isinstance(g, np.ndarray) else g.to_host()) for op, g in got.items()}
        for j in (0, 3):
            k = index[j]
            A = oracle.Ciphertext.from_array(opar, a[j], 0)
            B = oracle.Ciphertext.from_array(opar, b[j], 0)
            assert (oracle.Multiplicator.default(orks[k]).multiply(A, B).to_array() == got["mul"][j]).all(), j
            C3 = oracle.Ciphertext.from_array(opar, c3[j], 0)
            assert (orks[k].relinearizes(C3).to_array() == got["relin"][j]).all(), j
            assert (ogk(k, 3).relinearize(A).to_array() == got["galois"][j]).all(), j
            gks = {degree + 1: ogk(k, degree + 1), degree // 2 + 1: ogk(k, degree // 2 + 1)}
            for i, o in enumerate(oracle.expands(opar, gks, A, SIZE)):
                assert (o.to_array() == got["expand"][i * 4 + j]).all(), (j, i)


def _clients(F, degree, t, sizes, ct_level, key_level, n, size):
    par = F.BfvParameters(degree, t, moduli_sizes=sizes, device=0)
    sks = F.SecretKey.random_vec(par, n, seed=bytes(range(32)))
    level = max(0, (size - 1).bit_length())
    eks = [F.EvaluationKeyBuilder.new_leveled(sk, ct_level, key_level).enable_expansion(level).build(
        seed=bytes([i + 1]) * 32) for i, sk in enumerate(sks)]
    rks = [F.RelinearizationKey.new_leveled(sk, ct_level, key_level, seed=bytes([i + 101]) * 32)
           for i, sk in enumerate(sks)]
    return par, sks, eks, rks, level


def _merge(F, par, parts, level):
    """one batch holding ciphertext j of client c at position j * n + c (clients interleaved)"""
    words = np.stack([p.to_host() for p in parts], axis=1)
    return F.Ciphertext.from_host(par, words.reshape((-1,) + words.shape[2:]), level=level)


@pytest.mark.parametrize("shape", ["mulpir", "set_c"])
def test_multi_client_server(F, shape):
    """8 clients with device-generated keys; their queries interleaved in one batch: one expands_keyed and one
    multiply_keyed serve them all, each output decrypts under its own client's key, and a wrong index does not"""
    if shape == "mulpir":
        degree, t, sizes, ct_level, key_level, size = 8192, MULPIR_T, [50, 55, 55], 1, 0, 13
    else:
        degree, t, sizes, ct_level, key_level, size = 1 << 15, 65537, [62] * 14, 0, 0, 4
    n = 8
    par, sks, eks, rks, level = _clients(F, degree, t, sizes, ct_level, key_level, n, size)
    inv = pow(1 << level, -1, t)
    enc = F.Encoding.poly_at_level(ct_level)
    queries, chosen = [], []
    for c, sk in enumerate(sks):
        pt = np.zeros(degree, np.uint64)
        chosen.append(c % size)
        pt[chosen[-1]] = inv
        queries.append(sk.try_encrypt(F.PlaintextVec.try_encode(pt, enc, par), seed=bytes([c + 201]) * 32))
    Q = _merge(F, par, queries, ct_level)
    index = list(range(n))
    outs = F.expands_keyed(Q, eks, index, size)
    for i, o in enumerate(outs):
        for c in range(n):
            dec = sks[c].try_decrypt(o.take(c, 1)).try_decode(enc)
            assert int(dec[0]) == (1 if i == chosen[c] else 0) and not dec[1:].any(), (i, c)
    # products: client c multiplies its own x_c * y_c (2 ciphertexts per client)
    rng = np.random.default_rng(3)
    xs = [rng.integers(0, t, (2, degree)).astype(np.uint64) for _ in range(n)]
    ys = [rng.integers(0, t, (2, degree)).astype(np.uint64) for _ in range(n)]
    A = _merge(F, par, [sk.try_encrypt(F.PlaintextVec.try_encode(xs[c].ravel(), enc, par), seed=bytes([c + 1, 7]) * 16)
                        for c, sk in enumerate(sks)], ct_level)
    B = _merge(F, par, [sk.try_encrypt(F.PlaintextVec.try_encode(ys[c].ravel(), enc, par), seed=bytes([c + 1, 9]) * 16)
                        for c, sk in enumerate(sks)], ct_level)
    index = [j % n for j in range(2 * n)]
    prod = F.multiply_keyed(A, B, rks, index)

    def negacyclic(x, y):   # N t^2 < 2^63 at both shapes
        full = np.convolve(x.astype(np.int64), y.astype(np.int64))
        res = full[:degree].copy()
        res[:degree - 1] -= full[degree:]
        return (res % t).astype(np.uint64)
    for j in (0, 5, 2 * n - 1):
        c, r = j % n, j // n
        dec = sks[c].try_decrypt(prod.take(j, 1)).try_decode(enc)
        assert (dec == negacyclic(xs[c][r], ys[c][r])).all(), j
    wrong = F.multiply_keyed(A, B, rks, [(j + 1) % n for j in range(2 * n)])
    dec = sks[0].try_decrypt(wrong.take(0, 1)).try_decode(enc)
    assert not (dec == negacyclic(xs[0][0], ys[0][0])).all()


def test_refusals_write_nothing_and_keep_no_memory(F):
    """every error code of the keyed calls; the output words and device memory are unchanged by each refusal"""
    import torch
    from fhe_rs_b200 import _capi
    import ctypes as C
    lib = _capi.lib()
    degree, t, sizes, _, _ = CASES["n13_2x62"]
    S = Setup(F, degree, t, sizes, 0, 0, 3, 4, 1)
    other = Setup(F, degree, t, sizes, 0, 0, 1, 4, 2)   # another parameter set
    lv1 = F.KeySwitchingKey.from_arrays(S.par, *rand_rows(np.random.default_rng(1), S.moduli, (2, 1), degree), 1, 0)
    # level-1 keys at key level 0 (one RNS digit) and key level 1 (two base-2^31 digits), and a level-1 batch
    l1k0 = F.KeySwitchingKey.from_arrays(S.par, *rand_rows(np.random.default_rng(2), S.moduli, (2, 1), degree), 1, 0)
    l1k1 = F.KeySwitchingKey.from_arrays(S.par, *rand_rows(np.random.default_rng(3), S.moduli[:1], (2, 2), degree), 1, 1)
    c3_l1 = F.Ciphertext.from_host(S.par, rand_rows(np.random.default_rng(4), S.moduli[:1], (4, 3), degree), level=1)
    out_l1 = F.Ciphertext(S.par, 4, 2, 1)
    out2 = F.Ciphertext(S.par, 4, 2)
    sentinel = out2.to_host()
    out_exp = F.Ciphertext(S.par, SIZE * 4, 2)
    sentinel_exp = out_exp.to_host()
    sentinel_l1 = out_l1.to_host()

    def arr(hs):
        a = (C.c_void_p * max(1, len(hs)))(*[getattr(h, "value", h) for h in hs])
        return C.cast(a, C.POINTER(C.c_void_p))

    def ix(v):
        return (C.c_uint32 * max(1, len(v)))(*v)
    k = [x._h for x in S.ksks]
    good = ix([0, 1, 2, 0])
    cases = [
        ("null list", lambda: lib.fhe_b200_relinearize_keyed(S.C3._h, None, 3, good, out2._h, None), _capi.INVALID_ARGUMENT),
        ("no keys", lambda: lib.fhe_b200_relinearize_keyed(S.C3._h, arr(k), 0, good, out2._h, None), _capi.INVALID_ARGUMENT),
        ("null index", lambda: lib.fhe_b200_mul_relin_keyed(S.A._h, S.B._h, arr(k), 3, None, 0, out2._h, None),
         _capi.INVALID_ARGUMENT),
        ("null key", lambda: lib.fhe_b200_galois_keyed(S.A._h, 3, arr([k[0], None, k[2]]), 3, good, out2._h, None),
         _capi.INVALID_ARGUMENT),
        ("index beyond", lambda: lib.fhe_b200_mul_relin_keyed(S.A._h, S.B._h, arr(k), 3, ix([0, 1, 3, 0]), 0, out2._h,
                                                              None), _capi.INVALID_ARGUMENT),
        ("other parameters", lambda: lib.fhe_b200_galois_keyed(S.A._h, 3, arr(k + [other.ksks[0]._h]), 4, good, out2._h,
                                                              None), _capi.CONTEXT_MISMATCH),
        ("other level", lambda: lib.fhe_b200_relinearize_keyed(S.C3._h, arr(k + [lv1._h]), 4, good, out2._h, None),
         _capi.INVALID_LEVEL),
        ("key levels differ", lambda: lib.fhe_b200_relinearize_keyed(c3_l1._h, arr([l1k0._h, l1k1._h]), 2,
                                                                     ix([0, 1, 0, 1]), out_l1._h, None),
         _capi.INVALID_ARGUMENT),
        ("key switch output level", lambda: lib.fhe_b200_key_switch_keyed(S.P._h, 1, arr(k), 3, good, out_l1._h, None),
         _capi.INVALID_LEVEL),
        ("batch shape", lambda: lib.fhe_b200_relinearize_keyed(S.A._h, arr(k), 3, good, out2._h, None),
         _capi.BAD_POLY_COUNT),
        ("representation", lambda: lib.fhe_b200_galois_keyed(S.P._h, 3, arr(k), 3, good, out2._h, None),
         _capi.INVALID_REPRESENTATION),
        ("even exponent", lambda: lib.fhe_b200_galois_keyed(S.A._h, 4, arr(k), 3, good, out2._h, None),
         _capi.INVALID_EXPONENT),
        ("mod-switch output level", lambda: lib.fhe_b200_mul_relin_keyed(S.A._h, S.B._h, arr(k), 3, good, 1, out2._h, None),
         _capi.INVALID_LEVEL),
        ("expand n_gks", lambda: lib.fhe_b200_expand_keyed(S.A._h, SIZE, arr(k), 1, 3, good, out_exp._h, None),
         _capi.INVALID_ARGUMENT),
        ("expand no sets", lambda: lib.fhe_b200_expand_keyed(S.A._h, SIZE, arr(k + k), 2, 0, good, out_exp._h, None),
         _capi.INVALID_ARGUMENT),
        ("expand null index", lambda: lib.fhe_b200_expand_keyed(S.A._h, SIZE, arr(k + k), 2, 3, None, out_exp._h, None),
         _capi.INVALID_ARGUMENT),
        ("expand set beyond", lambda: lib.fhe_b200_expand_keyed(S.A._h, SIZE, arr(k + k), 2, 3, ix([0, 3, 0, 0]),
                                                                out_exp._h, None), _capi.INVALID_ARGUMENT),
        ("expand null key", lambda: lib.fhe_b200_expand_keyed(S.A._h, SIZE, arr([k[0], None, k[1], k[2]]), 2, 2,
                                                              ix([0, 1, 0, 1]), out_exp._h, None),
         _capi.INVALID_ARGUMENT),
        ("expand size", lambda: lib.fhe_b200_expand_keyed(S.A._h, 0, arr(k + k), 2, 3, good, out_exp._h, None),
         _capi.INVALID_ARGUMENT),
        ("key switch part", lambda: lib.fhe_b200_key_switch_keyed(S.P._h, 2, arr(k), 3, good, out2._h, None),
         _capi.BAD_POLY_COUNT),
    ]
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    for what, call, code in cases:
        got = call()
        assert got == code, (what, got, lib.fhe_b200_last_error())
    torch.cuda.synchronize()
    assert abs(torch.cuda.mem_get_info()[0] - free0) < 4 << 20
    assert (out2.to_host() == sentinel).all() and (out_exp.to_host() == sentinel_exp).all()
    assert (out_l1.to_host() == sentinel_l1).all()


def test_external_products_keyed(F):
    degree, t, sizes, _, _ = CASES["n13_2x62"]
    S = Setup(F, degree, t, sizes, 0, 0, 3, 5, 4)
    rg = [F.RGSWCiphertext(S.ksks[k], S.ksks[(k + 1) % 3]) for k in range(3)]
    index = [2, 2, 0, 1, 0]
    got = F.external_products_keyed(S.A, rg, index).to_host()
    for j in range(5):
        assert (got[j] == rg[index[j]].external_product(S.A.take(j, 1)).to_host()[0]).all(), j


def test_cpp_mirror(F, tmp_path):
    """the C++ mirror's keyed calls give the Python mirror's words"""
    degree, t, sizes = 1 << 13, 1153, [62, 62]
    S = Setup(F, degree, t, sizes, 0, 0, 3, 6, 8)
    index = [2, 0, 0, 1, 2, 1]
    lines = ["%d %d %d %d %d" % (degree, t, len(S.moduli), 6, 3), " ".join(map(str, S.moduli)),
             " ".join(map(str, index))]
    for k, ksk in enumerate(S.ksks):
        c0, c1 = ksk.arrays()
        c0.tofile(str(tmp_path / ("k%d_c0.bin" % k)))
        c1.tofile(str(tmp_path / ("k%d_c1.bin" % k)))
    (tmp_path / "args.txt").write_text("\n".join(lines) + "\n")
    S.A.to_host().tofile(str(tmp_path / "a.bin"))
    S.B.to_host().tofile(str(tmp_path / "b.bin"))
    exe = str(tmp_path / "keyed_test")
    lib_dir = os.path.join(ROOT, "fhe_rs_b200")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "cpp", "keyed_test.cpp"), "-o", exe,
                           "-L", lib_dir, "-lfhe_b200", "-Wl,-rpath," + lib_dir])
    out = subprocess.run([exe, str(tmp_path)], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0 and out.stdout.startswith("OK"), out.stdout + out.stderr
    rg = [F.RGSWCiphertext(k, k) for k in S.ksks]
    want = {"mul": S.keyed("mul", index).to_host(), "relin": S.keyed("relin", index).to_host(),
            "galois": S.keyed("galois", index).to_host(), "ks": S.keyed("ks", index).to_host(),
            "ext": F.external_products_keyed(S.A, rg, index).to_host(), "expand": S.keyed("expand", index).to_host()}
    for name, w in want.items():
        assert (np.fromfile(str(tmp_path / ("out_%s.bin" % name)), np.uint64) == w.ravel()).all(), name


SWITCHES = {"tma": {"FHE_B200_KSMAC": "tma"}, "classic": {"FHE_B200_KSMAC": "classic"},
            "stages3_cols2": {"FHE_B200_KS_STAGES": "3", "FHE_B200_TMA_COLS": "2"},
            "chunk1": {"FHE_B200_CHUNK": "1"}, "streams1": {"FHE_B200_STREAMS": "1"},
            "streams4": {"FHE_B200_STREAMS": "4"}}


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
