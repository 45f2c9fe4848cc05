"""The server's batched calls at their edges, device against the CPU oracle word for word: hoisted rotations
(fhe_b200_galois_many_hoisted, and galois_many beside it), linear transforms (fhe_b200_linear_transform, fused and
unfused), ciphertext dot products (fhe_b200_dot_product, _keyed), per-client products (fhe_b200_mul_relin_keyed) and
the inner sum (fhe_b200_inner_sum, _keyed), at
  (a) the boundary primes: each as q_0, all three after a generated prime, and an all-Barrett basis;
  (b) the lazy-bound bases, with all-(q - 1) digits under, at and near 8x the reduce-on-load bound, through both the
      hoisted digits (c1 all q - 1) and the reference's (sigma_e(c1) all q - 1, pre-substituted);
  (c) the modulus-width sweep at level 0, a middle level (keys at the ciphertext level and leveled keys) and the
      single-modulus last level (base-2^b keys, which are never hoisted);
  (d) 31 moduli at N = 2^13 and N = 2^16, with crafted zeros in the last limb, at s = N - 1 and where s e >= 2^32;
  (e) the large plaintext moduli of tests/bigt_reference.py at every level, Q_l < t included;
with random and all-(q - 1) keys and ciphertexts.  tests/test_server_edges_cpu.py shows the crafted inputs reach the
decisions they target.

What each check compares with:
  * rotations: GaloisKey.relinearize of the oracle for every output of a crafted or oracle-sized batch; in the larger
    batches, for source 0 (and the sources that repeat it word for word), the other outputs against galois_many;
  * n_hoisted and n_fallback: the CPU zero predicate (hoisting_reference.hoisted_count / needs_fallback), 0 and
    count * (b - 1) with base-2^b or leveled keys;
  * linear transforms: linear_transform_reference.linear_transform on the oracle for one or two ciphertexts (every
    ciphertext when a batch repeats one), the other ciphertexts against test_gpu_linear_transform's composition;
  * dot products and per-client products: the oracle's loop of mul, add, relinearizes and switch_to_level (and
    Multiplicator.default), every group; where a batch repeats one group, that group's oracle result;
  * inner sums: oracle.computes_inner_sum for every ciphertext;
  * large t: the same loop, and on one set decryption with bigt_reference's client to sum_i m_i * m'_i mod t.
test_switch_reruns reruns a subset under the transform, key-switch, arithmetic and chunking switches.  Run with
`-m gpu`."""
import os
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TESTS = os.path.join(ROOT, "tests")
for p in (ROOT, TESTS, os.path.join(ROOT, "oracle")):
    if p not in sys.path:
        sys.path.insert(0, p)

import bigt_reference as BR   # noqa: E402
import edge_inputs as E   # noqa: E402
import hoisting_reference as H   # noqa: E402
import linear_transform_reference as LR   # noqa: E402
from test_gpu_linear_transform import composition   # noqa: E402
from test_gpu_rotations import inner_sum_exponents   # noqa: E402
from test_server_edges_cpu import boundary_bases, crafted_c1, presubstituted_max, wide_exponents   # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def F():
    from conftest import has_gpu
    if not has_gpu():
        pytest.skip("no CUDA device")
    import fhe_rs_b200
    return fhe_rs_b200


def rand_rows(rng, moduli, prefix, degree):
    a = np.zeros(tuple(prefix) + (len(moduli), degree), np.uint64)
    for i, q in enumerate(moduli):
        a[..., i, :] = rng.integers(0, q, size=tuple(prefix) + (degree,), dtype=np.uint64)
    return a


def max_rows(moduli, prefix, degree):
    q = np.array(moduli, np.uint64)[:, None] - np.uint64(1)
    return np.ascontiguousarray(np.broadcast_to(q, tuple(prefix) + (len(moduli), degree)))


class Case:
    """one basis on the oracle and on the device, and keys and ciphertexts built from the same words on both"""

    def __init__(self, oracle, F, degree, t, moduli, seed=1):
        self.O, self.F, self.N = oracle, F, degree
        self.opar = oracle.BfvParameters(degree, t, moduli=moduli)
        self.gpar = F.BfvParameters(degree, t, moduli=self.opar.moduli, device=0)
        self.moduli = [int(q) for q in self.opar.moduli]
        self.rng = np.random.default_rng(seed)

    def mods(self, level):
        return self.moduli[:len(self.moduli) - level]

    def key_words(self, level, key_level, kind):
        """[2][digits][key limbs][N]: base-2^b digits when the key level has one modulus"""
        km = self.mods(key_level)
        if len(km) == 1:
            lq = (km[0] - 1).bit_length()
            n_dig = -(-lq // (lq // 2))
        else:
            n_dig = len(self.mods(level))
        if kind == "max":
            return max_rows(km, (2, n_dig), self.N).copy()
        return rand_rows(self.rng, km, (2, n_dig), self.N)

    def galois(self, e, level, key_level, kind):
        """(device GaloisKey, oracle GaloisKey) of exponent e (the device's unreduced)"""
        c = self.key_words(level, key_level, kind)
        g = self.F.GaloisKey(e, self.F.KeySwitchingKey.from_arrays(self.gpar, c[0], c[1], level, key_level))
        o = self.O.GaloisKey.__new__(self.O.GaloisKey)
        o.exponent = e % (2 * self.N)
        o.ksk = self.O.KeySwitchingKey.from_arrays(self.opar, c[0], c[1], level, key_level)
        return g, o

    def relin(self, level, key_level, kind):
        c = self.key_words(level, key_level, kind)
        g = self.F.RelinearizationKey.from_arrays(self.gpar, c[0], c[1], ciphertext_level=level, key_level=key_level)
        return g, self.O.RelinearizationKey.from_ksk(self.O.KeySwitchingKey.from_arrays(self.opar, c[0], c[1], level,
                                                                                          key_level))

    def ntt(self, level, rows):
        return self.O.Poly(self.opar.context_at_level(level), self.O.POWER_BASIS, rows.copy()).into_ntt().c

    def cts(self, level, c1_power, c0=None):
        """[count][2][L][N] NTT words with the given power-basis c1 rows [count][L][N] (random c0 by default)"""
        count = len(c1_power)
        c0 = rand_rows(self.rng, self.mods(level), (count,), self.N) if c0 is None else c0
        c1 = np.stack([self.ntt(level, r) for r in c1_power])
        return np.ascontiguousarray(np.stack([c0, c1], axis=1))

    def batch(self, words, level):
        return self.F.Ciphertext.from_host(self.gpar, words, level=level)

    def octs(self, words, level):
        return [self.O.Ciphertext.from_array(self.opar, w.copy(), level) for w in words]


# ------------------------------------------------------------------------------------------------------ checks

def check_hoisted(C, words, c1_power, level, keys, index, source, oracle_sources):
    """galois_many_hoisted: every output against galois_many, the outputs of oracle_sources against the oracle, and
    n_hoisted against the CPU predicate (0 with base-2^b keys)"""
    F = C.F
    A = C.batch(words, level)
    gks = [g for g, _ in keys]
    got, nh = F.galois_many_hoisted(A, gks, index, source)
    got = got.to_host()
    many = F.galois_many(A, gks, index, source).to_host()
    octs = C.octs(words, level)
    for j, (k, s) in enumerate(zip(index, source)):
        assert (got[j] == many[j]).all(), ("galois_many", j)
        if s in oracle_sources:
            assert (got[j] == keys[k][1].relinearize(octs[s]).to_array()).all(), ("oracle", j)
    exps = [keys[k][1].exponent for k in index]
    single = keys[0][1].ksk.log_base != 0
    expected = 0 if single else H.hoisted_count(list(c1_power), exps, source)
    assert nh == expected, (nh, expected)
    return nh


def check_lt(C, words, c1_power, level, keys, n, baby, oracle_cts, fused):
    """linear_transform of shared random diagonals: the oracle restatement for oracle_cts, the device composition
    for the others, and n_fallback against the CPU predicate (count * (b - 1) on the unfused route)"""
    F, O = C.F, C.O
    A = C.batch(words, level)
    steps = LR.steps(n, baby)
    step_key = dict(zip(steps, keys))
    diags = rand_rows(C.rng, C.mods(level), (n, 1), C.N)
    D = C.batch(diags, level)
    got, nf = F.linear_transform(A, D, baby, [g for g, _ in keys], n)
    got = got.to_host()
    ctx = C.opar.context_at_level(level)
    od = [O.Poly(ctx, O.NTT, d[0].copy()) for d in diags]
    octs = C.octs(words, level)
    rest = [c for c in range(len(words)) if c not in oracle_cts]
    want = composition(F, A, D, n, baby, {s: g for s, (g, _) in step_key.items()}, False) if rest else None
    for c in range(len(words)):
        if c in oracle_cts:
            exp = LR.linear_transform(octs[c], od, baby, {s: o for s, (_, o) in step_key.items()}).to_array()
        else:
            exp = want[c]
        assert (got[c] == exp).all(), ("linear transform", c, n, baby)
    if fused:
        expected = sum(1 for c in range(len(words)) for i in range(1, baby)
                       if H.needs_fallback(c1_power[c], pow(3, i, 2 * C.N)))
    else:
        expected = len(words) * (baby - 1)
    assert nf == expected, (nf, expected)
    return nf


def oracle_sums(C, a, b, level, n_terms, groups):
    """the 3-part sum_i a_i * b_i of each group on the oracle"""
    oa, ob = C.octs(a, level), C.octs(b, level)
    out = []
    for g in range(groups):
        acc = None
        for i in range(g * n_terms, (g + 1) * n_terms):
            p = oa[i].mul(ob[i])
            acc = p if acc is None else acc.add(p)
        out.append(acc)
    return out


def check_dot(C, level, key_level, kind, n_terms, groups, out_levels, operands="random"):
    """dot_product without a key and with one, and dot_product_keyed with one key per group, switched to each of
    out_levels, against the oracle's loop for every group"""
    F = C.F
    mods = C.mods(level)
    if operands == "max":
        a = b = max_rows(mods, (groups * n_terms, 2), C.N).copy()
    else:
        a, b = rand_rows(C.rng, mods, (groups * n_terms, 2), C.N), rand_rows(C.rng, mods, (groups * n_terms, 2), C.N)
    A, B = C.batch(a, level), C.batch(b, level)
    sums = oracle_sums(C, a, b, level, n_terms, groups)
    rks = [C.relin(level, key_level, kind) for _ in range(groups)]
    index = [(g + 1) % groups for g in range(groups)]
    for out_level in out_levels:
        got = F.dot_product(A, B, n_terms, None, level=out_level).to_host()
        one = F.dot_product(A, B, n_terms, rks[0][0], level=out_level).to_host()
        keyed = F.dot_product_keyed(A, B, n_terms, [g for g, _ in rks], index, level=out_level).to_host()
        for g in range(groups):
            assert (got[g] == sums[g].copy().switch_to_level(out_level).to_array()).all(), ("no key", g, out_level)
            exp = rks[0][1].relinearizes(sums[g]).switch_to_level(out_level).to_array()
            assert (one[g] == exp).all(), ("key", g, out_level)
            exp = rks[index[g]][1].relinearizes(sums[g]).switch_to_level(out_level).to_array()
            assert (keyed[g] == exp).all(), ("keyed", g, out_level)


def check_inner_sum(C, words, level, key_level, kind, n_clients):
    """computes_inner_sum_keyed with n_clients key sets (fhe_b200_inner_sum for one), every ciphertext against
    oracle.computes_inner_sum with its set"""
    F, O = C.F, C.O
    eks, oks = [], []
    for _ in range(n_clients):
        ek = F.EvaluationKey(C.gpar, level, key_level)
        ok = {}
        for e in inner_sum_exponents(C.N):
            g, o = C.galois(e, level, key_level, kind)
            ek.add_galois_key(g)
            ok[o.exponent] = o
        eks.append(ek)
        oks.append(ok)
    index = [(c + 1) % n_clients for c in range(len(words))]
    got = F.computes_inner_sum_keyed(C.batch(words, level), eks, index).to_host()
    for c, oct_ in enumerate(C.octs(words, level)):
        assert (got[c] == O.computes_inner_sum(C.opar, oks[index[c]], oct_).to_array()).all(), ("inner sum", c)


def all_pairs(n_src, n_exp):
    """source-major outputs: every source by every key"""
    return [k for _ in range(n_src) for k in range(n_exp)], [s for s in range(n_src) for _ in range(n_exp)]


# ----------------------------------------------------------------------------------------------- (a) boundary

@pytest.mark.parametrize("name", ["q0_solinas_max_c", "q0_non_solinas_min", "q0_above_2_61", "after_gen62",
                                  "all_barrett"])
def test_boundary_primes(oracle, F, name):
    """N = 2^13 over each boundary basis, random and all-(q - 1) keys, random and all-(q - 1) c1: 3 sources x 3
    exponents hoisted, a fused linear transform (n = 7, b = 3: G = 3), a dot product (2 groups of 3 terms) switched to
    the last level, and the inner sum of two ciphertexts.  All-(q - 1) c1 has no zero: every candidate is hoisted and
    nothing falls back, so the hoisted kernels computed those words."""
    degree = 1 << 13
    C = Case(oracle, F, degree, 786433, boundary_bases(degree)[name], seed=len(name))
    L = len(C.moduli)
    exps = [3, 2 * degree - 1, pow(3, 7, 2 * degree)]
    for key_kind in ("random", "max"):
        for c1_kind in ("random", "max"):
            if c1_kind == "max":   # three copies of one ciphertext: every output against the oracle
                one = C.cts(0, max_rows(C.moduli, (1,), degree))
                words, c1 = np.concatenate([one] * 3), max_rows(C.moduli, (3,), degree)
            else:
                c1 = rand_rows(C.rng, C.moduli, (3,), degree)
                words = C.cts(0, c1)
            keys = [C.galois(e, 0, 0, key_kind) for e in exps]
            index, source = all_pairs(3, 3)
            nh = check_hoisted(C, words, c1, 0, keys, index, source, {0, 1, 2} if c1_kind == "max" else {0})
            if c1_kind == "max":
                assert nh == 9
            steps = LR.steps(7, 3)
            lt_keys = [C.galois(pow(3, s, 2 * degree), 0, 0, key_kind) for s in steps]
            nf = check_lt(C, words, c1, 0, lt_keys, 7, 3, {0, 1, 2} if c1_kind == "max" else {0}, fused=True)
            if c1_kind == "max":
                assert nf == 0
            check_dot(C, 0, 0, key_kind, 3, 2, [0, L - 1], operands=c1_kind)
            if c1_kind == key_kind:
                check_inner_sum(C, words[:2], 0, 0, key_kind, 1)


# --------------------------------------------------------------------------------------------- (b) lazy bound

@pytest.mark.parametrize("base", ["unreduced", "reduced", "reduced_8x"])
def test_lazy_bound(oracle, F, base):
    """N = 2^13, tests/edge_inputs.lazy_bound_bases: 8 ciphertexts (24 digit rows per limb: the TMA digit transform),
    four with c1 all q - 1 (the hoisted digits at the bound) and four with sigma_3(c1) all q - 1 (the reference's
    digits at the bound), c0 all q - 1; rotations by 3 and by 9, 27 and 2N - 1 from every source, and a fused linear
    transform (n = 8, b = 4) whose baby steps include 3, with all-(q - 1) and random keys, every output against the
    oracle (the four copies of each kind against one oracle result)"""
    degree = 1 << 13
    C = Case(oracle, F, degree, 786433, E.lazy_bound_bases(degree)[base], seed=13)
    ctx = C.opar.context_at_level(0)
    mx = max_rows(C.moduli, (), degree).copy()
    c1 = np.stack([mx] * 4 + [presubstituted_max(oracle, ctx, 3)] * 4)
    words = C.cts(0, c1, c0=np.stack([mx] * 8))
    exps = [3, 9, 27, 2 * degree - 1]
    for kind in ("max", "random"):
        keys = [C.galois(e, 0, 0, kind) for e in exps]
        index, source = all_pairs(8, 4)
        octs = C.octs(words[[0, 4]], 0)
        got, nh = F.galois_many_hoisted(C.batch(words, 0), [g for g, _ in keys], index, source)
        assert nh == 32
        got = got.to_host()
        want = {(s, k): keys[k][1].relinearize(octs[s]).to_array() for s in range(2) for k in range(4)}
        for j, (k, s) in enumerate(zip(index, source)):
            assert (got[j] == want[(s // 4, k)]).all(), (base, kind, j)
        lt_keys = [C.galois(pow(3, s, 2 * degree), 0, 0, kind) for s in LR.steps(8, 4)]
        assert check_lt(C, words, c1, 0, lt_keys, 8, 4, set(range(8)), fused=True) == 0


# -------------------------------------------------------------------------------------------- (c) width sweep

@pytest.mark.parametrize("name", list(E.WIDTH_SETS))
def test_width_sweep(oracle, F, name):
    """tests/edge_inputs.WIDTH_SETS at level 0 and the middle level, with keys at the ciphertext level and (middle
    level) level-0 keys: galois_many and galois_many_hoisted (2 sources x 3 exponents), the linear transform (n = 7,
    b = 3; fused with keys at the ciphertext level, unfused with leveled keys), dot_product and dot_product_keyed
    switched to every lower level, and the keyed inner sum of two clients.  At the single-modulus last level the same
    calls with base-2^b keys: nothing hoisted, every baby step falls back."""
    degree, t, sizes = E.WIDTH_SETS[name]
    C = Case(oracle, F, degree, t, oracle.BfvParameters.generate_moduli(sizes, degree), seed=degree + sizes[0])
    L = len(C.moduli)
    exps = [3, 2 * degree - 1, degree + 1]
    for level in (0, L // 2, L - 1):
        for key_level in sorted({level, 0}) if level < L - 1 else [level]:
            mods = C.mods(level)
            c1 = rand_rows(C.rng, mods, (2,), degree)
            words = C.cts(level, c1)
            keys = [C.galois(e, level, key_level, "random") for e in exps]
            index, source = all_pairs(2, 3)
            nh = check_hoisted(C, words, c1, level, keys, index, source, {0, 1})
            assert (nh == 0) == (level == L - 1), nh
            lt_keys = [C.galois(pow(3, s, 2 * degree), level, key_level, "random") for s in LR.steps(7, 3)]
            fused = key_level == level and level < L - 1
            nf = check_lt(C, words, c1, level, lt_keys, 7, 3, {0, 1}, fused=fused)
            if not fused:
                assert nf == 2 * 2
            check_dot(C, level, key_level, "random", 2, 2, list(range(level, L)))
            if key_level == level:
                check_inner_sum(C, words, level, key_level, "random", 2)


# ---------------------------------------------------------------------------------------- (d) largest shapes

@pytest.mark.parametrize("name", ["l31", "n2_16"])
def test_largest_shapes(oracle, F, name):
    """31 moduli at N = 2^13 and 3 at N = 2^16 (tests/edge_inputs.CLIENT_SHAPES), with the crafted zeros of
    test_server_edges_cpu.crafted_c1 (one zero per source in the last limb: at s = N - 1, at a position the first
    exponent negates and at one it keeps, at N = 2^16 where s e >= 2^32): hoisted rotations of 3 sources by an
    exponent >= 2^16 (N = 2^16) or >= 3N/2, 2N - 1 and 2^17 + 5, n_hoisted equal to the predicate's 4; a linear
    transform (n = 8, b = 3) whose step 1 falls back for one ciphertext; a dot product of 3 terms switched one level
    down; at N = 2^16 the inner sum.  Every word against the oracle."""
    degree, _ = E.CLIENT_SHAPES[name]
    C = Case(oracle, F, degree, 786433, E.client_moduli(name), seed=degree)
    exps = wide_exponents(degree)
    c1, _ = crafted_c1(C.moduli, degree, exps, 3)
    words = C.cts(0, c1)
    keys = [C.galois(e, 0, 0, "random") for e in exps]
    index, source = all_pairs(3, 3)
    assert check_hoisted(C, words, c1, 0, keys, index, source, {0, 1, 2}) == 4
    c1, _ = crafted_c1(C.moduli, degree, [3, 9], 4)
    words = C.cts(0, c1)
    lt_keys = [C.galois(pow(3, s, 2 * degree), 0, 0, "random") for s in LR.steps(8, 3)]
    assert check_lt(C, words, c1, 0, lt_keys, 8, 3, {0, 1, 2}, fused=True) == 1
    check_dot(C, 0, 0, "random", 3, 1, [1])
    if degree == 1 << 16:
        check_inner_sum(C, words[:1], 0, 0, "random", 1)


# ------------------------------------------------------------------------------------------------- (e) large t

def bigt_levels(name, n_moduli):
    return [1, n_moduli - 1] if name == "set_c_near_q" else list(range(n_moduli))


@pytest.mark.parametrize("name", list(BR.BIGT_SETS))
def test_large_t(oracle, F, name):
    """tests/bigt_reference.BIGT_SETS at every level (set C: levels 1 and the last), the levels with Q_l < t
    included: dot_product of 3 groups x 2 terms (the groups repeat one) without a key and with one at the ciphertext
    level (base-2^b at a single modulus), dot_product_keyed with 3 clients' keys, and mul_relin_keyed of 3 pairs
    with 3 clients' keys (with modulus switching below the last level), against the oracle"""
    degree, t, moduli = BR.bigt_set(name)
    C = Case(oracle, F, degree, t, moduli, seed=len(name))
    L0 = len(C.moduli)
    assert BR.levels_t_above_q(t, C.moduli)
    for level in bigt_levels(name, L0):
        mods = C.mods(level)
        a1, b1 = rand_rows(C.rng, mods, (2, 2), degree), rand_rows(C.rng, mods, (2, 2), degree)
        a, b = np.concatenate([a1] * 3), np.concatenate([b1] * 3)
        A, B = C.batch(a, level), C.batch(b, level)
        s = oracle_sums(C, a1, b1, level, 2, 1)[0]
        rks = [C.relin(level, level, "random") for _ in range(3)]
        index = [2, 0, 1]
        got = F.dot_product(A, B, 2, None).to_host()
        one = F.dot_product(A, B, 2, rks[0][0]).to_host()
        keyed = F.dot_product_keyed(A, B, 2, [g for g, _ in rks], index).to_host()
        for g in range(3):
            assert (got[g] == s.to_array()).all(), (name, level, "no key", g)
            assert (one[g] == rks[0][1].relinearizes(s).to_array()).all(), (name, level, "key", g)
            assert (keyed[g] == rks[index[g]][1].relinearizes(s).to_array()).all(), (name, level, "keyed", g)
        if len(mods) == 1:   # Multiplicator.default takes no base-2^b key
            continue
        ms = level < L0 - 1
        prod = F.multiply_keyed(C.batch(np.stack([a1[0]] * 3), level), C.batch(np.stack([b1[0]] * 3), level),
                                [g for g, _ in rks], index, mod_switch=ms).to_host()
        oa, ob = C.octs(a1[:1], level)[0], C.octs(b1[:1], level)[0]
        for g in range(3):
            om = oracle.Multiplicator.default(rks[index[g]][1])
            if ms:
                om.enable_mod_switching()
            assert (prod[g] == om.multiply(oa, ob).to_array()).all(), (name, level, "mul_relin_keyed", g)


def test_large_t_dot_product_decrypts(oracle, F):
    """t = 2^127 - 1 (biguint.rs): ciphertexts the big-integer client encrypted, a dot product of 3 terms with a real
    relinearization key decrypts to sum_i m_i * m'_i mod t, as do both groups of the keyed call with the same key and
    the 3-part sum without one"""
    degree, t, moduli = BR.bigt_set("m127")
    opar = oracle.BfvParameters(degree, t, moduli=moduli)
    gpar = F.BfvParameters(degree, t, moduli=moduli, device=0)
    rng = np.random.default_rng(127)
    sk = oracle.SecretKey(opar, rng)
    ork = oracle.RelinearizationKey(sk, rng)
    grk = F.RelinearizationKey.from_arrays(gpar, *ork.ksk.arrays())
    msgs = [([int(rng.integers(0, 1 << 62)) * t >> 62 for _ in range(degree)],
             [int(rng.integers(0, 1 << 62)) * t >> 62 for _ in range(degree)]) for _ in range(3)]
    msgs[0] = ([10] + [0] * (degree - 1), [t - 20] + [0] * (degree - 1))
    cts = [(BR.encrypt(sk, BR.encode(opar, x), 0, rng), BR.encrypt(sk, BR.encode(opar, y), 0, rng)) for x, y in msgs]
    A = F.Ciphertext.from_host(gpar, np.stack([x.to_array() for x, _ in cts] * 2))
    B = F.Ciphertext.from_host(gpar, np.stack([y.to_array() for _, y in cts] * 2))
    want = [sum(v) % t for v in zip(*[BR.negacyclic(x, y, t) for x, y in msgs])]
    outs = {"relinearized": F.dot_product(A, B, 3, grk).to_host(), "keyed": F.dot_product_keyed(A, B, 3, [grk], [0, 0]).to_host(),
            "3 parts": F.dot_product(A, B, 3).to_host()}
    for what, got in outs.items():
        for g in range(2):
            dec = BR.decode(opar, BR.decrypt(sk, oracle.Ciphertext.from_array(opar, got[g], 0)))
            assert dec == want, (what, g)


# -------------------------------------------------------------------------------------------- (f) switch reruns

SWITCHES = {"no_solinas": {"FHE_B200_NO_SOLINAS": "1"}, "ntt_fast": {"FHE_B200_NTT": "fast"},
            "ntt_tma": {"FHE_B200_NTT": "tma"}, "ksmac_tma": {"FHE_B200_KSMAC": "tma"},
            "ksmac_classic": {"FHE_B200_KSMAC": "classic"},
            "chunk3_streams1": {"FHE_B200_CHUNK": "3", "FHE_B200_STREAMS": "1"},
            "chunk3_streams4": {"FHE_B200_CHUNK": "3", "FHE_B200_STREAMS": "4"}}
QUICK = ("test_boundary_primes and (non_solinas or all_barrett) or test_lazy_bound or "
         "test_width_sweep and (n64_up_10 or n2_13) or test_largest_shapes or test_large_t and (m127 or tma_200)")


def test_switch_reruns(F):
    """a subset of this module -- two boundary bases, the lazy-bound bases, two width sets, the largest shapes and
    two large-t sets -- under each switch, one process per switch (the switches are read once per process), side by
    side"""
    cmd = [sys.executable, "-m", "pytest", "-q", "-x", "-m", "gpu", "tests/test_gpu_server_edges.py",
           "-p", "no:cacheprovider", "-k", "(%s) and not test_switch_reruns" % QUICK]
    runs = [(name, subprocess.Popen(cmd, cwd=ROOT, env=dict(os.environ, **env), stdout=subprocess.PIPE,
                                    stderr=subprocess.STDOUT, text=True)) for name, env in SWITCHES.items()]
    failed = {}
    try:
        for name, p in runs:
            out = p.communicate(timeout=1800)[0]
            if p.returncode != 0:
                failed[name] = out[-3000:]
    finally:   # a timeout leaves no process behind
        for _, p in runs:
            if p.poll() is None:
                p.kill()
                p.wait()
    assert not failed, failed
