"""Pins the CPU oracle (oracle/fhe_oracle.{c,py}) against every known-answer
vector and property oracle the reference's own tests hold for the hot path
(SURVEY.md section 8c).  CPU only."""
import random

import numpy as np
import pytest

NFL_62 = [
    4611686018326724609, 4611686018309947393, 4611686018282684417, 4611686018257518593,
    4611686018232352769, 4611686018171535361, 4611686018106523649, 4611686018058289153,
    4611686018051997697, 4611686017974403073, 4611686017812922369, 4611686017781465089,
    4611686017773076481, 4611686017678704641, 4611686017666121729, 4611686017647247361,
    4611686017590624257, 4611686017554972673, 4611686017529806849, 4611686017517223937]

# SURVEY.md section 8: moduli of the three BASELINE.json parameter sets
SET_C_Q = [4611686018427322369, 4611686018425815041, 4611686018423390209, 4611686018423062529,
           4611686018422669313, 4611686018421293057, 4611686018418147329, 4611686018416115713,
           4611686018413166593, 4611686018408316929, 4611686018408120321, 4611686018407661569,
           4611686018407137281, 4611686018406940673]
SET_A_Q = [4611686018427322369, 4611686018427289601]
SET_A_EXT = [4611686018427215873, 4611686018427199489, 4611686018426953729]


def test_nfl_62bit_primes(oracle):
    """zq/primes.rs:68-101"""
    out, ub = [], (2**64 - 1) >> 2
    while len(out) != 20:
        ub = oracle.generate_prime(62, 2 * 1048576, ub)
        assert ub is not None
        out.append(ub)
    assert out == NFL_62


def test_ciphertext_moduli_kat(oracle):
    """bfv/parameters.rs:846-856"""
    assert oracle.BfvParameters.generate_moduli([62, 62, 62, 61, 60, 11], 16) == [
        4611686018427387617, 4611686018427387329, 4611686018427387073,
        2305843009213693921, 1152921504606845473, 2017]


def test_baseline_parameter_sets(oracle):
    assert oracle.BfvParameters.generate_moduli([62] * 14, 1 << 15) == SET_C_Q
    par = oracle.BfvParameters(1 << 12, 1032193, moduli_sizes=[62, 62])
    assert par.moduli == SET_A_Q
    assert par.extended_basis == SET_A_EXT
    assert all(oracle.supports_opt(q) for q in SET_C_Q)


def test_is_prime_kats(oracle):
    """fhe-util/src/lib.rs:252-267 style"""
    assert oracle.is_prime(2) and oracle.is_prime(3) and oracle.is_prime(4611686018326724609)
    assert not oracle.is_prime(0) and not oracle.is_prime(1) and not oracle.is_prime(4611686018326724607)


def test_rns_project_lift(oracle):
    """rns/mod.rs:212-249"""
    rns = oracle.RnsContext([4, 15, 1153])
    prod = 4 * 15 * 1153
    assert rns.product == prod
    for a, r in [(0, [0, 0, 0]), (4, [0, 4, 4]), (15, [3, 0, 15]), (1153, [1, 13, 0]),
                 (prod - 1, [3, 14, 1152])]:
        assert rns.project(a) == r
        assert rns.lift(r) == a
    with pytest.raises(ValueError):
        oracle.RnsContext([4, 4])


def test_zq_ops_against_bigint(oracle):
    """zq/mod.rs:842-1068: every modular op equals the exact integer formula."""
    rnd = random.Random(7)
    for p in [2, 3, 1153, 4611686018326724609, 4611686018427387903, (1 << 48) + 21 * (1 << 15) + 1]:
        m = oracle.Modulus(p)
        L = oracle.lib()
        for _ in range(300):
            a, b = rnd.randrange(p), rnd.randrange(p)
            assert L.orc_zq_mul(m.ref(), a, b) == a * b % p
            if m.supports_opt:
                assert L.orc_zq_mul_opt(m.ref(), a, b) == a * b % p
            bs = L.orc_zq_shoup(m.ref(), b)
            assert bs == (b << 64) // p
            x = rnd.randrange(1 << 64)  # lazy input
            assert L.orc_zq_mul_shoup(m.ref(), x, b, bs) == x * b % p
            r = L.orc_zq_lazy_mul_shoup(m.ref(), x, b, bs)
            assert r < 2 * p and r % p == x * b % p
            assert L.orc_zq_reduce(m.ref(), x) == x % p
            hi = rnd.randrange(1 << 64)
            assert L.orc_zq_reduce_u128(m.ref(), x, hi) == ((hi << 64) | x) % p
            e = rnd.randrange(p)
            assert L.orc_zq_pow(m.ref(), a, e) == pow(a, e, p)


def test_supports_opt_rule(oracle):
    """zq/primes.rs:10-24"""
    assert oracle.supports_opt(4611686018326724609)
    assert not oracle.supports_opt((1 << 63) + 1)
    assert not oracle.supports_opt(1153)


@pytest.mark.parametrize("n,p", [(8, 1153), (16, 4611686018427387617), (32, 4611686018326724609),
                                 (1024, 4611686018326724609)])
def test_ntt_is_negacyclic_evaluation(oracle, n, p):
    """ntt/mod.rs:50-82 + SURVEY appendix A-1: forward(a)[i] = a(psi^(2*bitrev(i)+1)),
    backward(forward(a)) == a, lazy forward < 4p and congruent."""
    rnd = np.random.default_rng(n)
    op = oracle.NttOperator(oracle.Modulus(p), n)
    a = rnd.integers(0, p, size=n, dtype=np.uint64)
    f = a.copy()
    op.forward(f)
    logn = n.bit_length() - 1
    if n <= 32:
        for i in range(n):
            x = pow(op.psi, 2 * oracle.bitrev(i, logn) + 1, p)
            assert int(f[i]) == sum(int(a[k]) * pow(x, k, p) for k in range(n)) % p
    lz = a.copy()
    op.forward_lazy(lz)
    assert all(int(v) < 4 * p for v in lz)
    assert ((lz % np.uint64(p)) == f).all()
    b = f.copy()
    op.backward(b)
    assert (b == a).all()
    # convolution theorem: backward(forward(a)*forward(b)) is the negacyclic product
    if n <= 32:
        c = rnd.integers(0, p, size=n, dtype=np.uint64)
        g = c.copy()
        op.forward(g)
        h = np.array([int(x) * int(y) % p for x, y in zip(f, g)], dtype=np.uint64)
        op.backward(h)
        exp = [0] * n
        for i in range(n):
            for j in range(n):
                k, v = i + j, int(a[i]) * int(c[j])
                if k < n:
                    exp[k] = (exp[k] + v) % p
                else:
                    exp[k - n] = (exp[k - n] - v) % p
        assert [int(x) for x in h] == exp


def _expected_scale(x_lift, Qfrom, n, d, Qto):
    """rns/scaler.rs:397-414 (the reference test's own BigUint rule)."""
    sign = x_lift >= (Qfrom >> 1)
    if sign:
        x_lift = Qfrom - x_lift
        if d % 2 == 0:
            return Qto - ((x_lift * n + ((d >> 1) - 1)) // d) % Qto
        return Qto - ((x_lift * n + (d >> 1)) // d) % Qto
    return (x_lift * n + (d >> 1)) // d


def test_scaler_same_context(oracle):
    """rns/scaler.rs:380-419"""
    rnd = random.Random(3)
    q = oracle.RnsContext([4, 4611686018326724609, 1153])
    for n in [1, 2, 3, 100, 1000, 4611686018326724610]:
        for d in [1, 2, 3, 4, 100, 101, 1000, 1001, 4611686018326724610]:
            s = oracle.RnsScaler(q, q, oracle.ScalingFactor(n, d))
            for _ in range(60):
                x = [rnd.randrange(m) for m in q.moduli_u64]
                z = s.scale_one(x, 3)
                assert z == q.project(_expected_scale(q.lift(x), q.product, n, d, q.product))


def test_scaler_different_contexts(oracle):
    """rns/scaler.rs:422-473"""
    rnd = random.Random(4)
    q = oracle.RnsContext([4, 4611686018326724609, 1153])
    r = oracle.RnsContext([4, 4611686018326724609, 1153] + NFL_62[1:8])
    for n in [1, 2, 3, 100, 1000, 4611686018326724610]:
        for d in [1, 2, 3, 4, 100, 101, 1000, 1001, 4611686018326724610]:
            s = oracle.RnsScaler(q, r, oracle.ScalingFactor(n, d))
            for _ in range(20):
                x = [rnd.randrange(m) for m in q.moduli_u64]
                y = s.scale_one(x, len(r.moduli))
                assert y == r.project(_expected_scale(q.lift(x), q.product, n, d, r.product))


def test_scaler_multiplication_bases(oracle):
    """SURVEY appendix A-3: the mul extender (factor 1, start=L) and down-scaler (t/Q) at
    62-bit bases obey the same centered-rounding rule."""
    rnd = random.Random(5)
    par = oracle.BfvParameters(16, 1153, moduli_sizes=[62] * 5)
    mp = par.level(0).mul_params
    frm, to = mp.frm.rns, mp.to.rns
    L = len(frm.moduli)
    assert mp.extender.number_common_moduli == L
    for _ in range(200):
        x = [rnd.randrange(m) for m in frm.moduli_u64]
        got = mp.extender.scaler.scale_one(x, len(to.moduli) - L, L)
        exp = to.project(_expected_scale(frm.lift(x), frm.product, 1, 1, to.product))
        assert got == exp[L:]
        y = [rnd.randrange(m) for m in to.moduli_u64]
        got = mp.down_scaler.scaler.scale_one(y, L, 0)
        exp = frm.project(_expected_scale(to.lift(y), to.product, par.plaintext, frm.product, frm.product))
        assert got == exp


def test_boundary_primes(oracle):
    """the boundary primes of tests/edge_inputs.py are primes == 1 mod 2^16, on the stated side of the Solinas rule
    (p = 2^62 - c, c < 2^28), and not reachable from 2^62 by the prime generator within a few steps"""
    import edge_inputs as E
    for name, p in E.BOUNDARY_PRIMES.items():
        assert oracle.is_prime(p) and p % (1 << 16) == 1 and p.bit_length() == 62, name
        c = (1 << 62) - p
        assert (c < (1 << 28)) == (name == "solinas_max_c"), name
    gen, ub = [], 1 << 62
    for _ in range(64):
        ub = oracle.generate_prime(62, 1 << 16, ub)
        gen.append(ub)
    assert not set(gen) & set(E.BOUNDARY_PRIMES.values())


# multiplication bases of the edge tests: name -> (degree, t, moduli sizes); the comments give the down scaler's
# theta_garner_shift
SCALER_BASES = {
    "set_a": (1 << 12, 1032193, [62] * 2),       # down 5 -> 2, shift 126
    "set_c": (1 << 15, 786433, [62] * 14),       # extension 14 -> 15, down 29 -> 14, shift 124
    "l31": (1 << 13, 786433, [62] * 31),         # down 63 -> 31: shift 123, the lowest the device kernels accept
    "small": (16, 1153, [40, 30]),               # extender 2 -> 3 with a small modulus: shift 127
}
_EPS = 2.0 ** -40


def _scale_branch(x, F, n, d, Qto, negative):
    """_expected_scale with the sign branch forced"""
    if negative:
        x = F - x
        r = (x * n + ((d >> 1) - 1 if d % 2 == 0 else d >> 1)) // d
        return (Qto - r % Qto) % Qto
    return ((x * n + (d >> 1)) // d) % Qto


def _windows(x, F, n, d):
    """(near a rounding tie of n x / d, near the sign boundary F / 2)"""
    from fractions import Fraction
    frac = Fraction(x * n % d, d)
    return abs(frac - Fraction(1, 2)) < _EPS, abs(Fraction(x, F) - Fraction(1, 2)) < _EPS


def _scaler_cases(oracle, name):
    """(scaler, from context, to context, factor, start, n_out, inputs) for the extender and the down scaler"""
    import edge_inputs as E
    degree, t, sizes = SCALER_BASES[name]
    par = oracle.BfvParameters(degree, t, moduli_sizes=sizes)
    mp = par.level(0).mul_params
    frm, to = mp.frm.rns, mp.to.rns
    L, K = len(frm.moduli), len(to.moduli)
    Q, F = frm.product, to.product
    rng = np.random.default_rng(len(sizes))
    rnd = [int(rng.integers(0, 1 << 62)) * F // (1 << 62) for _ in range(16)]
    down = E.scaler_near_ties(F, t, Q, rng) + E.sign_boundary(F) + rnd
    ext = E.extender_edges(Q) + E.sign_boundary(Q) + E.scaler_near_ties(Q, 1, 1, rng)[:7] + [x % Q for x in rnd]
    return [(mp.extender.scaler, frm, to, 1, 1, L, K - L, ext), (mp.down_scaler.scaler, to, frm, t, Q, 0, L, down)]


@pytest.mark.parametrize("name", sorted(SCALER_BASES))
def test_scaler_transcription_matches_oracle(oracle, name):
    """tests/scaler_reference.py (a plain-integer restatement of rns/scaler.rs:249-352) equals the oracle's C scaler on
    every crafted input: rounding ties, the sign boundary and the extender's edges."""
    import scaler_reference
    for sc, frm, to, n, d, start, n_out, xs in _scaler_cases(oracle, name):
        assert sc.theta_garner_shift == {"set_a": (127, 126), "set_c": (125, 124), "l31": (124, 123),
                                         "small": (127, 126)}[name][0 if n == 1 else 1]
        for x in xs:
            r = frm.project(x)
            assert scaler_reference.scale(sc, r, n_out, start) == sc.scale_one(r, n_out, start), (name, x)
    # residue vectors whose w sum sits between 2^190 and 2^191, where only bit 191 decides the sign of w (whether the
    # sum can get there depends on the basis; the 63 source limbs of l31 reach it)
    import edge_inputs as E
    sc, frm = _scaler_cases(oracle, name)[1][:2]
    wide = E.wide_w_sums(sc, frm.moduli_u64, np.random.default_rng(1), 32)
    if name == "l31":
        assert len(wide) == 32
    for r in wide:
        assert scaler_reference.scale(sc, r, len(sc.to.moduli)) == sc.scale_one(r, len(sc.to.moduli)), (name, r)


@pytest.mark.parametrize("name", sorted(SCALER_BASES))
def test_scaler_rounding_envelope(oracle, name):
    """The reference's fixed-point scaler is exact centered rounding (_expected_scale) except inside two windows: num x
    / den within 2^-40 of a half-integer, where it may round up by one, and x within 2^-40 F of F / 2, where it may
    take the other sign branch (again possibly plus one).  This pins where the reference -- and so every device
    kernel -- departs from exact rounding; any widening of these windows fails here."""
    seen = {"tie_plus_one": 0, "other_branch": 0}
    for sc, frm, to, n, d, start, n_out, xs in _scaler_cases(oracle, name):
        Qto = to.product

        def limbs(v):   # the limbs this scaler writes (the extender copies the first `start` ones)
            return to.project(v % Qto)[start:start + n_out]
        for x in xs:
            got = sc.scale_one(frm.project(x), n_out, start)
            exp = _expected_scale(x, frm.product, n, d, Qto)
            if got == limbs(exp):
                continue
            near_tie, near_sign = _windows(x, frm.product, n, d)
            if near_tie and got == limbs(exp + 1):
                seen["tie_plus_one"] += 1
                continue
            other = _scale_branch(x, frm.product, n, d, Qto, x < frm.product // 2)
            assert near_sign and got in (limbs(other), limbs(other + 1)), (name, x, near_tie, near_sign)
            seen["other_branch"] += 1
    # the crafted inputs do reach the departures (otherwise this test would check nothing)
    assert seen["other_branch"] > 0, seen
    if name != "small":
        assert seen["tie_plus_one"] > 0, seen


def test_poly_scaler_and_switch_down(oracle):
    """rq/scaler.rs:153-204 and rq/mod.rs:1040-1066: poly-level scale == per-coefficient BigUint rule;
    switch_down == round(x / q_last) with the reference's rounding."""
    rng = np.random.default_rng(11)
    ctx = oracle.Context(NFL_62[:4], 16)
    p = oracle.Poly.random(ctx, oracle.POWER_BASIS, rng)
    big = p.to_bigints()
    q_last = ctx.moduli[-1]
    sd = p.copy().switch_down()
    nxt = ctx.next_context
    for j, x in enumerate(big):
        exp = ((x + (q_last >> 1)) // q_last) % nxt.modulus()   # rq/mod.rs:1057-1066
        assert sd.ctx.rns.lift([int(v) for v in sd.c[:, j]]) == exp
    # Ntt-representation scale == PowerBasis scale then NTT
    to = oracle.Context(NFL_62[:4] + NFL_62[6:9], 16)
    sc = oracle.Scaler(ctx, to, oracle.ScalingFactor.one())
    pn = p.copy().into_ntt()
    a = sc.scale(pn).into_power_basis()
    b = sc.scale(p)
    assert (a.c == b.c).all()


def test_substitute_ntt_matches_power_basis(oracle):
    """rq/mod.rs:973-982 and SURVEY appendix A-2"""
    rng = np.random.default_rng(12)
    ctx = oracle.Context(NFL_62[:2], 16)
    p = oracle.Poly.random(ctx, oracle.POWER_BASIS, rng)
    for e in (3, 5, 9, 31):
        a = p.substitute(e).into_ntt()
        b = p.copy().into_ntt().substitute(e)
        assert (a.c == b.c).all()
    with pytest.raises(ValueError):
        p.substitute(2)


def _negacyclic(a, b, t):
    n = len(a)
    r = [0] * n
    for i in range(n):
        for j in range(n):
            k, v = i + j, int(a[i]) * int(b[j])
            if k < n:
                r[k] = (r[k] + v) % t
            else:
                r[k - n] = (r[k - n] - v) % t
    return np.array(r, dtype=np.uint64)


@pytest.mark.parametrize("nmod", [2, 3, 5])
def test_multiply_decrypts_to_product(oracle, nmod):
    """ops/mul.rs:263-294 (default multiplicator), :296-330 (mod switch), ops/mod.rs mul + relinearizes"""
    rng = np.random.default_rng(100 + nmod)
    par = oracle.BfvParameters(16, 1153, moduli_sizes=[62] * nmod)
    sk = oracle.SecretKey(par, rng)
    a, b = rng.integers(0, 1153, 16), rng.integers(0, 1153, 16)
    cta, ctb = sk.encrypt(a, 0, rng), sk.encrypt(b, 0, rng)
    assert (sk.decrypt(cta) == a).all()
    rk = oracle.RelinearizationKey(sk, rng)
    m = oracle.Multiplicator.default(rk)
    ct = m.multiply(cta, ctb)
    exp = _negacyclic(a, b, 1153)
    assert (sk.decrypt(ct) == exp).all()
    c3 = cta.mul(ctb)
    assert len(c3.c) == 3 and (sk.decrypt(c3) == exp).all()
    assert (rk.relinearizes(c3).to_array() == ct.to_array()).all()
    m.enable_mod_switching()
    ct2 = m.multiply(cta, ctb)
    assert ct2.level == 1 and (sk.decrypt(ct2) == exp).all()
    # add / sub / neg
    assert (sk.decrypt(cta.add(ctb)) == (a + b) % 1153).all()
    assert (sk.decrypt(cta.sub(ctb)) == (a + 1153 - b) % 1153).all()
    assert (sk.decrypt(cta.neg()) == (1153 - a) % 1153).all()


def test_second_multiplication_strategy(oracle):
    """ops/mul.rs:369-418 `different_mul_strategy`: the second strategy of ePrint 2021/204 (rhs scaled by P/Q into the
    extended basis, product scaled by t/P), built with Multiplicator::new; decrypts to the product with and without
    modulus switching."""
    rng = np.random.default_rng(204)
    t = 1153
    par = oracle.BfvParameters(16, t, moduli_sizes=[62] * 3)
    basis = list(par.moduli)
    for _ in range(3):
        basis.append(oracle.generate_prime(62, 2 * par.degree, basis[-1]))
    P = 1
    for q in basis[3:]:
        P *= q
    Q = par.context_at_level(0).modulus()
    for _ in range(3):
        sk = oracle.SecretKey(par, rng)
        a = rng.integers(0, t, 16)
        ct1, ct2 = sk.encrypt(a, 0, rng), sk.encrypt(a, 0, rng)
        m = oracle.Multiplicator(par, oracle.ScalingFactor.one(), oracle.ScalingFactor(P, Q), basis,
                                 oracle.ScalingFactor(t, P))
        assert m.extender_lhs.number_common_moduli == 3 and m.extender_rhs.number_common_moduli == 0
        ct3 = m.multiply(ct1, ct2)
        assert len(ct3.c) == 3
        exp = _negacyclic(a, a, t)
        assert (sk.decrypt(ct3) == exp).all()
        m.enable_mod_switching()
        ct3 = m.multiply(ct1, ct2)
        assert ct3.level == 1 and (sk.decrypt(ct3) == exp).all()


def test_dot_product_scalar(oracle):
    """bfv/ops/dot_product.rs:186-260 `test_dot_product_scalar`: empty input is an error; the result equals the sum of
    the ct * pt products and decrypts to the SIMD dot product."""
    rng = np.random.default_rng(77)
    t = 1153
    par = oracle.BfvParameters(16, t, moduli_sizes=[62] * 2)
    with pytest.raises(ValueError):
        oracle.dot_product_scalar([], [])
    sk = oracle.SecretKey(par, rng)
    for size in (1, 2, 7, 20):
        vals_c = rng.integers(0, t, size=(size, 16))
        vals_p = rng.integers(0, t, size=(size, 16))
        cts = [sk.encrypt(oracle.simd_encode(par, v), 0, rng) for v in vals_c]
        ctx = par.context_at_level(0)   # Plaintext::poly_ntt: the encoded message itself, transformed (no delta)
        pts = [oracle.Poly.from_u64(ctx, oracle.simd_encode(par, v), oracle.NTT) for v in vals_p]
        r = oracle.dot_product_scalar(cts, pts)
        exp = None
        for c, p in zip(cts, pts):
            term = oracle.Ciphertext(par, [x.mul(p) for x in c.c], 0)
            exp = term if exp is None else exp.add(term)
        assert (r.to_array() == exp.to_array()).all()
        dec = oracle.simd_decode(par, sk.decrypt(r))
        assert (dec.astype(np.int64) == (vals_c * vals_p).sum(axis=0) % t).all()
    with pytest.raises(ValueError):
        oracle.dot_product_scalar(cts, pts[:-1])


def test_key_switch_noise_and_galois(oracle):
    """key_switching_key.rs:532-560 (noise <= 70 bits), galois_key.rs:211-230 (slot permutation)"""
    rng = np.random.default_rng(21)
    par = oracle.BfvParameters(16, 1153, moduli_sizes=[62] * 3)
    sk = oracle.SecretKey(par, rng)
    ctx = par.context_at_level(0)
    # key switch noise
    frm = oracle.Poly.from_i64(ctx, rng.integers(-1, 2, 16))
    ksk = oracle.KeySwitchingKey(sk, frm, 0, 0, rng)
    inp = oracle.Poly.random(ctx, oracle.POWER_BASIS, rng)
    c0, c1 = ksk.key_switch(inp)
    s = sk.s_ntt(ctx)
    c0.iadd(c1.mul(s))
    c0.isub(inp.copy().into_ntt().mul(frm.copy().into_ntt()))
    Q = ctx.modulus()
    noise = max(min(v.bit_length(), (Q - v).bit_length()) for v in c0.into_power_basis().to_bigints())
    assert noise <= 70
    # galois: column rotation by one and row swap on SIMD slots
    v = rng.integers(0, 1153, 16)
    ct = sk.encrypt(oracle.simd_encode(par, v), 0, rng)
    row = 8
    gk = oracle.GaloisKey(sk, 3, rng)
    got = oracle.simd_decode(par, sk.decrypt(gk.relinearize(ct)))
    exp = np.concatenate([np.roll(v[:row], -1), np.roll(v[row:], -1)])
    assert (got == exp).all()
    gk = oracle.GaloisKey(sk, 2 * 16 - 1, rng)
    got = oracle.simd_decode(par, sk.decrypt(gk.relinearize(ct)))
    assert (got == np.concatenate([v[row:], v[:row]])).all()


def test_key_switch_decomposition(oracle):
    """keys/key_switching_key.rs:595-627 `key_switch_decomposition`: a key at a single-modulus level (6 moduli, level
    5) uses the base-2^(log q / 2) decomposition; c0 + c1*s - input*p stays below (bits(q) / 2) + 10 bits."""
    rng = np.random.default_rng(595)
    par = oracle.BfvParameters(16, 1153, moduli_sizes=[62] * 6)
    ctx = par.context_at_level(5)
    q = ctx.moduli[0]
    for _ in range(10):
        sk = oracle.SecretKey(par, rng)
        p = oracle.Poly.from_i64(ctx, oracle.sample_vec_cbd(16, 10, rng))
        ksk = oracle.KeySwitchingKey(sk, p, 5, 5, rng)
        assert ksk.log_base == 31 and len(ksk.c0) == 2
        inp = oracle.Poly.random(ctx, oracle.POWER_BASIS, rng)
        c0, c1 = ksk.key_switch(inp)
        c2 = c0.copy().iadd(c1.copy().imul(sk.s_ntt(ctx))).into_power_basis()
        c3 = inp.copy().into_ntt().imul(p.copy().into_ntt()).into_power_basis()
        for a, b in zip(c2.c[0], c3.c[0]):
            d = (int(a) - int(b)) % q
            assert min(d.bit_length(), (q - d).bit_length()) <= q.bit_length() // 2 + 10


def test_leveled_keys(oracle):
    """relinearization_key.rs:226-290: ciphertext at level 1, key at level 0 (switch down after key switch)"""
    rng = np.random.default_rng(31)
    par = oracle.BfvParameters(16, 1153, moduli_sizes=[62] * 4)
    sk = oracle.SecretKey(par, rng)
    a, b = rng.integers(0, 1153, 16), rng.integers(0, 1153, 16)
    cta, ctb = sk.encrypt(a, 1, rng), sk.encrypt(b, 1, rng)
    rk = oracle.RelinearizationKey(sk, rng, ciphertext_level=1, key_level=0)
    ct = rk.relinearizes(cta.mul(ctb))
    assert ct.level == 1 and (sk.decrypt(ct) == _negacyclic(a, b, 1153)).all()


def test_transcode_roundtrip(oracle):
    """fhe-util/src/lib.rs:323-372: transcode self-consistency, known 4-bit round trip, empty input"""
    rnd = random.Random(9)
    for size in (1, 2, 7, 8, 33, 100):
        vals = [rnd.randrange(1 << 64) for _ in range(size)]
        for nbits in (1, 4, 7, 8, 13, 36, 49, 61, 62):
            masked = [v & ((1 << nbits) - 1) for v in vals]
            b = oracle.transcode_to_bytes(masked, nbits)
            assert len(b) == -(-size * nbits // 8)
            assert oracle.transcode_from_bytes(b, nbits)[:size] == masked
    assert oracle.transcode_from_bytes(oracle.transcode_to_bytes([1, 2, 3, 4, 5, 6, 7, 8], 4), 4) == [1, 2, 3, 4, 5, 6, 7, 8]
    assert oracle.transcode_to_bytes([1, 2, 3, 4], 4) == bytes([0x21, 0x43])      # LSB-first nibbles
    assert oracle.transcode_to_bytes([], 8) == b"" and oracle.transcode_from_bytes(b"", 8) == []
    # Rq coefficients blob of a polynomial round-trips through both representations
    ctx = oracle.Context(NFL_62[:2], 16)
    p = oracle.Poly.random(ctx, oracle.NTT, np.random.default_rng(5))
    blob = oracle.poly_to_rq_coefficients(p)
    assert len(blob) == 2 * 62 * 16 // 8
    assert (oracle.poly_from_rq_coefficients(ctx, blob, oracle.NTT).c == p.c).all()


def test_inner_sum_and_expansion_semantics(oracle):
    """evaluation_key.rs tests (:600-760): inner sum puts the slot sum in every slot; oblivious expansion of
    Enc(sum_k m_k x^k) to `size` ciphertexts gives Enc(2^level * m_k) (constant polynomials)."""
    degree, t = 16, 1153
    rng = np.random.default_rng(77)
    par = oracle.BfvParameters(degree, t, moduli_sizes=[62] * 3)
    sk = oracle.SecretKey(par, rng)
    exps = sorted({pow(3, 1 << k, 2 * degree) for k in range(3)} | {2 * degree - 1} | {(degree >> l) + 1 for l in range(2)})
    gks = {e: oracle.GaloisKey(sk, e, rng) for e in exps}
    v = rng.integers(0, t, degree)
    ct = sk.encrypt(oracle.simd_encode(par, v), 0, rng)
    dec = oracle.simd_decode(par, sk.decrypt(oracle.computes_inner_sum(par, gks, ct)))
    assert (dec == np.full(degree, int(v.sum()) % t, dtype=np.uint64)).all()
    m = np.zeros(degree, dtype=np.int64)
    m[:4] = rng.integers(0, t, 4)      # the query polynomial carries one value per expanded ciphertext
    ct = sk.encrypt(m, 0, rng)
    outs = oracle.expands(par, gks, ct, 4)
    for k in range(4):
        d = sk.decrypt(outs[k])
        assert int(d[0]) == (4 * int(m[k])) % t and not d[1:].any()


def test_rgsw_external_product(oracle):
    """rgsw_ciphertext.rs tests (:200-245): Dec(ct * RGSW(m2)) == m1 (*) m2 (negacyclic product mod t)"""
    degree, t = 16, 1153
    rng = np.random.default_rng(88)
    par = oracle.BfvParameters(degree, t, moduli_sizes=[62] * 3)
    sk = oracle.SecretKey(par, rng)
    m1, m2 = rng.integers(0, t, degree), rng.integers(0, t, degree)
    ct = sk.encrypt(m1, 0, rng)
    pt_ntt = oracle.Poly.from_u64(par.context_at_level(0), m2.astype(np.uint64), oracle.NTT)  # Plaintext.poly_ntt
    rgsw = oracle.RGSWCiphertext(sk, pt_ntt, 0, rng)
    out = rgsw.external_product(ct)
    assert (sk.decrypt(out) == _negacyclic(m1, m2, t)).all()
