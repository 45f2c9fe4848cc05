"""GPU parity tests: every C-ABI operation of libfhe_b200.so (driven through the host
mirror fhe_rs_b200.bfv, i.e. through the C ABI) must be BIT-EXACT against the CPU oracle
on identical inputs.  Mirrors the reference's own tests (ntt/mod.rs:50-82,
rq/scaler.rs:153-204, bfv/ops/mul.rs:263-330, keys/*.rs tests).  Run with `-m gpu`."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def F():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import fhe_rs_b200
    return fhe_rs_b200


def make_pair(oracle, F, degree, nmod, t, seed, sizes=None):
    opar = oracle.BfvParameters(degree, t, moduli_sizes=sizes or [62] * nmod)
    gpar = F.BfvParameters(degree, t, moduli=opar.moduli, device=0)
    assert gpar.moduli() == opar.moduli
    assert gpar.mul_basis(0) == opar.level(0).mul_params.to.moduli
    return opar, gpar, np.random.default_rng(seed)


def rand_ct(oracle, opar, rng, count, parts=2, level=0):
    ctx = opar.context_at_level(level)
    arr = np.zeros((count, parts, len(ctx.moduli), opar.degree), np.uint64)
    for i, q in enumerate(ctx.moduli):
        arr[:, :, i, :] = rng.integers(0, q, size=(count, parts, opar.degree), dtype=np.uint64)
    return arr


@pytest.mark.parametrize("logn,nmod", [(3, 2), (4, 3), (6, 2), (9, 2), (10, 3), (11, 2), (12, 2), (13, 2), (14, 3),
                                        (15, 2), (16, 1)])
def test_ntt_forward_backward(oracle, F, logn, nmod):
    """NttOperator::forward/backward (ntt/native.rs:77-233) on every row of a batch."""
    n = 1 << logn
    opar, gpar, rng = make_pair(oracle, F, n, nmod, 1153 if logn < 12 else 786433, 10 + logn)
    ctx = opar.context_at_level(0)
    x = rand_ct(oracle, opar, rng, 3)
    ct = F.Ciphertext.from_host(gpar, x, repr=F.POWER_BASIS)
    got = ct.into_ntt().to_host()
    exp = x.copy()
    for c in range(3):
        for p in range(2):
            for i, op in enumerate(ctx.ops):
                op.forward(exp[c, p, i])
    assert (got == exp).all()
    back = ct.into_power_basis().to_host()
    assert (back == x).all()
    # an odd number of polynomials per limb (three 1-part polynomials): the TMA rows pass cannot pair them and takes
    # its one-tile kernel (under FHE_B200_NTT=tma at 2^13 <= N <= 2^15)
    odd = F.Ciphertext.from_host(gpar, x[:, :1], repr=F.POWER_BASIS)
    assert (odd.into_ntt().to_host() == exp[:, :1]).all()
    assert (odd.into_power_basis().to_host() == x[:, :1]).all()
    # backward on arbitrary (reduced) NTT-domain input
    ct2 = F.Ciphertext.from_host(gpar, x, repr=F.NTT)
    got = ct2.into_power_basis().to_host()
    exp = x.copy()
    for c in range(3):
        for p in range(2):
            for i, op in enumerate(ctx.ops):
                op.backward(exp[c, p, i])
    assert (got == exp).all()
    with pytest.raises(F.FheError) as e:
        ct2.into_power_basis()
    assert e.value.code == -8


def test_add_sub_neg(oracle, F):
    """ops/mod.rs:15-227"""
    opar, gpar, rng = make_pair(oracle, F, 64, 3, 1153, 1)
    a, b = rand_ct(oracle, opar, rng, 5), rand_ct(oracle, opar, rng, 5)
    A, B = F.Ciphertext.from_host(gpar, a), F.Ciphertext.from_host(gpar, b)
    q = np.array(opar.moduli, dtype=object)[None, None, :, None]
    ao, bo = a.astype(object), b.astype(object)
    assert ((A + B).to_host().astype(object) == (ao + bo) % q).all()
    assert ((A - B).to_host().astype(object) == (ao - bo) % q).all()
    assert ((-A).to_host().astype(object) == (-ao) % q).all()
    # mismatched levels are rejected (ops/mod.rs:28)
    C1 = F.Ciphertext(gpar, 5, 2, level=1)
    with pytest.raises(F.FheError) as e:
        A += C1
    assert e.value.code == -6


@pytest.mark.parametrize("degree,nmod", [(16, 2), (16, 5), (64, 3), (4096, 2)])
def test_scalers(oracle, F, degree, nmod):
    """rq::scaler::Scaler::scale (rq/scaler.rs:55-127) with the multiplication scalers."""
    t = 1153 if degree < 4096 else 1032193
    opar, gpar, rng = make_pair(oracle, F, degree, nmod, t, 2 + nmod)
    mp = opar.level(0).mul_params
    x = rand_ct(oracle, opar, rng, 2)
    ct = F.Ciphertext.from_host(gpar, x)
    up = ct.scale(0)
    got = up.to_host()
    for c in range(2):
        for p in range(2):
            exp = mp.extender.scale(oracle.Poly(mp.frm, oracle.NTT, x[c, p])).c
            assert (got[c, p] == exp).all()
    # down scaler on random data in the multiplication basis
    K = len(mp.to.moduli)
    y = np.zeros((2, 2, K, degree), np.uint64)
    for i, q in enumerate(mp.to.moduli):
        y[:, :, i, :] = rng.integers(0, q, size=(2, 2, degree), dtype=np.uint64)
    cty = F.Ciphertext.from_host(gpar, y, mul_basis=True)
    got = cty.scale(1).to_host()
    for c in range(2):
        for p in range(2):
            exp = mp.down_scaler.scale(oracle.Poly(mp.to, oracle.NTT, y[c, p])).c
            assert (got[c, p] == exp).all()


def _keys(oracle, F, opar, gpar, rng, exponents=(), ct_level=0, key_level=0):
    sk = oracle.SecretKey(opar, rng)
    ork = oracle.RelinearizationKey(sk, rng, ct_level, key_level)
    grk = F.RelinearizationKey.from_arrays(gpar, *ork.ksk.arrays(), ciphertext_level=ct_level, key_level=key_level)
    ogk, ggk = {}, {}
    for e in exponents:
        ogk[e] = oracle.GaloisKey(sk, e, rng, ct_level, key_level)
        ggk[e] = F.GaloisKey.from_arrays(gpar, e, *ogk[e].ksk.arrays(), ciphertext_level=ct_level, key_level=key_level)
    return sk, ork, grk, ogk, ggk


@pytest.mark.parametrize("degree,nmod,t", [(16, 2, 1153), (16, 3, 1153), (16, 5, 1153), (128, 3, 1153),
                                           (4096, 2, 1032193)])
def test_mul_relin_against_oracle(oracle, F, degree, nmod, t):
    """&ct * &ct (ops/mod.rs:259-358), RelinearizationKey::relinearizes (relinearization_key.rs:70-103),
    Multiplicator::multiply with and without mod switching (mul.rs:165-243): bit-exact, and the
    result decrypts to the negacyclic product (mul.rs:263-330)."""
    opar, gpar, rng = make_pair(oracle, F, degree, nmod, t, 40 + nmod)
    sk, ork, grk, _, _ = _keys(oracle, F, opar, gpar, rng)
    count = 3
    msgs_a = rng.integers(0, t, size=(count, degree))
    msgs_b = rng.integers(0, t, size=(count, degree))
    octa = [sk.encrypt(m, 0, rng) for m in msgs_a]
    octb = [sk.encrypt(m, 0, rng) for m in msgs_b]
    a = np.stack([c.to_array() for c in octa])
    b = np.stack([c.to_array() for c in octb])
    A, B = F.Ciphertext.from_host(gpar, a), F.Ciphertext.from_host(gpar, b)

    C3 = A * B
    assert len(C3) == 3
    got3 = C3.to_host()
    for i in range(count):
        assert (got3[i] == octa[i].mul(octb[i]).to_array()).all()

    got2 = grk.relinearizes(C3).to_host()
    om = oracle.Multiplicator.default(ork)
    gm = F.Multiplicator.default(grk)
    gotm = gm.multiply(A, B).to_host()
    for i in range(count):
        exp = om.multiply(octa[i], octb[i])
        assert (gotm[i] == exp.to_array()).all()
        assert (got2[i] == exp.to_array()).all()
    # decrypt-correctness of the GPU result (schoolbook check only at small degree)
    if degree <= 128:
        res = oracle.Ciphertext.from_array(opar, gotm[0], 0)
        dec = sk.decrypt(res)
        exp = np.zeros(degree, dtype=object)
        for x in range(degree):
            for y in range(degree):
                k, v = x + y, int(msgs_a[0][x]) * int(msgs_b[0][y])
                if k < degree:
                    exp[k] = (exp[k] + v) % t
                else:
                    exp[k - degree] = (exp[k - degree] - v) % t
        assert (dec.astype(object) == exp).all()
    # with modulus switching (mul.rs:296-330)
    om.enable_mod_switching()
    gm.enable_mod_switching()
    out = gm.multiply(A, B)
    assert out.level == 1
    gotms = out.to_host()
    for i in range(count):
        assert (gotms[i] == om.multiply(octa[i], octb[i]).to_array()).all()
    # error behaviour: wrong part count / level (mul.rs:168-189)
    with pytest.raises(F.FheError) as e:
        gm.multiply(C3, B)
    assert e.value.code == -7
    with pytest.raises(F.FheError) as e:
        gm.multiply(out, out)
    assert e.value.code == -6


@pytest.mark.parametrize("degree,nmod", [(16, 3), (128, 2)])
def test_mul_general_part_counts(oracle, F, degree, nmod):
    """&ct * &ct with n x m parts (ops/mod.rs:259-358: c[i+j] += a_i * b_j over the extended basis), including the
    product of a 3-part (unrelinearized) ciphertext with a fresh one and a 1-part operand."""
    opar, gpar, rng = make_pair(oracle, F, degree, nmod, 1153, 77)
    for na, nb in [(3, 2), (2, 3), (1, 2), (3, 3), (4, 1)]:
        a, b = rand_ct(oracle, opar, rng, 2, na), rand_ct(oracle, opar, rng, 2, nb)
        got = (F.Ciphertext.from_host(gpar, a) * F.Ciphertext.from_host(gpar, b)).to_host()
        assert got.shape[1] == na + nb - 1
        for i in range(2):
            exp = oracle.Ciphertext.from_array(opar, a[i], 0).mul(oracle.Ciphertext.from_array(opar, b[i], 0))
            assert (got[i] == exp.to_array()).all()


@pytest.mark.parametrize("degree,nmod", [(16, 3), (64, 2), (4096, 2)])
def test_custom_multiplication_strategy(oracle, F, degree, nmod):
    """Multiplicator::new / new_leveled (mul.rs:37-98) and the reference's `different_mul_strategy` test
    (mul.rs:369-418): lhs factor one, rhs factor P/Q, post factor t/P over base + extra primes; with and without
    relinearization and modulus switching; and the default strategy rebuilt through the custom entry point equals
    the fused default path."""
    t = 1153 if degree < 4096 else 1032193
    opar, gpar, rng = make_pair(oracle, F, degree, nmod, t, 900 + degree)
    sk, ork, grk, _, _ = _keys(oracle, F, opar, gpar, rng)
    basis = list(opar.moduli)
    for _ in range(nmod):
        basis.append(oracle.generate_prime(62, 2 * degree, basis[-1]))
    P = 1
    for q in basis[nmod:]:
        P *= q
    Q = opar.context_at_level(0).modulus()
    count = 2
    msgs = rng.integers(0, t, size=(count, degree))
    octa = [sk.encrypt(m, 0, rng) for m in msgs]
    octb = [sk.encrypt(m, 0, rng) for m in msgs]
    A = F.Ciphertext.from_host(gpar, np.stack([c.to_array() for c in octa]))
    B = F.Ciphertext.from_host(gpar, np.stack([c.to_array() for c in octb]))

    om = oracle.Multiplicator(opar, oracle.ScalingFactor.one(), oracle.ScalingFactor(P, Q), basis,
                              oracle.ScalingFactor(t, P))
    gm = F.Multiplicator.new(F.ScalingFactor.one(), F.ScalingFactor(P, Q), basis, F.ScalingFactor(t, P), gpar)
    out = gm.multiply(A, B)
    assert len(out) == 3 and out.level == 0
    got = out.to_host()
    for i in range(count):
        assert (got[i] == om.multiply(octa[i], octb[i]).to_array()).all()
    if degree <= 64:   # decrypt-correctness of the device result
        res = oracle.Ciphertext.from_array(opar, got[0], 0)
        exp = np.zeros(degree, dtype=object)
        for x in range(degree):
            for y in range(degree):
                k, v = x + y, int(msgs[0][x]) * int(msgs[0][y])
                if k < degree:
                    exp[k] = (exp[k] + v) % t
                else:
                    exp[k - degree] = (exp[k - degree] - v) % t
        assert (sk.decrypt(res).astype(object) == exp).all()
    # + relinearization (enable_relinearization, mul.rs:141-151)
    om.enable_relinearization(ork)
    gm.enable_relinearization(grk)
    got = gm.multiply(A, B).to_host()
    for i in range(count):
        assert (got[i] == om.multiply(octa[i], octb[i]).to_array()).all()
    # + modulus switching (mul.rs:411-416)
    om.enable_mod_switching()
    gm.enable_mod_switching()
    out = gm.multiply(A, B)
    assert out.level == 1 and len(out) == 2
    got = out.to_host()
    for i in range(count):
        assert (got[i] == om.multiply(octa[i], octb[i]).to_array()).all()
    # without relinearization but with modulus switching: three parts one level down
    om2 = oracle.Multiplicator(opar, oracle.ScalingFactor.one(), oracle.ScalingFactor(P, Q), basis,
                               oracle.ScalingFactor(t, P))
    om2.enable_mod_switching()
    gm2 = F.Multiplicator.new(F.ScalingFactor.one(), F.ScalingFactor(P, Q), basis, F.ScalingFactor(t, P), gpar)
    gm2.enable_mod_switching()
    out = gm2.multiply(A, B)
    assert out.level == 1 and len(out) == 3
    got = out.to_host()
    for i in range(count):
        assert (got[i] == om2.multiply(octa[i], octb[i]).to_array()).all()
    # the default strategy through the custom entry point == the fused default path
    dflt = gpar.mul_basis(0)
    gd = F.Multiplicator.new(F.ScalingFactor.one(), F.ScalingFactor.one(), dflt, F.ScalingFactor(t, Q), gpar)
    gd.enable_relinearization(grk)
    assert (gd.multiply(A, B).to_host() == F.Multiplicator.default(grk).multiply(A, B).to_host()).all()
    # both extenders with a non-unit factor (no common prefix on either side), non-62-bit extra prime in the basis
    basis3 = basis + [oracle.generate_prime(50, 2 * degree, 1 << 50)]
    P3 = P * basis3[-1]
    om3 = oracle.Multiplicator(opar, oracle.ScalingFactor(3, 1), oracle.ScalingFactor(P3, 3 * Q), basis3,
                               oracle.ScalingFactor(t, P3))
    gm3 = F.Multiplicator.new(F.ScalingFactor(3, 1), F.ScalingFactor(P3, 3 * Q), basis3, F.ScalingFactor(t, P3), gpar)
    got = gm3.multiply(A, B).to_host()
    for i in range(count):
        assert (got[i] == om3.multiply(octa[i], octb[i]).to_array()).all()
    # error behaviour
    with pytest.raises(F.FheError) as e:   # level out of range (context_at_level)
        F.Multiplicator.new_leveled(F.ScalingFactor.one(), F.ScalingFactor.one(), dflt, F.ScalingFactor(t, Q), nmod, gpar)
    assert e.value.code == -6
    with pytest.raises(F.FheError) as e:   # duplicate modulus in the basis
        F.Multiplicator.new(F.ScalingFactor.one(), F.ScalingFactor.one(), dflt + [dflt[0]], F.ScalingFactor(t, Q), gpar)
    assert e.value.code == -2
    with pytest.raises(F.FheError) as e:   # not NTT friendly
        F.Multiplicator.new(F.ScalingFactor.one(), F.ScalingFactor.one(), dflt + [113], F.ScalingFactor(t, Q), gpar)
    assert e.value.code == -4


@pytest.mark.parametrize("degree,nmod", [(16, 3), (64, 2), (4096, 2)])
def test_galois_and_key_switch(oracle, F, degree, nmod):
    """GaloisKey::relinearize (galois_key.rs:63-86), Poly::substitute (rq/mod.rs:360-389),
    KeySwitchingKey::key_switch (key_switching_key.rs:241-270), rotation semantics (:211-230)."""
    t = 1153 if degree < 4096 else 1032193
    opar, gpar, rng = make_pair(oracle, F, degree, nmod, t, 60 + nmod)
    exps = (3, 2 * degree - 1, 9)
    sk, ork, grk, ogk, ggk = _keys(oracle, F, opar, gpar, rng, exps)
    count = 2
    vals = rng.integers(0, t, size=(count, degree))
    octs = [sk.encrypt(oracle.simd_encode(opar, v), 0, rng) for v in vals]
    x = np.stack([c.to_array() for c in octs])
    X = F.Ciphertext.from_host(gpar, x)
    for e in exps:
        got = ggk[e].relinearize(X).to_host()
        for i in range(count):
            assert (got[i] == ogk[e].relinearize(octs[i]).to_array()).all()
        sub = X.substitute(e).to_host()
        for i in range(count):
            for p in range(2):
                assert (sub[i, p] == octs[i].c[p].substitute(e).c).all()
    with pytest.raises(F.FheError) as err:
        X.substitute(4)
    assert err.value.code == -10
    # the PowerBasis branch (rq/mod.rs:390-408): signed coefficient permutation; substitution commutes with the NTT
    PB = X.clone().into_power_basis()
    for e in exps + (2 * degree + 3,):
        sub = PB.substitute(e)
        assert sub.representation == F.POWER_BASIS
        got = sub.to_host()
        for i in range(count):
            for p in range(2):
                assert (got[i, p] == octs[i].c[p].copy().into_power_basis().substitute(e).c).all()
        assert (sub.into_ntt().to_host() == X.substitute(e).to_host()).all()
    # EvaluationKey rotations decrypt to the expected slot permutation
    ek = F.EvaluationKey(gpar)
    for e in exps:
        ek.add_galois_key(ggk[e])
    row = degree // 2
    got = ek.rotates_columns_by(X, 1).to_host()
    dec = oracle.simd_decode(opar, sk.decrypt(oracle.Ciphertext.from_array(opar, got[0], 0)))
    assert (dec == np.concatenate([np.roll(vals[0][:row], -1), np.roll(vals[0][row:], -1)])).all()
    got = ek.rotates_rows(X).to_host()
    dec = oracle.simd_decode(opar, sk.decrypt(oracle.Ciphertext.from_array(opar, got[0], 0)))
    assert (dec == np.concatenate([vals[0][row:], vals[0][:row]])).all()
    # raw key switch of a power-basis polynomial
    pb = F.Ciphertext.from_host(gpar, x).into_power_basis()
    ks = grk.ksk.key_switch(pb, part=1).to_host()
    for i in range(count):
        p = octs[i].c[1].copy().into_power_basis()
        c0, c1 = ork.ksk.key_switch(p)
        assert (ks[i, 0] == c0.c).all() and (ks[i, 1] == c1.c).all()


def test_switch_down(oracle, F):
    """Ciphertext::switch_down (ciphertext.rs:148-161, rq/mod.rs:433-492)"""
    opar, gpar, rng = make_pair(oracle, F, 32, 4, 1153, 77)
    x = rand_ct(oracle, opar, rng, 3)
    X = F.Ciphertext.from_host(gpar, x)
    X.switch_down()
    assert X.level == 1 and X.limbs == 3
    got = X.to_host()
    for i in range(3):
        exp = oracle.Ciphertext.from_array(opar, x[i], 0).switch_down()
        assert (got[i] == exp.to_array()).all()
    X.switch_down().switch_down()
    with pytest.raises(F.FheError) as e:
        X.switch_down()
    assert e.value.code == -9
    # Ciphertext::switch_to_level (ciphertext.rs:164-184)
    Y = F.Ciphertext.from_host(gpar, x)
    assert Y.max_switchable_level() == 3
    Y.switch_to_level(2)
    assert Y.level == 2 and Y.limbs == 2
    got = Y.to_host()
    for i in range(3):
        assert (got[i] == oracle.Ciphertext.from_array(opar, x[i], 0).switch_to_level(2).to_array()).all()
    for bad in (1, 4):   # moving up, or past the last level
        with pytest.raises(F.FheError) as e:
            Y.switch_to_level(bad)
        assert e.value.code == -6


def test_mixed_modulus_sizes(oracle, F):
    """non-62-bit moduli (default_parameters_128 style, parameters.rs:224-250): generic Barrett/Shoup path."""
    moduli = [0xffffee001, 0xffffc4001, 0x1ffffe0001]
    t = 65537
    opar = oracle.BfvParameters(4096, t, moduli=moduli)
    gpar = F.BfvParameters(4096, t, moduli=moduli)
    rng = np.random.default_rng(5)
    sk, ork, grk, _, _ = _keys(oracle, F, opar, gpar, rng)
    ma, mb = rng.integers(0, t, 4096), rng.integers(0, t, 4096)
    ca, cb = sk.encrypt(ma, 0, rng), sk.encrypt(mb, 0, rng)
    A = F.Ciphertext.from_host(gpar, ca.to_array()[None])
    B = F.Ciphertext.from_host(gpar, cb.to_array()[None])
    got = F.Multiplicator.default(grk).multiply(A, B).to_host()
    assert (got[0] == oracle.Multiplicator.default(ork).multiply(ca, cb).to_array()).all()


def test_golden_fixture(oracle, F):
    """committed golden vectors (tests/golden/make_golden.py): GPU == stored outputs, no oracle involved"""
    import os
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "golden_n16_l3.npz"))
    gpar = F.BfvParameters(int(g["degree"]), int(g["t"]), moduli=[int(x) for x in g["moduli"]],
                           psi=[int(x) for x in g["psi"]])
    A, B = F.Ciphertext.from_host(gpar, g["a"]), F.Ciphertext.from_host(gpar, g["b"])
    rk = F.RelinearizationKey.from_arrays(gpar, g["rk_c0"], g["rk_c1"])
    gk = F.GaloisKey.from_arrays(gpar, 3, g["gk_c0"], g["gk_c1"])
    assert ((A + B).to_host() == g["add"]).all()
    assert ((A * B).to_host() == g["mul3"]).all()
    m = F.Multiplicator.default(rk)
    assert (m.multiply(A, B).to_host() == g["mul_relin"]).all()
    assert (m.enable_mod_switching().multiply(A, B).to_host() == g["mul_relin_ms"]).all()
    assert (gk.relinearize(A).to_host() == g["galois3"]).all()
    assert (F.Ciphertext.from_host(gpar, g["a"]).into_power_basis().to_host() == g["a_pb"]).all()


def test_wide_golden_fixture(F):
    """committed golden vectors of the operations around the core (tests/golden/make_golden_wide.py): device ==
    stored outputs, no oracle involved"""
    import os
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "golden_n16_l3_wide.npz"))
    t = int(g["t"])
    gpar = F.BfvParameters(int(g["degree"]), t, moduli=[int(x) for x in g["moduli"]])
    A, B = F.Ciphertext.from_host(gpar, g["a"]), F.Ciphertext.from_host(gpar, g["b"])
    assert ((A - B).to_host() == g["sub"]).all() and ((-A).to_host() == g["neg"]).all()
    assert (A.clone().switch_down().to_host() == g["switch_down"]).all()
    assert (A.clone().switch_to_level(2).to_host() == g["switch_to_2"]).all()
    assert (A.clone().add_plain(g["pt_to_poly"]).to_host() == g["add_plain"]).all()
    assert (A.clone().sub_plain(g["pt_to_poly"]).to_host() == g["sub_plain"]).all()
    assert (A.clone().mul_plain(g["pt_poly_ntt"]).to_host() == g["mul_plain"]).all()
    assert (F.dot_product_scalar(A, g["dot_pts"], 2).to_host() == g["dot"]).all()
    assert (((A * B) * B).to_host() == g["mul_3x2"]).all()
    basis = [int(x) for x in g["basis"]]
    P, Q = 1, 1
    for q in basis[3:]:
        P *= q
    for q in basis[:3]:
        Q *= q
    m2 = F.Multiplicator.new(F.ScalingFactor.one(), F.ScalingFactor(P, Q), basis, F.ScalingFactor(t, P), gpar)
    assert (m2.multiply(A, B).to_host() == g["strategy2"]).all()
    m2.enable_relinearization(F.RelinearizationKey.from_arrays(gpar, g["rk_c0"], g["rk_c1"]))
    assert (m2.multiply(A, B).to_host() == g["strategy2_relin"]).all()
    k2 = F.KeySwitchingKey.from_arrays(gpar, g["k2_c0"], g["k2_c1"], ciphertext_level=2, key_level=2)
    X = F.Ciphertext.from_host(gpar, g["k2_in"][:, None], level=2, repr=F.POWER_BASIS)
    assert (k2.key_switch(X, 0).to_host() == g["k2_out"]).all()
    assert (A.to_packed()[0] == g["packed"]).all()


@pytest.mark.parametrize("env", [{"FHE_B200_SOLINAS_NTT": "1"}, {"FHE_B200_NO_SOLINAS": "1"}, {"FHE_B200_GENERIC_NTT": "1"},
                                 {"FHE_B200_CHUNK": "1"}, {"FHE_B200_NTT": "tma"}, {"FHE_B200_NTT": "fast"},
                                 {"FHE_B200_NTT": "tma", "FHE_B200_CHUNK": "1"}, {"FHE_B200_SCALER": "classic"}, {"FHE_B200_KSMAC": "classic"}, {"FHE_B200_NO_TENSOR_FUSION": "1"},
                                 {"FHE_B200_NTT": "tma", "FHE_B200_TMA_COLS": "2", "FHE_B200_SCALE_UNROLL": "4",
                                  "FHE_B200_KS_STAGES": "3"}])
def test_alternate_code_paths(F, env):
    """the optional arithmetic / kernel variants (Solinas twiddle pairs, Barrett-only folds, generic tile NTT,
    one-ciphertext chunks, the TMA kernels' ring depth and unroll alternatives) must be bit-identical too: rerun the
    set-A multiply + the 2^13 NTT test under each switch"""
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    out = subprocess.run([sys.executable, "-m", "pytest", "-q", "-x", "-m", "gpu", "tests/test_gpu_parity.py", "-k",
                          "test_mul_relin_against_oracle and 4096 or test_ntt_forward_backward and 13-2 or "
                          "test_ntt_forward_backward and 14-3 or test_ntt_forward_backward and 15-2 or "
                          "test_golden_fixture or test_full_size_set_c or test_set_b_ntt_config or test_scalers"],
                         cwd=root, env=dict(os.environ, **env), capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, out.stdout[-2000:] + out.stderr[-2000:]


@pytest.mark.parametrize("degree,nmod,ct_level,key_level", [(16, 4, 1, 0), (64, 4, 2, 0), (4096, 3, 1, 0), (32, 3, 1, 1)])
def test_leveled_keys(oracle, F, degree, nmod, ct_level, key_level):
    """keys generated at a lower level number than the ciphertext (relinearization_key.rs:226-290,
    galois_key.rs:69-76, mul.rs:215-222): key switch at the key level, switch_down_to the ciphertext level."""
    t = 1153 if degree < 4096 else 1032193
    opar, gpar, rng = make_pair(oracle, F, degree, nmod, t, 90 + nmod + ct_level)
    sk, ork, grk, ogk, ggk = _keys(oracle, F, opar, gpar, rng, (3,), ct_level, key_level)
    count = 2
    ma, mb = rng.integers(0, t, size=(count, degree)), rng.integers(0, t, size=(count, degree))
    octa = [sk.encrypt(m, ct_level, rng) for m in ma]
    octb = [sk.encrypt(m, ct_level, rng) for m in mb]
    A = F.Ciphertext.from_host(gpar, np.stack([c.to_array() for c in octa]), level=ct_level)
    B = F.Ciphertext.from_host(gpar, np.stack([c.to_array() for c in octb]), level=ct_level)
    C3 = A * B
    got = grk.relinearizes(C3).to_host()
    om = oracle.Multiplicator.default(ork)
    gm = F.Multiplicator.default(grk)
    gotm = gm.multiply(A, B).to_host()
    gotg = ggk[3].relinearize(A).to_host()
    for i in range(count):
        exp = ork.relinearizes(octa[i].mul(octb[i]))
        assert (got[i] == exp.to_array()).all()
        assert (gotm[i] == om.multiply(octa[i], octb[i]).to_array()).all()
        assert (gotg[i] == ogk[3].relinearize(octa[i]).to_array()).all()
    # wrong level for this key
    if ct_level > 0:
        A0 = F.Ciphertext(gpar, count, 2, level=0)
        with pytest.raises(F.FheError) as e:
            ggk[3].relinearize(A0)
        assert e.value.code == -6


def test_full_size_set_c(oracle, F):
    """BASELINE configs 3/4 shape: N = 2^15, 14 x 62-bit.  One product and one rotation bit-exact against the
    oracle, plus size-independent properties on a batch: commutativity of the product (canonical outputs),
    backward(forward(x)) == x, and (a + b) - b == a."""
    degree, t, L = 1 << 15, 786433, 14
    opar = oracle.BfvParameters(degree, t, moduli_sizes=[62] * L)
    gpar = F.BfvParameters(degree, t, moduli_sizes=[62] * L)
    assert gpar.moduli() == opar.moduli
    rng = np.random.default_rng(2024)
    ctx = opar.context_at_level(0)

    def rnd(n, parts):
        a = np.zeros((n, parts, L, degree), np.uint64)
        for i, q in enumerate(ctx.moduli):
            a[:, :, i, :] = rng.integers(0, q, size=(n, parts, degree), dtype=np.uint64)
        return a
    kc = rnd(2, L)          # random key material is enough for bit-exactness
    gc = rnd(2, L)
    ork = oracle.RelinearizationKey.from_ksk(oracle.KeySwitchingKey.from_arrays(opar, kc[0], kc[1]))
    grk = F.RelinearizationKey.from_arrays(gpar, kc[0], kc[1])
    count = 3
    a, b = rnd(count, 2), rnd(count, 2)
    A, B = F.Ciphertext.from_host(gpar, a), F.Ciphertext.from_host(gpar, b)
    gm = F.Multiplicator.default(grk)
    P = gm.multiply(A, B).to_host()
    exp = oracle.Multiplicator.default(ork).multiply(oracle.Ciphertext.from_array(opar, a[0], 0),
                                                     oracle.Ciphertext.from_array(opar, b[0], 0))
    assert (P[0] == exp.to_array()).all()
    assert (gm.multiply(B, A).to_host() == P).all()
    # rotation (config 4)
    ogk = oracle.GaloisKey.__new__(oracle.GaloisKey)
    ogk.exponent, ogk.ksk = 3, oracle.KeySwitchingKey.from_arrays(opar, gc[0], gc[1])
    ggk = F.GaloisKey.from_arrays(gpar, 3, gc[0], gc[1])
    R = ggk.relinearize(A).to_host()
    assert (R[0] == ogk.relinearize(oracle.Ciphertext.from_array(opar, a[0], 0)).to_array()).all()
    # NTT round trip and add/sub on the batch
    X = F.Ciphertext.from_host(gpar, a)
    assert (X.into_power_basis().into_ntt().to_host() == a).all()
    S = A + B
    S -= B
    assert (S.to_host() == a).all()


@pytest.mark.parametrize("degree,sizes", [(16, [62, 62, 62]), (64, [50, 36, 20]), (4096, [62, 62])])
def test_wire_format(oracle, F, degree, sizes):
    """From<&Poly> for Rq / TryConvertFrom<&Rq> (rq/convert.rs:17-131): bit-packed power-basis coefficients"""
    t = 1153 if degree < 4096 else 1032193
    opar, gpar, rng = make_pair(oracle, F, degree, len(sizes), t, 7, sizes)
    ctx = opar.context_at_level(0)
    x = rand_ct(oracle, opar, rng, 3)
    X = F.Ciphertext.from_host(gpar, x)                     # NTT batch
    blobs = X.to_packed()
    assert blobs.shape[2] == sum((q - 1).bit_length() * degree // 8 for q in ctx.moduli)
    for c in range(3):
        for p in range(2):
            exp = oracle.poly_to_rq_coefficients(oracle.Poly(ctx, oracle.NTT, x[c, p]))
            assert blobs[c, p].tobytes() == exp
    Y = F.Ciphertext.from_packed(gpar, blobs, repr=F.NTT)
    assert (Y.to_host() == x).all()
    # power-basis batch: packing is the plain transcode of the stored words
    Z = F.Ciphertext.from_host(gpar, x, repr=F.POWER_BASIS)
    zb = Z.to_packed()
    for c in range(3):
        for p in range(2):
            assert zb[c, p].tobytes() == oracle.poly_to_rq_coefficients(oracle.Poly(ctx, oracle.POWER_BASIS, x[c, p]))
    W = F.Ciphertext.from_packed(gpar, zb, repr=F.POWER_BASIS)
    assert (W.to_host() == x).all()
    with pytest.raises(F.FheError):
        F.Ciphertext.from_packed(gpar, zb[:, :, :-1], repr=F.NTT)


@pytest.mark.parametrize("degree,nmod,n_terms,groups", [(16, 2, 1, 1), (16, 3, 7, 3), (64, 2, 20, 2), (4096, 2, 5, 2)])
def test_dot_product_scalar(oracle, F, degree, nmod, n_terms, groups):
    """dot_product_scalar (bfv/ops/dot_product.rs:55-184, tests :186-260): bit-exact against the oracle for several
    independent dot products per call, with the ciphertext or the plaintext operand shared across them, on 2- and
    3-part ciphertexts; error behaviour of the reference."""
    t = 1153
    opar, gpar, rng = make_pair(oracle, F, degree, nmod, t, 31 + n_terms)
    ctx = opar.context_at_level(0)
    for parts in (2, 3):
        carr = rand_ct(oracle, opar, rng, groups * n_terms, parts)
        parr = rand_ct(oracle, opar, rng, groups * n_terms, 1)[:, 0]
        octs = [oracle.Ciphertext.from_array(opar, a, 0) for a in carr]
        opts = [oracle.Poly(ctx, oracle.NTT, a.copy()) for a in parr]
        X = F.Ciphertext.from_host(gpar, carr)
        got = F.dot_product_scalar(X, parr, n_terms).to_host()
        assert got.shape[0] == groups
        for g in range(groups):
            sl = slice(g * n_terms, (g + 1) * n_terms)
            assert (got[g] == oracle.dot_product_scalar(octs[sl], opts[sl]).to_array()).all()
        # shared ciphertexts (the PIR query), per-group plaintexts; then the other way round
        Xs = F.Ciphertext.from_host(gpar, carr[:n_terms])
        got = F.dot_product_scalar(Xs, parr, n_terms).to_host()
        for g in range(groups):
            sl = slice(g * n_terms, (g + 1) * n_terms)
            assert (got[g] == oracle.dot_product_scalar(octs[:n_terms], opts[sl]).to_array()).all()
        got = F.dot_product_scalar(X, parr[:n_terms], n_terms).to_host()
        for g in range(groups):
            sl = slice(g * n_terms, (g + 1) * n_terms)
            assert (got[g] == oracle.dot_product_scalar(octs[sl], opts[:n_terms]).to_array()).all()
    # one dot product over the whole batch (n_terms defaults to the batch size)
    got = F.dot_product_scalar(X, parr).to_host()
    assert got.shape[0] == 1 and (got[0] == oracle.dot_product_scalar(octs, opts).to_array()).all()
    # errors (dot_product.rs:60-70, :93-101)
    with pytest.raises(F.FheError) as e:
        F.dot_product_scalar(X, np.zeros((0, nmod, degree), np.uint64))
    assert e.value.code == -1
    if groups * n_terms > 2:
        with pytest.raises(F.FheError) as e:   # operand counts do not match
            F.dot_product_scalar(X, parr[:groups * n_terms - 1], groups * n_terms)
        assert e.value.code == -1
    if nmod >= 2:
        with pytest.raises(F.FheError) as e:   # plaintext at another level
            lower = F.Ciphertext(gpar, groups * n_terms, 1, level=1)
            F.dot_product_scalar(X, lower, n_terms)
        assert e.value.code == -6


@pytest.mark.parametrize("degree,sizes", [(16, [62, 62, 62]), (64, [62, 50]), (4096, [62])])
def test_single_modulus_key_switch(oracle, F, degree, sizes):
    """KeySwitchingKey at a level with one modulus (key_switching_key.rs:92-110): base-2^(log q / 2) decomposition,
    key_switch_decomposition (:323-362); and the RGSW external product at that level (rgsw_ciphertext.rs:122-155)."""
    t = 1153
    opar = oracle.BfvParameters(degree, t, moduli_sizes=sizes)
    gpar = F.BfvParameters(degree, t, moduli=opar.moduli, device=0)
    rng = np.random.default_rng(5 + degree)
    last = len(sizes) - 1
    ctx = opar.context_at_level(last)
    sk = oracle.SecretKey(opar, rng)
    frm = oracle.Poly.random(ctx, oracle.POWER_BASIS, rng)
    ok = oracle.KeySwitchingKey(sk, frm, last, last, rng)
    assert ok.log_base > 0 and len(ok.c0) in (2, 3)
    gk = F.KeySwitchingKey.from_arrays(gpar, *ok.arrays(), ciphertext_level=last, key_level=last)
    x = rand_ct(oracle, opar, rng, 3, 2, level=last)
    X = F.Ciphertext.from_host(gpar, x, level=last, repr=F.POWER_BASIS)
    for part in (0, 1):
        got = gk.key_switch(X, part).to_host()
        for i in range(3):
            c0, c1 = ok.key_switch(oracle.Poly(ctx, oracle.POWER_BASIS, x[i, part].copy()))
            assert (got[i, 0] == c0.c).all() and (got[i, 1] == c1.c).all()
    # wrong digit count / a single-modulus key for a ciphertext level with more limbs
    with pytest.raises(F.FheError) as e:
        F.KeySwitchingKey.from_arrays(gpar, ok.arrays()[0][:1], ok.arrays()[1][:1], ciphertext_level=last, key_level=last)
    assert e.value.code == -5
    if degree <= 64:   # RGSW external product at the last level decrypts to the product (rgsw_ciphertext.rs tests)
        m1, m2 = rng.integers(0, t, degree), rng.integers(0, t, degree)
        ct = sk.encrypt(oracle.simd_encode(opar, m1), last, rng)
        m2_ntt = oracle.Poly.from_u64(ctx, oracle.simd_encode(opar, m2), oracle.NTT)
        org = oracle.RGSWCiphertext(sk, m2_ntt, last, rng)
        grg = F.RGSWCiphertext.from_arrays(gpar, *org.ksk0.arrays(), *org.ksk1.arrays(), level=last)
        CT = F.Ciphertext.from_host(gpar, ct.to_array()[None], level=last)
        got = grg.external_product(CT).to_host()[0]
        assert (got == org.external_product(ct).to_array()).all()
        dec = oracle.simd_decode(opar, sk.decrypt(oracle.Ciphertext.from_array(opar, got, last)))
        assert (dec.astype(np.int64) == (m1 * m2) % t).all()


def test_mul_plain_inner_sum_expand(oracle, F):
    """Ciphertext * Plaintext (ops/mod.rs:229-238), EvaluationKey::computes_inner_sum (evaluation_key.rs:56-100)
    and EvaluationKey::expands (:192-256) -- the PIR examples' loops, built from the same kernels"""
    degree, t = 16, 1153
    opar, gpar, rng = make_pair(oracle, F, degree, 3, t, 123)
    exps = sorted({pow(3, 1 << k, 2 * degree) for k in range(3)} | {2 * degree - 1} | {(degree >> l) + 1 for l in range(2)})
    sk, ork, grk, ogk, ggk = _keys(oracle, F, opar, gpar, rng, exps)
    vals = rng.integers(0, t, size=(2, degree))
    octs = [sk.encrypt(oracle.simd_encode(opar, v), 0, rng) for v in vals]
    X = F.Ciphertext.from_host(gpar, np.stack([c.to_array() for c in octs]))
    # ct * pt
    pt = oracle.plaintext_to_poly(opar, rng.integers(0, t, degree), 0)    # any NTT-domain polynomial of the level
    got = X.clone().mul_plain(pt.c).to_host()
    for i in range(2):
        assert (got[i] == np.stack([p.mul(pt).c for p in octs[i].c])).all()
    per_ct = np.stack([oracle.Poly.random(opar.context_at_level(0), oracle.NTT, rng).c for _ in range(2)])
    got = X.clone().mul_plain(per_ct).to_host()
    for i in range(2):
        w = oracle.Poly(opar.context_at_level(0), oracle.NTT, per_ct[i])
        assert (got[i] == np.stack([p.mul(w).c for p in octs[i].c])).all()
    # ct + pt, ct - pt (ops/mod.rs:88-97, :188-197): part 0 +/- Plaintext::to_poly(); decrypts to the slot-wise sum
    pv = rng.integers(0, t, degree)
    dp = oracle.plaintext_to_poly(opar, oracle.simd_encode(opar, pv), 0)
    got_add = X.clone().add_plain(dp.c).to_host()
    got_sub = X.clone().sub_plain(dp.c).to_host()
    for i in range(2):
        ea = octs[i].copy(); ea.c[0] = ea.c[0].copy().iadd(dp)
        es = octs[i].copy(); es.c[0] = es.c[0].copy().isub(dp)
        assert (got_add[i] == ea.to_array()).all() and (got_sub[i] == es.to_array()).all()
        dec = oracle.simd_decode(opar, sk.decrypt(oracle.Ciphertext.from_array(opar, got_add[i], 0)))
        assert (dec.astype(np.int64) == (vals[i] + pv) % t).all()
        dec = oracle.simd_decode(opar, sk.decrypt(oracle.Ciphertext.from_array(opar, got_sub[i], 0)))
        assert (dec.astype(np.int64) == (vals[i] - pv) % t).all()
    # inner sum
    ek = F.EvaluationKey(gpar)
    for e in exps:
        ek.add_galois_key(ggk[e])
    assert ek.supports_inner_sum()
    got = ek.computes_inner_sum(X).to_host()
    for i in range(2):
        exp = oracle.computes_inner_sum(opar, ogk, octs[i])
        assert (got[i] == exp.to_array()).all()
        dec = oracle.simd_decode(opar, sk.decrypt(oracle.Ciphertext.from_array(opar, got[i], 0)))
        assert (dec == np.full(degree, int(vals[i].sum()) % t, dtype=np.uint64)).all()
    # oblivious expansion to 4 ciphertexts
    monos = [oracle.expansion_monomial(opar, l).c for l in range(2)]
    outs = ek.expands(X, 4, monos)
    for i in range(2):
        exp = oracle.expands(opar, ogk, octs[i], 4)
        for k in range(4):
            assert (outs[k].to_host()[i] == exp[k].to_array()).all()


def test_rgsw_external_product(oracle, F):
    """&Ciphertext * &RGSWCiphertext (rgsw_ciphertext.rs:122-155) through the key-switch primitive"""
    degree, t = 64, 1153
    opar, gpar, rng = make_pair(oracle, F, degree, 3, t, 321)
    sk = oracle.SecretKey(opar, rng)
    m2 = rng.integers(0, t, degree)
    pt_ntt = oracle.Poly.from_u64(opar.context_at_level(0), m2.astype(np.uint64), oracle.NTT)
    org = oracle.RGSWCiphertext(sk, pt_ntt, 0, rng)
    grg = F.RGSWCiphertext.from_arrays(gpar, *org.ksk0.arrays(), *org.ksk1.arrays())
    octs = [sk.encrypt(rng.integers(0, t, degree), 0, rng) for _ in range(3)]
    X = F.Ciphertext.from_host(gpar, np.stack([c.to_array() for c in octs]))
    got = grg.external_product(X).to_host()
    for i in range(3):
        assert (got[i] == org.external_product(octs[i]).to_array()).all()


def _rand_rows(rng, moduli, shape_prefix, degree):
    a = np.zeros(tuple(shape_prefix) + (len(moduli), degree), np.uint64)
    for i, q in enumerate(moduli):
        a[..., i, :] = rng.integers(0, q, size=tuple(shape_prefix) + (degree,), dtype=np.uint64)
    return a


@pytest.mark.parametrize("variant", ["plain", "mod_switch", "key_level_0_ct_level_1"])
def test_set_c_across_chunk_boundary(oracle, F, variant):
    """The shape the headline number is measured on (N = 2^15, 14 x 62-bit) with MORE ciphertexts than one internal
    chunk (256): products 0, 255, 256, 257 of a 258-pair batch and rotations 0 / 256 / 257 are compared with the
    oracle, so the chunk loop, its tail chunk and every per-chunk offset of mul_relin / galois are covered --
    plain, with modulus switching (mul.rs:296-330), and with a level-0 key serving level-1 ciphertexts
    (relinearization_key.rs:88-95, galois_key.rs:69-76)."""
    degree, t, L = 1 << 15, 786433, 14
    opar = oracle.BfvParameters(degree, t, moduli_sizes=[62] * L)
    gpar = F.BfvParameters(degree, t, moduli_sizes=[62] * L)
    rng = np.random.default_rng(77)
    ct_level = 1 if variant == "key_level_0_ct_level_1" else 0
    key_mod = opar.context_at_level(0).moduli
    ct_mod = opar.context_at_level(ct_level).moduli
    n_dig = len(ct_mod)
    kc = _rand_rows(rng, key_mod, (2, n_dig), degree)      # [c0|c1][digit][key limb][N]
    gc = _rand_rows(rng, key_mod, (2, n_dig), degree)
    oksk = oracle.KeySwitchingKey.from_arrays(opar, kc[0], kc[1], ct_level, 0)
    ork = oracle.RelinearizationKey.from_ksk(oksk)
    grk = F.RelinearizationKey.from_arrays(gpar, kc[0], kc[1], ciphertext_level=ct_level, key_level=0)
    ogk = oracle.GaloisKey.__new__(oracle.GaloisKey)
    ogk.exponent, ogk.ksk = 3, oracle.KeySwitchingKey.from_arrays(opar, gc[0], gc[1], ct_level, 0)
    ggk = F.GaloisKey.from_arrays(gpar, 3, gc[0], gc[1], ciphertext_level=ct_level, key_level=0)
    count = 258
    a = _rand_rows(rng, ct_mod, (count, 2), degree)
    b = _rand_rows(rng, ct_mod, (count, 2), degree)
    A = F.Ciphertext.from_host(gpar, a, level=ct_level)
    B = F.Ciphertext.from_host(gpar, b, level=ct_level)
    om, gm = oracle.Multiplicator.default(ork), F.Multiplicator.default(grk)
    if variant == "mod_switch":
        om.enable_mod_switching()
        gm.enable_mod_switching()
    out = gm.multiply(A, B)
    assert out.level == ct_level + (1 if variant == "mod_switch" else 0)
    P = out.to_host()
    for i in (0, 255, 256, 257):
        exp = om.multiply(oracle.Ciphertext.from_array(opar, a[i], ct_level),
                          oracle.Ciphertext.from_array(opar, b[i], ct_level))
        assert (P[i] == exp.to_array()).all(), "product %d differs" % i
    R = ggk.relinearize(A).to_host()
    for i in (0, 256, 257):
        exp = ogk.relinearize(oracle.Ciphertext.from_array(opar, a[i], ct_level))
        assert (R[i] == exp.to_array()).all(), "rotation %d differs" % i
    if variant == "plain":
        # &ct * &ct then relinearizes, across the boundary as well
        C3 = A * B
        R2 = grk.relinearizes(C3).to_host()
        assert (R2 == P).all()


def test_set_b_ntt_config(oracle, F):
    """BASELINE configs[1]: N = 2^14, 8 x 62-bit.  (a) the full [256][8][2^14] buffer the roofline leg of bench.py
    times: backward(forward(x)) == x on every word, and rows of forward(x) equal to the oracle's transform;
    (b) one ct x ct mul + relinearize and one rotation against the oracle (ntt/mod.rs:50-82, mul.rs:263-330)."""
    degree, t, L = 1 << 14, 786433, 8
    opar = oracle.BfvParameters(degree, t, moduli_sizes=[62] * L)
    gpar = F.BfvParameters(degree, t, moduli_sizes=[62] * L)
    assert gpar.moduli() == opar.moduli
    ctx = opar.context_at_level(0)
    rng = np.random.default_rng(14)
    x = _rand_rows(rng, ctx.moduli, (256, 1), degree)
    X = F.Ciphertext.from_host(gpar, x, repr=F.POWER_BASIS)
    fwd = X.into_ntt().to_host()
    for c in (0, 100, 255):
        for i, op in enumerate(ctx.ops):
            e = x[c, 0, i].copy()
            op.forward(e)
            assert (fwd[c, 0, i] == e).all()
    assert (X.into_power_basis().to_host() == x).all()
    # mul + relin and rotation
    kc, gc = _rand_rows(rng, ctx.moduli, (2, L), degree), _rand_rows(rng, ctx.moduli, (2, L), degree)
    ork = oracle.RelinearizationKey.from_ksk(oracle.KeySwitchingKey.from_arrays(opar, kc[0], kc[1]))
    grk = F.RelinearizationKey.from_arrays(gpar, kc[0], kc[1])
    a, b = _rand_rows(rng, ctx.moduli, (3, 2), degree), _rand_rows(rng, ctx.moduli, (3, 2), degree)
    A, B = F.Ciphertext.from_host(gpar, a), F.Ciphertext.from_host(gpar, b)
    P = F.Multiplicator.default(grk).multiply(A, B).to_host()
    om = oracle.Multiplicator.default(ork)
    for i in (0, 2):
        exp = om.multiply(oracle.Ciphertext.from_array(opar, a[i], 0), oracle.Ciphertext.from_array(opar, b[i], 0))
        assert (P[i] == exp.to_array()).all()
    ogk = oracle.GaloisKey.__new__(oracle.GaloisKey)
    ogk.exponent, ogk.ksk = 3, oracle.KeySwitchingKey.from_arrays(opar, gc[0], gc[1])
    R = F.GaloisKey.from_arrays(gpar, 3, gc[0], gc[1]).relinearize(A).to_host()
    assert (R[1] == ogk.relinearize(oracle.Ciphertext.from_array(opar, a[1], 0)).to_array()).all()


def test_two_devices_one_process(oracle, F):
    """One host process driving parameter sets on two devices (a Rust host holding one Arc<BfvParameters> per GPU):
    kernels that need the opt-in shared-memory size (4096-word NTT tiles at N = 2^16, the TMA kernels at N = 2^15)
    must get it on every device, the caller's current device is left alone, and both devices give the oracle's
    words.  Skipped on a one-GPU box."""
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two CUDA devices")
    torch.cuda.set_device(0)
    rng = np.random.default_rng(31)
    for logn, nmod in ((16, 1), (15, 2)):
        n = 1 << logn
        opar = oracle.BfvParameters(n, 786433, moduli_sizes=[62] * nmod)
        ctx = opar.context_at_level(0)
        x = _rand_rows(rng, ctx.moduli, (8, 2), n)
        exp = x.copy()
        for i, op in enumerate(ctx.ops):
            op.forward(exp[0, 0, i])
        for dev in (0, 1, 0):
            gpar = F.BfvParameters(n, 786433, moduli=opar.moduli, device=dev)
            ct = F.Ciphertext.from_host(gpar, x, repr=F.POWER_BASIS)
            got = ct.into_ntt().to_host()
            assert (got[0, 0] == exp[0, 0]).all(), "device %d" % dev
            assert (ct.into_power_basis().to_host() == x).all()
            assert torch.cuda.current_device() == 0, "the library changed the caller's current device"
    # set A multiply on device 1 against the oracle
    degree, t = 1 << 12, 1032193
    opar = oracle.BfvParameters(degree, t, moduli_sizes=[62, 62])
    gpar = F.BfvParameters(degree, t, moduli=opar.moduli, device=1)
    sk = oracle.SecretKey(opar, rng)
    ork = oracle.RelinearizationKey(sk, rng)
    grk = F.RelinearizationKey.from_arrays(gpar, *ork.ksk.arrays())
    ca, cb = sk.encrypt(rng.integers(0, t, degree), 0, rng), sk.encrypt(rng.integers(0, t, degree), 0, rng)
    A = F.Ciphertext.from_host(gpar, ca.to_array()[None])
    B = F.Ciphertext.from_host(gpar, cb.to_array()[None])
    got = F.Multiplicator.default(grk).multiply(A, B).to_host()[0]
    assert (got == oracle.Multiplicator.default(ork).multiply(ca, cb).to_array()).all()
    assert torch.cuda.current_device() == 0


def test_packed_mul_basis_batch(oracle, F):
    """pack / unpack of a batch over the multiplication basis (L + E limbs): the host buffer is sized per batch
    (fhe_b200_batch_packed_bytes), and the blobs decode back to the same words"""
    opar, gpar, rng = make_pair(oracle, F, 64, 3, 1153, 5)
    mp = opar.level(0).mul_params
    K = len(mp.to.moduli)
    y = np.zeros((2, 2, K, 64), np.uint64)
    for i, q in enumerate(mp.to.moduli):
        y[:, :, i, :] = rng.integers(0, q, size=(2, 2, 64), dtype=np.uint64)
    Y = F.Ciphertext.from_host(gpar, y, mul_basis=True, repr=F.POWER_BASIS)
    blobs = Y.to_packed()
    assert blobs.shape[2] == sum((q - 1).bit_length() * 64 // 8 for q in mp.to.moduli)
    for i, q in enumerate(mp.to.moduli):
        off = sum((qq - 1).bit_length() * 8 for qq in mp.to.moduli[:i])
        nb = (q - 1).bit_length()
        assert oracle.transcode_from_bytes(bytes(blobs[1, 0, off:off + nb * 8]), nb)[:64] == [int(v) for v in y[1, 0, i]]


def test_mixed_sizes_through_tma_kernels(oracle, F):
    """N = 2^13 with moduli of very different sizes: the key-switch digits (below the largest modulus) exceed four
    times the smallest one, so the digit transform must reduce its source words as it reads them (zq/mod.rs:756,
    rq/mod.rs:563-586) -- the REDUCE variant of the TMA cols kernel -- and the scaler's output limbs are not all
    Solinas primes (per-tile scaler kernel).  Multiply + relinearize and a rotation against the oracle."""
    degree, t, sizes = 1 << 13, 65537, [62, 40, 30]
    opar = oracle.BfvParameters(degree, t, moduli_sizes=sizes)
    gpar = F.BfvParameters(degree, t, moduli=opar.moduli)
    rng = np.random.default_rng(813)
    ctx = opar.context_at_level(0)
    L = len(sizes)
    kc, gc = _rand_rows(rng, ctx.moduli, (2, L), degree), _rand_rows(rng, ctx.moduli, (2, L), degree)
    ork = oracle.RelinearizationKey.from_ksk(oracle.KeySwitchingKey.from_arrays(opar, kc[0], kc[1]))
    grk = F.RelinearizationKey.from_arrays(gpar, kc[0], kc[1])
    count = 5
    a, b = _rand_rows(rng, ctx.moduli, (count, 2), degree), _rand_rows(rng, ctx.moduli, (count, 2), degree)
    A, B = F.Ciphertext.from_host(gpar, a), F.Ciphertext.from_host(gpar, b)
    P = F.Multiplicator.default(grk).multiply(A, B).to_host()
    om = oracle.Multiplicator.default(ork)
    for i in (0, count - 1):
        exp = om.multiply(oracle.Ciphertext.from_array(opar, a[i], 0), oracle.Ciphertext.from_array(opar, b[i], 0))
        assert (P[i] == exp.to_array()).all()
    ogk = oracle.GaloisKey.__new__(oracle.GaloisKey)
    ogk.exponent, ogk.ksk = 3, oracle.KeySwitchingKey.from_arrays(opar, gc[0], gc[1])
    R = F.GaloisKey.from_arrays(gpar, 3, gc[0], gc[1]).relinearize(A).to_host()
    for i in (0, count - 1):
        assert (R[i] == ogk.relinearize(oracle.Ciphertext.from_array(opar, a[i], 0)).to_array()).all()


@pytest.mark.parametrize("degree,nmod", [(16, 6), (64, 3), (8192, 2)])
def test_messages_against_oracle(oracle, F, degree, nmod):
    """The protobuf messages either side of the path (SURVEY 8f row 1): `Ciphertext::{to_bytes, from_bytes}`
    (bfv/ciphertext.rs:230-317), key-switching / relinearization / Galois keys and RGSW ciphertexts
    (keys/key_switching_key.rs:365-482, relinearization_key.rs:113-141, galois_key.rs:146-173,
    rgsw_ciphertext.rs:30-71): bytes produced by the oracle are consumed by the device path and give the oracle's
    words and results; bytes produced by the device path are the oracle's bytes."""
    import fhe_wire as ow
    t = 65537
    opar, gpar, rng = make_pair(oracle, F, degree, nmod, t, 300 + degree)
    sk = oracle.SecretKey(opar, rng)
    last = nmod - 1

    cts = [sk.encrypt(rng.integers(0, t, degree), 0, rng) for _ in range(3)]
    for batch in (cts, [c.mul(c) for c in cts[:2]], [c.copy().switch_to_level(1) for c in cts]):
        msgs = [ow.ciphertext_to_bytes(c) for c in batch]
        G = F.Ciphertext.from_bytes(gpar, msgs)
        assert G.level == batch[0].level and len(G) == len(batch[0].c)
        assert (G.to_host() == np.stack([c.to_array() for c in batch])).all()
        assert G.to_bytes() == msgs
    # seeded ciphertexts: the last polynomial travels as a seed and is expanded by the host
    seeded = [ow.ciphertext_to_bytes(c, seed=bytes([i]) * 32) for i, c in enumerate(cts)]
    G = F.Ciphertext.from_bytes(gpar, seeded, seeded_halves=np.stack([c.c[1].c for c in cts]))
    assert (G.to_host() == np.stack([c.to_array() for c in cts])).all()
    with pytest.raises(F.WireError) as e:
        F.Ciphertext.from_bytes(gpar, seeded)
    assert e.value.variant == "SeedExpansion" and e.value.code == -11

    # keys from their messages: the results of the path are the oracle's
    ork = oracle.RelinearizationKey(sk, rng)
    ogk = oracle.GaloisKey(sk, 3, rng)
    grk = F.RelinearizationKey.from_bytes(gpar, ow.relin_key_to_bytes(ork))
    ggk = F.GaloisKey.from_bytes(gpar, ow.galois_key_to_bytes(ogk))
    assert grk.to_bytes() == ow.relin_key_to_bytes(ork) and ggk.to_bytes() == ow.galois_key_to_bytes(ogk)
    A = F.Ciphertext.from_bytes(gpar, [ow.ciphertext_to_bytes(c) for c in cts[:2]])
    B = F.Ciphertext.from_bytes(gpar, [ow.ciphertext_to_bytes(c) for c in cts[1:]])
    out = F.Multiplicator.default(grk).multiply(A, B)
    om = oracle.Multiplicator.default(ork)
    assert out.to_bytes() == [ow.ciphertext_to_bytes(om.multiply(cts[i], cts[i + 1])) for i in range(2)]
    assert ggk.relinearize(A).to_bytes() == [ow.ciphertext_to_bytes(ogk.relinearize(c)) for c in cts[:2]]
    # a seeded key: c1 row from the host
    seeded_key = ow.ksk_to_bytes(ork.ksk, seed=b"k" * 32)
    k2 = F.KeySwitchingKey.from_bytes(gpar, seeded_key, seeded_c1=np.stack([p.c for p in ork.ksk.c1]))
    assert k2.to_bytes() == ow.ksk_to_bytes(ork.ksk)
    # the last level has one modulus: base-2^31 digits (key_switching_key.rs:92-110, :401-409), RGSW at that level
    m = oracle.Poly.random(opar.context_at_level(last), oracle.NTT, rng)
    org = oracle.RGSWCiphertext(sk, m, last, rng)
    grg = F.RGSWCiphertext.from_bytes(gpar, ow.rgsw_to_bytes(org))
    assert grg.to_bytes() == ow.rgsw_to_bytes(org)
    low = cts[0].copy().switch_to_level(last)
    got = grg.external_product(F.Ciphertext.from_bytes(gpar, [ow.ciphertext_to_bytes(low)]))
    assert got.to_bytes() == [ow.ciphertext_to_bytes(org.external_product(low))]

    # rejections carry the reference's variant names (the oracle raises the same ones on the same bytes)
    def both(variant, data, gpu_call, oracle_call):
        with pytest.raises(F.WireError) as e:
            gpu_call(data)
        assert e.value.variant == variant
        with pytest.raises(ow.WireError, match=variant):
            oracle_call(data)

    good = ow.CiphertextProto()
    good.ParseFromString(ow.ciphertext_to_bytes(cts[0]))
    rq = ow.Rq()
    rq.ParseFromString(good.c[0])
    for change, variant in ((dict(representation=0), "UnknownRepresentation"), (dict(representation=1), "RepresentationMismatch"),
                            (dict(degree=6), "InvalidDegree"), (dict(coefficients=rq.coefficients[:-1]), "InvalidCoefficientCount"),
                            (dict(degree=degree * 2), "InvalidCoefficientCount")):
        bad_rq = ow.Rq()
        bad_rq.CopyFrom(rq)
        for k, v in change.items():
            setattr(bad_rq, k, v)
        bad = ow.CiphertextProto()
        bad.CopyFrom(good)
        bad.c[0] = bad_rq.SerializeToString()
        both(variant, bad.SerializeToString(), lambda d: F.Ciphertext.from_bytes(gpar, [d]),
             lambda d: ow.ciphertext_from_bytes(opar, d))
    bad = ow.CiphertextProto()
    bad.CopyFrom(good)
    bad.level = nmod
    both("InvalidLevel", bad.SerializeToString(), lambda d: F.Ciphertext.from_bytes(gpar, [d]),
         lambda d: ow.ciphertext_from_bytes(opar, d))
    both("InvalidCiphertextPolynomialCount", ow.CiphertextProto(c=[good.c[0]]).SerializeToString(),
         lambda d: F.Ciphertext.from_bytes(gpar, [d]), lambda d: ow.ciphertext_from_bytes(opar, d))
    both("Decode", ow.ciphertext_to_bytes(cts[0])[:-5], lambda d: F.Ciphertext.from_bytes(gpar, [d]),
         lambda d: ow.ciphertext_from_bytes(opar, d))
    key = ow.KeySwitchingKeyProto()
    key.ParseFromString(ow.ksk_to_bytes(ork.ksk))
    del key.c0[-1]
    both("WrongPolynomialCount", key.SerializeToString(), lambda d: F.KeySwitchingKey.from_bytes(gpar, d),
         lambda d: ow.ksk_from_bytes(opar, d))
    key.ParseFromString(ow.ksk_to_bytes(ork.ksk))
    key.log_base = 31
    both("InvalidKeySwitchingDecompositionLevels", key.SerializeToString(), lambda d: F.KeySwitchingKey.from_bytes(gpar, d),
         lambda d: ow.ksk_from_bytes(opar, d))
    gal = ow.GaloisKeyProto()
    gal.ParseFromString(ow.galois_key_to_bytes(ogk))
    gal.exponent = 2 * degree + 4
    both("InvalidSubstitutionExponent", gal.SerializeToString(), lambda d: F.GaloisKey.from_bytes(gpar, d),
         lambda d: ow.galois_key_from_bytes(opar, d))
    both("MissingField", b"", lambda d: F.RelinearizationKey.from_bytes(gpar, d), lambda d: ow.relin_key_from_bytes(opar, d))
    if degree == 16:   # one modulus: a shorter polynomial is a low-order one, zero-extended (rq/convert.rs:160-183)
        ctx8 = oracle.Context(opar.moduli[:1], 8)
        short = [oracle.Poly.random(ctx8, oracle.NTT, rng) for _ in range(2)]
        data = ow.CiphertextProto(c=[ow.poly_to_bytes(p) for p in short], level=last).SerializeToString()
        got = F.Ciphertext.from_bytes(gpar, [data])
        assert (got.to_host()[0] == ow.ciphertext_from_bytes(opar, data).to_array()).all()


@pytest.mark.parametrize("env", [{"FHE_B200_CHUNK": "2"}, {"FHE_B200_CHUNK": "3", "FHE_B200_STREAMS": "3"},
                                 {"FHE_B200_CHUNK": "4", "FHE_B200_STREAMS": "4"}, {"FHE_B200_CHUNK": "2", "FHE_B200_STREAMS": "1"}])
def test_chunk_runner_entry_points(F, env):
    """capi.cu::ChunkRunner: a batched call deals its chunks over side streams of the parameter set; every chunked entry
    point, on a batch of several chunks, equals the same call on one-ciphertext batches (tests/chunk_runner_probe.py).
    Oracle parity across the chunk boundary at the benchmarked size is test_set_c_across_chunk_boundary."""
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    out = subprocess.run([sys.executable, os.path.join(root, "tests", "chunk_runner_probe.py")], cwd=root,
                         env=dict(os.environ, **env), capture_output=True, text=True, timeout=600)
    assert out.returncode == 0 and "chunk runner probe ok" in out.stdout, out.stdout[-2000:] + out.stderr[-2000:]
