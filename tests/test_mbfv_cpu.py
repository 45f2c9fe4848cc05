"""CPU tests of multiparty BFV (fhe::mbfv): the reference's protocol tests run on tests/mbfv_reference.py's restatement
over the oracle, the stream roles of the new calls, the from_shares lift against try_decrypt's, and the refusals and
symbols that need no device."""
import ctypes as C
import os
import re

import numpy as np
import pytest

import encrypt_reference as R
import mbfv_reference as M

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
VAR = 10
# BfvParameters::default_arc(num_moduli, degree) (parameters.rs:299-309): t = 1153, 62-bit moduli
SHAPES = [(1, 16), (6, 32), (3, 16)]


@pytest.fixture(scope="module")
def F():
    import fhe_rs_b200
    return fhe_rs_b200


def default_arc(oracle, n_moduli, degree):
    return oracle.BfvParameters(degree, 1153, moduli_sizes=[62] * n_moduli)


def seeds(rng, n):
    return [rng.integers(0, 256, size=32, dtype=np.uint8).tobytes() for _ in range(n)]


def summed_key(oracle, par, keys):
    """SecretKey(sum s_i), the key the parties' shares add up to"""
    k = object.__new__(oracle.SecretKey)
    k.par, k.coeffs = par, np.sum([s.coeffs for s in keys], axis=0).astype(np.int64)
    return k


def collective_pk(oracle, par, parties, rng):
    """PublicKeyShare of every party for one CRP, aggregated"""
    a = M.crp(par, seeds(rng, 1)[0], 1)[0]
    shares = [M.pk_share(sk, [a], sd, VAR)[0] for sk, sd in zip(parties, seeds(rng, len(parties)))]
    return M.pk_aggregate(par, shares, a)


def encrypt_values(oracle, par, pk, rng, level):
    values = rng.integers(0, par.plaintext, size=par.degree, dtype=np.uint64)
    m = R.to_poly(par, values, level)
    return R.encrypt_pk(par, pk, seeds(rng, 1)[0], 1, level, VAR, [m])[0], values


def collective_decrypt(parties, ct, rng):
    hs = [M.sks_share(sk, None, [ct], sd, VAR)[0] for sk, sd in zip(parties, seeds(rng, len(parties)))]
    return M.from_shares(ct, hs)[1]


@pytest.mark.parametrize("shape", SHAPES)
def test_protocol_creates_valid_pk(oracle, shape):
    """public_key_gen.rs tests: encryptions under the aggregated key decrypt under SecretKey(sum s_i)"""
    par = default_arc(oracle, *shape)
    rng = np.random.default_rng(shape[0] * 100 + shape[1])
    for level in range(par.max_level() + 1):
        parties = [oracle.SecretKey(par, rng) for _ in range(5)]
        pk = collective_pk(oracle, par, parties, rng)
        ct, values = encrypt_values(oracle, par, pk, rng, level)
        assert (summed_key(oracle, par, parties).decrypt(ct) == values).all(), level


@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("n_parties", [5, 11])
def test_encrypt_decrypt(oracle, shape, n_parties):
    """secret_key_switch.rs encrypt_decrypt: the collective decryption gives the plaintext"""
    par = default_arc(oracle, *shape)
    rng = np.random.default_rng(shape[0] * 7 + n_parties)
    for level in range(par.max_level() + 1):
        parties = [oracle.SecretKey(par, rng) for _ in range(n_parties)]
        ct, values = encrypt_values(oracle, par, collective_pk(oracle, par, parties, rng), rng, level)
        assert (collective_decrypt(parties, ct, rng) == values).all(), level


@pytest.mark.parametrize("shape", SHAPES)
def test_sks_encrypt_keyswitch_decrypt(oracle, shape):
    """secret_key_switch.rs encrypt_keyswitch_decrypt: switch to a second set of parties, who decrypt collectively"""
    par = default_arc(oracle, *shape)
    rng = np.random.default_rng(shape[0] * 11 + shape[1])
    for level in range(par.max_level() + 1):
        ins = [oracle.SecretKey(par, rng) for _ in range(5)]
        outs = [oracle.SecretKey(par, rng) for _ in range(5)]
        ct1, values = encrypt_values(oracle, par, collective_pk(oracle, par, ins, rng), rng, level)
        hs = [M.sks_share(i, o, [ct1], sd, VAR)[0] for i, o, sd in zip(ins, outs, seeds(rng, 5))]
        ct2 = M.sks_aggregate(ct1, hs)
        assert (collective_decrypt(outs, ct2, rng) == values).all(), level


@pytest.mark.parametrize("shape", SHAPES)
def test_pks_encrypt_keyswitch_decrypt(oracle, shape):
    """public_key_switch.rs encrypt_keyswitch_decrypt: switch to the holder of another public key"""
    par = default_arc(oracle, *shape)
    rng = np.random.default_rng(shape[0] * 13 + shape[1])
    for level in range(par.max_level() + 1):
        ins = [oracle.SecretKey(par, rng) for _ in range(5)]
        ct1, values = encrypt_values(oracle, par, collective_pk(oracle, par, ins, rng), rng, level)
        out_sk = oracle.SecretKey(par, rng)
        out_pk = R.encrypt_sk(out_sk, seeds(rng, 1)[0], 1, 0, VAR)[0]     # PublicKey::new
        shares = [M.pks_share(sk, out_pk, [ct1], sd, VAR)[0] for sk, sd in zip(ins, seeds(rng, 5))]
        ct2 = M.pks_aggregate(ct1, shares)
        assert (out_sk.decrypt(ct2) == values).all(), level


def collective_relin_key(oracle, par, parties, rng):
    """RelinKeyGenerator of every party on the same CRPs: round 1, its aggregate, round 2, RelinearizationKey"""
    crps = M.crp(par, seeds(rng, 1)[0], len(par.moduli))
    us = [M.rkg_u(par, sd, VAR) for sd in seeds(rng, len(parties))]
    r1 = M.rkg_r1_aggregate([M.rkg_round1(sk, crps, u, sd, VAR) for sk, u, sd in zip(parties, us, seeds(rng, len(parties)))])
    r2 = [M.rkg_round2(sk, u, r1[0], r1[1], sd, VAR) for sk, u, sd in zip(parties, us, seeds(rng, len(parties)))]
    c0, c1 = M.rkg_aggregate(r2, r1[1])
    return oracle.RelinearizationKey.from_ksk(oracle.KeySwitchingKey.from_arrays(par, c0, c1))


@pytest.mark.parametrize("shape", [(3, 16), (6, 32)])
@pytest.mark.parametrize("n_parties", [5, 11])
def test_relinearization_works(oracle, shape, n_parties):
    """relin_key_gen.rs relinearization_works: the collective relinearization key drives Multiplicator::default with
    mod switching, and the collective decryption of the product is the slot-wise product"""
    par = default_arc(oracle, *shape)
    rng = np.random.default_rng(shape[0] * 17 + n_parties)
    t = par.plaintext
    parties = [oracle.SecretKey(par, rng) for _ in range(n_parties)]
    pk = collective_pk(oracle, par, parties, rng)
    rk = collective_relin_key(oracle, par, parties, rng)
    v1, v2 = (rng.integers(0, t, size=par.degree, dtype=np.uint64) for _ in range(2))
    cts = [R.encrypt_pk(par, pk, sd, 1, 0, VAR, [R.to_poly(par, oracle.simd_encode(par, v), 0)])[0]
           for v, sd in zip((v1, v2), seeds(rng, 2))]
    m = oracle.Multiplicator.default(rk)
    m.enable_mod_switching()
    ct = m.multiply(cts[0], cts[1])
    assert len(ct.c) == 2 and ct.level == 1
    w = collective_decrypt(parties, ct, rng)
    assert (oracle.simd_decode(par, w) == (v1 * v2) % np.uint64(t)).all()


def test_roles_are_distinct_and_positional(oracle):
    """the new roles draw other words than roles 0-6 for the same (seed, index, limb), and a row depends only on its
    position: CRP k of a call of 3 is CRP k whatever the call's size"""
    seed = bytes(range(5, 37))
    rows = {r: R.row_values(seed, 2, r, [0, 1], 64) for r in range(7)}
    for r in M.ROLES + (M.ROLE_RKG_U, M.ROLE_RKG_R1_E0, M.ROLE_RKG_R1_E1, M.ROLE_RKG_R2_E0, M.ROLE_RKG_R2_E1):
        lo, hi = R.row_values(seed, 2, r, [0, 1], 64)
        for o, (olo, ohi) in rows.items():
            assert not (lo == olo).all() and not (hi == ohi).all(), (r, o)
        rows[r] = (lo, hi)
    blk = np.frombuffer(R.chacha20_block(seed, 5, 2, (M.ROLE_CRP << 8) | 1, 0), "<u8")
    assert rows[M.ROLE_CRP][0][1, 20] == blk[0] and rows[M.ROLE_CRP][1][1, 20] == blk[1]
    par = oracle.BfvParameters(16, 1153, moduli_sizes=[62, 62, 62])
    three = M.crp(par, seed, 3, 1)
    assert (three[2].c == M.crp(par, seed, 3, 1)[2].c).all()
    assert all((three[k].c == M.crp(par, seed, k + 1, 1)[k].c).all() for k in range(3))
    assert not (three[0].c == three[1].c).all()


def band_params(oracle, q0_bits=30):
    """q_0 of q0_bits bits, t = q_0 - 2 (so q_0 / 2 < t < q_0), and a 62-bit modulus: two plaintext-context moduli"""
    q0 = oracle.generate_prime(q0_bits, 32, 1 << q0_bits)
    par = oracle.BfvParameters(16, q0 - 2, moduli=[q0] + oracle.BfvParameters.generate_moduli([62], 16))
    assert len(par.plaintext_context.moduli) == 2
    return par


def test_from_shares_lift_differs_from_try_decrypt_in_the_band(oracle):
    """inside q_0 / 2 < t < q_0 with a two-moduli plaintext context from_shares gives v mod t for the centred scaled
    value v (|v| <= t / 2), try_decrypt ((v + t) mod q_0) mod t: they differ exactly for q_0 - t <= v <= t / 2; outside
    the band they agree"""
    rng = np.random.default_rng(3)
    par = band_params(oracle)
    t, q0 = par.plaintext, par.moduli[0]
    osk = oracle.SecretKey(par, rng)
    values = np.array([0, 1, 2, 3, t - 1, t - 2, t // 2, t // 2 + 1, 5, t // 2 - 1] + [0] * 6, dtype=np.uint64)
    ct = R.encrypt_sk(osk, seeds(rng, 1)[0], 1, 0, VAR, [R.to_poly(par, values, 0)])[0]
    shared = collective_decrypt([osk], ct, rng)
    assert (shared == values).all()
    direct = osk.decrypt(ct)
    centred = [v if v <= t // 2 else v - t for v in values.tolist()]
    for v, d in zip(centred, direct.tolist()):
        assert d == ((v % q0 + t) % q0) % t
    differ = sum(1 for v in centred if q0 - t <= v)
    assert (direct != values).sum() == differ > 0
    assert all(M.lift_from_limb0(v % q0, t, q0, 2) == v % t for v in centred)
    # outside the band: t = 1153
    par = default_arc(oracle, 2, 16)
    osk = oracle.SecretKey(par, rng)
    values = rng.integers(0, 1153, size=16, dtype=np.uint64)
    ct = R.encrypt_sk(osk, seeds(rng, 1)[0], 1, 0, VAR, [R.to_poly(par, values, 0)])[0]
    assert (collective_decrypt([osk], ct, rng) == osk.decrypt(ct)).all()


@pytest.mark.parametrize("kind", ["band", "one_plain_modulus", "default"])
def test_device_lift_equals_literal_from_shares(oracle, kind):
    """the device's lift from limb 0 (mbfv_reference.lift_from_limb0) equals the literal BigUint lift of from_shares
    for uniformly random phases, at every level"""
    par = {"band": lambda: band_params(oracle), "one_plain_modulus": lambda: default_arc(oracle, 1, 16),
           "default": lambda: default_arc(oracle, 3, 16)}[kind]()
    rng = np.random.default_rng(9)
    t, q0, n_plain = par.plaintext, par.moduli[0], len(par.plaintext_context.moduli)
    for level in range(par.max_level() + 1):
        ctx = par.context_at_level(level)
        for _ in range(4):
            c = [oracle.Poly.random(ctx, oracle.NTT, rng) for _ in range(2)]
            ct = oracle.Ciphertext(par, c, level)
            zero = oracle.Poly(ctx, oracle.NTT)
            _, w = M.from_shares(ct, [zero])
            r = par.level(level).scaler.scale(c[0].copy().into_power_basis()).c[0]
            assert [M.lift_from_limb0(int(x), t, q0, n_plain) for x in r] == w.tolist()


NEW = ["fhe_b200_crp_generate", "fhe_b200_pk_share", "fhe_b200_pk_aggregate", "fhe_b200_shares_sum",
       "fhe_b200_sks_share", "fhe_b200_sks_aggregate", "fhe_b200_pks_share", "fhe_b200_pks_aggregate",
       "fhe_b200_decryption_aggregate", "fhe_b200_rkg_create", "fhe_b200_rkg_free", "fhe_b200_rkg_round1",
       "fhe_b200_rkg_round2", "fhe_b200_rkg_aggregate"]


def test_symbols_declared_and_bound():
    from fhe_rs_b200 import _capi
    header = open(os.path.join(ROOT, "include", "fhe_b200.h")).read()
    for name in NEW:
        m = re.search(r"\bint %s\(([^)]*)\)" % name, header)
        assert m, name
        assert name in _capi.SYMBOLS and hasattr(_capi.lib(), name)
        assert len(m.group(1).split(",")) == len(_capi.SYMBOLS[name][1]), name
    assert "not audited" in header


def test_refusals_without_a_device(F, oracle):
    from fhe_rs_b200 import _capi
    lib = _capi.lib()
    seed = bytes(32)
    gpar = F.BfvParameters(16, 1153, moduli=default_arc(oracle, 2, 16).moduli, device=-1)
    assert lib.fhe_b200_crp_generate(gpar._h, seed, None, None) == _capi.NO_DEVICE
    assert lib.fhe_b200_decryption_aggregate(gpar.encoder(), None, None, 0, None, None) == _capi.NO_DEVICE
    with pytest.raises(F.FheError) as e:
        F.mbfv.CommonRandomPoly.new(gpar, seed)
    assert e.value.code == _capi.NO_DEVICE
    for v in (0, 33):
        assert lib.fhe_b200_pk_share(None, None, v, seed, None, None) == _capi.INVALID_ARGUMENT
        assert b"InvalidVariance" in lib.fhe_b200_last_error()
        assert lib.fhe_b200_sks_share(None, None, None, v, seed, None, None) == _capi.INVALID_ARGUMENT
        assert lib.fhe_b200_pks_share(None, None, None, v, seed, None, None) == _capi.INVALID_ARGUMENT
    assert lib.fhe_b200_crp_generate(None, seed, None, None) == _capi.INVALID_ARGUMENT
    assert lib.fhe_b200_shares_sum(None, 0, None, None) == _capi.INVALID_ARGUMENT
    assert lib.fhe_b200_pk_aggregate(None, 0, None, None, None) == _capi.INVALID_ARGUMENT
    assert lib.fhe_b200_sks_aggregate(None, None, 0, None, None) == _capi.INVALID_ARGUMENT
    assert lib.fhe_b200_pks_aggregate(None, None, 0, None, None) == _capi.INVALID_ARGUMENT
    for v in (0, 33):
        assert lib.fhe_b200_rkg_create(None, None, v, seed, None, None) == _capi.INVALID_ARGUMENT
    assert lib.fhe_b200_rkg_round1(None, seed, None, None, None) == _capi.INVALID_ARGUMENT
    assert lib.fhe_b200_rkg_round2(None, None, None, seed, None, None, None) == _capi.INVALID_ARGUMENT
    assert lib.fhe_b200_rkg_aggregate(None, None, 0, None, None, None) == _capi.INVALID_ARGUMENT
    assert lib.fhe_b200_rkg_free(None) == _capi.OK
    # MultipartyError::NoShares before any device work
    with pytest.raises(F.FheError) as e:
        F.mbfv.aggregate([])
    assert e.value.code == _capi.INVALID_ARGUMENT and "NoShares" in str(e.value)
