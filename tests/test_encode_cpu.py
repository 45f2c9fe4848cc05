"""CPU tests of the plaintext encoders: the encoder tables of fhe_b200_encoder_create on host-only parameter sets against
the oracle, the oracle's encoders against the properties the reference's tests check (plaintext.rs:478-597, :690,
plaintext_vec.rs:175-215), and the host-only refusal of fhe_b200_encode."""
import ctypes as C

import numpy as np
import pytest

import encode_reference as R


@pytest.fixture(scope="module")
def F():
    import fhe_rs_b200
    return fhe_rs_b200


def _other_root(t, n, psi):
    """another primitive 2N-th root of unity mod t (an odd power of one is one)"""
    return pow(psi, 3, t)


@pytest.mark.parametrize("degree,sizes", [(16, [62, 62, 62]), (1 << 12, [62, 62]), (1 << 15, [62, 50, 62])])
@pytest.mark.parametrize("custom_psi", [False, True])
def test_encoder_tables_match_oracle(F, oracle, degree, sizes, custom_psi):
    t = 786433
    psi_t = _other_root(t, degree, oracle.default_psi(t, degree)) if custom_psi else None
    opar = oracle.BfvParameters(degree, t, moduli_sizes=sizes, psi={t: psi_t} if custom_psi else None)
    gpar = F.BfvParameters(degree, t, moduli=opar.moduli, device=-1, plaintext_psi=psi_t)
    op = oracle._ntt_op(t, degree, psi_t)
    for level in range(len(sizes)):
        tb = gpar.encoder_tables(level)
        assert list(tb["index_map"]) == opar.matrix_reps_index_map
        assert (tb["omegas"] == op.omegas).all() and (tb["zetas_inv"] == op.zetas_inv).all()
        lvl = opar.level(level)
        assert tb["q_mod_t"] == lvl.q_mod_t
        assert [int(x) for x in tb["delta"]] == lvl.delta_rests


def test_encoder_without_ntt_for_t(F, oracle):
    """t = 1153 is prime but not 1 mod 2N at N = 2^12: the handle is created, without NTT tables"""
    opar = oracle.BfvParameters(1 << 12, 1153, moduli_sizes=[62, 62])
    gpar = F.BfvParameters(1 << 12, 1153, moduli=opar.moduli, device=-1)
    tb = gpar.encoder_tables(1)
    assert tb["omegas"] is None
    assert list(tb["index_map"]) == opar.matrix_reps_index_map
    assert tb["q_mod_t"] == opar.level(1).q_mod_t


def test_encode_needs_a_device(F):
    from fhe_rs_b200 import _capi
    gpar = F.BfvParameters(16, 1153, moduli_sizes=[62, 62], device=-1)
    vals = np.arange(16, dtype=np.uint64)
    for kind in (_capi.ENCODING_POLY, _capi.ENCODING_SIMD):
        code = _capi.lib().fhe_b200_encode(gpar.encoder(), kind, 0, vals.ctypes.data, 16, None, None)
        assert code == _capi.NO_DEVICE
    with pytest.raises(F.FheError) as e:
        F.Plaintext.try_encode(vals, F.Encoding.simd(), gpar)
    assert e.value.code == _capi.NO_DEVICE


@pytest.mark.parametrize("degree,t,level", [(16, 1153, 0), (16, 1153, 2), (1 << 12, 1032193, 0), (1 << 12, 1032193, 1)])
def test_oracle_encoders_decode_to_their_values(oracle, degree, t, level):
    """decode(encode(v)) == v for Poly and SIMD, u64 and i64, from poly_ntt at the encoding level
    (plaintext.rs:478-597, :690; plaintext_vec.rs:175-215)"""
    opar = oracle.BfvParameters(degree, t, moduli_sizes=[62] * 3 if degree == 16 else [62, 62])
    rng = np.random.default_rng(degree + level)
    L = len(opar.moduli) - level
    for n in (0, 1, degree - 1, degree, 3 * degree):
        u = rng.integers(0, t, size=n, dtype=np.uint64)
        s = rng.integers(-(1 << 62), 1 << 62, size=n, dtype=np.int64)
        for simd in (False, True):
            for vals, signed in ((u, False), (s, True)):
                pts = R.try_encode(opar, vals, simd, level, signed)
                assert pts.shape == (max(1, -(-n // degree)), L, degree)
                want = np.zeros(pts.shape[0] * degree, np.uint64)
                want[:n] = R.reduce_i64(vals, t) if signed else vals
                for k in range(pts.shape[0]):
                    c = R.coefficients(opar, pts[k], level)
                    got = oracle.simd_decode(opar, c) if simd else c
                    assert (got == want[k * degree:(k + 1) * degree]).all(), (n, simd, signed, k)


def test_oracle_to_poly_matches_plaintext_to_poly(oracle):
    """to_poly from poly_ntt equals the oracle's value-side Plaintext::to_poly"""
    opar = oracle.BfvParameters(64, 1153, moduli_sizes=[62, 62])
    rng = np.random.default_rng(5)
    v = rng.integers(0, 1153, size=64, dtype=np.uint64)
    for level in (0, 1):
        pt = R.try_encode(opar, v, False, level)[0]
        assert (R.to_poly(opar, pt, level) == oracle.plaintext_to_poly(opar, v, level).c).all()
