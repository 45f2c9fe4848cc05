"""Linear transforms without a device: the restatement of tests/linear_transform_reference.py against a literal
sum_k d_k (.) rot_k(v) on decrypted slots (the oracle's keys and encryption), encode_diagonals' slot permutation
against the numpy construction of the hand-built baby-step/giant-step test, linear_transform_steps, the C ABI symbol
and argtypes, and every refusal that needs no device."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TESTS = os.path.join(ROOT, "tests")
if TESTS not in sys.path:
    sys.path.insert(0, TESTS)


@pytest.fixture(scope="module")
def F():
    from fhe_rs_b200 import build
    build.build()
    import fhe_rs_b200
    return fhe_rs_b200


@pytest.fixture(scope="module")
def R(oracle):
    import linear_transform_reference
    return linear_transform_reference


def _diag_poly(O, par, slots, level=0):
    """a SIMD plaintext's poly_ntt at `level`: the encoded coefficients lifted to every modulus, then NTT"""
    return O.Poly.from_u64(par.context_at_level(level), O.simd_encode(par, slots), O.POWER_BASIS).into_ntt()


@pytest.mark.parametrize("degree,n,baby", [(16, 1, 1), (16, 5, 2), (16, 8, 3), (16, 8, 8), (16, 7, 1),
                                           (64, 16, 4), (64, 32, 5)])
def test_restatement_is_the_literal_sum(oracle, R, degree, n, baby):
    """decrypt(restatement with pre-rotated diagonals) == decrypt(sum_k d_k (.) rot_k(ct)) == M v mod t, both rows"""
    O = oracle
    t, half = 1153, degree // 2
    rng = np.random.default_rng(degree * 100 + n * 10 + baby)
    par = O.BfvParameters(degree, t, moduli_sizes=[62, 62])
    sk = O.SecretKey(par, rng)
    M = rng.integers(0, t, (2, half, half)).astype(np.int64)
    M[:, np.arange(half)[:, None], (np.arange(half)[:, None] + np.arange(n, half)[None, :]) % half] = 0   # n diagonals
    v = rng.integers(0, t, (2, half)).astype(np.int64)
    ct = sk.encrypt(O.simd_encode(par, v.reshape(-1)), 0, rng)
    need = sorted(set(R.steps(n, baby)) | set(range(1, n)))
    gks = {k: O.GaloisKey(sk, O.rotation_exponent(par, k), rng) for k in need}
    pre = np.stack([R.slot_diagonals(M[q], n, baby) for q in range(2)], axis=1)   # [n][2][half]
    got = R.linear_transform(ct, [_diag_poly(O, par, pre[k].reshape(-1)) for k in range(n)], baby, gks)
    plain = np.stack([R.slot_diagonals(M[q], n, n) for q in range(2)], axis=1)    # not rotated
    literal = None
    for k in range(n):
        x = ct if k == 0 else gks[k].relinearize(ct)
        d = _diag_poly(O, par, plain[k].reshape(-1))
        term = O.Ciphertext(par, [p.mul(d) for p in x.c], 0)
        literal = term if literal is None else literal.add(term)
    want = np.stack([(M[q] @ v[q]) % t for q in range(2)]).astype(np.uint64)
    dec = O.simd_decode(par, sk.decrypt(got)).reshape(2, half)
    assert (dec == want).all()
    assert (O.simd_decode(par, sk.decrypt(literal)).reshape(2, half) == want).all()
    assert len(R.steps(n, baby)) == (baby - 1) + (-(-n // baby) - 1)


def test_encode_diagonals_permutation(F, R):
    """bfv.diagonals (the host side of encode_diagonals) against the numpy construction of the hand-built test, for
    one matrix, a pair and a stack of pairs; entries beyond n_diags must be zero"""
    half = 32
    rng = np.random.default_rng(3)
    for n, baby in ((32, 8), (7, 3), (16, 4), (1, 1), (5, 5)):
        M = rng.integers(0, 1153, (3, 2, half, half)).astype(np.int64)
        mask = ((np.arange(half)[None, :] - np.arange(half)[:, None]) % half) < n   # M[r][c] on diagonal (c - r)
        M = M * mask
        got = F.bfv.diagonals(M, half, n, baby)
        assert got.shape == (3, n, 2 * half)
        for c in range(3):
            for q in range(2):
                assert (got[c, :, q * half:(q + 1) * half] == R.slot_diagonals(M[c, q], n, baby)).all(), (n, baby)
        assert (F.bfv.diagonals(M[0], half, n, baby) == got[:1]).all()
        one = F.bfv.diagonals(M[0, 0], half, n, baby)
        assert (one[0, :, :half] == one[0, :, half:]).all() and (one[0, :, :half] == got[0, :, :half]).all()
    # the construction of test_baby_step_giant_step_matrix_times_vector, literally
    M = rng.integers(0, 1153, (half, half)).astype(np.int64)
    n1 = 8
    d = F.bfv.diagonals(M, half, half, n1)[0]
    for g in range(half // n1):
        for j in range(n1):
            i = g * n1 + j
            ref = np.roll(np.array([M[r][(r + i) % half] for r in range(half)], np.int64), g * n1)
            assert (d[i] == np.concatenate([ref, ref])).all()
    with pytest.raises(F.FheError) as e:
        F.bfv.diagonals(M, half, 31, 4)   # diagonal 31 of a full matrix is not zero
    assert e.value.code == F._capi.INVALID_ARGUMENT and "n_diags" in str(e.value)


def test_diagonals_refusals(F):
    half = 8
    M = np.ones((half, half), np.int64)
    for call in (lambda: F.bfv.diagonals(np.ones((half, half - 1), np.int64), half, 1, 1),
                 lambda: F.bfv.diagonals(np.ones((3, half, half), np.int64), half, 8, 1),
                 lambda: F.bfv.diagonals(M.astype(np.float64), half, 8, 1),
                 lambda: F.bfv.diagonals(M, half, 0, 1),
                 lambda: F.bfv.diagonals(M, half, 9, 1),
                 lambda: F.bfv.diagonals(M, half, 8, 0),
                 lambda: F.bfv.diagonals(M, half, 8, 9)):
        with pytest.raises(F.FheError) as e:
            call()
        assert e.value.code == F._capi.INVALID_ARGUMENT


def test_linear_transform_steps(F, R):
    assert F.linear_transform_steps(64, 8) == list(range(1, 8)) + [8, 16, 24, 32, 40, 48, 56]
    assert F.linear_transform_steps(7, 3) == [1, 2, 3, 6]
    assert F.linear_transform_steps(1, 1) == []
    assert F.linear_transform_steps(16, 1) == list(range(1, 16))
    assert F.linear_transform_steps(16, 16) == list(range(1, 16))
    assert F.linear_transform_steps(17, 4) == [1, 2, 3, 4, 8, 12, 16]
    for n in range(1, 40):
        for b in range(1, n + 1):
            assert F.linear_transform_steps(n, b) == R.steps(n, b)
    for n, b in ((5, 0), (5, 6), (0, 1)):
        with pytest.raises(F.FheError) as e:
            F.linear_transform_steps(n, b)
        assert e.value.code == F._capi.INVALID_ARGUMENT


def test_symbol_argtypes_and_mirrors(F):
    from fhe_rs_b200 import _capi
    f = _capi.lib().fhe_b200_linear_transform
    u32, pu32, pp, vp = C.c_uint32, C.POINTER(C.c_uint32), C.POINTER(C.c_void_p), C.c_void_p
    assert f.restype is C.c_int and list(f.argtypes) == [vp, vp, u32, u32, pp, pu32, u32, vp, pu32, vp]
    for name in ("linear_transform", "linear_transform_steps", "encode_diagonals"):
        assert callable(getattr(F, name)) and name in F.bfv.__all__, name
    assert callable(F.EvaluationKey.linear_transform)


def test_argument_checks(F):
    """NULL batches, a NULL key list with keys, NULL keys: INVALID_ARGUMENT before anything else; n_fallback is not
    written"""
    from fhe_rs_b200 import _capi
    lib, bad = _capi.lib(), _capi.INVALID_ARGUMENT
    keys = (C.c_void_p * 2)(None, None)
    kp = C.cast(keys, C.POINTER(C.c_void_p))
    ex = (C.c_uint32 * 2)(3, 9)
    nf = C.c_uint32(77)
    for n, b in ((0, 0), (1, 1), (8, 3)):
        assert lib.fhe_b200_linear_transform(None, None, n, b, None, None, 0, None, C.byref(nf), None) == bad
        assert lib.fhe_b200_linear_transform(None, None, n, b, None, ex, 2, None, C.byref(nf), None) == bad
        assert lib.fhe_b200_linear_transform(None, None, n, b, kp, None, 2, None, C.byref(nf), None) == bad
        assert lib.fhe_b200_linear_transform(None, None, n, b, kp, ex, 2, None, C.byref(nf), None) == bad
    assert nf.value == 77
    assert b"null" in lib.fhe_b200_last_error()
