"""CPU tests of SecretKey::random on the device: the role-18 stream that fhe_b200_secret_keys_random draws, restated in
tests/secret_key_reference.py on top of the ChaCha20 block function pinned to RFC 8439, follows the centred binomial
law of sample_vec_cbd (fhe-util/src/lib.rs:22-67) for variance 1, 10 and 32; and the refusals that need no device."""
import ctypes as C

import numpy as np
import pytest
from scipy import stats

import encrypt_reference as R
import secret_key_reference as S

SEED = bytes(range(32))


@pytest.fixture(scope="module")
def F():
    import fhe_rs_b200
    return fhe_rs_b200


def test_role_18_rows_follow_the_stream_layout():
    """coefficient 4b + m of key k is value m (u64 words 2m, 2m + 1) of block (b, k, 18 << 8 | 0, 0)"""
    variance, degree = 10, 64
    add = (1 << (2 * variance)) - 1
    sub = add << (2 * variance)
    for k in (0, 1, 7):
        got = S.secret_key_coeffs(SEED, k, variance, degree)
        for i in (0, 1, 2, 3, 4, 33, 63):
            b, m = divmod(i, 4)
            w = np.frombuffer(R.chacha20_block(SEED, b, k, S.ROLE_S << 8, 0), "<u4").astype(object)
            v = int(w[4 * m]) | int(w[4 * m + 1]) << 32 | int(w[4 * m + 2]) << 64 | int(w[4 * m + 3]) << 96
            assert got[i] == bin(v & add).count("1") - bin(v & sub).count("1"), (k, i)


def _binomial_chi2(x: np.ndarray, variance: int) -> float:
    """p-value of Pearson's chi-square test of x + 2 variance ~ Binomial(4 variance, 1/2), tails pooled so that every
    bin expects at least 5 samples"""
    n = 4 * variance
    counts = np.bincount(x + 2 * variance, minlength=n + 1).astype(float)
    assert counts.size == n + 1, "a sample outside [-2 variance, 2 variance]"
    expected = stats.binom.pmf(np.arange(n + 1), n, 0.5) * x.size
    obs, exp, acc_o, acc_e = [], [], 0.0, 0.0
    for o, e in zip(counts, expected):
        acc_o, acc_e = acc_o + o, acc_e + e
        if acc_e >= 5:
            obs.append(acc_o)
            exp.append(acc_e)
            acc_o = acc_e = 0.0
    obs[-1] += acc_o
    exp[-1] += acc_e
    exp = np.array(exp) * (sum(obs) / sum(exp))
    return stats.chisquare(obs, exp).pvalue


@pytest.mark.parametrize("variance", [1, 10, 32])
def test_cbd_histogram_matches_the_binomial_law(variance):
    degree = 1 << 13
    x = np.concatenate([S.secret_key_coeffs(SEED, k, variance, degree) for k in range(8)])
    assert x.min() >= -2 * variance and x.max() <= 2 * variance
    assert _binomial_chi2(x, variance) > 1e-3
    assert abs(x.mean()) < 4 * np.sqrt(variance / x.size)
    assert abs(x.var() / variance - 1) < 0.05


def test_keys_of_a_call_are_independent_and_repeatable():
    degree = 1 << 10
    keys = [S.secret_key_coeffs(SEED, k, 10, degree) for k in range(4)]
    for i in range(4):
        for j in range(i):
            assert (keys[i] != keys[j]).any()
            assert abs(np.corrcoef(keys[i], keys[j])[0, 1]) < 0.15
    assert (S.secret_key_coeffs(SEED, 2, 10, degree) == keys[2]).all()
    assert (S.secret_key_coeffs(bytes(32), 2, 10, degree) != keys[2]).any()
    # role 18 is its own row: not the encryption error of ciphertext k (role 1)
    assert (R.cbd(SEED, 0, R.ROLE_E, 10, degree) != keys[0]).any()


def test_refusals_without_a_device(F, oracle):
    from fhe_rs_b200 import _capi
    lib = _capi.lib()
    moduli = oracle.BfvParameters.generate_moduli([62, 62], 1 << 12)
    par = F.BfvParameters(1 << 12, 1032193, moduli=moduli, device=-1)
    hs = (C.c_void_p * 2)()
    out = C.cast(hs, C.POINTER(C.c_void_p))

    def call(p=par._h, n=2, v=10, seed=SEED, o=out):
        code = lib.fhe_b200_secret_keys_random(p, n, v, seed, o, None)
        assert not hs[0] and not hs[1]
        return code
    assert call() == _capi.NO_DEVICE
    for v in (0, 33):
        assert call(v=v) == _capi.INVALID_ARGUMENT and "InvalidVariance" in _capi.lib().fhe_b200_last_error().decode()
    assert call(n=0) == _capi.INVALID_ARGUMENT
    assert call(seed=None) == _capi.INVALID_ARGUMENT
    assert call(o=None) == _capi.INVALID_ARGUMENT
    assert call(p=None) == _capi.INVALID_ARGUMENT
    with pytest.raises(F.FheError) as e:
        F.SecretKey.random(par)
    assert e.value.code == _capi.NO_DEVICE
    with pytest.raises(F.FheError) as e:
        F.SecretKey.random_vec(par, 3, seed=b"short")
    assert e.value.code == _capi.INVALID_ARGUMENT
    # t beyond a u64 Modulus, as fhe_b200_secret_key_create
    big = F.BfvParameters(16, 340282366920938463463374607431768211507, moduli_sizes=[62] * 5, device=-1)
    assert call(p=big._h) == _capi.UNSUPPORTED
    assert lib.fhe_b200_secret_key_coeffs(None, np.zeros(16, np.int64).ctypes.data, None) == _capi.INVALID_ARGUMENT
