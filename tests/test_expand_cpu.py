"""CPU-side tests of oblivious expansion (fhe_b200_expand): the monomial tables the library derives from the parameter
set's roots equal the reference's -x^(N - 2^l) in the NTT domain (evaluation_key.rs:465-474, restated by the oracle) at
every level, and the new entry points need a device."""
import ctypes as C

import numpy as np
import pytest


@pytest.fixture(scope="module")
def F():
    from fhe_rs_b200 import build
    build.build()
    import fhe_rs_b200
    return fhe_rs_b200


def _monomial(F, gpar, level, l):
    from fhe_rs_b200 import _capi
    out = np.zeros((len(gpar.moduli()) - level, gpar.degree()), np.uint64)
    F.bfv.check(_capi.lib().fhe_b200_debug_expansion_monomial(gpar._h, level, l, out.ctypes.data))
    return out


@pytest.mark.parametrize("degree,sizes,t", [(16, [62, 62, 62], 1153),
                                            (8192, [50, 55, 55], (1 << 20) + (1 << 19) + (1 << 17) + (1 << 16) + (1 << 14) + 1),
                                            (1 << 15, [62] * 14, 65537)])
def test_expansion_monomials_match_oracle(F, oracle, degree, sizes, t):
    opar = oracle.BfvParameters(degree, t, moduli_sizes=sizes)
    gpar = F.BfvParameters(degree, t, moduli=opar.moduli, device=-1)
    for level in range(len(sizes)):
        for l in range(degree.bit_length() - 1):
            exp = oracle.expansion_monomial(opar, l, level).c
            assert (_monomial(F, gpar, level, l) == exp).all(), (level, l)


def test_expansion_monomial_arguments(F):
    from fhe_rs_b200 import _capi
    gpar = F.BfvParameters(16, 1153, moduli_sizes=[62, 62], device=-1)
    out = np.zeros((2, 16), np.uint64)
    assert _capi.lib().fhe_b200_debug_expansion_monomial(gpar._h, 0, 4, out.ctypes.data) == _capi.INVALID_ARGUMENT
    assert _capi.lib().fhe_b200_debug_expansion_monomial(gpar._h, 2, 0, out.ctypes.data) == _capi.INVALID_LEVEL
    assert _capi.lib().fhe_b200_debug_expansion_monomial(gpar._h, 0, 0, None) == _capi.INVALID_ARGUMENT


def test_expansion_needs_a_device(F):
    """no CPU fallback: on a host-only parameter set neither the batches nor the keys that fhe_b200_expand and
    fhe_b200_batch_copy_range take can be created (NO_DEVICE), and the calls refuse NULL handles"""
    from fhe_rs_b200 import _capi
    L = _capi.lib()
    gpar = F.BfvParameters(16, 1153, moduli_sizes=[62, 62], device=-1)
    with pytest.raises(F.FheError) as e:
        F.Ciphertext(gpar, 2)
    assert e.value.code == _capi.NO_DEVICE
    with pytest.raises(F.FheError) as e:
        F.GaloisKey.from_arrays(gpar, 17, np.zeros((2, 2, 16), np.uint64), np.zeros((2, 2, 16), np.uint64))
    assert e.value.code == _capi.NO_DEVICE
    assert L.fhe_b200_expand(None, 2, None, 0, None, None) == _capi.INVALID_ARGUMENT
    assert L.fhe_b200_batch_copy_range(None, 0, None, 0, 1, 1, None) == _capi.INVALID_ARGUMENT
    ek = F.EvaluationKey(gpar)
    assert ek.supports_expansion(0) and not ek.supports_expansion(1)
