"""Per-ciphertext Galois exponents and the batched inner sum without a device: the three symbols and their argtypes,
the mirrors' names, NO_DEVICE for the batches and keys the calls take on a host-only parameter set, and every argument
check that needs no device (NULL lists and batches, no keys, no key sets, the mirrors' index and source lengths)."""
import ctypes as C

import numpy as np
import pytest

NEW = ("fhe_b200_galois_many", "fhe_b200_inner_sum", "fhe_b200_inner_sum_keyed")


@pytest.fixture(scope="module")
def F():
    from fhe_rs_b200 import build
    build.build()
    import fhe_rs_b200
    return fhe_rs_b200


def test_symbols_and_argtypes(F):
    from fhe_rs_b200 import _capi
    lib = _capi.lib()
    u32, pu32, pp, vp = C.c_uint32, C.POINTER(C.c_uint32), C.POINTER(C.c_void_p), C.c_void_p
    want = {
        "fhe_b200_galois_many": [vp, pu32, pp, pu32, u32, pu32, vp, vp],
        "fhe_b200_inner_sum": [vp, pp, u32, vp, vp],
        "fhe_b200_inner_sum_keyed": [vp, pp, u32, u32, pu32, vp, vp],
    }
    for name in NEW:
        f = getattr(lib, name)
        assert f.restype is C.c_int and list(f.argtypes) == want[name], name
    for name in ("galois_many", "computes_inner_sum_keyed"):
        assert callable(getattr(F, name)) and name in F.bfv.__all__, name
    assert callable(F.EvaluationKey.rotates_columns_by_many)


def test_host_only_parameters_give_no_device(F):
    from fhe_rs_b200 import _capi
    par = F.BfvParameters(16, 1153, moduli_sizes=[62, 62], device=-1)
    with pytest.raises(F.FheError) as e:
        F.Ciphertext(par, 2)
    assert e.value.code == _capi.NO_DEVICE
    z = np.zeros((2, 2, 16), np.uint64)
    with pytest.raises(F.FheError) as e:
        F.GaloisKey.from_arrays(par, 3, z, z)
    assert e.value.code == _capi.NO_DEVICE


def test_argument_checks(F):
    """NULL batches, key lists, exponent lists and indices, no keys and no key sets: INVALID_ARGUMENT before anything
    else"""
    from fhe_rs_b200 import _capi
    lib, bad = _capi.lib(), _capi.INVALID_ARGUMENT
    one = (C.c_uint32 * 1)(0)
    three = (C.c_uint32 * 1)(3)
    keys = (C.c_void_p * 1)(None)
    kp = C.cast(keys, C.POINTER(C.c_void_p))
    for n_keys, k, ex, ix in ((1, None, three, one), (0, kp, three, one), (1, kp, None, one), (1, kp, three, None),
                              (1, kp, three, one)):
        assert lib.fhe_b200_galois_many(None, None, k, ex, n_keys, ix, None, None) == bad
        assert lib.fhe_b200_galois_many(None, one, k, ex, n_keys, ix, None, None) == bad
    for n_gks in (0, 4):
        assert lib.fhe_b200_inner_sum(None, kp, n_gks, None, None) == bad
        assert lib.fhe_b200_inner_sum(None, None, n_gks, None, None) == bad
        for n_sets, ix in ((0, one), (1, None), (1, one)):
            assert lib.fhe_b200_inner_sum_keyed(None, kp, n_gks, n_sets, ix, None, None) == bad
    assert b"null" in lib.fhe_b200_last_error()


class _Batch:
    """what the mirrors read of a batch before they reach the device"""

    def __init__(self, par, count):
        self.par, self.count, self.level, self.stream = par, count, 0, 0

    def __len__(self):
        return 2


def test_mirrors_check_lengths_and_keys(F):
    """one key index per output (per source entry when a source list is given), sources in range, and an
    EvaluationKey that supports the inner sum or the rotation, checked before the library is called"""
    from fhe_rs_b200 import _capi
    par = F.BfvParameters(16, 1153, moduli_sizes=[62, 62], device=-1)
    ct = _Batch(par, 3)
    ek = F.EvaluationKey(par)
    for call in (lambda: F.galois_many(ct, [], [0, 0]),
                 lambda: F.galois_many(ct, [], [0, 0, 0], [0, 1]),
                 lambda: F.galois_many(ct, [], [0], [-1]),
                 lambda: F.computes_inner_sum_keyed(ct, [], [0, 0]),
                 lambda: F.computes_inner_sum_keyed(ct, [ek], [0, 0, 0]),
                 lambda: ek.computes_inner_sum(ct),
                 lambda: ek.rotates_columns_by_many(ct, [1, 2])):
        with pytest.raises(F.FheError) as e:
            call()
        assert e.value.code == _capi.INVALID_ARGUMENT
