"""Ciphertext dot products and batch sums without a device: the three symbols and their argtypes, the mirrors' names,
NO_DEVICE for the batches and keys the calls take on a host-only parameter set, and every argument check that needs no
device (NULL batches, key lists and indices, no terms, no keys, the mirrors' run lengths and key indices)."""
import ctypes as C

import numpy as np
import pytest

NEW = ("fhe_b200_batch_sum", "fhe_b200_dot_product", "fhe_b200_dot_product_keyed")


@pytest.fixture(scope="module")
def F():
    from fhe_rs_b200 import build
    build.build()
    import fhe_rs_b200
    return fhe_rs_b200


def test_symbols_and_argtypes(F):
    from fhe_rs_b200 import _capi
    lib = _capi.lib()
    u32, pu32, pp, vp, i = C.c_uint32, C.POINTER(C.c_uint32), C.POINTER(C.c_void_p), C.c_void_p, C.c_int
    want = {
        "fhe_b200_batch_sum": [vp, u32, i, vp, vp],
        "fhe_b200_dot_product": [vp, vp, u32, vp, vp, vp],
        "fhe_b200_dot_product_keyed": [vp, vp, u32, pp, u32, pu32, vp, vp],
    }
    for name in NEW:
        f = getattr(lib, name)
        assert f.restype is C.c_int and list(f.argtypes) == want[name], name
    f = lib.fhe_b200_ntt_row_count
    assert f.restype is C.c_uint64 and list(f.argtypes) == [C.c_int]
    assert f(0) >= 0 and f(1) >= 0
    for name in ("dot_product", "dot_product_keyed"):
        assert callable(getattr(F, name)) and name in F.bfv.__all__, name
    assert callable(F.Ciphertext.sum)


def test_host_only_parameters_give_no_device(F):
    from fhe_rs_b200 import _capi
    par = F.BfvParameters(16, 1153, moduli_sizes=[62, 62], device=-1)
    with pytest.raises(F.FheError) as e:
        F.Ciphertext(par, 2)
    assert e.value.code == _capi.NO_DEVICE
    z = np.zeros((2, 2, 16), np.uint64)
    with pytest.raises(F.FheError) as e:
        F.RelinearizationKey.from_arrays(par, z, z)
    assert e.value.code == _capi.NO_DEVICE


def test_argument_checks(F):
    """NULL batches, key lists and indices, and no keys: INVALID_ARGUMENT before anything else"""
    from fhe_rs_b200 import _capi
    lib, bad = _capi.lib(), _capi.INVALID_ARGUMENT
    one = (C.c_uint32 * 1)(0)
    keys = (C.c_void_p * 1)(None)
    kp = C.cast(keys, C.POINTER(C.c_void_p))
    for n_terms in (0, 1, 5):
        for acc in (0, 1):
            assert lib.fhe_b200_batch_sum(None, n_terms, acc, None, None) == bad
        assert lib.fhe_b200_dot_product(None, None, n_terms, None, None, None) == bad
        for k, n_keys, ix in ((None, 1, one), (kp, 0, one), (kp, 1, None), (kp, 1, one)):
            assert lib.fhe_b200_dot_product_keyed(None, None, n_terms, k, n_keys, ix, None, None) == bad
    assert b"null" in lib.fhe_b200_last_error()


class _Batch:
    """what the mirrors read of a batch before they reach the device"""

    def __init__(self, par, count):
        self.par, self.count, self.level, self.stream = par, count, 0, 0

    def __len__(self):
        return 2


def test_mirrors_check_lengths_and_keys(F):
    """runs that do not divide the batch, no terms, and one key index per group (not per term), checked before the
    library is called"""
    from fhe_rs_b200 import _capi
    par = F.BfvParameters(16, 1153, moduli_sizes=[62, 62], device=-1)
    a, b, shared = _Batch(par, 6), _Batch(par, 6), _Batch(par, 3)
    for call in (lambda: F.dot_product(a, b, 0),
                 lambda: F.dot_product(a, b, 4),
                 lambda: F.dot_product(a, shared, 5),
                 lambda: F.dot_product_keyed(a, b, 0, [], []),
                 lambda: F.dot_product_keyed(a, b, 3, [], [0]),
                 lambda: F.dot_product_keyed(a, shared, 3, [], [0, 0, 0, 0, 0, 0]),
                 lambda: F.dot_product_keyed(a, b, 3, [], [0, -1])):
        with pytest.raises(F.FheError) as e:
            call()
        assert e.value.code == _capi.INVALID_ARGUMENT
    for n in (0, -1, 4):
        with pytest.raises(F.FheError) as e:
            F.Ciphertext.sum(a, n)
        assert e.value.code == _capi.INVALID_ARGUMENT
