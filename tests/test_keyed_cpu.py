"""Per-ciphertext keys without a device: the five fhe_b200_*_keyed symbols and their argtypes, NO_DEVICE for the
batches and keys a keyed call takes on a host-only parameter set, and every argument check that needs no device
(NULL key lists, indices and batches, an empty key list, the mirrors' index length)."""
import ctypes as C

import numpy as np
import pytest

KEYED = ("fhe_b200_key_switch_keyed", "fhe_b200_relinearize_keyed", "fhe_b200_mul_relin_keyed",
         "fhe_b200_galois_keyed", "fhe_b200_expand_keyed")


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
        "fhe_b200_key_switch_keyed": [vp, u32, pp, u32, pu32, vp, vp],
        "fhe_b200_relinearize_keyed": [vp, pp, u32, pu32, vp, vp],
        "fhe_b200_mul_relin_keyed": [vp, vp, pp, u32, pu32, C.c_int, vp, vp],
        "fhe_b200_galois_keyed": [vp, u32, pp, u32, pu32, vp, vp],
        "fhe_b200_expand_keyed": [vp, u32, pp, u32, u32, pu32, vp, vp],
    }
    for name in KEYED:
        f = getattr(lib, name)
        assert f.restype is C.c_int and list(f.argtypes) == want[name], name
    for name in ("key_switch_keyed", "relinearizes_keyed", "multiply_keyed", "galois_keyed", "rotates_columns_by_keyed",
                 "rotates_rows_keyed", "expands_keyed", "expands_batch_keyed", "external_products_keyed"):
        assert callable(getattr(F, name)) and name in F.bfv.__all__, name


def test_host_only_parameters_give_no_device(F):
    """a keyed call needs batches and keys, and neither exists on a host-only parameter set"""
    from fhe_rs_b200 import _capi
    par = F.BfvParameters(16, 1153, moduli_sizes=[62, 62], device=-1)
    with pytest.raises(F.FheError) as e:
        F.Ciphertext(par, 2)
    assert e.value.code == _capi.NO_DEVICE
    z = np.zeros((2, 2, 16), np.uint64)
    for make in (lambda: F.RelinearizationKey.from_arrays(par, z, z), lambda: F.GaloisKey.from_arrays(par, 3, z, z),
                 lambda: F.KeySwitchingKey.from_arrays(par, z, z)):
        with pytest.raises(F.FheError) as e:
            make()
        assert e.value.code == _capi.NO_DEVICE


def test_argument_checks(F):
    """NULL batches, key lists and indices, and an empty key list: INVALID_ARGUMENT before anything else"""
    from fhe_rs_b200 import _capi
    lib, bad = _capi.lib(), _capi.INVALID_ARGUMENT
    one = (C.c_uint32 * 1)(0)
    keys = (C.c_void_p * 1)(None)
    kp = C.cast(keys, C.POINTER(C.c_void_p))
    for n_keys, k, ix in ((1, None, one), (0, kp, one), (1, kp, None), (1, kp, one)):
        assert lib.fhe_b200_key_switch_keyed(None, 0, k, n_keys, ix, None, None) == bad
        assert lib.fhe_b200_relinearize_keyed(None, k, n_keys, ix, None, None) == bad
        assert lib.fhe_b200_mul_relin_keyed(None, None, k, n_keys, ix, 0, None, None) == bad
        assert lib.fhe_b200_galois_keyed(None, 3, k, n_keys, ix, None, None) == bad
        assert lib.fhe_b200_expand_keyed(None, 2, k, 1, n_keys, ix, None, None) == bad
    assert b"null" in lib.fhe_b200_last_error()


class _Batch:
    """what the mirrors read of a batch before they reach the device"""

    def __init__(self, par, count):
        self.par, self.count, self.level, self.stream = par, count, 0, 0

    def __len__(self):
        return 2


def test_mirrors_check_the_index_length(F):
    """one index per ciphertext (per query for expands_keyed), checked before the library is called"""
    from fhe_rs_b200 import _capi
    par = F.BfvParameters(16, 1153, moduli_sizes=[62, 62], device=-1)
    ct = _Batch(par, 3)
    for call in (lambda: F.relinearizes_keyed(ct, [], [0, 0]),
                 lambda: F.key_switch_keyed(ct, 0, [], [0, 0, 0, 0]),
                 lambda: F.galois_keyed(ct, [], []),
                 lambda: F.multiply_keyed(ct, ct, [], [-1, 0, 0])):
        with pytest.raises(F.FheError) as e:
            call()
        assert e.value.code == _capi.INVALID_ARGUMENT
    with pytest.raises(F.FheError) as e:
        F.expands_keyed(ct, [], [0, 0, 0], 0)
    assert e.value.code == _capi.INVALID_ARGUMENT
