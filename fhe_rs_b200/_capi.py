"""ctypes binding of include/fhe_b200.h (the C ABI of libfhe_b200.so).

This is the same binding a foreign host would write (INTEGRATION.md shows the Rust
`extern "C"` equivalent).  There is no fallback: if the shared library is missing the
import fails loudly."""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("FHE_B200_LIB") or os.path.join(_HERE, "libfhe_b200.so")   # (override: A/B of two builds)

# fhe_b200_status
OK = 0
INVALID_ARGUMENT, INVALID_MODULUS, INVALID_DEGREE, NTT_UNAVAILABLE = -1, -2, -3, -4
CONTEXT_MISMATCH, INVALID_LEVEL, BAD_POLY_COUNT, INVALID_REPRESENTATION = -5, -6, -7, -8
NO_MORE_CONTEXT, INVALID_EXPONENT, UNSUPPORTED = -9, -10, -11
CUDA_ERROR, OUT_OF_MEMORY, NO_DEVICE = -20, -21, -22
POWER_BASIS, NTT = 0, 1
ENCODING_POLY, ENCODING_SIMD = 0, 1

# every symbol declared in include/fhe_b200.h: name -> (restype, argtypes)
_u32, _u64, _vp, _i = C.c_uint32, C.c_uint64, C.c_void_p, C.c_int
_pu32, _pu64, _pu8 = C.POINTER(C.c_uint32), C.POINTER(C.c_uint64), C.POINTER(C.c_uint8)
_pp = C.POINTER(C.c_void_p)
SYMBOLS = {
    "fhe_b200_version": (C.c_char_p, []),
    "fhe_b200_last_error": (C.c_char_p, []),
    "fhe_b200_params_create": (_i, [_i, _u32, _vp, _u32, _vp, _u32, _vp, _pp]),
    "fhe_b200_params_create_from_sizes": (_i, [_i, _u32, _vp, _u32, _vp, _u32, _pp]),
    "fhe_b200_params_destroy": (_i, [_vp]),
    "fhe_b200_params_degree": (_u32, [_vp]),
    "fhe_b200_params_n_moduli": (_u32, [_vp]),
    "fhe_b200_params_moduli": (_i, [_vp, _vp]),
    "fhe_b200_params_mul_basis": (_i, [_vp, _u32, _vp, _pu32]),
    "fhe_b200_params_psi": (_i, [_vp, _u64, _pu64]),
    "fhe_b200_batch_alloc": (_i, [_vp, _u32, _u32, _u32, _i, _pp]),
    "fhe_b200_batch_alloc_mul_basis": (_i, [_vp, _u32, _u32, _u32, _i, _pp]),
    "fhe_b200_batch_free": (_i, [_vp]),
    "fhe_b200_batch_info": (_i, [_vp, _pu32, _pu32, _pu32, _pu32, C.POINTER(_i)]),
    "fhe_b200_batch_upload": (_i, [_vp, _u32, _u32, _vp, _vp]),
    "fhe_b200_batch_download": (_i, [_vp, _u32, _u32, _vp, _vp]),
    "fhe_b200_batch_download_async": (_i, [_vp, _u32, _u32, _vp, _vp]),
    "fhe_b200_batch_copy": (_i, [_vp, _vp, _vp]),
    "fhe_b200_batch_copy_range": (_i, [_vp, _u32, _vp, _u32, _u32, _u32, _vp]),
    "fhe_b200_host_alloc": (_i, [C.c_size_t, _i, _pp]),
    "fhe_b200_host_free": (_i, [_vp]),
    "fhe_b200_batch_device_ptr": (_i, [_vp, _pp, C.POINTER(C.c_size_t)]),
    "fhe_b200_ksk_upload": (_i, [_vp, _u32, _u32, _vp, _vp, _u32, _pp]),
    "fhe_b200_ksk_free": (_i, [_vp]),
    "fhe_b200_ksk_download": (_i, [_vp, _vp, _vp, _vp]),
    "fhe_b200_ntt_forward": (_i, [_vp, _vp]),
    "fhe_b200_ntt_backward": (_i, [_vp, _vp]),
    "fhe_b200_add": (_i, [_vp, _vp, _vp]),
    "fhe_b200_sub": (_i, [_vp, _vp, _vp]),
    "fhe_b200_neg": (_i, [_vp, _vp]),
    "fhe_b200_mul_plain": (_i, [_vp, _vp, _u32, _vp]),
    "fhe_b200_add_plain": (_i, [_vp, _vp, _u32, _i, _vp]),
    "fhe_b200_dot_product_scalar": (_i, [_vp, _vp, _u32, _vp, _vp]),
    "fhe_b200_encoder_create": (_i, [_vp, _vp, _pp]),
    "fhe_b200_encoder_free": (_i, [_vp]),
    "fhe_b200_encode": (_i, [_vp, _i, _i, _vp, C.c_size_t, _vp, _vp]),
    "fhe_b200_mul_plain_batch": (_i, [_vp, _vp, _vp]),
    "fhe_b200_add_plain_batch": (_i, [_vp, _vp, _i, _vp]),
    "fhe_b200_secret_key_create": (_i, [_vp, _vp, _pp]),
    "fhe_b200_secret_key_free": (_i, [_vp]),
    "fhe_b200_secret_keys_random": (_i, [_vp, _u32, _u32, _vp, _pp, _vp]),
    "fhe_b200_secret_key_coeffs": (_i, [_vp, _vp, _vp]),
    "fhe_b200_decrypt": (_i, [_vp, _vp, _vp, _vp]),
    "fhe_b200_decode": (_i, [_vp, _i, _i, _vp, _vp, C.c_size_t, _vp]),
    "fhe_b200_measure_noise": (_i, [_vp, _vp, _vp, _vp]),
    "fhe_b200_encrypt_sk": (_i, [_vp, _vp, _u32, _vp, _vp, _vp]),
    "fhe_b200_encrypt_pk": (_i, [_vp, _vp, _u32, _vp, _vp, _vp]),
    "fhe_b200_relin_key_generate": (_i, [_vp, _u32, _u32, _u32, _vp, _pp, _vp]),
    "fhe_b200_galois_keys_generate": (_i, [_vp, _vp, _u32, _u32, _u32, _u32, _vp, _pp, _vp]),
    "fhe_b200_rgsw_encrypt": (_i, [_vp, _vp, _u32, _vp, _pp, _vp]),
    "fhe_b200_crp_generate": (_i, [_vp, _vp, _vp, _vp]),
    "fhe_b200_pk_share": (_i, [_vp, _vp, _u32, _vp, _vp, _vp]),
    "fhe_b200_pk_aggregate": (_i, [_pp, _u32, _vp, _vp, _vp]),
    "fhe_b200_shares_sum": (_i, [_pp, _u32, _vp, _vp]),
    "fhe_b200_sks_share": (_i, [_vp, _vp, _vp, _u32, _vp, _vp, _vp]),
    "fhe_b200_sks_aggregate": (_i, [_vp, _pp, _u32, _vp, _vp]),
    "fhe_b200_pks_share": (_i, [_vp, _vp, _vp, _u32, _vp, _vp, _vp]),
    "fhe_b200_pks_aggregate": (_i, [_vp, _pp, _u32, _vp, _vp]),
    "fhe_b200_decryption_aggregate": (_i, [_vp, _vp, _pp, _u32, _vp, _vp]),
    "fhe_b200_rkg_create": (_i, [_vp, _vp, _u32, _vp, _pp, _vp]),
    "fhe_b200_rkg_free": (_i, [_vp]),
    "fhe_b200_rkg_round1": (_i, [_vp, _vp, _vp, _vp, _vp]),
    "fhe_b200_rkg_round2": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "fhe_b200_rkg_aggregate": (_i, [_pp, _pp, _u32, _vp, _pp, _vp]),
    "fhe_b200_mul": (_i, [_vp, _vp, _vp, _vp]),
    "fhe_b200_relinearize": (_i, [_vp, _vp, _vp, _vp]),
    "fhe_b200_mul_relin": (_i, [_vp, _vp, _vp, _i, _vp, _vp]),
    "fhe_b200_multiplicator_create": (_i, [_vp, _u32, _vp, _u32, _vp, _u32, _vp, _u32, _vp, _u32, _vp, _u32, _vp,
                                           _vp, _u32, _vp, _u32, _vp]),
    "fhe_b200_multiplicator_free": (_i, [_vp]),
    "fhe_b200_multiplicator_multiply": (_i, [_vp, _vp, _vp, _vp, _i, _vp, _vp]),
    "fhe_b200_galois": (_i, [_vp, _u32, _vp, _vp, _vp]),
    "fhe_b200_expand": (_i, [_vp, _u32, _pp, _u32, _vp, _vp]),
    "fhe_b200_substitute": (_i, [_vp, _u32, _vp, _vp]),
    "fhe_b200_switch_down": (_i, [_vp, _vp]),
    "fhe_b200_key_switch": (_i, [_vp, _u32, _vp, _vp, _vp]),
    "fhe_b200_key_switch_keyed": (_i, [_vp, _u32, _pp, _u32, _pu32, _vp, _vp]),
    "fhe_b200_relinearize_keyed": (_i, [_vp, _pp, _u32, _pu32, _vp, _vp]),
    "fhe_b200_mul_relin_keyed": (_i, [_vp, _vp, _pp, _u32, _pu32, _i, _vp, _vp]),
    "fhe_b200_galois_keyed": (_i, [_vp, _u32, _pp, _u32, _pu32, _vp, _vp]),
    "fhe_b200_expand_keyed": (_i, [_vp, _u32, _pp, _u32, _u32, _pu32, _vp, _vp]),
    "fhe_b200_galois_many": (_i, [_vp, _pu32, _pp, _pu32, _u32, _pu32, _vp, _vp]),
    "fhe_b200_galois_many_hoisted": (_i, [_vp, _pu32, _pp, _pu32, _u32, _pu32, _vp, _pu32, _vp]),
    "fhe_b200_linear_transform": (_i, [_vp, _vp, _u32, _u32, _pp, _pu32, _u32, _vp, _pu32, _vp]),
    "fhe_b200_inner_sum": (_i, [_vp, _pp, _u32, _vp, _vp]),
    "fhe_b200_inner_sum_keyed": (_i, [_vp, _pp, _u32, _u32, _pu32, _vp, _vp]),
    "fhe_b200_batch_sum": (_i, [_vp, _u32, _i, _vp, _vp]),
    "fhe_b200_dot_product": (_i, [_vp, _vp, _u32, _vp, _vp, _vp]),
    "fhe_b200_dot_product_keyed": (_i, [_vp, _vp, _u32, _pp, _u32, _pu32, _vp, _vp]),
    "fhe_b200_scale": (_i, [_vp, _i, _vp, _vp]),
    "fhe_b200_poly_packed_bytes": (_i, [_vp, _u32, C.POINTER(C.c_size_t)]),
    "fhe_b200_batch_packed_bytes": (_i, [_vp, C.POINTER(C.c_size_t)]),
    "fhe_b200_batch_pack": (_i, [_vp, _u32, _u32, _vp, _vp]),
    "fhe_b200_batch_unpack": (_i, [_vp, _u32, _u32, _vp, _vp]),
    "fhe_b200_transcode": (_i, [_vp, _vp, _u32, C.c_size_t, C.c_size_t, _u32, _vp, _u32, C.c_size_t, C.c_size_t,
                                _u32, _u32, _vp]),
    "fhe_b200_fold": (_i, [_vp, _u32, _u32, _vp, _vp]),
    "fhe_b200_sync": (_i, [_vp]),
    "fhe_b200_launch_count": (_u64, []),
    "fhe_b200_ntt_row_count": (_u64, [_i]),
    "fhe_b200_debug_scaler_tables": (_i, [_vp, _u32, _i, _pu32, _pu32, _pu32] + [_vp] * 8),
    "fhe_b200_debug_ntt_tables": (_i, [_vp, _u64, _vp, _vp, _vp, _vp, _pu64]),
    "fhe_b200_debug_expansion_monomial": (_i, [_vp, _u32, _u32, _vp]),
    "fhe_b200_debug_encoder_tables": (_i, [_vp, _u32, _vp, _vp, _vp, _pu64, _vp]),
}

_lib = None


def lib() -> C.CDLL:
    """Load libfhe_b200.so.  Raises if the CUDA extension has not been built
    (`python -m fhe_rs_b200.build`): the product has no CPU fallback."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError(
                "fhe_rs_b200: %s is missing -- build it with `python -m fhe_rs_b200.build` "
                "(there is no CPU fallback)" % LIB_PATH)
        _lib = C.CDLL(LIB_PATH)
        for name, (res, args) in SYMBOLS.items():
            f = getattr(_lib, name)
            f.restype, f.argtypes = res, args
    return _lib


class FheError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__("fhe_b200 error %d: %s" % (code, msg))
        self.code = code


def check(code: int) -> None:
    if code != OK:
        raise FheError(code, lib().fhe_b200_last_error().decode())
