"""SecretKey::random on the device (fhe_b200_secret_keys_random) restated on the oracle.

Key k of a call is sample_vec_cbd(N, variance) drawn from the seeded ChaCha20 stream of include/fhe_b200.h as role 18,
limb 0, word 13 = k, word 15 = 0: coefficient 4b + m takes value m of block b, and the 128-bit value v gives
popc(v & mask_add) - popc(v & mask_sub), exactly as the errors of tests/encrypt_reference.py.
"""
from __future__ import annotations

import numpy as np

import encrypt_reference as R

ROLE_S = 18


def secret_key_coeffs(seed: bytes, k: int, variance: int, degree: int) -> np.ndarray:
    """the signed coefficients of key k of a call: int64 [degree]"""
    return R.cbd(seed, k, ROLE_S, variance, degree)
