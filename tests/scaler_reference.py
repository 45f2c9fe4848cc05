"""A plain-integer transcription of `RnsScaler::scale` (fhe-math rns/scaler.rs:249-352).

It is a third implementation of the exact scaler next to the oracle's C (oracle/fhe_oracle.c) and the device kernels
(scale_kernel, scale_tma_kernel and scale_small_kernel in fhe_rs_b200/csrc/kernels.cu).  The fixed-point steps are kept
as the reference codes them -- the U256 wrapping sums, the `>> (shift - 1)` and `div_ceil(2)` of v, the sign taken from
bit 191 and the `!sum >> 126` branch of w -- because these steps, not exact rounding, are what the device has to match.
The tables (theta_garner, theta_omega with signs, theta_gamma, omega, gamma, the shift) are taken from the oracle's
`RnsScaler`; only the arithmetic of `scale` is restated here.
"""
from __future__ import annotations

from typing import List, Sequence

M64 = (1 << 64) - 1
M128 = (1 << 128) - 1
M256 = (1 << 256) - 1


def _lazy_mul_shoup(p: int, a: int, b: int, b_shoup: int) -> int:
    """zq/mod.rs:224-234: [0, 2p)"""
    q = (a * b_shoup) >> 64
    return (a * b - q * p) & M64


def _lazy_reduce_u128(p: int, barrett: int, a: int) -> int:
    """zq/mod.rs:693-707: [0, 2p)"""
    b_lo, b_hi = barrett & M64, barrett >> 64
    a_lo, a_hi = a & M64, a >> 64
    p_lo_lo = (a_lo * b_lo) >> 64
    p_hi_lo = a_hi * b_lo
    p_lo_hi = a_lo * b_hi
    q = (((p_lo_hi + p_hi_lo + p_lo_lo) >> 64) + a_hi * b_hi) & M128
    return ((a - q * p) & M128) & M64


def _reduce_u128(p: int, barrett: int, a: int) -> int:
    """zq/mod.rs:594-596"""
    r = _lazy_reduce_u128(p, barrett, a)
    return r - p if r >= p else r


def v_and_w_sum(sc, rests: Sequence[int]):
    """(v, sum_theta_omega) of RnsScaler::scale: the rounded Garner quotient and the U256 sum whose bit 191 is the sign
    of w (sum_theta_omega is None for a scaling factor of one)."""
    rests = [int(r) for r in rests]
    # :260-268  sum_theta_garner = sum r_i * theta_garner_i  (U256 wrapping_add)
    s = 0
    for lo, hi, r in zip(sc.theta_garner_lo, sc.theta_garner_hi, rests):
        s = (s + r * (int(lo) | (int(hi) << 64))) & M256
    # :270  sum_theta_garner >>= shift - 1
    s >>= sc.theta_garner_shift - 1
    # :271  v = sum.as_u128().div_ceil(2)
    v = -(-(s & M128) // 2)
    if sc.factor.is_one:
        return v, None
    # :278-292  sum_theta_omega = sum +/- r_i * theta_omega_i  (U256 wrapping_add / wrapping_sub)
    so = 0
    for lo, hi, sign, r in zip(sc.theta_omega_lo, sc.theta_omega_hi, sc.theta_omega_sign, rests):
        product = r * (int(lo) | (int(hi) << 64))
        so = (so - product) & M256 if sign else (so + product) & M256
    # :294-302  -/+ v * theta_gamma
    vtg = v * (sc.theta_gamma_lo | (sc.theta_gamma_hi << 64))
    so = (so + vtg) & M256 if sc.theta_gamma_sign else (so - vtg) & M256
    return v, so


def scale(sc, rests: Sequence[int], out_len: int, starting_index: int = 0) -> List[int]:
    """RnsScaler::scale of one residue vector; `sc` is an oracle `RnsScaler` (its tables only)."""
    rests = [int(r) for r in rests]
    is_one = sc.factor.is_one
    v, so = v_and_w_sum(sc, rests)
    # :273-276
    w_sign = False
    w = 0
    if not is_one:
        # :304-305  w_sign = (sum >> (63 + 128)) > 0
        w_sign = (so >> 191) > 0
        if w_sign:
            # :307-309  w = ((!sum) >> 126).as_u128() + 1; w /= 2
            w = ((((~so) & M256) >> 126) & M128) + 1
            w //= 2
        else:
            # :310-312  w = (sum >> 126).as_u128().div_ceil(2)
            w = ((so >> 126) & M128)
            w = -(-w // 2)
    out = []
    for i in range(out_len):
        # :316-350
        j = starting_index + i
        qi = sc.to.moduli_u64[j]
        barrett = (1 << 128) // qi
        gamma_i, gamma_shoup_i = int(sc.gamma[j]), int(sc.gamma_shoup[j])
        yi = qi * 2 - _lazy_mul_shoup(qi, _reduce_u128(qi, barrett, v), gamma_i, gamma_shoup_i)
        if not is_one:
            wi = _lazy_reduce_u128(qi, barrett, w)
            yi += qi * 2 - wi if w_sign else wi
        for r, om, om_s in zip(rests, sc.omega[j], sc.omega_shoup[j]):
            yi += _lazy_mul_shoup(qi, r, int(om), int(om_s))
        out.append(_reduce_u128(qi, barrett, yi & M128))
    return out
