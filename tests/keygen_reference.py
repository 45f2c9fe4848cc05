"""Key generation on the device (fhe_b200_relin_key_generate, fhe_b200_galois_keys_generate, fhe_b200_rgsw_encrypt)
restated on the oracle the reference's way, without the device's NTT-domain shortcut.

The stream is the one of encrypt_reference.py with two more roles.  Block b of the row (key k, role, limb, digit i)
is the ChaCha20 block of the state (constants, seed, b, k, role << 8 | limb, i):
  * c1_i (role 5, limb j of the key level): (hi 2^64 + lo) mod q_j, as NTT words;
  * e_i (role 6, limb 0): the centred binomial sample of the variance.
KeySwitchingKey::new (key_switching_key.rs:71-238) then builds b = e_i - INTT(c1_i s) + g_i from in the power basis,
with g_i the Garner coefficient of the ciphertext basis (RnsContext.garner) or 2^(i log_base), and transforms it.
`from` is built as the reference does: s s, s substituted, or the plaintext (times s), switched up with Switcher.
"""
from __future__ import annotations

from typing import List, Sequence

import numpy as np

import encrypt_reference as R
import fhe_oracle as O

ROLE_C1, ROLE_KEY_E = 5, 6


def row_values(seed: bytes, key: int, role: int, limbs: Sequence[int], digit: int, degree: int):
    """(lo, hi) uint64 [len(limbs)][degree] of the rows (key, role, limb, digit)"""
    b = np.arange(degree // 4, dtype=np.uint32)[None, :]
    w14 = np.array([(role << 8) | j for j in limbs], dtype=np.uint32)[:, None]
    blk = R.chacha20_blocks(seed, b, key, w14, digit).astype(np.uint64)
    lo = blk[..., 0::4] | (blk[..., 1::4] << np.uint64(32))
    hi = blk[..., 2::4] | (blk[..., 3::4] << np.uint64(32))
    return lo.reshape(len(limbs), degree), hi.reshape(len(limbs), degree)


def c1_ntt(seed: bytes, key: int, digit: int, ctx: "O.Context") -> "O.Poly":
    lo, hi = row_values(seed, key, ROLE_C1, range(len(ctx.moduli)), digit, ctx.degree)
    p = O.Poly(ctx, O.NTT)
    for j, q in enumerate(ctx.moduli):
        p.c[j] = (((hi[j].astype(object) << 64) | lo[j].astype(object)) % q).astype(np.uint64)
    return p


def error(seed: bytes, key: int, digit: int, variance: int, degree: int) -> np.ndarray:
    """e_i: the signed centred binomial coefficients, int64 [degree]"""
    lo, hi = row_values(seed, key, ROLE_KEY_E, [0], digit, degree)
    (alo, ahi), (slo, shi) = R.cbd_masks(variance)
    pc = lambda v: np.bitwise_count(v).astype(np.int64)
    return (pc(lo[0] & alo) + pc(hi[0] & ahi)) - (pc(lo[0] & slo) + pc(hi[0] & shi))


def gadget(par: "O.BfvParameters", ciphertext_level: int, ksk_level: int) -> List[int]:
    """g_i of every digit: the Garner coefficients of the ciphertext basis, or 2^(i log_base) for a single-modulus
    key level"""
    ctx_ksk = par.context_at_level(ksk_level)
    log_base, n_dec = O._ksk_log_base(ctx_ksk)
    if log_base:
        return [1 << (i * log_base) for i in range(n_dec)]
    return list(O.RnsContext(par.moduli[:len(par.context_at_level(ciphertext_level).moduli)]).garner)


def key_digit(osk: "O.SecretKey", frm: "O.Poly", ciphertext_level: int, ksk_level: int, seed: bytes, key: int,
              i: int, variance: int):
    """digit i of KeySwitchingKey::new from `frm` (power basis at the key level), key index `key` of the call:
    (c0_i, c1_i) as NTT words [key limbs][N]"""
    par = osk.par
    ctx = par.context_at_level(ksk_level)
    assert frm.ctx == ctx and frm.rep == O.POWER_BASIS
    a = c1_ntt(seed, key, i, ctx)
    b = O.Poly.from_i64(ctx, error(seed, key, i, variance, ctx.degree))
    b.isub(a.mul(osk.s_ntt(ctx)).into_power_basis())
    b.iadd(frm.mul_scalar_big(gadget(par, ciphertext_level, ksk_level)[i]))
    return b.into_ntt().c, a.c


def key_switching_key(osk: "O.SecretKey", frm: "O.Poly", ciphertext_level: int, ksk_level: int, seed: bytes,
                      key: int, variance: int) -> "O.KeySwitchingKey":
    """KeySwitchingKey::new from `frm` (power basis at the key level) with key index `key` of the call"""
    n = len(gadget(osk.par, ciphertext_level, ksk_level))
    c0, c1 = zip(*[key_digit(osk, frm, ciphertext_level, ksk_level, seed, key, i, variance) for i in range(n)])
    return O.KeySwitchingKey.from_arrays(osk.par, np.stack(c0), np.stack(c1), ciphertext_level, ksk_level)


def relin_from(osk, ciphertext_level: int, key_level: int) -> "O.Poly":
    """relinearization_key.rs:56-62: s s switched up to the key level"""
    par = osk.par
    ctx_ct, ctx_rk = par.context_at_level(ciphertext_level), par.context_at_level(key_level)
    s = osk.s_ntt(ctx_ct)
    return O.Switcher(ctx_ct, ctx_rk).switch(s.mul(s).into_power_basis())


def galois_from(osk, exponent: int, ciphertext_level: int, key_level: int) -> "O.Poly":
    """galois_key.rs:36-46: s substituted, switched up to the key level"""
    par = osk.par
    ctx_ct, ctx_gk = par.context_at_level(ciphertext_level), par.context_at_level(key_level)
    return O.Switcher(ctx_ct, ctx_gk).switch(O.Poly.from_i64(ctx_ct, osk.coeffs).substitute(exponent))


def rgsw_from(osk, m: "O.Poly", level: int, times_s: bool) -> "O.Poly":
    """rgsw_ciphertext.rs:106-113: m (ksk0) or m s (ksk1) in the power basis, m = pt.poly_ntt"""
    if times_s:
        return osk.s_ntt(osk.par.context_at_level(level)).imul(m).into_power_basis()
    return m.copy().into_power_basis()


def relinearization_key(osk, seed: bytes, ciphertext_level: int, key_level: int, variance: int):
    """RelinearizationKey::new_leveled (relinearization_key.rs:43-65): from = s s switched up"""
    up = relin_from(osk, ciphertext_level, key_level)
    return O.RelinearizationKey.from_ksk(key_switching_key(osk, up, ciphertext_level, key_level, seed, 0, variance))


def galois_keys(osk, exponents: Sequence[int], seed: bytes, ciphertext_level: int, key_level: int,
                variance: int) -> List["O.GaloisKey"]:
    """GaloisKey::new (galois_key.rs:26-60) for key k = exponents[k] of one call"""
    par = osk.par
    out = []
    for k, e in enumerate(exponents):
        up = galois_from(osk, e, ciphertext_level, key_level)
        gk = O.GaloisKey.__new__(O.GaloisKey)
        gk.exponent = e % (2 * par.degree)
        gk.ksk = key_switching_key(osk, up, ciphertext_level, key_level, seed, k, variance)
        out.append(gk)
    return out


def rgsw(osk, ms: Sequence["O.Poly"], level: int, seed: bytes, variance: int) -> List["O.RGSWCiphertext"]:
    """SecretKey::try_encrypt into RGSWCiphertext (rgsw_ciphertext.rs:94-120) of each plaintext's poly_ntt (NTT at
    `level`): ksk0 = key 2p from m, ksk1 = key 2p + 1 from m s"""
    out = []
    for p, m in enumerate(ms):
        r = O.RGSWCiphertext.__new__(O.RGSWCiphertext)
        r.level = level
        r.ksk0 = key_switching_key(osk, rgsw_from(osk, m, level, False), level, level, seed, 2 * p, variance)
        r.ksk1 = key_switching_key(osk, rgsw_from(osk, m, level, True), level, level, seed, 2 * p + 1, variance)
        out.append(r)
    return out


def switch_up_closed_form(x_ntt: "O.Poly", ctx_key: "O.Context") -> "O.Poly":
    """the device's form of Switcher(ctx_ct, ctx_key).switch(x): x (Q_key / Q_ct) on the ciphertext limbs, 0 on the
    others (NTT words in, NTT words out)"""
    L = len(x_ntt.ctx.moduli)
    P = ctx_key.modulus() // x_ntt.ctx.modulus()
    out = O.Poly(ctx_key, O.NTT)
    for j, q in enumerate(ctx_key.moduli[:L]):
        out.c[j] = ((x_ntt.c[j].astype(object) * (P % q)) % q).astype(np.uint64)
    return out


def evaluation_key_exponents(degree: int, inner_sum=False, row_rotation=False, expansion_level=0,
                             column_rotation=()) -> List[int]:
    """EvaluationKeyBuilder::build's index set (evaluation_key.rs:439-463), ascending"""
    idx = {pow(3, i, 2 * degree) for i in column_rotation}
    if row_rotation or inner_sum:
        idx.add(2 * degree - 1)
    if inner_sum:
        i = 1
        while i < degree // 2:
            idx.add(pow(3, i, 2 * degree))
            i *= 2
    idx.update((degree >> l) + 1 for l in range(expansion_level))
    return sorted(idx)
