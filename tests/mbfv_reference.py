"""The multiparty BFV calls of include/fhe_b200.h (fhe::mbfv) restated on the oracle.

The algebra is the reference's (crates/fhe/src/mbfv: crp.rs, public_key_gen.rs, secret_key_switch.rs,
public_key_switch.rs), built from the oracle's Poly / Scaler operations; the random words are those of
encrypt_reference.py's stream with word 15 = 0 and word 13 = the index within the call:
  * role 7: the CRP, (hi 2^64 + lo) mod q_j of limb j's row, drawn directly as NTT words;
  * role 8: e of PublicKeyShare;  role 14: e of SecretKeySwitchShare / DecryptionShare;
  * roles 15, 16, 17: u, e0, e1 of PublicKeySwitchShare;
the small polynomials come from limb 0's row and are lifted to every limb.  `from_shares` performs the reference's
Plaintext::from_shares literally: the CRT lift of the scaled polynomial over the plaintext context, + t, mod Q_p, mod t.
"""
from __future__ import annotations

from typing import List, Optional, Sequence

import numpy as np

import encrypt_reference as R
import fhe_oracle as O

ROLE_CRP, ROLE_PK_E, ROLE_SKS_E, ROLE_PKS_U, ROLE_PKS_E0, ROLE_PKS_E1 = 7, 8, 14, 15, 16, 17
ROLES = (ROLE_CRP, ROLE_PK_E, ROLE_SKS_E, ROLE_PKS_U, ROLE_PKS_E0, ROLE_PKS_E1)


def crp(par: "O.BfvParameters", seed: bytes, count: int, level: int = 0) -> List["O.Poly"]:
    """fhe_b200_crp_generate: CRP k of the call at `level` (CommonRandomPoly::new_leveled, crp.rs:35-43)"""
    ctx = par.context_at_level(level)
    out = []
    for k in range(count):
        lo, hi = R.row_values(seed, k, ROLE_CRP, range(len(ctx.moduli)), ctx.degree)
        p = O.Poly(ctx, O.NTT)
        for j, q in enumerate(ctx.moduli):
            v = (hi[j].astype(object) << 64) | lo[j].astype(object)
            p.c[j] = (v % q).astype(np.uint64)
        out.append(p)
    return out


def _sum(polys: Sequence["O.Poly"]) -> "O.Poly":
    acc = polys[0].copy()
    for p in polys[1:]:
        acc.iadd(p)
    return acc


def pk_share(osk: "O.SecretKey", crps: Sequence["O.Poly"], seed: bytes, variance: int) -> List["O.Poly"]:
    """fhe_b200_pk_share: p0_k = -crp_k s + e_k (public_key_gen.rs:32-58)"""
    ctx = osk.par.context_at_level(0)
    s = osk.s_ntt(ctx)
    out = []
    for k, a in enumerate(crps):
        p0 = a.neg()
        p0.imul(s)
        p0.iadd(R.small_ntt(seed, k, ROLE_PK_E, variance, ctx))
        out.append(p0)
    return out


def pk_aggregate(par: "O.BfvParameters", shares: Sequence["O.Poly"], a: "O.Poly") -> "O.Ciphertext":
    """PublicKey::from_shares (public_key_gen.rs:60-77): c = (sum p0_i, crp)"""
    return O.Ciphertext(par, [_sum(shares), a.copy()], 0)


def sks_share(osk_in: "O.SecretKey", osk_out: Optional["O.SecretKey"], cts: Sequence["O.Ciphertext"], seed: bytes,
              variance: int) -> List["O.Poly"]:
    """fhe_b200_sks_share: h_k = (s_in - s_out) c1_k + e_k (secret_key_switch.rs:38-96); osk_out None is
    DecryptionShare's zero key (:133-143)"""
    out = []
    for k, ct in enumerate(cts):
        assert len(ct.c) == 2
        ctx = ct.c[0].ctx
        h = osk_in.s_ntt(ctx)
        if osk_out is not None:
            h.isub(osk_out.s_ntt(ctx))
        h.imul(ct.c[1])
        h.iadd(R.small_ntt(seed, k, ROLE_SKS_E, variance, ctx))
        out.append(h)
    return out


def sks_aggregate(ct: "O.Ciphertext", hs: Sequence["O.Poly"]) -> "O.Ciphertext":
    """Ciphertext::from_shares of SecretKeySwitchShares (secret_key_switch.rs:98-115): (c0 + sum h, c1)"""
    return O.Ciphertext(ct.par, [ct.c[0].copy().iadd(_sum(hs)), ct.c[1].copy()], ct.level)


def pks_share(osk: "O.SecretKey", pk: "O.Ciphertext", cts: Sequence["O.Ciphertext"], seed: bytes,
              variance: int) -> List["O.Ciphertext"]:
    """fhe_b200_pks_share: (u pk0 + s c1 + e0, u pk1 + e1), pk switched down to the ciphertext's level
    (public_key_switch.rs:33-93)"""
    out = []
    for k, ct in enumerate(cts):
        c = pk.copy().switch_to_level(ct.level)
        ctx = ct.c[0].ctx
        u = R.small_ntt(seed, k, ROLE_PKS_U, variance, ctx)
        h0 = c.c[0].mul(u)
        h0.iadd(osk.s_ntt(ctx).mul(ct.c[1]))
        h0.iadd(R.small_ntt(seed, k, ROLE_PKS_E0, variance, ctx))
        h1 = c.c[1].mul(u)
        h1.iadd(R.small_ntt(seed, k, ROLE_PKS_E1, variance, ctx))
        out.append(O.Ciphertext(ct.par, [h0, h1], ct.level))
    return out


def pks_aggregate(ct: "O.Ciphertext", shares: Sequence["O.Ciphertext"]) -> "O.Ciphertext":
    """Ciphertext::from_shares of PublicKeySwitchShares (public_key_switch.rs:95-112): (c0 + sum h0, sum h1)"""
    return O.Ciphertext(ct.par, [ct.c[0].copy().iadd(_sum([s.c[0] for s in shares])), _sum([s.c[1] for s in shares])],
                        ct.level)


def lift_from_limb0(r: int, t: int, q0: int, n_plain: int) -> int:
    """the device's from_shares lift from the residue r modulo q_0 of the scaled value v (|v| <= t / 2, t < q_0) with
    n_plain plaintext-context moduli: try_decrypt's ((r + t) mod q_0) mod t for one, else v mod t, v < 0 exactly when
    r > q_0 / 2"""
    if n_plain == 1:
        return ((r + t) % q0) % t
    return (r + t - (q0 if r > q0 // 2 else 0)) % t


def from_shares(ct: "O.Ciphertext", hs: Sequence["O.Poly"]):
    """Plaintext::from_shares (secret_key_switch.rs:145-186), literally: returns (poly_ntt, the coefficients w)"""
    par = ct.par
    c = sks_aggregate(ct, hs).c[0].into_power_basis()
    d = par.level(ct.level).scaler.scale(c)
    t = par.plaintext
    v = [vi + t for vi in d.to_bigints()]
    q_poly = d.ctx.modulus()
    w = [(wi % q_poly) % t for wi in v[:par.degree]]
    poly = O.Poly(c.ctx, O.POWER_BASIS)
    for j, q in enumerate(c.ctx.moduli):
        poly.c[j] = np.array([x % q for x in w], dtype=np.uint64)
    return poly.into_ntt(), np.array(w, dtype=np.uint64)


# ---- RelinKeyGenerator (relin_key_gen.rs): u (role 9, word 15 = 0), the errors of round 1 (roles 10, 11) and round 2
# (roles 12, 13) with word 13 = 0 and word 15 = the CRP / digit index i
ROLE_RKG_U, ROLE_RKG_R1_E0, ROLE_RKG_R1_E1, ROLE_RKG_R2_E0, ROLE_RKG_R2_E1 = 9, 10, 11, 12, 13


def small_digit(seed: bytes, role: int, digit: int, variance: int, ctx: "O.Context") -> "O.Poly":
    """the centred binomial polynomial of the row (0, role, limb 0, digit), lifted and transformed"""
    b = np.arange(ctx.degree // 4, dtype=np.uint32)
    blk = R.chacha20_blocks(seed, b, 0, role << 8, digit).astype(np.uint64)
    lo = (blk[..., 0::4] | (blk[..., 1::4] << np.uint64(32))).reshape(ctx.degree)
    hi = (blk[..., 2::4] | (blk[..., 3::4] << np.uint64(32))).reshape(ctx.degree)
    (alo, ahi), (slo, shi) = R.cbd_masks(variance)
    pc = lambda v: np.bitwise_count(v).astype(np.int64)  # noqa: E731
    x = (pc(lo & alo) + pc(hi & ahi)) - (pc(lo & slo) + pc(hi & shi))
    return O.Poly.from_i64(ctx, x, O.NTT)


def rkg_u(par: "O.BfvParameters", seed: bytes, variance: int) -> "O.Poly":
    """fhe_b200_rkg_create: u of RelinKeyGenerator::new (relin_key_gen.rs:76-96)"""
    return small_digit(seed, ROLE_RKG_U, 0, variance, par.context_at_level(0))


def rkg_round1(osk: "O.SecretKey", crps: Sequence["O.Poly"], u: "O.Poly", seed: bytes, variance: int):
    """RelinKeyShare<R1>::new (relin_key_gen.rs:112-198): h0_i = -a_i u + w_i s + e, h1_i = a_i s + e"""
    ctx = osk.par.context_at_level(0)
    s = osk.s_ntt(ctx)
    garner = O.RnsContext(ctx.moduli).garner
    h0, h1 = [], []
    for i, a in enumerate(crps):
        h = a.neg()
        h.imul(u)
        h.iadd(s.mul_scalar_big(garner[i]))
        h.iadd(small_digit(seed, ROLE_RKG_R1_E0, i, variance, ctx))
        h0.append(h)
        h1.append(a.mul(s).iadd(small_digit(seed, ROLE_RKG_R1_E1, i, variance, ctx)))
    return h0, h1


def rkg_r1_aggregate(shares):
    """RelinKeyShare<R1Aggregated>::from_shares (relin_key_gen.rs:200-222): shares = [(h0, h1)] of every party"""
    L = len(shares[0][0])
    return [_sum([sh[0][i] for sh in shares]) for i in range(L)], [_sum([sh[1][i] for sh in shares]) for i in range(L)]


def rkg_round2(osk: "O.SecretKey", u: "O.Poly", r1_h0: Sequence["O.Poly"], r1_h1: Sequence["O.Poly"], seed: bytes,
               variance: int):
    """RelinKeyShare<R2>::new (relin_key_gen.rs:224-297): h0'_i = r1_h0_i s + e, h1'_i = r1_h1_i (u - s) + e"""
    ctx = osk.par.context_at_level(0)
    s = osk.s_ntt(ctx)
    u_s = u.copy().isub(s)
    h0 = [h.mul(s).iadd(small_digit(seed, ROLE_RKG_R2_E0, i, variance, ctx)) for i, h in enumerate(r1_h0)]
    h1 = [h.mul(u_s).iadd(small_digit(seed, ROLE_RKG_R2_E1, i, variance, ctx)) for i, h in enumerate(r1_h1)]
    return h0, h1


def rkg_aggregate(shares, r1_h1: Sequence["O.Poly"]):
    """RelinearizationKey::from_shares (relin_key_gen.rs:299-350): the key's (c0, c1) words [digit][limb][N] with
    c0_i = sum h0'_i + sum h1'_i and c1_i = r1_h1_i"""
    h0, h1 = rkg_r1_aggregate(shares)
    c0 = np.stack([a.copy().iadd(b).c for a, b in zip(h0, h1)])
    c1 = np.stack([h.c for h in r1_h1])
    return c0, c1
