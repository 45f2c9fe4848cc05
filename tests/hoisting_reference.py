"""Hoisted rotations restated on the CPU oracle (DESIGN §8), for tests/test_hoisted_cpu.py and the expected counts of
tests/test_gpu_hoisted.py.

GaloisKey::relinearize (galois_key.rs:63-86) key-switches the power-basis sigma_e(c1): digit k of the reference is its
residue row modulo q_k, which holds x at the coefficients sigma keeps and q_k - x (0 when x = 0) at those it negates.
sigma_e applied to the digit rows of c1 instead gives -x = q_j - x modulo q_j.  The two differ by exactly q_k at every
negated coefficient whose source residue is not zero, so with D_k[j] = NTT_j(lazy(x_k)) (rq/mod.rs:563-586), pi_e the
NTT-domain permutation of sigma_e (rq/mod.rs:360-389) and M_e[j] = NTT_j(N_e), N_e the 0/1 polynomial of the negated
coefficients (rq/mod.rs:390-408):

    key_switch(sigma_e(c1))_p[j] = sum_k key_p,k[j] (.) pi_e(D_k[j])  +  M_e[j] (.) sum_k [q_k]_{q_j} key_p,k[j]

modulo q_j, unless some negated coefficient s >= 1 has a zero residue in some row k (needs_fallback).  The second
term is the form the device kernel computes."""
from typing import List, Sequence

import numpy as np

import fhe_oracle as O


def negates(degree: int, e: int, s) -> np.ndarray:
    """whether sigma_e negates coefficient s: (s * e mod 2N) >= N"""
    return (np.asarray(s, dtype=np.int64) * (e % (2 * degree))) % (2 * degree) >= degree


def negation_row(degree: int, e: int) -> np.ndarray:
    """N_e: 1 at every destination x^d whose source x^s sigma_e negates"""
    s = np.arange(degree, dtype=np.int64)
    p = (s * (e % (2 * degree))) % (2 * degree)
    row = np.zeros(degree, np.uint64)
    row[p[p >= degree] - degree] = 1
    return row


def needs_fallback(c1_power: np.ndarray, e: int) -> bool:
    """the exact predicate of fhe_b200_galois_many_hoisted: some residue row of the power-basis c1 ([L][N]) is zero at
    a position s >= 1 that sigma_e negates"""
    degree = c1_power.shape[-1]
    zero = (c1_power == 0).any(axis=0)
    zero[0] = False
    return bool(negates(degree, e, np.nonzero(zero)[0]).any())


def hoisted_count(c1_power: Sequence[np.ndarray], exponents: Sequence[int], source: Sequence[int]) -> int:
    """how many outputs the hoisted call computes from shared digits: output j (exponent exponents[j], source
    source[j]) when its source has two or more outputs and needs no fallback; c1_power[s] is source s's [L][N]"""
    uses = np.bincount(np.asarray(source, dtype=np.int64), minlength=len(c1_power))
    return sum(1 for e, s in zip(exponents, source) if uses[s] >= 2 and not needs_fallback(c1_power[s], e))


def digits(ksk: "O.KeySwitchingKey", c1_power: "O.Poly") -> List["O.Poly"]:
    """D_k = the lazy transforms of the residue rows of c1 in the key's context, computed once for every exponent"""
    return [O.lazy_constant_ntt(c1_power.c[k], ksk.ctx_ksk) for k in range(len(ksk.c0))]


def hoisted_key_switch(ksk: "O.KeySwitchingKey", D: Sequence["O.Poly"], e: int):
    """(c0, c1) of KeySwitchingKey::key_switch(sigma_e(c1)) from the digits of c1, by the identity above"""
    ctx = ksk.ctx_ksk
    M = O.Poly(ctx, O.POWER_BASIS, np.tile(negation_row(ctx.degree, e), (len(ctx.moduli), 1))).into_ntt()
    out = []
    for key in (ksk.c0, ksk.c1):
        rows = []
        for j, q in enumerate(ctx.moduli):
            q = int(q)
            acc = np.zeros(ctx.degree, dtype=object)
            h = np.zeros(ctx.degree, dtype=object)
            for k, Dk in enumerate(D):
                t = O.Poly(ctx, O.NTT, Dk.c).substitute(e).c[j].astype(object)   # pi_e of the lazy words
                kw = key[k].c[j].astype(object)
                acc += t * kw
                h += (int(ctx.moduli[k]) % q) * kw
            rows.append(((acc + (h % q) * M.c[j].astype(object)) % q).astype(np.uint64))
        out.append(O.Poly(ctx, O.NTT, np.stack(rows)))
    return out[0], out[1]


def hoisted_relinearize(gk: "O.GaloisKey", ct: "O.Ciphertext", D=None) -> "O.Ciphertext":
    """GaloisKey::relinearize from the digits of ct's c1 (computed here when D is None)"""
    if D is None:
        D = digits(gk.ksk, ct.c[1].copy().into_power_basis())
    c0, c1 = hoisted_key_switch(gk.ksk, D, gk.exponent)
    c0, c1 = O._post_key_switch(c0, c1, ct.c[0].ctx)
    c0.iadd(ct.c[0].substitute(gk.exponent))
    return O.Ciphertext(ct.par, [c0, c1], gk.ksk.ciphertext_level)
