"""A plain-integer restatement of the reference's client for a plaintext modulus of any length (fhe/src/bfv at
e248cd28): encoding `&[BigUint]` and signed values, `Plaintext::to_poly`, encryption, `SecretKey::try_decrypt` and
decoding back to `Vec<BigUint>`.

The oracle's own client (fhe_oracle.plaintext_to_poly, SecretKey.decrypt) follows the small-t fast path, where t is a
`zq::Modulus`; the reference takes the branches restated here whenever t does not fit one (t >= 2^62), and this library
refuses every client entry point there.  A host that encrypts with the reference at such a t and runs the server path
on the device needs exactly these steps to check what the device computed.  Polynomials are oracle `Poly`s; every
coefficient is handled as a Python integer.  `decrypt_literal` is the definition the restated decryption has to agree
with: round(t * phase / Q_l) mod t.  BIGT_SETS holds the parameter sets the large-t tests share.
"""
from __future__ import annotations

from typing import List, Sequence

import numpy as np

import fhe_oracle as O


def is_small(t: int) -> bool:
    """PlaintextModulus::try_new (parameters.rs:35-49): t has a `small()` Modulus when it is a u64 that
    Modulus::new accepts (zq/mod.rs:32-45: 2 <= t < 2^62)"""
    return 2 <= t < 1 << 62


def _poly_from_bigints(ctx: O.Context, values: Sequence[int]) -> O.Poly:
    """Poly::<PowerBasis>::try_convert_from(&[BigUint], ctx) (rq/convert.rs:362-386): value mod q_i in limb i,
    zero-padded to N coefficients"""
    vals = [int(v) for v in values] + [0] * (ctx.degree - len(values))
    rows = np.array([[v % q for v in vals] for q in ctx.moduli], dtype=np.uint64)
    return O.Poly(ctx, O.POWER_BASIS, rows)


def encode(par: O.BfvParameters, values: Sequence[int], level: int = 0) -> O.Poly:
    """Plaintext::try_encode(&[BigUint], Encoding::poly_at_level(level)) (plaintext.rs:291-309 through
    plaintext_vec.rs:104-118): the values go into the polynomial as they are -- not reduced mod t -- and the
    plaintext is that polynomial in the NTT domain (`poly_ntt`)"""
    if len(values) > par.degree:
        raise ValueError("TooManyValues")
    return _poly_from_bigints(par.context_at_level(level), values).into_ntt()


def encode_signed(par: O.BfvParameters, values: Sequence[int], level: int = 0) -> O.Poly:
    """Plaintext::try_encode(&[i64]) (plaintext.rs:351-372): the `None` branch maps x to x mod t in [0, t) and
    encodes the result as `&[BigUint]`; the small branch (reduce_vec_i64) gives the same residues"""
    t = par.plaintext
    return encode(par, [int(x) % t for x in values], level)


def coefficients(par: O.BfvParameters, pt: O.Poly) -> List[int]:
    """Plaintext::coefficients (plaintext.rs:103-135): the power-basis words, reduced mod t.  With a small t below
    q_0 the reference reduces limb 0 only; otherwise it lifts every coefficient over the plaintext's context
    (Vec<BigUint>::from(&Poly)) and reduces the lift mod t."""
    t = par.plaintext
    pb = pt.copy().into_power_basis()
    if is_small(t) and t < pt.ctx.moduli[0]:
        return [int(v) % t for v in pb.c[0]]
    return [v % t for v in pb.to_bigints()]


def to_poly(par: O.BfvParameters, pt: O.Poly, level: int = 0) -> O.Poly:
    """Plaintext::to_poly (plaintext.rs:172-197): coefficients * (Q_l mod t) mod t (PlaintextModulus::scalar_mul_vec,
    parameters.rs:66-69, for `Large`; the same residues as Modulus::scalar_mul_vec for `Small`), into the level's
    context, transformed, times delta = (-t)^-1 mod q_i (parameters.rs:604-624)"""
    t = par.plaintext
    lvl = par.level(level)
    vals = [v * lvl.q_mod_t % t for v in coefficients(par, pt)]
    return _poly_from_bigints(lvl.poly_context, vals).into_ntt().imul(lvl.delta)


def encrypt(sk: O.SecretKey, pt: O.Poly, level: int, rng) -> O.Ciphertext:
    """SecretKey::try_encrypt (secret_key.rs:183-191): the oracle's encrypt_poly of to_poly"""
    return sk.encrypt_poly(to_poly(sk.par, pt, level), level, rng)


def decrypt_values(sk: O.SecretKey, ct: O.Ciphertext) -> List[int]:
    """try_decrypt (secret_key.rs:198-260) up to the polynomial it builds: the phase in the power basis, scaled by
    t / Q_l into the plaintext context (cipher_plain_context.scaler, parameters.rs:638-643), then
      * `Some(t)` (:229-238): v + t over the concatenated u64 words, the first N of them (limb 0) mod q_0, mod t;
      * `None` (:239-250): every coefficient lifted over the plaintext context, + t, mod Q_plain, mod t."""
    par = sk.par
    t = par.plaintext
    c_pb = sk.phase(ct).into_power_basis()
    d = par.level(ct.level).scaler.scale(c_pb)
    if is_small(t):
        q0 = par.moduli[0]
        return [((int(v) + t) % q0) % t for v in d.c[0]]
    q_plain = d.ctx.modulus()
    return [((v + t) % q_plain) % t for v in d.to_bigints()]


def decrypt(sk: O.SecretKey, ct: O.Ciphertext) -> O.Poly:
    """try_decrypt's plaintext (secret_key.rs:229-257): the values as a polynomial of the ciphertext's context, NTT"""
    return _poly_from_bigints(ct.c[0].ctx, decrypt_values(sk, ct)).into_ntt()


def decode(par: O.BfvParameters, pt: O.Poly) -> List[int]:
    """Vec<BigUint>::try_decode(pt, Encoding::poly()) (plaintext.rs:376-400): the coefficients"""
    return coefficients(par, pt)


def decrypt_literal(sk: O.SecretKey, ct: O.Ciphertext) -> List[int]:
    """The definition: round(t * phase / Q_l) mod t, phase in [0, Q_l).  t * phase / Q_l is never a half-integer
    (Q_l is odd), so the rounding is unambiguous."""
    t = sk.par.plaintext
    ph = sk.phase(ct).into_power_basis()
    Q = ph.ctx.modulus()
    return [((2 * t * x + Q) // (2 * Q)) % t for x in ph.to_bigints()]


def negacyclic(a: Sequence[int], b: Sequence[int], t: int) -> List[int]:
    """a * b in Z_t[x] / (x^N + 1)"""
    n = len(a)
    out = [0] * n
    for i, x in enumerate(a):
        if not x:
            continue
        for j, y in enumerate(b):
            k = i + j
            if k < n:
                out[k] += x * y
            else:
                out[k - n] -= x * y
    return [v % t for v in out]


# ------------------------------------------------------------------------------------------ parameter sets

def _product(moduli: Sequence[int]) -> int:
    out = 1
    for q in moduli:
        out *= int(q)
    return out


def prime_below(bound: int) -> int:
    """the largest (probable) prime below bound, any length"""
    p = bound - 1
    while not O.is_prime(p):
        p -= 1
    return p


def prime_at_or_above(bound: int) -> int:
    p = bound
    while not O.is_prime(p):
        p += 1
    return p


# name -> (degree, plaintext modulus, moduli sizes).  Every t is prime, hence coprime with every ciphertext modulus.
# t > Q_l at a level makes the down scaler's factor t / Q_l at least one.  The N = 16 sets take scale_small_kernel;
# tma_200 has only Solinas limbs (scale_tma_kernel), mixed_200 does not (scale_kernel).
BIGT_SETS = {
    "m127": (16, lambda: (1 << 127) - 1, [60] * 5),                    # biguint.rs; t > Q_l at levels 3, 4
    "wide_2_62": (16, lambda: prime_at_or_above((1 << 62) + 135), [62] * 3),   # t in [2^62, 2^64); t > Q_2
    "t62_above_q0": (64, lambda: prime_below(1 << 62), [62] * 3),     # t_small, but q_0 < t; t > Q_2
    # 8 limbs rather than 6: a product decrypts only when Q_l exceeds about t^2 N 2^10
    "tma_200": (1 << 13, lambda: prime_below(1 << 200), [62] * 8),    # t > Q_l at levels 5..7
    "mixed_200": (1 << 13, lambda: prime_below(1 << 200), [62, 62, 62, 40, 30, 50]),   # t > Q_l at levels 3..5
    "set_c_near_q": (1 << 15, None, [62] * 14),                        # t: 807 bits, t > Q_l from level 1 on
}


def bigt_set(name: str):
    """(degree, t, moduli) of BIGT_SETS[name]; set_c_near_q takes the largest prime below Q / 2^61"""
    degree, t, sizes = BIGT_SETS[name]
    moduli = O.BfvParameters.generate_moduli(sizes, degree)
    return degree, (t() if t is not None else prime_below(_product(moduli) >> 61)), moduli


def levels_t_above_q(t: int, moduli: Sequence[int]) -> List[int]:
    """the levels l whose modulus Q_l = q_0 ... q_{L-1-l} is below t"""
    return [l for l in range(len(moduli)) if _product(moduli[:len(moduli) - l]) < t]
