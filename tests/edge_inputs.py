"""Crafted inputs for the arithmetic's decision points and range limits.

Each coefficient of a polynomial is one independent scaler input, so the values are built as big integers and then
projected onto the limbs of a basis.  Uniform random residues land on these points with probability around 2^-60:
  * the exact scaler's rounding ties: num * x / den a hair away from a half-integer;
  * its sign boundary: x next to F/2, where F is the product of the source basis;
  * the extender (factor one) around (Q - 1)/2;
  * switch_down around the ties of round(x / q_last).
`residue_rows` gives rows that drive lazy sums to their extremes instead (all q - 1 and friends).
For the client side: `decrypt_phases` (decryption's ties, Q / 2 and the failure boundary), `noise_points` (the word
boundaries of Q), `key_extremes` (secret keys at the extremes), and the shapes and plaintext moduli of
CLIENT_SHAPES / `client_plaintexts`.
"""
from __future__ import annotations

from typing import Dict, List, Sequence

import numpy as np

D_RANGE = range(-3, 4)

# 62-bit primes at the edges of the device's limb modes, all == 1 mod 2^16 (NTT-friendly for any N <= 2^15).  A limb
# p = 2^62 - c takes the Solinas path when c < 2^28.
BOUNDARY_PRIMES = {
    "solinas_max_c": 0x3ffffffff00a0001,     # c = 0xff5ffff: the thinnest [0, 2p) margin of the Solinas folds
    "non_solinas_min": 0x3fffffffeff50001,   # c = 0x100affff: the largest 62-bit prime that is a Barrett limb
    "above_2_61": 0x20000000000b0001,        # a Barrett limb just above 2^61
}


def gen62(degree: int, k: int) -> int:
    """the k-th 62-bit NTT-friendly prime below 2^62 (the generator's order)"""
    import fhe_oracle as O
    ub = 1 << 62
    for _ in range(k + 1):
        ub = O.generate_prime(62, 2 * degree, ub)
    return ub


# decryption shapes: name -> (degree, moduli sizes, or the names of the first moduli followed by generated 62-bit
# ones).  With one output row (q_0) the scaler kernel is scale_small_kernel for N < 128, scale_tma_kernel when every
# modulus of the plaintext context is Solinas, scale_kernel otherwise.
CLIENT_SHAPES = {
    "n16_l5": (16, [62] * 5),
    "set_a": (1 << 12, [62] * 2),
    "set_c": (1 << 15, [62] * 14),
    "q0_barrett": (1 << 13, ["non_solinas_min", 0, 1]),
    "q0_above_2_61": (1 << 13, ["above_2_61", 0, 1]),
    "q0_solinas_max_c": (1 << 13, ["solinas_max_c", 0, 1]),
    "q1_barrett": (1 << 13, [0, "non_solinas_min", 1]),        # t = 1153: plaintext context (q_0, q_1)
    "l31": (1 << 13, [62] * 31),
    "n2_16": (1 << 16, [62] * 3),
    "ten_bit": (64, [62, 62, 10]),
}


def client_moduli(name: str) -> List[int]:
    import fhe_oracle as O
    degree, spec = CLIENT_SHAPES[name]
    if all(isinstance(s, int) and s >= 10 for s in spec):
        return O.BfvParameters.generate_moduli(spec, degree)
    return [BOUNDARY_PRIMES[s] if isinstance(s, str) else gen62(degree, s) for s in spec]


def coprime_below(bound: int, moduli: Sequence[int]) -> int:
    """the largest t < bound coprime with every modulus"""
    from math import gcd
    t = bound - 1
    while any(gcd(t, int(q)) != 1 for q in moduli):
        t -= 1
    return t


def client_plaintexts(degree: int, moduli: Sequence[int]) -> Dict[str, int]:
    """plaintext moduli for decryption: 2 (a one-modulus plaintext context with a 62-bit q_0), 1153, a 40-bit prime,
    the largest t below q_0, and the largest t the library takes (t < 2^62), which is above q_0"""
    import fhe_oracle as O
    return {"t2": 2, "t1153": 1153, "t40": O.generate_prime(40, 2 * degree, 1 << 40),
            "below_q0": coprime_below(int(moduli[0]), moduli), "max": coprime_below(1 << 62, moduli)}


def product(moduli: Sequence[int]) -> int:
    out = 1
    for q in moduli:
        out *= int(q)
    return out


def scaler_near_ties(F: int, num: int, den: int, rng: np.random.Generator, n_m: int = 4) -> List[int]:
    """x = floor((2m + 1) * den / (2 num)) + d, d in [-3, 3], for random m with x in both halves of [0, F):
    num * x / den is within a few num / den of m + 1/2."""
    m_max = num * F // den          # num * x / den < m_max for x < F
    out = []
    for half in (0, 1):
        lo, hi = (0, m_max // 2) if half == 0 else (m_max // 2, m_max)
        for _ in range(n_m):
            m = lo + int(rng.integers(0, 1 << 62)) * (hi - lo) // (1 << 62)
            base = (2 * m + 1) * den // (2 * num)
            out += [(base + d) % F for d in D_RANGE]
    return out


def sign_boundary(F: int) -> List[int]:
    """F/2 + d with d in [-3, 3], plus 0, 1 and F - 1"""
    return [(F // 2 + d) % F for d in D_RANGE] + [0, 1, F - 1]


def extender_edges(Q: int) -> List[int]:
    """(Q - 1)/2, (Q + 1)/2, (Q - 3)/2, 0 and Q - 1 (Q odd)"""
    return [(Q - 1) // 2, (Q + 1) // 2, (Q - 3) // 2, 0, Q - 1]


def switch_down_ties(Q: int, q_last: int, rng: np.random.Generator, n: int = 8) -> List[int]:
    """x with x mod q_last in {(q_last - 1)/2, (q_last + 1)/2, 0, q_last - 1} and a random quotient"""
    out = []
    for r in ((q_last - 1) // 2, (q_last + 1) // 2, 0, q_last - 1):
        for _ in range(n):
            k = int(rng.integers(0, 1 << 62)) * (Q // q_last) // (1 << 62)
            out.append(k * q_last + r)
    return out + [(q_last - 1) // 2, (q_last + 1) // 2, Q - 1 - (q_last - 1) // 2]


def wide_w_sums(sc, moduli: Sequence[int], rng: np.random.Generator, count: int, tries: int = 4000) -> List[List[int]]:
    """Residue vectors whose theta_omega sum (rns/scaler.rs:278-302) has a magnitude in [2^190, 2^191): bits 190 and
    191 of the U256 differ there, so only these inputs tell the sign test at bit 191 from one a bit lower.  The search
    gives the terms of one sign residues in [15q/16, q) and the others zero.  The sum reaches the range only with
    enough source limbs (29 at 62 bits do); with fewer, the search returns fewer vectors or none."""
    import scaler_reference
    signs = [int(s) for s in sc.theta_omega_sign]
    out = []
    for k in range(tries):
        neg = k % 2 == 1
        r = [int(q) - 1 - int(rng.integers(0, q >> 4)) if signs[i] == neg else 0 for i, q in enumerate(moduli)]
        _, so = scaler_reference.v_and_w_sum(sc, r)
        if ((so >> 190) & 1) != ((so >> 191) & 1) and so >> 192 in (0, (1 << 64) - 1):
            out.append(r)
            if len(out) == count:
                break
    return out


def polys_from_residues(cols: Sequence[Sequence[int]], degree: int) -> np.ndarray:
    """[count][limbs][N] with the given residue vectors as coefficients (repeated to fill the last polynomial)"""
    count = -(-len(cols) // degree)
    reps = -(-count * degree // len(cols))
    a = np.array([[int(v) for v in c] for c in cols], dtype=np.uint64)
    a = np.tile(a, (reps, 1))[: count * degree]
    return np.ascontiguousarray(a.reshape(count, degree, -1).transpose(0, 2, 1))


def polys_from_values(values: Sequence[int], moduli: Sequence[int], degree: int) -> np.ndarray:
    """[count][limbs][N] residues of the values, N per polynomial; the last polynomial is filled by repeating them"""
    vals = [int(v) for v in values]
    count = -(-len(vals) // degree)
    vals = (vals * (-(-count * degree // len(vals))))[: count * degree]
    out = np.zeros((count, len(moduli), degree), np.uint64)
    for i, q in enumerate(moduli):
        out[:, i, :] = np.array([v % int(q) for v in vals], dtype=np.uint64).reshape(count, degree)
    return out


def decrypt_phases(Q: int, t: int, rng: np.random.Generator, n_m: int = 4) -> List[int]:
    """phases x in [0, Q) where decryption decides something: the ties of t x / Q and the sign boundary Q / 2
    (scaler_near_ties, sign_boundary), and Delta m +/- floor(Q / 2t) + d (Delta = floor(Q / t), d in [-3, 3]) for
    m in {0, 1, t/2, t - 1} -- a ciphertext whose noise is at the decryption-failure boundary"""
    delta, half = Q // t, Q // (2 * t)
    out = scaler_near_ties(Q, t, Q, rng, n_m) + sign_boundary(Q)
    for m in sorted({0, 1, t // 2, t - 1}):
        for s in (-half, half):
            out += [(delta * m + s + d) % Q for d in D_RANGE]
    return out


def decrypt_windows(x: int, Q: int, t: int, eps: float = 2.0 ** -40):
    """(t x / Q within eps of a half-integer, x / Q within eps of 1/2): where the reference's fixed-point scaler may
    depart from round(t x / Q)"""
    from fractions import Fraction
    return (abs(Fraction(x * t % Q, Q) - Fraction(1, 2)) < eps, abs(Fraction(x, Q) - Fraction(1, 2)) < eps)


def decrypt_one(par, level: int, x: int) -> int:
    """the oracle's decryption of one phase coefficient x (its level scaler, then ((v + t) mod q_0) mod t)"""
    lv, t, q0 = par.level(level), par.plaintext, int(par.moduli[0])
    v0 = int(lv.scaler.scaler.scale_one(lv.poly_context.rns.project(x), 1, 0)[0])
    return ((v0 + t) % q0) % t


def noise_one(par, level: int, x: int) -> int:
    """measure_noise of a ciphertext whose phase is x at one coefficient and 0 elsewhere, in plain integers: the
    phase minus to_poly(decrypt) = x - (m q_mod_t mod t) (-t)^-1 mod Q, then min(bits(v), bits(Q - v))"""
    lv, t = par.level(level), par.plaintext
    Q = lv.poly_context.modulus()
    m = decrypt_one(par, level, x) * lv.q_mod_t % t
    v = (x - m * pow(-t % Q, -1, Q)) % Q
    return min(v.bit_length(), (Q - v).bit_length())


def noise_points(Q: int) -> List[int]:
    """phases for measure_noise's multi-word arithmetic: 2^k - 1, 2^k, 2^k + 1 and Q - 2^k at every 64-bit word
    boundary k below bits(Q), and floor(Q / 2), ceil(Q / 2)"""
    out = []
    for k in range(64, Q.bit_length(), 64):
        out += [(1 << k) - 1, 1 << k, (1 << k) + 1, Q - (1 << k)]
    out += [Q // 2, (Q + 1) // 2]
    return [x for x in out if 0 <= x < Q]


def key_extremes(degree: int, q0: int, rng: np.random.Generator) -> Dict[str, np.ndarray]:
    """secret-key coefficients [N] (int64) at the extremes: the constants -1 and 1 (every NTT word of s is q - 1,
    resp. 1), and i64 min / max, +/-(q_0 - 1), +/-q_0 at random positions among small random coefficients"""
    i64 = np.iinfo(np.int64)
    minus, plus = np.zeros(degree, np.int64), np.zeros(degree, np.int64)
    minus[0], plus[0] = -1, 1
    mixed = rng.integers(-16, 17, size=degree).astype(np.int64)
    special = [i64.min, i64.max, q0 - 1, -(q0 - 1), q0, -q0]
    pos = rng.permutation(degree)[:len(special)] if degree >= len(special) else np.arange(degree)
    for p, v in zip(pos, special):
        mixed[p] = v
    return {"minus_one": minus, "one": plus, "extremes": mixed}


def residue_rows(moduli: Sequence[int], degree: int) -> Dict[str, np.ndarray]:
    """[limbs][N] rows at the extremes: all 0, all q - 1, alternating 0 / q - 1, constant (q -/+ 1)/2, a single 1 at
    coefficient 0 or at N - 1"""
    L = len(moduli)
    q = np.array([int(x) for x in moduli], dtype=np.uint64)[:, None]
    one = np.ones((L, degree), np.uint64)
    alt = np.zeros((L, degree), np.uint64)
    alt[:, 1::2] = (q - np.uint64(1))[:, :1].repeat(degree // 2, axis=1)
    first = np.zeros((L, degree), np.uint64)
    first[:, 0] = 1
    last = np.zeros((L, degree), np.uint64)
    last[:, -1] = 1
    return {
        "zero": np.zeros((L, degree), np.uint64),
        "max": one * (q - np.uint64(1)),
        "alternating": alt,
        "half_down": one * ((q - np.uint64(1)) // np.uint64(2)),
        "half_up": one * ((q + np.uint64(1)) // np.uint64(2)),
        "one_first": first,
        "one_last": last,
    }


# ------------------------------------------------------------------------------------------------ modulus widths

def prime_of_width(bits: int, degree: int, k: int = 0) -> int:
    """the k-th NTT-friendly prime (== 1 mod 2N) of exactly `bits` bits, from the top (the generator's order)"""
    import fhe_oracle as O
    ub = 1 << bits
    for _ in range(k + 1):
        ub = O.generate_prime(bits, 2 * degree, ub)
    return ub


def decomposition_moduli(q0_bits: int, degree: int) -> List[int]:
    """a q_0 of the given width followed by two 62-bit moduli: the last level's key decomposes q_0 in base
    2^(bits / 2), in 3 digits when the width is odd and 2 when it is even"""
    import fhe_oracle as O
    return O.BfvParameters.generate_moduli([q0_bits, 62, 62], degree)


# name -> (degree, t, moduli sizes).  The N = 64 sets cover every width from 10 to 62 once; two start narrow (q_0 of
# 10 and 11 bits), two wide (60 and 61 bits); t = 257 is below every q_0 and a SIMD modulus at N = 64.
WIDTH_SETS = {
    "n64_up_10": (64, 257, list(range(10, 63, 4))),
    "n64_up_11": (64, 257, list(range(11, 63, 4))),
    "n64_down_60": (64, 257, list(range(60, 9, -4))),
    "n64_down_61": (64, 257, list(range(61, 9, -4))),
    "n2_13": (1 << 13, 786433, [61, 55, 47, 39, 31, 23, 17]),
}


def lazy_bound_bases(degree: int) -> Dict[str, List[int]]:
    """Bases around the reduce-on-load decision of the RNS-digit transform (a digit below q_i goes into the forward
    transform modulo q_j unreduced while max q_i <= 4 min q_j - 1):
      * "unreduced": q_j the first NTT-friendly prime above 2^60 and q_i primes just below 2^62: an all-(q_i - 1)
        digit sits a hair under 4 q_j, and the transform takes it as it is;
      * "reduced": q_j the first one below 2^60 with 4 q_j < q_i (q_i the same primes): the same digits are at or
        above 4 q_j, and are reduced on load;
      * "reduced_8x": q_j the first one above 2^59: the digits reach 8 q_j - 2^52, far above 4 q_j (and below the
        8 q_j a laxer threshold might allow).
    Only an unreduced digit >= 4 q_j would tell a skipped reduction, and the lazy forward transform keeps even those
    exact: its first butterfly subtracts 2p once (X < x), every output stays below max(x, 4p) < 2^64, the Shoup
    products are exact for any 64-bit operand, and the inner product after the transform reduces whatever it gets."""
    import fhe_oracle as O
    m = 2 * degree

    def first_above(x):
        p = x // m * m + 1
        while p < x or not O.is_prime(p):
            p += m
        return p
    up, up59 = first_above(1 << 60), first_above(1 << 59)
    big = [prime_of_width(62, degree, k) for k in range(2)]
    down = O.generate_prime(60, m, min(big) // 4 + 1)
    assert max(big) - 1 < 4 * up - 1 and 4 * down < min(big) and 4 * up59 < min(big) and max(big) < 8 * up59
    return {"unreduced": [big[0], up, big[1]], "reduced": [big[0], down, big[1]], "reduced_8x": [big[0], up59, big[1]]}


def pack_rows(q: int, degree: int, rng: np.random.Generator) -> Dict[str, np.ndarray]:
    """[N] power-basis rows for the bit packer of a modulus q: 0, q - 1, alternating 0 / q - 1, random below q; and
    fields no reduced word reaches, which a message may still carry (transcode_from_bytes yields up to 2^nbits - 1
    < 2q): q itself, all 2^nbits - 1, alternating q / 2^nbits - 1, random in [q, 2^nbits)"""
    top = (1 << (q - 1).bit_length()) - 1
    alt = np.zeros(degree, np.uint64)
    alt[1::2] = q - 1
    over = np.full(degree, q, np.uint64)
    over[1::2] = top
    return {
        "zero": np.zeros(degree, np.uint64),
        "max": np.full(degree, q - 1, np.uint64),
        "alternating": alt,
        "random": rng.integers(0, q, size=degree, dtype=np.uint64),
        "field_q": np.full(degree, q, np.uint64),
        "field_top": np.full(degree, top, np.uint64),
        "field_alternating": over,
        "field_random": rng.integers(q, top, size=degree, dtype=np.uint64, endpoint=True),
    }
