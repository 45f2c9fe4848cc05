"""The crafted inputs of tests/test_gpu_server_edges.py, checked without a device: each reaches the decision it targets,
so a passing device run means something.
  * the crafted-zero patterns of 31 moduli and N = 2^16 give the zero predicate (tests/hoisting_reference.py) the
    counts the device test expects: zeros in the last limb, at s = N - 1, and at N = 2^16 at positions with
    s e >= 2^32 that the exponent negates and that it keeps;
  * the 32-bit index arithmetic of hoist_zero_kernel, negation_rows_kernel and subst_source equals the exact 64-bit
    forms for every s < 2^16 and every odd e < 2^17 (N = 2^16), where s e wraps;
  * on the lazy-bound bases the all-(q - 1) digits lie on the intended side of 4 q_j, by a restatement of
    capi.cu's digit_reduce, and the pre-substituted c1 makes sigma_e(c1) all q - 1;
  * the hoisting identity equals GaloisKey.relinearize on the boundary-prime and lazy-bound bases at N = 16 and 64
    with all-(q - 1) keys.
The shared constructions (boundary_bases, wide_exponents, crafted_c1, presubstituted_max, digit_reduce) are imported
by the device module."""
import os
import sys
import time

import numpy as np
import pytest

TESTS = os.path.dirname(os.path.abspath(__file__))
if TESTS not in sys.path:
    sys.path.insert(0, TESTS)

import edge_inputs as E   # noqa: E402


# ---------------------------------------------------------------------------------------------- shared inputs

def next_barrett(degree: int) -> int:
    """the largest 62-bit NTT-friendly prime below BOUNDARY_PRIMES["non_solinas_min"]: another Barrett limb"""
    import fhe_oracle as O
    return O.generate_prime(62, max(2 * degree, 1 << 17), E.BOUNDARY_PRIMES["non_solinas_min"])


def boundary_bases(degree: int):
    """name -> moduli: each boundary prime as q_0 before two generated 62-bit primes, all three after one generated
    prime, and three Barrett limbs (no Solinas limb at all)"""
    bp = E.BOUNDARY_PRIMES
    g0, g1 = E.gen62(degree, 0), E.gen62(degree, 1)
    out = {"q0_" + k: [v, g0, g1] for k, v in bp.items()}
    out["after_gen62"] = [g0, bp["solinas_max_c"], bp["non_solinas_min"], bp["above_2_61"]]
    out["all_barrett"] = [bp["non_solinas_min"], next_barrett(degree), bp["above_2_61"]]
    return out


def is_solinas(q: int) -> bool:
    """a 62-bit limb p = 2^62 - c takes the Solinas path when c < 2^28 (edge_inputs.BOUNDARY_PRIMES)"""
    return q.bit_length() == 62 and (1 << 62) - q < 1 << 28


def wide_exponents(degree: int):
    """three Galois exponents for one source: the first 3^k mod 2N at or above 3N/2 (>= 2^16 at N = 2^16), the row
    rotation 2N - 1, and 2^17 + 5, which the call reduces to 5"""
    m = 2 * degree
    big = next(e for e in (pow(3, k, m) for k in range(1, degree)) if e >= 3 * degree // 2)
    return [big, m - 1, (1 << 17) + 5]


def crafted_c1(moduli, degree: int, exps, seed: int):
    """[3][L][N] power-basis c1 rows of non-zero random residues with one crafted zero each, in the last limb.  The
    row rotation 2N - 1 negates every s >= 1, so "the others" below leave it out:
      source 0: at s = N - 1 ("last"), negated by exactly the exponents whose reduced value is above N;
      source 1: at the largest s < N - 1 that exps[0] negates and the others keep ("negated");
      source 2: at the largest s that every exponent but 2N - 1 keeps ("kept"), with zeros at s = 0 in every limb,
                which nothing negates.
    Returns the rows and the positions {"last", "negated", "kept"}."""
    import hoisting_reference as H
    rng = np.random.default_rng(seed)
    L = len(moduli)
    rows = np.stack([np.stack([rng.integers(1, q, degree, dtype=np.uint64) for q in moduli]) for _ in range(3)])
    s = np.arange(1, degree - 1)
    neg = np.stack([H.negates(degree, e, s) for e in exps if e % (2 * degree) != 2 * degree - 1])
    pos = {"last": degree - 1, "negated": int(s[neg[0] & ~neg[1:].any(axis=0)].max()),
           "kept": int(s[~neg.any(axis=0)].max())}
    for src, name in enumerate(("last", "negated", "kept")):
        rows[src, L - 1, pos[name]] = 0
    rows[2, :, 0] = 0
    return rows, pos


def presubstituted_max(O, ctx, e: int) -> np.ndarray:
    """[L][N] power-basis c1 with sigma_e(c1) all q - 1: all q - 1 substituted by e^-1 (tests/test_gpu_widths.py's
    lazy_inputs).  Its own words are q - 1 where sigma_e keeps a coefficient and 1 where it negates one."""
    mx = np.stack([np.full(ctx.degree, q - 1, np.uint64) for q in ctx.moduli])
    return O.Poly(ctx, O.POWER_BASIS, mx).substitute(pow(e, -1, 2 * ctx.degree)).c.copy()


def digit_reduce(ct_moduli, key_moduli) -> bool:
    """capi.cu's digit_reduce: the digit transforms reduce on load when a digit (< max q_i of the ciphertext level)
    can reach 4 min q_j of the key level, or when every key modulus is below 2^8"""
    qmax, qmin = max(int(q) for q in ct_moduli), min(int(q) for q in key_moduli)
    return qmax > 4 * qmin - 1 or qmin < 1 << 8


# ------------------------------------------------------------------------------------------------- the tests

@pytest.fixture(scope="module")
def H(oracle):
    import hoisting_reference
    return hoisting_reference


def test_boundary_bases_reach_their_limb_modes(oracle):
    """q_0 of each boundary prime, all three after a generated prime, and an all-Barrett basis, valid up to
    N = 2^15"""
    for degree in (16, 64, 1 << 13):
        bases = boundary_bases(degree)
        for name, mods in bases.items():
            assert len(set(mods)) == len(mods) and all(oracle.is_prime(q) and q % (2 * degree) == 1 for q in mods)
        assert not any(is_solinas(q) for q in bases["all_barrett"])
        assert is_solinas(bases["q0_solinas_max_c"][0]) and not is_solinas(bases["q0_non_solinas_min"][0])
        assert [is_solinas(q) for q in bases["after_gen62"]] == [True, True, False, False]
        # the correction term's [q_k]_{q_j} is non-trivial only for q_k > q_j: each basis has such pairs
        for mods in bases.values():
            assert any(qk > qj for qk in mods for qj in mods)


@pytest.mark.parametrize("degree", [1 << 13, 1 << 16])
def test_crafted_zero_counts(H, degree):
    """the predicate counts of the crafted zeros at 3 sources x 3 exponents (the device test's layout): sources 0
    ("last") and 1 ("negated") fall back for exps[0] and 2N - 1, source 2 ("kept") for 2N - 1 only, 4 outputs
    hoisted, so each zero decides exps[0] on its own; at N = 2^16 all three sit where s e >= 2^32"""
    L = 31 if degree == 1 << 13 else 3
    moduli = [(1 << 62) - 57 - 2 * i for i in range(L)]   # any odd values: the predicate reads zeros only
    exps = wide_exponents(degree)
    red = [e % (2 * degree) for e in exps]
    assert any(e >= 1 << 16 for e in exps) and red[1] == 2 * degree - 1 and red[2] == 5 and red[0] > degree
    rows, pos = crafted_c1(moduli, degree, exps, 3)
    assert (rows[:, :L - 1, 1:] != 0).all() and (rows[:2, :, 0] != 0).all()   # the zeros of s >= 1: last limb only
    want = [[True, True, False], [True, True, False], [False, True, False]]
    for src in range(3):
        assert [H.needs_fallback(rows[src], e) for e in exps] == want[src], src
    assert H.hoisted_count(list(rows), exps * 3, [s for s in range(3) for _ in range(3)]) == 4
    assert H.negates(degree, red[0], pos["negated"]) and not H.negates(degree, red[0], pos["kept"])
    if degree == 1 << 16:
        for name in ("last", "negated", "kept"):
            assert pos[name] * red[0] >= 1 << 32, (name, pos[name])
    # the linear transform's baby steps 1 and 2 (exponents 3 and 9) keep N - 1: step 1 falls back for source 1 only
    lt_exps = [3, 9]
    rows, pos = crafted_c1(moduli, degree, lt_exps, 4)
    assert [[H.needs_fallback(r, e) for e in lt_exps] for r in rows] == [[False, False], [True, False], [False, False]]


def test_32_bit_index_arithmetic():
    """N = 2^16: for every s < 2^16 and odd e < 2^17 the uint32 product s e, as hoist_zero_kernel ((s e) & N) and
    negation_rows_kernel (destination (s e) & (N - 1)) use it, gives the exact 64-bit s e mod 2N; and subst_source's
    (j e + (e - 1) / 2) & (N - 1) gives the exact (j e + (e - 1) / 2) mod N.  j = brev(o) runs over [0, N) as o does,
    so j takes the values of s.  All three read the low logn + 1 bits of the product (subst_source after adding the
    same (e - 1) / 2 to both forms), so each equals its exact form exactly when the wrapped and the exact product agree
    modulo 2N: that is checked for every pair, in about 15 s.  About 1 in 7 of the products wraps."""
    t0 = time.time()
    N, block = 1 << 16, 4
    s32 = np.arange(N, dtype=np.uint32)
    s64 = s32.astype(np.int64)
    p32, p64 = np.empty((block, N), np.uint32), np.empty((block, N), np.int64)
    for e0 in range(1, 2 * N, 2 * block):
        e32 = np.arange(e0, e0 + 2 * block, 2, dtype=np.uint32)[:, None]
        np.multiply(s32[None], e32, out=p32)                  # mod 2^32, as the kernels multiply
        np.multiply(s64[None], e32.astype(np.int64), out=p64)   # exact: below 2^33
        np.subtract(p64, p32, out=p64)
        np.bitwise_and(p64, 2 * N - 1, out=p64)
        assert not p64.any(), e0
    # the pairs whose product wraps: s >= ceil(2^32 / e)
    wraps = sum(max(0, N - -(-(1 << 32) // e)) for e in range(1, 2 * N, 2))
    assert 0.1 < wraps / float(N * N) < 0.2, wraps
    p = (np.array([N - 1], np.uint32) * np.uint32(2 * N - 1))[0]   # the largest product wraps, keeps its low bits
    assert int(p) == ((N - 1) * (2 * N - 1)) % (1 << 32) and int(p) & (2 * N - 1) == ((N - 1) * (2 * N - 1)) % (2 * N)
    assert time.time() - t0 < 45


@pytest.mark.parametrize("degree", [16, 1 << 13])
def test_lazy_bound_digits(oracle, degree):
    """the all-(q - 1) digits of the lazy-bound bases against 4 q_j, and digit_reduce's decision: "unreduced" keeps
    every digit below 4 q_j and skips the reduction, "reduced" has digits at or above 4 q_j and reduces, "reduced_8x"
    has digits within 2^53 of 8 q_j and reduces.  The pre-substituted c1 makes sigma_e(c1) all q - 1, and its own
    words are q - 1 and 1."""
    bases = E.lazy_bound_bases(degree)
    for name, mods in bases.items():
        top = max(q - 1 for q in mods)
        qj = min(mods)
        if name == "unreduced":
            assert top < 4 * qj and not digit_reduce(mods, mods)
        else:
            assert top >= 4 * qj and digit_reduce(mods, mods)
        if name == "reduced_8x":
            assert 8 * qj - (1 << 53) < top < 8 * qj
        opar = oracle.BfvParameters(degree, 257, moduli=mods)
        ctx = opar.context_at_level(0)
        for e in (3, 2 * degree - 1, 9):
            pre = presubstituted_max(oracle, ctx, e)
            got = oracle.Poly(ctx, oracle.POWER_BASIS, pre.copy()).substitute(e).c
            assert (got == np.array(mods, np.uint64)[:, None] - np.uint64(1)).all(), (name, e)
            q = np.array(mods, np.uint64)[:, None]
            assert ((pre == q - np.uint64(1)) | (pre == 1)).all()
    # the boundary-prime bases and the width sweep: which side each takes
    for mods in boundary_bases(1 << 13).values():
        assert not digit_reduce(mods, mods)
    assert digit_reduce(oracle.BfvParameters.generate_moduli(E.WIDTH_SETS["n2_13"][2], 1 << 13),
                        oracle.BfvParameters.generate_moduli(E.WIDTH_SETS["n2_13"][2], 1 << 13))


def _identity_bases(degree):
    out = dict(boundary_bases(degree))
    out.update({"lazy_" + k: v for k, v in E.lazy_bound_bases(degree).items()})
    return out


@pytest.mark.parametrize("degree", [16, 64])
def test_identity_with_all_max_keys(oracle, H, degree):
    """hoisting_reference.hoisted_relinearize == GaloisKey.relinearize, word for word, on every boundary-prime and
    lazy-bound basis with all-(q - 1) keys, for random, all-(q - 1) and pre-substituted c1"""
    exps = [3, 2 * degree - 1, degree + 1, pow(3, 5, 2 * degree)]
    for name, mods in _identity_bases(degree).items():
        par = oracle.BfvParameters(degree, 257, moduli=mods)
        ctx = par.context_at_level(0)
        L = len(mods)
        k = np.ascontiguousarray(np.broadcast_to(np.array(mods, np.uint64)[:, None] - np.uint64(1), (L, L, degree)))
        ksk = oracle.KeySwitchingKey.from_arrays(par, k, k)
        rng = np.random.default_rng(L + degree)
        c0 = oracle.Poly.random(ctx, oracle.NTT, rng)
        mx = np.stack([np.full(degree, q - 1, np.uint64) for q in mods])
        kinds = {"random": oracle.Poly.random(ctx, oracle.POWER_BASIS, rng).c.copy(), "max": mx,
                 "pre": presubstituted_max(oracle, ctx, 3)}
        for kind, c1 in kinds.items():
            ct = oracle.Ciphertext(par, [c0.copy(), oracle.Poly(ctx, oracle.POWER_BASIS, c1.copy()).into_ntt()], 0)
            D = H.digits(ksk, oracle.Poly(ctx, oracle.POWER_BASIS, c1.copy()))
            for e in exps:
                if H.needs_fallback(c1, e):
                    continue
                g = oracle.GaloisKey.__new__(oracle.GaloisKey)
                g.exponent, g.ksk = e, ksk
                assert (H.hoisted_relinearize(g, ct, D).to_array() == g.relinearize(ct).to_array()).all(), \
                    (name, kind, e)
