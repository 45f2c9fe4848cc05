"""CPU restatement of the reference's plaintext encoders on top of the oracle's primitives (oracle/fhe_oracle.py), for
the encoder tests:
  - PlaintextVec::try_encode / encode_u64_chunk (plaintext_vec.rs:37-103), including the single-modulus branch of
    TryConvertFrom<Vec<u64>> (rq/convert.rs:150-159) that takes the N coefficient words unreduced;
  - the &[i64] encoders (plaintext.rs:347-372): Modulus::reduce_vec_i64 into [0, t) first;
  - Plaintext::coefficients (plaintext.rs:103-135, branch t < q_0) and Plaintext::to_poly (:172-197), both starting
    from poly_ntt."""
import numpy as np

import fhe_oracle as O


def encode_u64_chunk(par, values, simd: bool, level: int) -> np.ndarray:
    """poly_ntt words [limbs][N] of one plaintext"""
    n = par.degree
    ctx = par.context_at_level(level)
    coeffs = np.zeros(n, np.uint64)
    values = np.asarray(values, dtype=np.uint64)
    if simd:
        for i, v in enumerate(values):
            coeffs[par.matrix_reps_index_map[i]] = v
        O._ntt_op(par.plaintext, n, par.psi.get(par.plaintext)).backward(coeffs)
    else:
        coeffs[: len(values)] = values
    if len(ctx.moduli) == 1:   # coefficients.len() == q.len() * degree: the words are taken as they are
        p = O.Poly(ctx, O.POWER_BASIS, coeffs[None, :])
    else:
        p = O.Poly.from_u64(ctx, coeffs)
    return p.into_ntt().c


def reduce_i64(values, t: int) -> np.ndarray:
    return np.array([int(v) % t for v in values], dtype=np.uint64)


def try_encode(par, values, simd: bool, level: int = 0, signed: bool = False) -> np.ndarray:
    """poly_ntt words [count][limbs][N] of PlaintextVec::try_encode"""
    if signed:
        values = reduce_i64(values, par.plaintext)
    values = np.asarray(values, dtype=np.uint64)
    n = par.degree
    count = max(1, -(-len(values) // n))
    return np.stack([encode_u64_chunk(par, values[k * n:(k + 1) * n], simd, level) for k in range(count)])


def coefficients(par, poly_ntt: np.ndarray, level: int) -> np.ndarray:
    """Plaintext::coefficients for t < q_0: limb 0 of the power basis, reduced mod t"""
    p = O.Poly(par.context_at_level(level), O.NTT, poly_ntt.copy()).into_power_basis()
    assert par.plaintext < par.moduli[0]
    return p.c[0] % np.uint64(par.plaintext)


def to_poly(par, poly_ntt: np.ndarray, level: int) -> np.ndarray:
    """Plaintext::to_poly words [limbs][N]: coefficients * q_mod_t mod t, lifted, into_ntt, times delta"""
    lvl, t = par.level(level), par.plaintext
    v = np.array([(int(x) * lvl.q_mod_t) % t for x in coefficients(par, poly_ntt, level)], dtype=np.uint64)
    m = O.Poly.from_u64(lvl.poly_context, v, O.NTT)
    m.imul(lvl.delta)
    return m.c
