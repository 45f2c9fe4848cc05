"""Baby-step/giant-step linear transforms restated on the CPU oracle, for tests/test_linear_transform_cpu.py and the
expected words of tests/test_gpu_linear_transform.py.

For n diagonals D[0 .. n) and a baby step b (G = ceil(n / b) giant groups), every ciphertext x becomes

    out = sum_{g < G} rot_{g b}( sum_{i < b, g b + i < n} D[g b + i] (.) B_i(x) ),   B_0(x) = x,  B_i = rot_i

with rot_k = EvaluationKey::rotates_columns_by(k), i.e. GaloisKey::relinearize with exponent 3^k mod 2N
(evaluation_key.rs:145-170), (.) the NTT-domain product of Ciphertext *= &Plaintext (ops/mod.rs:229-238) and the sums
AddAssign (ops/mod.rs:54-69).  The rotation by 0 is no rotation.  Every step is exact modulo each q_j, so the order of
the sums does not change the words."""
from typing import Dict, List, Sequence

import numpy as np

import fhe_oracle as O


def steps(n_diags: int, baby: int) -> List[int]:
    """the column rotation steps the transform needs keys for: baby steps 1 .. b - 1, giant steps b, 2b, .."""
    return list(range(1, baby)) + list(range(baby, n_diags, baby))


def linear_transform(ct: "O.Ciphertext", diags: Sequence["O.Poly"], baby: int,
                     gks: Dict[int, "O.GaloisKey"]) -> "O.Ciphertext":
    """the composition above for one ciphertext; diags: NTT polys at ct's level, gks: step -> GaloisKey"""
    n = len(diags)
    acc = None
    baby_rot = [ct] + [gks[i].relinearize(ct) for i in range(1, min(baby, n))]
    for g in range(-(-n // baby)):
        part = None
        for i in range(min(baby, n - g * baby)):
            term = O.Ciphertext(ct.par, [p.mul(diags[g * baby + i]) for p in baby_rot[i].c], ct.level)
            part = term if part is None else part.add(term)
        if g:
            part = gks[g * baby].relinearize(part)
        acc = part if acc is None else acc.add(part)
    return acc


def slot_diagonals(M: np.ndarray, n_diags: int, baby: int) -> np.ndarray:
    """[n_diags][N/2] of one (N/2) x (N/2) matrix: diagonal k = M[r][(r + k) mod N/2], rotated right by its giant step
    (the construction of tests/test_gpu_hoisted.py's baby-step/giant-step test)"""
    half = M.shape[0]
    out = np.zeros((n_diags, half), M.dtype)
    for k in range(n_diags):
        d = np.array([M[r][(r + k) % half] for r in range(half)], M.dtype)
        out[k] = np.roll(d, (k // baby) * baby)
    return out
