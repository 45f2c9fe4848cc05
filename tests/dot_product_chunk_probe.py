"""Word checks of the ciphertext dot product and batch sum at group and term counts that cut chunks, streams and the
persistent kernels' work split (tests/work_split_cases.SHAPES).  Every output is compared with the same computation
from existing device calls: the batched product (fhe_b200_mul), a host sum modulo each limb, fhe_b200_relinearize and
fhe_b200_switch_down.  tests/test_gpu_dot_product.py runs it in one process per kernel or chunking switch (the
switches are read once per process):

    python tests/dot_product_chunk_probe.py        prints WORD CHECKS OK"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
TESTS = os.path.join(ROOT, "tests")
if TESTS not in sys.path:
    sys.path.insert(0, TESTS)

from work_split_cases import SHAPES   # noqa: E402


def rand_rows(rng, moduli, prefix, n):
    a = np.zeros(tuple(prefix) + (len(moduli), n), np.uint64)
    for i, q in enumerate(moduli):
        a[..., i, :] = rng.integers(0, q, size=tuple(prefix) + (n,), dtype=np.uint64)
    return a


def host_sum(words, moduli, n_terms):
    """words [groups * n_terms][parts][L][N] (canonical) -> [groups][parts][L][N], each limb summed modulo its prime"""
    w = words.reshape((-1, n_terms) + words.shape[1:])
    q = np.array(moduli[:words.shape[2]], np.uint64)[:, None]
    acc = np.zeros((w.shape[0],) + w.shape[2:], np.uint64)
    for i in range(n_terms):
        acc += w[:, i]
        acc = np.where(acc >= q, acc - q, acc)
    return acc


class DotSetup:
    """a parameter set, operands at `level` (a: groups * n_terms or n_terms entries, likewise b) and a random
    relinearization key of (ciphertext level, key level) when key_level is not None (bit-exactness needs no real
    keys), on a new parameter set or on `par`"""

    def __init__(self, F, degree, t, sizes, level, key_level, groups, n_terms, seed, moduli=None, shared=None,
                 par=None):
        self.F = F
        self.par = par or F.BfvParameters(degree, t, moduli=moduli, moduli_sizes=None if moduli else sizes, device=0)
        self.moduli = [int(q) for q in self.par.moduli()]
        self.level, self.groups, self.n_terms, self.degree = level, groups, n_terms, degree
        rng = np.random.default_rng(seed)
        ct_mod = self.moduli[:len(self.moduli) - level]
        na = n_terms if shared == "a" else groups * n_terms
        nb = n_terms if shared == "b" else groups * n_terms
        self.A = F.Ciphertext.from_host(self.par, rand_rows(rng, ct_mod, (na, 2), degree), level=level)
        self.B = F.Ciphertext.from_host(self.par, rand_rows(rng, ct_mod, (nb, 2), degree), level=level)
        self.rk = None
        if key_level is not None:
            key_mod = self.moduli[:len(self.moduli) - key_level]
            if len(key_mod) == 1:   # key_switching_key.rs:92-126: base 2^(log q / 2)
                lq = (self.moduli[0] - 1).bit_length()
                n_dig = -(-lq // (lq // 2))
            else:
                n_dig = len(ct_mod)
            c = rand_rows(rng, key_mod, (2, n_dig), degree)
            self.rk = F.RelinearizationKey.from_arrays(self.par, c[0], c[1], level, key_level)

    def full(self, X):
        """an operand with one entry per term of every group (a shared one repeated)"""
        if X.count == self.groups * self.n_terms:
            return X
        w = X.to_host()
        return self.F.Ciphertext.from_host(self.par, np.concatenate([w] * self.groups), level=self.level)

    def expected(self, out_level, rk="own"):
        """the reference's loop from existing device calls: mul, sum, relinearizes, switch_to_level"""
        rk = self.rk if rk == "own" else rk
        prods = (self.full(self.A) * self.full(self.B)).to_host()
        s = self.F.Ciphertext.from_host(self.par, host_sum(prods, self.moduli, self.n_terms), level=self.level)
        if rk is not None:
            s = rk.relinearizes(s)
        return s.switch_to_level(out_level).to_host()

    def got(self, out_level, rk="own"):
        rk = self.rk if rk == "own" else rk
        return self.F.dot_product(self.A, self.B, self.n_terms, rk, out_level).to_host()

    def check(self, out_level=None, with_key=True):
        out_level = self.level if out_level is None else out_level
        rk = self.rk if with_key else None
        got, exp = self.got(out_level, rk), self.expected(out_level, rk)
        bad = [g for g in range(got.shape[0]) if not (got[g] == exp[g]).all()]
        assert not bad, (self.degree, self.groups, self.n_terms, out_level, with_key, bad[:8])


# (shape, groups, n_terms): group and term counts that cut the default chunk of 256 over 2 streams (and every chunk
# of FHE_B200_CHUNK=1), one group's terms over several slices, and products counts off the kernels' wave sizes
CHUNK_RUNS = [("n13_2x62", 3, 7), ("n13_2x62", 1, 300), ("n13_2x62", 67, 5), ("n13_2x62", 2, 129),
              ("n13_62_40_30", 5, 7), ("n14_8x62", 3, 11), ("n15_14x62", 2, 3)]


def word_checks(F, quick=False):
    runs = CHUNK_RUNS[:3] + CHUNK_RUNS[4:5] if quick else CHUNK_RUNS
    for k, (name, groups, n_terms) in enumerate(runs):
        s = SHAPES[name]
        S = DotSetup(F, 1 << s["logn"], s["t"], s["sizes"], 0, 0, groups, n_terms, 100 + k)
        S.check()
        S.check(with_key=False)
        if k == 0:
            S.check(out_level=len(S.moduli) - 1)
            shared = DotSetup(F, 1 << s["logn"], s["t"], s["sizes"], 0, 0, groups, n_terms, 200, shared="b")
            shared.check()
    # batch sums across chunks
    par = F.BfvParameters(1 << 13, 786433, moduli_sizes=[62, 62], device=0)
    moduli = [int(q) for q in par.moduli()]
    rng = np.random.default_rng(7)
    for groups, n_terms in ((3, 65), (300, 2)):
        w = rand_rows(rng, moduli, (groups * n_terms, 2), 1 << 13)
        got = F.Ciphertext.from_host(par, w).sum(n_terms).to_host()
        assert (got == host_sum(w, moduli, n_terms)).all(), (groups, n_terms)


if __name__ == "__main__":
    import fhe_rs_b200
    word_checks(fhe_rs_b200, quick=os.environ.get("FHE_B200_CHUNK") == "1")
    print("WORD CHECKS OK")
