"""Run by tests/test_gpu_expand.py::test_expand_across_chunks in a subprocess with a tiny FHE_B200_CHUNK: an expansion of
Q = 7 queries, whose levels span several chunks dealt over the side streams, must give, entry for entry, what seven
expansions of one query give."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import fhe_rs_b200 as F  # noqa: E402

degree, nmod, t, count = 64, 3, 1153, 7
par = F.BfvParameters(degree, t, moduli_sizes=[62] * nmod, device=0)
moduli = par.moduli()
rng = np.random.default_rng(200)


def rnd(*prefix):
    a = np.zeros(tuple(prefix) + (nmod, degree), np.uint64)
    for i in range(nmod):
        a[..., i, :] = rng.integers(0, moduli[i], size=tuple(prefix) + (degree,), dtype=np.uint64)
    return a


ek = F.EvaluationKey(par)
for l in range(3):
    k = rnd(2, nmod)
    ek.add_galois_key(F.GaloisKey.from_arrays(par, (degree >> l) + 1, k[0], k[1]))
a = rnd(count, 2)
for size in (5, 8):   # 5: the last level spills three outputs of every query
    whole = ek.expands_batch(F.Ciphertext.from_host(par, a), size).to_host()
    for q in range(count):
        one = ek.expands_batch(F.Ciphertext.from_host(par, a[q:q + 1]), size).to_host()
        for i in range(size):
            assert (whole[i * count + q] == one[i]).all(), (size, q, i)
print("expand chunk probe ok", count, "queries, chunk", os.environ.get("FHE_B200_CHUNK"),
      "streams", os.environ.get("FHE_B200_STREAMS", "2"))
