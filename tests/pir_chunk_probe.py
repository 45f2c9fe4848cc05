"""Run by tests/test_gpu_pir.py::test_pir_across_chunks in a subprocess with a tiny FHE_B200_CHUNK: a fold of many
ciphertexts and a many-row transcode, both spanning several chunks dealt over the side streams, must equal, entry for
entry, the same calls made one ciphertext or one row at a time."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import fhe_rs_b200 as F  # noqa: E402

degree, nmod, count = 64, 3, 11
par = F.BfvParameters(degree, 1153, moduli_sizes=[62] * nmod, device=0)
rng = np.random.default_rng(300)

words = rng.integers(0, 1 << 64, size=(count, 2, nmod, degree), dtype=np.uint64)
for in_bits, out_bits in ((62, 20), (36, 7)):
    whole = F.Ciphertext.from_host(par, words).fold(in_bits, out_bits, 1).batch.to_host()
    P = whole.shape[0] // count
    for j in range(count):
        one = F.Ciphertext.from_host(par, words[j:j + 1]).fold(in_bits, out_bits, 1).batch.to_host()
        for i in range(P):
            assert (whole[i * count + j] == one[i]).all(), (in_bits, out_bits, i, j)

# rows of 3 000 words: a chunk stages at most chunk * 2 * 3 * 64 words, so a few rows per chunk
rows = rng.integers(0, 1 << 64, size=(37, 3000), dtype=np.uint64)
for in_bits, out_bits, out_len in ((62, 20, 9300), (13, 64, 500)):
    whole = F.transcode_bidirectional(par, rows, in_bits, out_bits, out_len=out_len)
    for r in range(rows.shape[0]):
        assert (whole[r] == F.transcode_bidirectional(par, rows[r], in_bits, out_bits, out_len=out_len)).all(), r
by = rng.integers(0, 256, size=(29, 5000), dtype=np.uint8)
whole = F.transcode_from_bytes(par, by, 20)
for r in range(by.shape[0]):
    assert (whole[r] == F.transcode_from_bytes(par, by[r], 20)).all(), r
print("pir chunk probe ok", count, "ciphertexts, chunk", os.environ.get("FHE_B200_CHUNK"),
      "streams", os.environ.get("FHE_B200_STREAMS", "2"))
