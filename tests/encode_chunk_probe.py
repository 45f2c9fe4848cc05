"""Run by tests/test_gpu_encode.py::test_encode_chunk_boundary in a subprocess with a small FHE_B200_CHUNK: encoding a
PlaintextVec that spans several chunks (dealt over the side streams), and ct +- pt / ct x pt with one plaintext per
ciphertext, must give entry by entry what one-plaintext calls give."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import fhe_rs_b200 as F  # noqa: E402

degree, t, count = 1 << 13, 786433, 7
par = F.BfvParameters(degree, t, moduli_sizes=[62] * 3, device=0)
moduli = par.moduli()
rng = np.random.default_rng(int(os.environ.get("FHE_B200_CHUNK", "0")) + 200)
n_vals = count * degree - 5
for enc in (F.Encoding.simd(), F.Encoding.poly()):
    for v in (rng.integers(0, t, size=n_vals, dtype=np.uint64), rng.integers(-t, t, size=n_vals, dtype=np.int64)):
        whole = F.PlaintextVec.try_encode(v, enc, par).poly_ntt()
        for k in range(count):
            one = F.Plaintext.try_encode(v[k * degree:(k + 1) * degree], enc, par).poly_ntt()
            assert (whole[k] == one[0]).all(), (enc, v.dtype, k)

x = np.zeros((count, 2, len(moduli), degree), np.uint64)
for i, q in enumerate(moduli):
    x[:, :, i] = rng.integers(0, q, size=(count, 2, degree), dtype=np.uint64)
P = F.PlaintextVec.try_encode(rng.integers(0, t, size=count * degree, dtype=np.uint64), F.Encoding.simd(), par)
words = P.poly_ntt()
for name, op in (("add", lambda c, p: c.add_plain(p)), ("sub", lambda c, p: c.add_plain(p, subtract=True)),
                 ("mul", lambda c, p: c.mul_plain(p))):
    whole = op(F.Ciphertext.from_host(par, x), P).to_host()
    for k in range(count):
        pk = F.PlaintextVec(F.Ciphertext.from_host(par, words[k:k + 1, None]), F.Encoding.simd())
        one = op(F.Ciphertext.from_host(par, x[k:k + 1]), pk).to_host()
        assert (whole[k] == one[0]).all(), (name, k)
print("encode chunk probe ok", count, "plaintexts, chunk", os.environ.get("FHE_B200_CHUNK"))
