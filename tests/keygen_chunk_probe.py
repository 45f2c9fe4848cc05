"""Run by tests/test_gpu_keygen.py::test_keygen_chunking in a subprocess with a small FHE_B200_CHUNK and 1, 2 or 4
FHE_B200_STREAMS: Galois keys and RGSW encryptions whose (key, digit) items span several chunks, with chunks that
start and end inside a key, must give the words the stream defines for the whole call; a temporary secret key is
released right after the enqueue-only call."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import keygen_reference as K  # noqa: E402
import fhe_oracle as orc  # noqa: E402
import fhe_rs_b200 as F  # noqa: E402

degree, t = 1 << 12, 1032193
opar = orc.BfvParameters(degree, t, moduli_sizes=[62] * 4)
par = F.BfvParameters(degree, t, moduli=opar.moduli, device=0)
rng = np.random.default_rng(int(os.environ.get("FHE_B200_CHUNK", "0")) + 500)
osk = orc.SecretKey(opar, rng)
sk = F.SecretKey(par, osk.coeffs)


def same(ksk, frm, seed, key):
    c0, c1 = ksk.arrays()
    for i in range(c0.shape[0]):
        w0, w1 = K.key_digit(osk, frm, ksk.ciphertext_level, ksk.ksk_level, seed, key, i, 10)
        assert (c0[i] == w0).all() and (c1[i] == w1).all(), (key, i)


exps = [3, 9, 2 * degree - 1, degree + 1, (degree >> 1) + 1]   # 5 keys x 4 digits
for c, k in ((0, 0), (1, 0)):
    seed = rng.integers(0, 256, 32, dtype=np.uint8).tobytes()
    for key, gk in enumerate(F.bfv._galois_keys(F.SecretKey.from_bytes(par, sk.to_bytes()), exps, c, k, seed)):
        same(gk.ksk, K.galois_from(osk, exps[key], c, k), seed, key)
values = rng.integers(0, t, size=3 * degree, dtype=np.uint64)
P = F.PlaintextVec.try_encode(values, F.Encoding.simd(), par)
ms = [orc.Poly(opar.context_at_level(0), orc.NTT, w.copy()) for w in P.batch.to_host()[:, 0]]
seed = rng.integers(0, 256, 32, dtype=np.uint8).tobytes()
for p, r in enumerate(sk.try_encrypt_rgsw(P, seed)):
    same(r.ksk0, K.rgsw_from(osk, ms[p], 0, False), seed, 2 * p)
    same(r.ksk1, K.rgsw_from(osk, ms[p], 0, True), seed, 2 * p + 1)
print("keygen chunk probe ok, chunk", os.environ.get("FHE_B200_CHUNK"), "streams", os.environ.get("FHE_B200_STREAMS"))
