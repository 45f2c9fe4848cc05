"""Run by tests/test_gpu_encrypt.py::test_encrypt_chunking in a subprocess with a small FHE_B200_CHUNK and 1, 2 or 4
FHE_B200_STREAMS: secret-key and public-key encryption of a batch that spans several chunks must give the words the
stream defines for the whole call (every block is addressed by the call-wide ciphertext index), also with a temporary
key released right after the enqueue-only call."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import encrypt_reference as R  # noqa: E402
import fhe_oracle as orc  # noqa: E402
import fhe_rs_b200 as F  # noqa: E402

degree, t, count = 1 << 12, 1032193, 11
opar = orc.BfvParameters(degree, t, moduli_sizes=[62] * 3)
par = F.BfvParameters(degree, t, moduli=opar.moduli, device=0)
rng = np.random.default_rng(int(os.environ.get("FHE_B200_CHUNK", "0")) + 400)
osk = orc.SecretKey(opar, rng)
sk = F.SecretKey(par, osk.coeffs)
for level in (0, 1):
    values = rng.integers(0, t, size=count * degree, dtype=np.uint64)
    P = F.PlaintextVec.try_encode(values, F.Encoding.simd_at_level(level), par)
    ms = [R.to_poly(opar, orc.simd_encode(opar, values[k * degree:(k + 1) * degree]), level) for k in range(count)]
    seed_pk, seed_sk, seed_enc = (rng.integers(0, 256, 32, dtype=np.uint8).tobytes() for _ in range(3))
    pk = F.PublicKey.new(sk, seed_pk)
    opk = R.encrypt_sk(osk, seed_pk, 1, 0, 10)[0]
    want_sk = np.stack([c.to_array() for c in R.encrypt_sk(osk, seed_sk, count, level, 10, ms)])
    want_pk = np.stack([c.to_array() for c in R.encrypt_pk(opar, opk, seed_enc, count, level, 10, ms)])
    assert (sk.try_encrypt(P, seed_sk).to_host() == want_sk).all(), level
    assert (pk.try_encrypt(P, seed_enc).to_host() == want_pk).all(), level
    # temporary keys, released as soon as the call has been enqueued
    data_sk, data_pk = sk.to_bytes(), pk.to_bytes()
    for _ in range(2):
        got_sk = F.SecretKey.from_bytes(par, data_sk).try_encrypt(P, seed_sk)
        got_pk = F.PublicKey.from_bytes(par, data_pk).try_encrypt(P, seed_enc)
        assert (got_sk.to_host() == want_sk).all() and (got_pk.to_host() == want_pk).all(), level
    assert (sk.try_decrypt(got_pk).try_decode(F.Encoding.simd_at_level(level)) == values).all()
print("encrypt chunk probe ok", count, "ciphertexts, chunk", os.environ.get("FHE_B200_CHUNK"),
      "streams", os.environ.get("FHE_B200_STREAMS"))
