"""Run by tests/test_gpu_decrypt.py::test_decrypt_chunking in a subprocess with a small FHE_B200_CHUNK and several
FHE_B200_STREAMS: decrypting, decoding and measuring the noise of a batch that spans several chunks (dealt over the side
streams) must give entry by entry what one-ciphertext calls give."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import fhe_oracle as orc  # noqa: E402
import fhe_rs_b200 as F  # noqa: E402

degree, t, count = 1 << 12, 1032193, 11
opar = orc.BfvParameters(degree, t, moduli_sizes=[62] * 3)
par = F.BfvParameters(degree, t, moduli=opar.moduli, device=0)
rng = np.random.default_rng(int(os.environ.get("FHE_B200_CHUNK", "0")) + 300)
osk = orc.SecretKey(opar, rng)
sk = F.SecretKey(par, osk.coeffs)
words = np.stack([osk.encrypt(rng.integers(0, t, size=degree), 0, rng).to_array() for _ in range(count)])
ct = F.Ciphertext.from_host(par, words)
whole = sk.try_decrypt(ct)
whole_ntt = whole.poly_ntt()
whole_simd = whole.try_decode(F.Encoding.simd())
whole_i64 = whole.try_decode(F.Encoding.poly(), signed=True)
whole_noise = sk.measure_noise(ct)
for k in range(count):
    one_ct = F.Ciphertext.from_host(par, words[k:k + 1])
    one = sk.try_decrypt(one_ct)
    assert (one.poly_ntt()[0] == whole_ntt[k]).all(), k
    assert (one.try_decode(F.Encoding.simd()) == whole_simd[k * degree:(k + 1) * degree]).all(), k
    assert (one.try_decode(F.Encoding.poly(), signed=True) == whole_i64[k * degree:(k + 1) * degree]).all(), k
    assert sk.measure_noise(one_ct)[0] == whole_noise[k], k
    assert whole_noise[k] == osk.measure_noise(orc.Ciphertext.from_array(opar, words[k], 0)), k
ctx = opar.context_at_level(0)
want = np.stack([orc.Poly.from_u64(ctx, osk.decrypt(orc.Ciphertext.from_array(opar, words[k], 0)), orc.NTT).c
                 for k in range(count)])
assert (whole_ntt == want).all()
# a temporary key is released as soon as the enqueue-only call returns, while its chunks may still be queued on the
# side streams (or on a caller's non-blocking stream): the release must not erase s under them
import torch  # noqa: E402
data = sk.to_bytes()
for stream in (0, torch.cuda.Stream().cuda_stream):
    for _ in range(3):
        pts = F.SecretKey.from_bytes(par, data).try_decrypt(F.Ciphertext.from_host(par, words, stream=stream))
        assert (pts.poly_ntt() == want).all(), stream
print("decrypt chunk probe ok", count, "ciphertexts, chunk", os.environ.get("FHE_B200_CHUNK"),
      "streams", os.environ.get("FHE_B200_STREAMS"))
