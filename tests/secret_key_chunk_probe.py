"""Run by tests/test_gpu_secret_key.py::test_secret_key_chunking in a subprocess with a small FHE_B200_CHUNK and 1, 2
or 4 FHE_B200_STREAMS: a call whose keys span several chunks gives every key the coefficients the stream defines for
the whole call (every block is addressed by the call-wide key index), and encryptions under them the same words."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import secret_key_reference as S  # noqa: E402
import fhe_oracle as orc  # noqa: E402
import fhe_rs_b200 as F  # noqa: E402

degree, t, count = 1 << 12, 1032193, 11
moduli = orc.BfvParameters.generate_moduli([62] * 3, degree)
par = F.BfvParameters(degree, t, moduli=moduli, device=0)
seed = bytes(range(100, 132))
keys = F.SecretKey.random_vec(par, count, seed)
enc_seed = bytes(32)
for k, sk in enumerate(keys):
    want = S.secret_key_coeffs(seed, k, par.variance, degree)
    assert (sk._download_coeffs() == want).all(), k
    host = F.SecretKey(par, want)
    assert (sk.try_encrypt(seed=enc_seed, count=2).to_host() == host.try_encrypt(seed=enc_seed, count=2).to_host()).all()
print("secret key chunk probe ok", count, "keys, chunk", os.environ.get("FHE_B200_CHUNK"),
      "streams", os.environ.get("FHE_B200_STREAMS"))
