"""Decryption, decoding and noise measurement at N = 2^13 (TMA-fed NTT and scaler kernels) and N = 16 (generic
kernels), small enough to run under `compute-sanitizer` (memcheck / racecheck): 2- and 3-part ciphertexts, a batch over
several chunks (FHE_B200_CHUNK=2, three side streams), Poly / SIMD decoding into host and device memory, checked
against the oracle."""
import os
import sys

os.environ.setdefault("FHE_B200_CHUNK", "2")
os.environ.setdefault("FHE_B200_STREAMS", "3")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import numpy as np  # noqa: E402
import fhe_oracle as O  # noqa: E402
import fhe_rs_b200 as F  # noqa: E402

for degree, t, sizes in ((1 << 13, 786433, [62] * 3), (16, 1153, [62, 62, 62])):
    opar = O.BfvParameters(degree, t, moduli_sizes=sizes)
    gpar = F.BfvParameters(degree, t, moduli=opar.moduli, device=0)
    rng = np.random.default_rng(degree)
    osk = O.SecretKey(opar, rng)
    sk = F.SecretKey(gpar, osk.coeffs)
    for level in (0, len(sizes) - 1):
        w = np.stack([osk.encrypt(rng.integers(0, t, size=degree), level, rng).to_array() for _ in range(5)])
        A = F.Ciphertext.from_host(gpar, w, level)
        for ct in (A, A * A):
            words = ct.to_host()
            pts = sk.try_decrypt(ct)
            poly = pts.try_decode(F.Encoding.poly_at_level(level))
            signed = pts.try_decode(F.Encoding.poly_at_level(level), signed=True)
            noise = sk.measure_noise(ct)
            for k in range(len(words)):
                oc = O.Ciphertext.from_array(opar, words[k], level)
                m = osk.decrypt(oc)
                assert (poly[k * degree:(k + 1) * degree] == m).all()
                assert int(noise[k]) == osk.measure_noise(oc)
            if degree > 16:
                import torch
                out = torch.empty(len(words) * degree, dtype=torch.int64, device="cuda")
                pts.try_decode(F.Encoding.simd_at_level(level), out=out)
                assert (out.cpu().numpy().view(np.uint64) == pts.try_decode(F.Encoding.simd_at_level(level))).all()
            assert (np.mod(signed, t).astype(np.uint64) == poly).all()
    del sk
print("sanitize decrypt probe ok")
