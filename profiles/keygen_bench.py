"""Key generation on the device at set C (N = 2^15, 14 x 62-bit moduli, t = 786433): relinearization keys, inner-sum
EvaluationKeyBuilder.build (15 Galois keys in one call) and RGSW encryptions, against the oracle's single-threaded
RelinearizationKey and the host route (the oracle's key, then fhe_b200_ksk_upload of its 2 x 14 x 14 x N words).
    python profiles/keygen_bench.py [out.json]
Rates are keys (or builds, or RGSW ciphertexts) per second, wall clock between device synchronisations after warm-up,
the median of three windows of at least a second each; the keys stay on the device and are released as the next one
is made.  Prints the card name and power limit with the numbers."""
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.join(ROOT, "profiles"))
import fhe_oracle as O  # noqa: E402
import fhe_rs_b200 as F  # noqa: E402
from encrypt_bench import card, rate  # noqa: E402


def main():
    degree, t, sizes = 1 << 15, 786433, [62] * 14
    opar = O.BfvParameters(degree, t, moduli_sizes=sizes)
    par = F.BfvParameters(degree, t, moduli=opar.moduli, device=0)
    rng = np.random.default_rng(1)
    osk = O.SecretKey(opar, rng)
    sk = F.SecretKey(par, osk.coeffs)
    seed = bytes(range(32))
    res = {"card": card(), "degree": degree, "moduli": len(opar.moduli), "t": t}
    keep = []

    def relin():
        keep[:] = [F.RelinearizationKey.new(sk, seed)]
    res["relin_keys_per_s"] = rate(relin, 1)
    builder = F.EvaluationKeyBuilder(sk).enable_inner_sum()
    res["inner_sum_galois_keys"] = len(builder.exponents())

    def build():
        keep[:] = [builder.build(seed)]
    res["inner_sum_builds_per_s"] = rate(build, 1)
    batch = 16
    pts = F.PlaintextVec.try_encode(rng.integers(0, t, size=batch * degree, dtype=np.uint64), F.Encoding.simd(), par)

    def rgsw():
        keep[:] = sk.try_encrypt_rgsw(pts, seed)
    res["rgsw_batch"] = batch
    res["rgsw_per_s"] = rate(rgsw, batch)
    keep.clear()
    # the oracle's key on one CPU thread, and the host route (that key, then its upload)
    t0 = time.perf_counter()
    ork = O.RelinearizationKey(osk, rng)
    oracle_s = time.perf_counter() - t0
    c0, c1 = ork.ksk.arrays()
    F.RelinearizationKey.from_arrays(par, c0, c1)
    t0 = time.perf_counter()
    for _ in range(3):
        F.RelinearizationKey.from_arrays(par, c0, c1)
    upload_s = (time.perf_counter() - t0) / 3
    res["oracle_relin_keys_per_s"] = 1.0 / oracle_s
    res["host_route_relin_keys_per_s"] = 1.0 / (oracle_s + upload_s)
    res["relin_key_upload_mb"] = 2 * c0.nbytes / 1e6
    print(json.dumps(res, indent=1))
    if len(sys.argv) > 1:
        with open(sys.argv[1], "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
