"""Decryption on the device: fhe_b200_decrypt, fhe_b200_decrypt + fhe_b200_decode (SIMD, u64) and
fhe_b200_measure_noise at set C (N = 2^15, 14 x 62-bit moduli, t = 786433), batch 256, against the oracle's
single-threaded SecretKey.decrypt on a few ciphertexts.
    python profiles/decrypt_bench.py [out.json]
Two inputs: fresh ciphertexts (2 parts, level 0) and the output of Multiplicator::default(rk).multiply (relinearized,
2 parts, level 0).  Key, ciphertexts and relinearization key are random words: the timing does not depend on them.
Rates are ciphertexts per second, wall clock between device synchronisations after warm-up, the median of three
windows of at least a second each; outputs stay on the device
(the decoded values go to a CUDA buffer).  Prints the card name and power limit with the numbers."""
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import fhe_oracle as O  # noqa: E402
import fhe_rs_b200 as F  # noqa: E402

L = F._capi.lib()
check = F._capi.check


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception as e:  # noqa: BLE001
        return "unknown (%s)" % e


def rate(fn, count, window_s=1.0):
    """calls per timed window chosen so that every window lasts at least window_s; median of three windows"""
    fn()
    check(L.fhe_b200_sync(None))
    t0 = time.perf_counter()
    for _ in range(3):
        fn()
    check(L.fhe_b200_sync(None))
    reps = max(1, int(np.ceil(window_s / ((time.perf_counter() - t0) / 3))))
    best = []
    for _ in range(3):
        t0 = time.perf_counter()
        for _ in range(reps):
            fn()
        check(L.fhe_b200_sync(None))
        best.append(count * reps / (time.perf_counter() - t0))
    return float(np.median(best))


def main():
    import torch
    degree, t, sizes, batch = 1 << 15, 786433, [62] * 14, 256
    opar = O.BfvParameters(degree, t, moduli_sizes=sizes)
    par = F.BfvParameters(degree, t, moduli=opar.moduli, device=0)
    moduli = par.moduli()
    Lc = len(moduli)
    rng = np.random.default_rng(1)
    coeffs = rng.integers(-10, 11, size=degree, dtype=np.int64)
    sk = F.SecretKey(par, coeffs)
    w = np.zeros((batch, 2, Lc, degree), np.uint64)
    for j, q in enumerate(moduli):
        w[:, :, j] = rng.integers(0, q, size=(batch, 2, degree), dtype=np.uint64)
    k = np.zeros((2, Lc, Lc, degree), np.uint64)
    for j, q in enumerate(moduli):
        k[:, :, j] = rng.integers(0, q, size=(2, Lc, degree), dtype=np.uint64)
    rk = F.RelinearizationKey.from_arrays(par, k[0], k[1])
    fresh = F.Ciphertext.from_host(par, w)
    inputs = {"fresh": fresh, "mul_relin": F.Multiplicator.default(rk).multiply(fresh, F.Ciphertext.from_host(par, w))}
    out = F.Ciphertext(par, batch, 1, 0)
    values = torch.empty(batch * degree, dtype=torch.int64, device="cuda")
    noise = torch.empty(batch, dtype=torch.int32, device="cuda")
    enc = par.encoder()
    res = {"card": card(), "degree": degree, "moduli": Lc, "t": t, "batch": batch}
    for name, ct in inputs.items():
        dec = lambda: check(L.fhe_b200_decrypt(sk._h, ct._h, out._h, None))  # noqa: E731

        def dec_decode():
            dec()
            check(L.fhe_b200_decode(enc, 1, 0, out._h, values.data_ptr(), batch * degree, None))
        nz = lambda: check(L.fhe_b200_measure_noise(sk._h, ct._h, noise.data_ptr(), None))  # noqa: E731
        res[name] = {"decrypt_per_s": rate(dec, batch), "decrypt_decode_simd_per_s": rate(dec_decode, batch),
                     "measure_noise_per_s": rate(nz, batch)}
    # the oracle on a few ciphertexts (the host route: download the words, decrypt on the CPU)
    osk = O.SecretKey(opar, rng)
    osk.coeffs = coeffs
    done, t0 = 0, time.perf_counter()
    while done < 4 or time.perf_counter() - t0 < 1.0:   # at least four ciphertexts and one second
        osk.decrypt(O.Ciphertext.from_array(opar, w[done % batch], 0))
        done += 1
    res["oracle_decrypt_per_s"] = done / (time.perf_counter() - t0)
    res["oracle_decrypt_ciphertexts"] = done
    print(json.dumps(res, indent=1))
    if len(sys.argv) > 1:
        with open(sys.argv[1], "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
