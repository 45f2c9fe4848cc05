"""Encryption on the device: fhe_b200_encrypt_sk and fhe_b200_encrypt_pk at set C (N = 2^15, 14 x 62-bit moduli,
t = 786433), batch 256, from device plaintexts and from host values including the SIMD encode, against the oracle's
single-threaded encryption and against today's host route (encrypt on the CPU, then upload the 2 L N words).
    python profiles/encrypt_bench.py [out.json]
Rates are ciphertexts per second, wall clock between device synchronisations after warm-up, the median of three
windows of at least a second each; the ciphertexts stay on the device.  The host route is the oracle's
SecretKey.encrypt (numpy randomness, C arithmetic) per ciphertext plus one upload of the batch.  Prints the card name
and power limit with the numbers."""
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
    degree, t, sizes, batch = 1 << 15, 786433, [62] * 14, 256
    opar = O.BfvParameters(degree, t, moduli_sizes=sizes)
    par = F.BfvParameters(degree, t, moduli=opar.moduli, device=0)
    rng = np.random.default_rng(1)
    osk = O.SecretKey(opar, rng)
    sk = F.SecretKey(par, osk.coeffs)
    pk = F.PublicKey.new(sk, bytes(32))
    values = rng.integers(0, t, size=batch * degree, dtype=np.uint64)
    pts = F.PlaintextVec.try_encode(values, F.Encoding.simd(), par)
    out = F.Ciphertext(par, batch, 2, 0)
    seed = bytes(range(32))
    enc = par.encoder()
    res = {"card": card(), "degree": degree, "moduli": len(opar.moduli), "t": t, "batch": batch}
    for name, fn, key in (("sk", L.fhe_b200_encrypt_sk, sk._h), ("pk", L.fhe_b200_encrypt_pk, pk.c._h)):
        from_device = lambda: check(fn(key, pts.batch._h, 10, seed, out._h, None))  # noqa: E731

        def from_host():
            check(L.fhe_b200_encode(enc, 1, 0, values.ctypes.data, values.size, pts.batch._h, None))
            from_device()
        res[name] = {"encrypt_per_s": rate(from_device, batch), "encode_encrypt_from_host_per_s": rate(from_host, batch)}
    # the host route: the oracle encrypts one ciphertext at a time, then the batch is uploaded
    level0 = [O.plaintext_to_poly(opar, O.simd_encode(opar, values[k * degree:(k + 1) * degree]), 0) for k in range(4)]
    done, words, t0 = 0, [], time.perf_counter()
    while done < 4 or time.perf_counter() - t0 < 1.0:
        words.append(osk.encrypt_poly(level0[done % 4], 0, rng).to_array())
        done += 1
    oracle_s = (time.perf_counter() - t0) / done
    host = np.stack([words[k % done] for k in range(batch)])
    out.upload(host)
    t0 = time.perf_counter()
    for _ in range(3):
        out.upload(host)
    upload_s = (time.perf_counter() - t0) / 3 / batch
    res["oracle_encrypt_sk_per_s"] = 1.0 / oracle_s
    res["oracle_encrypt_ciphertexts"] = done
    res["host_route_encrypt_upload_per_s"] = 1.0 / (oracle_s + upload_s)
    print(json.dumps(res, indent=1))
    if len(sys.argv) > 1:
        with open(sys.argv[1], "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
