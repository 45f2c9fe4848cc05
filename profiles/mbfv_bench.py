"""Multiparty BFV on the device at set C (N = 2^15, 14 x 62-bit moduli, t = 786433): one party's decryption shares
for C = 256 ciphertexts, and the aggregator's work for P = 16 parties.
    python profiles/mbfv_bench.py [out.json]
Rates are wall clock between device synchronisations after warm-up, the median of three windows of at least a second
each.  The aggregation bandwidth counts the bytes the sum has to move, (P + 1) x C x 14 x N x 8 (P share reads and one
write; with the c0 base of a switch, P + 2), over the time of the call, against the H100 SXM's 3.35 TB/s.  Prints the
card name and power limit with the numbers."""
import ctypes as C
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.join(ROOT, "profiles"))
import fhe_oracle as O  # noqa: E402
import fhe_rs_b200 as F  # noqa: E402
from encrypt_bench import card, rate  # noqa: E402
from fhe_rs_b200 import _capi  # noqa: E402

HBM = 3.35e12


def main():
    degree, t, sizes, cts, parties = 1 << 15, 786433, [62] * 14, 256, 16
    opar = O.BfvParameters(degree, t, moduli_sizes=sizes)
    par = F.BfvParameters(degree, t, moduli=opar.moduli, device=0)
    rng = np.random.default_rng(1)
    sk = F.SecretKey(par, O.SecretKey(opar, rng).coeffs)
    seed = bytes(range(32))
    ct = sk.try_encrypt(count=cts, seed=seed)
    res = {"card": card(), "degree": degree, "moduli": len(sizes), "ciphertexts": cts, "parties": parties}
    keep = []

    def share():
        keep[:] = [F.mbfv.DecryptionShare(sk, ct, seed)]
    res["decryption_shares_per_s"] = rate(share, cts)
    shares = [F.mbfv.DecryptionShare(sk, ct, bytes([p]) * 32) for p in range(parties)]
    keep.clear()
    share_bytes = cts * len(sizes) * degree * 8
    out = F.Ciphertext(par, cts, 1, 0)
    hs = (C.c_void_p * parties)(*[s.h_share._h for s in shares])
    lib = _capi.lib()

    def total():
        _capi.check(lib.fhe_b200_shares_sum(hs, parties, out._h, None))
    calls = rate(total, 1)
    res["shares_sum_gb_per_s"] = calls * (parties + 1) * share_bytes / 1e9
    res["shares_sum_share_of_hbm"] = res["shares_sum_gb_per_s"] * 1e9 / HBM
    sw = F.Ciphertext(par, cts, 2, 0)

    def sks_aggregate():
        _capi.check(lib.fhe_b200_sks_aggregate(ct._h, hs, parties, sw._h, None))
    calls = rate(sks_aggregate, 1)
    res["sks_aggregate_gb_per_s"] = calls * (parties + 4) * share_bytes / 1e9   # + c0 read, c0 + c1 write, c1 read
    pts = F.Ciphertext(par, cts, 1, 0)

    def decrypt_aggregate():
        _capi.check(lib.fhe_b200_decryption_aggregate(par.encoder(), ct._h, hs, parties, pts._h, None))
    res["decryption_aggregates_per_s"] = rate(decrypt_aggregate, cts)
    print(json.dumps(res, indent=1))
    if len(sys.argv) > 1:
        with open(sys.argv[1], "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
