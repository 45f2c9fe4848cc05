"""Timings of the other operations of the path at set C (N = 2^15, 14 x 62-bit), device-resident operands, through
the host mirror (so each call also allocates its result batch).
    python profiles/secondary_bench.py [batch]
Not a bench.py line: context for DESIGN.md (rotation = BASELINE config 4; add is the HBM-bound member of the family)."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch
import fhe_rs_b200 as F
from bench import fill_uniform, DEGREE, N_MODULI, PLAINTEXT, peaks

B = int(sys.argv[1]) if len(sys.argv) > 1 else 256
par = F.BfvParameters(DEGREE, PLAINTEXT, moduli_sizes=[62] * N_MODULI, device=0)
moduli = par.moduli()
A = F.Ciphertext(par, B, 2)
Bt = F.Ciphertext(par, B, 2)
fill_uniform(torch, A, moduli, 1)
fill_uniform(torch, Bt, moduli, 2)
rng = np.random.default_rng(7)
kc = np.zeros((2, N_MODULI, N_MODULI, DEGREE), np.uint64)
for i, q in enumerate(moduli):
    kc[:, :, i, :] = rng.integers(0, q, size=(2, N_MODULI, DEGREE), dtype=np.uint64)
rk = F.RelinearizationKey.from_arrays(par, kc[0], kc[1])
gk = F.GaloisKey.from_arrays(par, 3, kc[0], kc[1])
ct_bytes = 2 * N_MODULI * DEGREE * 8
hbm, _ = peaks()


def timed(fn, reps=5, warm=2):
    """seconds per call: wall clock between two device synchronisations (the calls are asynchronous)"""
    import time
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(reps):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / reps


out = {"batch": B, "set": "C: n=2^15, 14x62-bit", "hbm_peak_gbs": hbm}
s = timed(lambda: A.__iadd__(Bt))
out["add"] = {"ct_per_s": B / s, "gbs": 3 * B * ct_bytes / s / 1e9, "hbm_frac": 3 * B * ct_bytes / s / 1e9 / hbm,
              "bytes": "2 reads + 1 write of a ciphertext (SURVEY 8d: 22.0 MB per ct + ct)"}
s = timed(lambda: gk.relinearize(A))
out["rotate_columns_by_1"] = {"ct_per_s": B / s, "ms_per_ct": s / B * 1e3, "what": "GaloisKey::relinearize, exponent 3 (BASELINE config 4)"}
s = timed(lambda: A * Bt)
out["mul_no_relin"] = {"ct_per_s": B / s}
C3 = A * Bt
s = timed(lambda: rk.relinearizes(C3))
out["relinearize"] = {"ct_per_s": B / s}
s = timed(lambda: (A.into_power_basis(), A.into_ntt()))
out["ntt_fwd_plus_inv"] = {"us_per_limb_ntt": s / (2 * B * 2 * N_MODULI) * 1e6,
                           "alg_gbs": 2 * B * 2 * N_MODULI * 16 * DEGREE / s / 1e9}
n_terms = 64
pts = F.Ciphertext(par, B, 1)
fill_uniform(torch, pts, moduli, 5)
s = timed(lambda: F.dot_product_scalar(A, pts, n_terms))
rd = B * (ct_bytes + ct_bytes // 2)
out["dot_product_scalar"] = {"terms_per_s": B / s, "n_terms": n_terms, "gbs": rd / s / 1e9, "hbm_frac": rd / s / 1e9 / hbm}
s = timed(lambda: A.to_packed(), reps=2, warm=1)
out["wire_pack_to_host"] = {"ct_per_s": B / s, "note": "inverse NTT + 62-bit packing + download to pageable host memory"}

# plaintexts: B SIMD plaintexts of N slot values (B*N u64) against the B*L*N poly_ntt words they encode to
from fhe_rs_b200 import _capi  # noqa: E402
lib = _capi.lib()
n_vals = B * DEGREE
slots = torch.from_numpy(rng.integers(0, PLAINTEXT, size=n_vals, dtype=np.int64))
slots_pinned, slots_dev = slots.pin_memory(), slots.cuda()
PT = F.Ciphertext(par, B, 1)
enc = par.encoder()
for name, src in (("encode_simd_pinned_host", slots_pinned), ("encode_simd_device", slots_dev)):
    s = timed(lambda: _capi.check(lib.fhe_b200_encode(enc, _capi.ENCODING_SIMD, 1, src.data_ptr(), n_vals, PT._h, 0)))
    out[name] = {"pt_per_s": B / s, "input_mb": n_vals * 8 / 1e6}
words_pinned = torch.empty(B * N_MODULI * DEGREE, dtype=torch.int64).pin_memory()
s = timed(lambda: _capi.check(lib.fhe_b200_batch_upload(PT._h, 0, B, words_pinned.data_ptr(), 0)))
out["upload_host_encoded_poly_ntt_pinned"] = {"pt_per_s": B / s, "input_mb": B * N_MODULI * DEGREE * 8 / 1e6,
                                              "note": "today's route without the CPU encode: poly_ntt words from pinned memory"}
P = F.PlaintextVec(PT, F.Encoding.simd())
s = timed(lambda: A.mul_plain(P))
out["mul_plain_batch"] = {"ct_per_s": B / s, "plaintexts": B}
s = timed(lambda: A.add_plain(P))
out["add_plain_batch"] = {"ct_per_s": B / s, "plaintexts": B, "note": "to_poly derived from poly_ntt on the device"}
import subprocess  # noqa: E402
out["gpu"] = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                            capture_output=True, text=True).stdout.strip()
print(json.dumps(out, indent=1))
