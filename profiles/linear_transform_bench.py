"""Baby-step/giant-step matrix x vector products: fhe_b200_linear_transform against the composition of existing calls
on the same inputs, the two alternating in one run.
    python profiles/linear_transform_bench.py [out.json]
Workloads, all at set C (N = 2^15, 14 x 62-bit moduli, t = 786433) with n = 64 diagonals and baby step b = 8 (G = 8
giant groups): batches of 1, 16 and 64 ciphertexts with the diagonals shared, and 16 ciphertexts with one set of
diagonals per ciphertext.
The composition: galois_many_hoisted of the b baby steps of every ciphertext (step 0 through a key of exponent 1),
one dot_product_scalar per giant group, the G - 1 giant rotations of every ciphertext in one galois_many call and
their sum with the group-0 partial by batch_sum.
Keys are generated on the device from one secret key, so both routes must decrypt to the same slots, which is asserted
before timing (their words differ: the composition key-switches step 0).  Each route is timed with CUDA events in
windows of at least one second, five windows per route, alternating; the spread is the windows' minimum and maximum.
hoist_dot_kernel's device time is read with torch.profiler and set against the traffic model: the bytes the kernel
must move per call, from the shapes (keys of the b - 1 baby steps once per chunk of ciphertexts, every ciphertext's
digits and words, the diagonals, the correction rows and the partial sums written), at 3.35 TB/s."""
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "profiles"))
import fhe_rs_b200 as F  # noqa: E402
from expand_bench import gpu_info  # noqa: E402

L = F._capi.lib()
WINDOW_S, WINDOWS, HBM = 1.0, 5, 3.35e12


def event_ms(fn, n):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(n):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b)


def timed(routes):
    """routes: name -> (call, products per call)"""
    res, calls = {}, {}
    for name, (fn, units) in routes.items():
        fn()
        torch.cuda.synchronize()
        c0 = L.fhe_b200_launch_count()
        one = event_ms(fn, 1)
        calls[name] = max(1, int(np.ceil(WINDOW_S * 1e3 / one)))
        res[name] = {"launches_per_call": L.fhe_b200_launch_count() - c0, "calls_per_window": calls[name], "ms": []}
    for _ in range(WINDOWS):
        for name, (fn, _) in routes.items():
            res[name]["ms"].append(event_ms(fn, calls[name]) / calls[name])
    for name, (_, units) in routes.items():
        ms = res[name].pop("ms")
        med = float(np.median(ms))
        res[name].update(ms_per_call=med, ms_min=min(ms), ms_max=max(ms), products_per_s=units / (med * 1e-3),
                         products_per_s_min=units / (max(ms) * 1e-3), products_per_s_max=units / (min(ms) * 1e-3))
    return res


def traffic_bytes(count, n, b, L_, N, per_ct, chunk=256):
    """the bytes hoist_dot_kernel must move per call"""
    G = -(-n // b)
    chunks = -(-count // max(1, chunk // G))
    row = N * 8
    keys = chunks * (b - 1) * 2 * L_ * L_ * row
    digits = count * L_ * L_ * row
    cts = count * 2 * L_ * row
    diags = (count if per_ct else 1) * n * L_ * row
    mrows = chunks * b * L_ * row
    partial = count * G * 2 * L_ * row
    return keys + digits + cts + diags + mrows + partial


def kernel_us(fn, name="hoist_dot_kernel"):
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    times = [e.device_time_total for e in prof.key_averages() if name in e.key]
    return float(sum(times)) if times else None


class Keys:
    def __init__(self, par, n, b, seed):
        self.par = par
        self.sk = F.SecretKey.random_vec(par, 1, seed=bytes([seed]) * 32)[0]
        bld = F.EvaluationKeyBuilder.new(self.sk)
        for s in F.linear_transform_steps(n, b):
            bld.enable_column_rotation(s)
        self.ek = bld.build(seed=bytes([seed + 1]) * 32)
        self.id = F.GaloisKey.new(self.sk, 1, seed=bytes([seed + 2]) * 32)


def workload(name, K, count, n, b, per_ct, seed):
    par, ek, sk = K.par, K.ek, K.sk
    degree, half, t = par.degree(), par.degree() // 2, par.plaintext()
    G = -(-n // b)
    rng = np.random.default_rng(seed)
    enc = F.Encoding.simd()
    v = rng.integers(0, t, (count, 2 * half)).astype(np.uint64)
    ct = sk.try_encrypt(F.PlaintextVec.try_encode(v.reshape(-1), enc, par), seed=bytes([seed]) * 32)
    # a banded matrix by its n diagonals, raw[m][k][q][r] = M_q[r][(r + k) mod N/2] (the (N/2)^2 matrices themselves
    # would not fit in host memory at set C), then rotated right by each diagonal's giant step as encode_diagonals does
    m = count if per_ct else 1
    raw = rng.integers(0, t, (m, n, 2, half)).astype(np.int64)
    d = np.stack([np.roll(raw[:, k], (k // b) * b, axis=-1) for k in range(n)], axis=1).reshape(m, n, 2 * half)
    diags = F.PlaintextVec.try_encode(d.reshape(-1), enc, par)
    diags.n_diags = n
    group_pts = [F.PlaintextVec.try_encode(d[:, g * b:(g + 1) * b].reshape(-1), enc, par) for g in range(G)]
    two_n = 2 * degree
    baby_keys = [K.id] + [ek.gk[pow(3, i, two_n)] for i in range(1, b)]
    giant_keys = [ek.gk[pow(3, g * b, two_n)] for g in range(1, G)]
    baby_index = [i for _ in range(count) for i in range(b)]
    baby_source = [c for c in range(count) for _ in range(b)]
    giant_index = [g - 1 for _ in range(count) for g in range(1, G)]
    giant_source = [g * count + c for c in range(count) for g in range(1, G)]

    def composition():
        baby, _ = F.galois_many_hoisted(ct, baby_keys, baby_index, baby_source)
        parts = F.Ciphertext(par, G * count, 2)
        for g in range(G):
            p = F.dot_product_scalar(baby, group_pts[g], b)
            F.bfv.check(L.fhe_b200_batch_copy_range(parts._h, g * count, p._h, 0, 1, count, 0))
        out = parts.take(0, count)
        if G > 1:
            F.galois_many(parts, giant_keys, giant_index, giant_source).sum(G - 1, out=out)
        return out

    def call():
        return ek.linear_transform(ct, diags, b)
    slots_a = sk.try_decrypt(composition()).try_decode(enc)
    slots_b = sk.try_decrypt(call()).try_decode(enc)
    assert (slots_a == slots_b).all(), name
    vv = v.reshape(count, 2, half).astype(np.int64)
    want = np.zeros((count, 2, half), np.int64)
    for k in range(n):   # (M v)[r] = sum_k M[r][(r + k) mod N/2] v[(r + k) mod N/2]
        want = (want + raw[:, k] * np.roll(vv, -k, axis=-1)) % t
    want = want.reshape(-1).astype(np.uint64)
    assert (slots_b == want).all(), name
    res = timed({"composition": (composition, count), "linear_transform": (call, count)})
    us = kernel_us(call)
    model = traffic_bytes(count, n, b, len(par.moduli()), degree, per_ct)
    return dict(workload=name, N=degree, moduli=len(par.moduli()), ciphertexts=count, n_diags=n, baby=b,
                per_ciphertext_diagonals=per_ct, slots_equal=True, hoist_dot_us=us, traffic_model_bytes=model,
                traffic_floor_us=model / HBM * 1e6, **res)


def main():
    out = sys.argv[1] if len(sys.argv) > 1 else None
    info = gpu_info()
    print("gpu:", info, flush=True)
    par = F.BfvParameters(1 << 15, 786433, moduli_sizes=[62] * 14, device=0)
    n, b = 64, 8
    K = Keys(par, n, b, 41)
    rows = []
    for count, per_ct in ((1, False), (16, False), (64, False), (16, True)):
        rows.append(workload("set_c_%d_ciphertexts%s" % (count, "_per_ciphertext" if per_ct else ""), K, count, n, b,
                             per_ct, 50 + count))
        print(json.dumps(rows[-1]), flush=True)
    if out:
        with open(out, "w") as f:
            json.dump({"gpu": info, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
