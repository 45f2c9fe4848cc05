"""Oblivious expansion (EvaluationKey::expands): fhe_b200_expand -- one batched Galois call and one butterfly kernel per
level -- against the host loop the Python mirror ran before it (per output: one Galois call, clone, -=, mul_plain with a
host monomial, +=), alternating the two routes in one run.
    python profiles/expand_bench.py [out.json]
Shapes: MulPIR (examples/mulpir.rs: N = 8192, moduli 50/55/55, query at level 1 with keys at level 0, size 115 =
dim1 + dim2 of its 65 536 x 1 024-byte database) and Set C (N = 2^15, 14 x 62-bit, size 256), each with Q = 1 and 16
queries per call.  Keys and ciphertexts are random words: the timing does not depend on them, and both routes get the
same ones.  Reports expansions per second and ms per expansion (wall clock between device synchronisations, after
warm-up) and kernel launches per expansion; checks that both routes give equal outputs (every output of the last query)."""
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import fhe_rs_b200 as F  # noqa: E402

L = F._capi.lib()
MULPIR_T = (1 << 20) + (1 << 19) + (1 << 17) + (1 << 16) + (1 << 14) + 1


def sync():
    F._capi.check(L.fhe_b200_sync(None))


def host_loop(ek, ct, size, monos):
    """the parent's EvaluationKey.expands: 2^l one-batch Galois calls per level and four element-wise calls per output"""
    n = ek.par.degree()
    level = (size - 1).bit_length()
    out = [None] * (1 << level)
    out[0] = ct.clone()
    for l in range(level):
        gk = ek.gk[(n >> l) + 1]
        step = 1 << l
        for i in range(step):
            sub = gk.relinearize(out[i])
            j = step | i
            if j < size:
                tgt = out[i].clone()
                tgt -= sub
                tgt.mul_plain(monos[l])
                out[j] = tgt
            out[i] += sub
    return out[:size]


def measure(name, degree, t, sizes, ct_level, key_level, size, queries, reps):
    par = F.BfvParameters(degree, t, moduli_sizes=sizes, device=0)
    moduli = par.moduli()
    rng = np.random.default_rng(degree + size)
    Lc, Lk = len(moduli) - ct_level, len(moduli) - key_level
    level = (size - 1).bit_length()
    ek = F.EvaluationKey(par)
    for l in range(level):
        k = np.zeros((2, Lc, Lk, degree), np.uint64)
        for j in range(Lk):
            k[:, :, j] = rng.integers(0, moduli[j], size=(2, Lc, degree), dtype=np.uint64)
        ek.add_galois_key(F.GaloisKey.from_arrays(par, (degree >> l) + 1, k[0], k[1], ciphertext_level=ct_level,
                                                  key_level=key_level))
    monos = []
    for l in range(level):
        m = np.zeros((Lc, degree), np.uint64)
        F._capi.check(L.fhe_b200_debug_expansion_monomial(par._h, ct_level, l, m.ctypes.data))
        monos.append(m)
    rows = []
    for q in (1, queries):
        w = np.zeros((q, 2, Lc, degree), np.uint64)
        for j in range(Lc):
            w[:, :, j] = rng.integers(0, moduli[j], size=(q, 2, degree), dtype=np.uint64)
        X = F.Ciphertext.from_host(par, w, level=ct_level)
        routes = {"host_loop": lambda: host_loop(ek, X, size, monos), "fhe_b200_expand": lambda: ek.expands_batch(X, size)}
        # equality: every output of the last query
        fast = routes["fhe_b200_expand"]()
        sample = np.stack([fast.to_host(np.empty((1, 2, Lc, degree), np.uint64), i * q + q - 1)[0] for i in range(size)])
        del fast
        slow = routes["host_loop"]()
        equal = all((slow[i].to_host(np.empty((1, 2, Lc, degree), np.uint64), q - 1)[0] == sample[i]).all()
                    for i in range(size))
        del slow, sample
        res = {name_: {"seconds": 0.0} for name_ in routes}
        for name_, fn in routes.items():   # warm-up and launch counts
            fn()
            sync()
            c0 = L.fhe_b200_launch_count()
            fn()
            sync()
            res[name_]["launches_per_expansion"] = (L.fhe_b200_launch_count() - c0) / q
        for _ in range(reps):             # alternate the routes
            for name_, fn in routes.items():
                sync()
                t0 = time.perf_counter()
                r = fn()
                sync()
                res[name_]["seconds"] += time.perf_counter() - t0
                del r
        for name_ in routes:
            s = res[name_].pop("seconds") / reps
            res[name_].update(ms_per_call=s * 1e3, ms_per_expansion=s * 1e3 / q, expansions_per_s=q / s)
        rows.append(dict(shape=name, N=degree, moduli_bits=sizes, ct_level=ct_level, key_level=key_level, size=size,
                         queries=q, outputs_equal=bool(equal),
                         speedup=res["fhe_b200_expand"]["expansions_per_s"] / res["host_loop"]["expansions_per_s"],
                         **res))
        print(json.dumps(rows[-1]), flush=True)
    return rows


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader",
                              "-i", os.environ.get("CUDA_VISIBLE_DEVICES", "0").split(",")[0]],
                             capture_output=True, text=True, timeout=60).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = ""
    return out


if __name__ == "__main__":
    info = gpu_info()
    print(json.dumps({"gpu": info}), flush=True)
    rows = measure("MulPIR", 8192, MULPIR_T, [50, 55, 55], 1, 0, 115, 16, reps=5)
    rows += measure("Set C", 1 << 15, 65537, [62] * 14, 0, 0, 256, 16, reps=3)
    result = {"gpu": info, "rows": rows}
    if len(sys.argv) > 1:
        os.makedirs(os.path.dirname(os.path.abspath(sys.argv[1])), exist_ok=True)
        with open(sys.argv[1], "w") as f:
            json.dump(result, f, indent=1)
