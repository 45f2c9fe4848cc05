"""Hoisted rotations (fhe_b200_galois_many_hoisted) against fhe_b200_galois_many on the same seeded inputs, the two
calls alternating in one run.
    python profiles/hoisted_bench.py [out.json]
Workloads:
  * d = 16 and 64 column rotations of one ciphertext (steps 1..d), at N = 2^13 with the MulPIR moduli (50/55/55) and at
    set C (N = 2^15, 14 x 62-bit): the workloads of rotations_bench.py, where every output shares its source.
  * Set C, 16 ciphertexts x 8 shared steps (128 outputs, 8 keys): many sources, each hoisted once for 8 outputs.
  * Set C, 64 ciphertexts x 1 step each (16 distinct steps): no source has two outputs, so nothing is hoisted and the
    call is galois_many's path; its rate must match.
Keys and ciphertexts are random words (the timing does not depend on them).  Both calls are checked word for word,
and n_hoisted against the workload's expectation, before timing.  Each call is warmed up, then timed with CUDA events
in windows of at least one second (the call count per window comes from the warm-up), five windows per call,
alternating the calls; the spread is the windows' minimum and maximum.  The card's name, power limit and nominal SM
clock are read in the same run."""
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
from rotations_bench import MULPIR_T, KeyWords, words  # noqa: E402

L = F._capi.lib()
WINDOW_S, WINDOWS = 1.0, 5


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
    """routes: name -> (call, outputs per call)"""
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
        res[name].update(ms_per_call=med, ms_min=min(ms), ms_max=max(ms), units_per_s=units / (med * 1e-3),
                         units_per_s_min=units / (max(ms) * 1e-3), units_per_s_max=units / (min(ms) * 1e-3))
    return res


def workload(name, degree, t, sizes, n_ct, steps, source, expect_hoisted):
    """output j rotates ciphertext source[j] by steps[j]"""
    par = F.BfvParameters(degree, t, moduli_sizes=sizes, device=0)
    rng = np.random.default_rng(degree + len(steps) + n_ct)
    kw = KeyWords(par, rng)
    distinct = sorted(set(steps))
    gks = [kw.gk(pow(3, i, 2 * degree)) for i in distinct]
    index = [distinct.index(i) for i in steps]
    ct = F.Ciphertext.from_host(par, words(rng, par.moduli(), (n_ct, 2), degree))
    many = F.galois_many(ct, gks, index, source)
    hoisted, nh = F.galois_many_hoisted(ct, gks, index, source)
    assert (many.to_host() == hoisted.to_host()).all(), name
    assert nh == expect_hoisted, (name, nh)
    del many, hoisted
    routes = {"galois_many": (lambda: F.galois_many(ct, gks, index, source), len(steps)),
              "galois_many_hoisted": (lambda: F.galois_many_hoisted(ct, gks, index, source), len(steps))}
    return dict(workload=name, N=degree, moduli_bits=sizes, ciphertexts=n_ct, outputs=len(steps),
                distinct_steps=len(distinct), n_hoisted=nh, unit="rotation", words_equal=True, **timed(routes))


def main():
    out = sys.argv[1] if len(sys.argv) > 1 else None
    info = gpu_info()
    print("gpu:", info, flush=True)
    set_c = (1 << 15, 786433, [62] * 14)
    rows = []
    for d in (16, 64):
        for name, shape in (("mulpir", (8192, MULPIR_T, [50, 55, 55])), ("set_c", set_c)):
            rows.append(workload("%s_rotations_%d" % (name, d), *shape, 1, list(range(1, d + 1)), [0] * d, d))
            print(json.dumps(rows[-1]), flush=True)
    rows.append(workload("set_c_16_ciphertexts_x_8_steps", *set_c, 16, [1 + j % 8 for j in range(128)],
                         [j // 8 for j in range(128)], 128))
    print(json.dumps(rows[-1]), flush=True)
    rows.append(workload("set_c_64_ciphertexts_x_1_step", *set_c, 64, [1 + j % 16 for j in range(64)], list(range(64)),
                         0))
    print(json.dumps(rows[-1]), flush=True)
    if out:
        with open(out, "w") as f:
            json.dump({"gpu": info, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
