"""Per-kernel device-time shares of the hot path, from torch.profiler's CUDA activity trace (no Nsight needed).

    python profiles/kernel_shares.py [mulrelin|rotate] [batch] [--steps S] [--json OUT]

Runs the operation once untimed (tables, pools, tensor maps), then S times under the profiler, and prints every
kernel name with its total device time, launch count and share of the summed kernel time.  The card name and its
power limit are printed with the table: they are part of the numbers.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch
from torch.profiler import ProfilerActivity, profile

import fhe_rs_b200 as F
from bench import DEGREE, N_MODULI, PLAINTEXT, fill_uniform


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip().split(", ")
        return {"gpu": q[0], "power_limit_w": float(q[1])}
    except Exception:   # noqa: BLE001 -- the table is still useful without it
        return {"gpu": torch.cuda.get_device_name(0), "power_limit_w": None}


def short(name):
    # template arguments identify the variant; the namespace and the argument list do not
    name = name.replace("(anonymous namespace)::", "").replace("void ", "").replace("fhe_b200::", "")
    return name.split("(")[0] or name


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("what", nargs="?", default="mulrelin", choices=["mulrelin", "rotate"])
    ap.add_argument("batch", nargs="?", type=int, default=256)
    ap.add_argument("--steps", type=int, default=2)
    ap.add_argument("--json", help="also write the table as JSON")
    a = ap.parse_args()

    par = F.BfvParameters(DEGREE, PLAINTEXT, moduli_sizes=[62] * N_MODULI, device=0)
    moduli = par.moduli()
    A = F.Ciphertext(par, a.batch, 2)
    fill_uniform(torch, A, moduli, 1)
    rng = np.random.default_rng(7)
    kc = np.zeros((2, N_MODULI, N_MODULI, DEGREE), np.uint64)
    for i, q in enumerate(moduli):
        kc[:, :, i, :] = rng.integers(0, q, size=(2, N_MODULI, DEGREE), dtype=np.uint64)
    if a.what == "mulrelin":
        B = F.Ciphertext(par, a.batch, 2)
        fill_uniform(torch, B, moduli, 2)
        m = F.Multiplicator.default(F.RelinearizationKey.from_arrays(par, kc[0], kc[1]))
        op = lambda: m.multiply(A, B)   # noqa: E731
    else:
        gk = F.GaloisKey.from_arrays(par, 3, kc[0], kc[1])
        op = lambda: gk.relinearize(A)   # noqa: E731
    op().sync()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(a.steps):
            out = op()
        out.sync()
        torch.cuda.synchronize()

    per = {}
    for ev in prof.events():
        if ev.device_type != torch.autograd.DeviceType.CUDA:
            continue
        k = short(ev.name)
        t, c = per.get(k, (0.0, 0))
        per[k] = (t + ev.time_range.elapsed_us(), c + 1)
    total = sum(t for t, _ in per.values())
    rows = sorted(((k, t, c) for k, (t, c) in per.items()), key=lambda r: -r[1])
    info = card()
    print("%s, power limit %s W; %s batch %d, %d steps; summed kernel time %.2f ms per step"
          % (info["gpu"], info["power_limit_w"], a.what, a.batch, a.steps, total / 1e3 / a.steps))
    print("%8s %6s %7s  %s" % ("ms/step", "share", "launch", "kernel"))
    for k, t, c in rows:
        print("%8.3f %5.1f%% %7.1f  %s" % (t / 1e3 / a.steps, 100.0 * t / total, c / a.steps, k))
    if a.json:
        with open(a.json, "w") as f:
            json.dump({**info, "what": a.what, "batch": a.batch, "steps": a.steps,
                       "kernel_ms_per_step": total / 1e3 / a.steps,
                       "kernels": [{"name": k, "ms_per_step": t / 1e3 / a.steps, "share": t / total,
                                    "launches_per_step": c / a.steps} for k, t, c in rows]}, f, indent=1)


if __name__ == "__main__":
    main()
