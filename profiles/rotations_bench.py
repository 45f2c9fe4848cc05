"""Many rotations per call (fhe_b200_galois_many) and the batched inner sum (fhe_b200_inner_sum, _keyed) against the
one-call-per-step routes they replace, alternating the routes in one run.
    python profiles/rotations_bench.py [out.json]
Workloads:
  * d = 16 and 64 column rotations of one ciphertext (steps 1..d, the rotations of a diagonal matrix-vector product):
    one galois_many call against d fhe_b200_galois calls, at N = 2^13 with the MulPIR moduli (50/55/55) and at set C
    (N = 2^15, 14 x 62-bit).
  * Inner sums at set C, batches of 1, 16 and 256: one fhe_b200_inner_sum against the loop the mirrors ran before it
    (log2 N fhe_b200_galois calls, each followed by fhe_b200_add), with the kernel launches per inner sum.
  * Sixteen clients' inner sums at N = 2^14, 8 x 62-bit, one ciphertext and one key set each: one
    fhe_b200_inner_sum_keyed call against sixteen fhe_b200_inner_sum calls.
Keys and ciphertexts are random words (the timing does not depend on them).  Each route is warmed up, then timed with
CUDA events on the stream the library calls use; both routes of a workload are checked word for word before timing.
The card's name, power limit and nominal SM clock are read in the same run."""
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
MULPIR_T = (1 << 20) + (1 << 19) + (1 << 17) + (1 << 16) + (1 << 14) + 1


def words(rng, moduli, prefix, degree):
    a = np.zeros(tuple(prefix) + (len(moduli), degree), np.uint64)
    for j, q in enumerate(moduli):
        a[..., j, :] = rng.integers(0, q, size=tuple(prefix) + (degree,), dtype=np.uint64)
    return a


class KeyWords:
    """random key words, repeating every 8 keys to spare host memory (each key is a device buffer of its own)"""

    def __init__(self, par, rng):
        self.par, m = par, par.moduli()
        self.pool = [words(rng, m, (2, len(m)), par.degree()) for _ in range(8)]
        self.n = 0

    def gk(self, exponent):
        c = self.pool[self.n % 8]
        self.n += 1
        return F.GaloisKey(exponent, F.KeySwitchingKey.from_arrays(self.par, c[0], c[1]))


def inner_sum_ek(par, kw):
    n = par.degree()
    ek = F.EvaluationKey(par)
    for e in [pow(3, 1 << l, 2 * n) for l in range(n.bit_length() - 2)] + [2 * n - 1]:
        ek.add_galois_key(kw.gk(e))
    return ek


def loop_inner_sum(ek, ct):
    out = ct.clone()
    for g in ek.inner_sum_keys():
        out += g.relinearize(out)
    return out


def timed(routes, reps):
    res = {}
    for name, (fn, units) in routes.items():   # warm-up, launch count
        fn()
        torch.cuda.synchronize()
        c0 = L.fhe_b200_launch_count()
        fn()
        torch.cuda.synchronize()
        res[name] = {"launches_per_unit": (L.fhe_b200_launch_count() - c0) / units, "ms": []}
    for _ in range(reps):
        for name, (fn, _) in routes.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            a.record()
            fn()
            b.record()
            b.synchronize()
            res[name]["ms"].append(a.elapsed_time(b))
    for name, (_, units) in routes.items():
        ms = res[name].pop("ms")
        med = float(np.median(ms))
        res[name].update(ms_per_call=med, ms_min=min(ms), ms_max=max(ms), units_per_s=units / (med * 1e-3))
    return res


def same(a, b):
    return bool((a.to_host() == b.to_host()).all())


def rotations(name, degree, t, sizes, d, reps):
    par = F.BfvParameters(degree, t, moduli_sizes=sizes, device=0)
    rng = np.random.default_rng(degree + d)
    kw = KeyWords(par, rng)
    ek = F.EvaluationKey(par)
    steps = list(range(1, d + 1))
    for i in steps:
        ek.add_galois_key(kw.gk(pow(3, i, 2 * degree)))
    ct = F.Ciphertext.from_host(par, words(rng, par.moduli(), (1, 2), degree))
    many = ek.rotates_columns_by_many(ct, steps).to_host()
    for k, i in enumerate(steps):
        assert (ek.rotates_columns_by(ct, i).to_host()[0] == many[k]).all(), i
    routes = {"galois_many": (lambda: ek.rotates_columns_by_many(ct, steps), d),
              "single_calls": (lambda: [ek.rotates_columns_by(ct, i) for i in steps], d)}
    return dict(workload=name, N=degree, moduli_bits=sizes, steps=d, unit="rotation", **timed(routes, reps))


def inner_sums(batch, reps):
    degree, sizes = 1 << 15, [62] * 14
    par = F.BfvParameters(degree, 786433, moduli_sizes=sizes, device=0)
    rng = np.random.default_rng(batch)
    ek = inner_sum_ek(par, KeyWords(par, rng))
    ct = F.Ciphertext.from_host(par, words(rng, par.moduli(), (batch, 2), degree))
    assert same(ek.computes_inner_sum(ct), loop_inner_sum(ek, ct))
    routes = {"inner_sum": (lambda: ek.computes_inner_sum(ct), batch),
              "galois_add_loop": (lambda: loop_inner_sum(ek, ct), batch)}
    return dict(workload="set_c_inner_sum_batch_%d" % batch, N=degree, moduli_bits=sizes, batch=batch,
                unit="inner sum", **timed(routes, reps))


def clients(reps):
    degree, sizes, n = 1 << 14, [62] * 8, 16
    par = F.BfvParameters(degree, 786433, moduli_sizes=sizes, device=0)
    rng = np.random.default_rng(16)
    kw = KeyWords(par, rng)
    eks = [inner_sum_ek(par, kw) for _ in range(n)]
    ct = F.Ciphertext.from_host(par, words(rng, par.moduli(), (n, 2), degree))
    singles = [ct.take(c, 1) for c in range(n)]
    keyed = F.computes_inner_sum_keyed(ct, eks, list(range(n))).to_host()
    for c in range(n):
        assert (eks[c].computes_inner_sum(singles[c]).to_host()[0] == keyed[c]).all(), c
    routes = {"inner_sum_keyed": (lambda: F.computes_inner_sum_keyed(ct, eks, list(range(n))), n),
              "per_client_inner_sum": (lambda: [eks[c].computes_inner_sum(singles[c]) for c in range(n)], n)}
    return dict(workload="inner_sum_16_clients", N=degree, moduli_bits=sizes, clients=n, unit="inner sum",
                **timed(routes, reps))


def main():
    out = sys.argv[1] if len(sys.argv) > 1 else None
    info = gpu_info()
    print("gpu:", info, flush=True)
    rows = []
    for d in (16, 64):
        rows.append(rotations("mulpir_rotations_%d" % d, 8192, MULPIR_T, [50, 55, 55], d, 20))
        print(json.dumps(rows[-1]), flush=True)
        rows.append(rotations("set_c_rotations_%d" % d, 1 << 15, 786433, [62] * 14, d, 10))
        print(json.dumps(rows[-1]), flush=True)
    for batch, reps in ((1, 20), (16, 10), (256, 3)):
        rows.append(inner_sums(batch, reps))
        print(json.dumps(rows[-1]), flush=True)
    rows.append(clients(10))
    print(json.dumps(rows[-1]), flush=True)
    if out:
        with open(out, "w") as f:
            json.dump({"gpu": info, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
