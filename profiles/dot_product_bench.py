"""Ciphertext dot products (fhe_b200_dot_product, _keyed) and batch sums (fhe_b200_batch_sum) against the routes they
replace, alternating the routes in one run.
    python profiles/dot_product_bench.py [out.json]
Workloads:
  * Set C (N = 2^15, 14 x 62-bit), n_terms 16 with 1 and 16 groups, 128 with 1 and 4, relinearized, three routes:
      mul_add_loop_relin: one batched fhe_b200_mul, a loop of take + fhe_b200_add per group, fhe_b200_relinearize;
      mul_batch_sum_relin: one batched fhe_b200_mul, one fhe_b200_batch_sum, fhe_b200_relinearize;
      dot_product: one fhe_b200_dot_product.
  * The MulPIR response shape (N = 2^13, 50/55/55 bits, level 1, dim2 = 16 terms, level-1 key, switched to level 2)
    for 16 clients: one fhe_b200_dot_product_keyed call against sixteen per-client loops and sixteen
    fhe_b200_dot_product calls.
  * fhe_b200_batch_sum throughput: bytes read and written over kernel time, against the H100 SXM's 3.35 TB/s.
Keys and ciphertexts are random words (the timing does not depend on them).  Each route is warmed up, then timed with
CUDA events; the routes of a workload are checked word for word against each other before timing.  The card's name,
power limit and nominal SM clock are read in the same run."""
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
from rotations_bench import MULPIR_T, same, timed, words  # noqa: E402

HBM_TBS = 3.35


def rk_of(par, rng, level=0, key_level=0):
    m = par.moduli()
    c = words(rng, m[:len(m) - key_level], (2, len(m) - level), par.degree())
    return F.RelinearizationKey.from_arrays(par, c[0], c[1], level, key_level)


def pooled(par, rng, count, level=0):
    """count ciphertexts at `level` cycling through 16 random ones (host memory stays small at set C)"""
    m = par.moduli()
    pool = words(rng, m[:len(m) - level], (min(count, 16), 2), par.degree())
    return F.Ciphertext.from_host(par, np.resize(pool, (count,) + pool.shape[1:]), level=level)


def loop_route(A, B, n, groups, rk, level=None):
    prods = A * B
    outs = []
    for g in range(groups):
        acc = prods.take(g * n, 1)
        for i in range(1, n):
            acc += prods.take(g * n + i, 1)
        acc = rk.relinearizes(acc)
        outs.append(acc if level is None else acc.switch_to_level(level))
    return outs


def sum_route(A, B, n, rk):
    return rk.relinearizes((A * B).sum(n))


def set_c(n, groups, reps):
    degree, sizes = 1 << 15, [62] * 14
    par = F.BfvParameters(degree, 786433, moduli_sizes=sizes, device=0)
    rng = np.random.default_rng(n * 100 + groups)
    rk = rk_of(par, rng)
    A = pooled(par, rng, groups * n)
    B = pooled(par, rng, groups * n)
    dot = F.dot_product(A, B, n, rk).to_host()
    assert same(sum_route(A, B, n, rk), F.dot_product(A, B, n, rk))
    for g, o in enumerate(loop_route(A, B, n, groups, rk)):
        assert (o.to_host()[0] == dot[g]).all(), g
    routes = {"mul_add_loop_relin": (lambda: loop_route(A, B, n, groups, rk), groups),
              "mul_batch_sum_relin": (lambda: sum_route(A, B, n, rk), groups),
              "dot_product": (lambda: F.dot_product(A, B, n, rk), groups)}
    return dict(workload="set_c_dot_%d_terms_%d_groups" % (n, groups), N=degree, moduli_bits=sizes, n_terms=n,
                groups=groups, unit="relinearized dot product", **timed(routes, reps))


def mulpir_clients(reps):
    degree, sizes, n, clients, level = 8192, [50, 55, 55], 16, 16, 1
    par = F.BfvParameters(degree, MULPIR_T, moduli_sizes=sizes, device=0)
    rng = np.random.default_rng(16)
    rks = [rk_of(par, rng, level, level) for _ in range(clients)]
    A = pooled(par, rng, clients * n, level)
    B = pooled(par, rng, clients * n, level)
    As = [A.take(c * n, n) for c in range(clients)]
    Bs = [B.take(c * n, n) for c in range(clients)]
    idx = list(range(clients))
    keyed = F.dot_product_keyed(A, B, n, rks, idx, level=2).to_host()
    for c in range(clients):
        assert (F.dot_product(As[c], Bs[c], n, rks[c], 2).to_host()[0] == keyed[c]).all(), c
        assert (loop_route(As[c], Bs[c], n, 1, rks[c], 2)[0].to_host()[0] == keyed[c]).all(), c
    routes = {"dot_product_keyed": (lambda: F.dot_product_keyed(A, B, n, rks, idx, level=2), clients),
              "per_client_dot_product": (lambda: [F.dot_product(As[c], Bs[c], n, rks[c], 2) for c in range(clients)],
                                         clients),
              "per_client_loop": (lambda: [loop_route(As[c], Bs[c], n, 1, rks[c], 2) for c in range(clients)],
                                  clients)}
    return dict(workload="mulpir_response_16_clients", N=degree, moduli_bits=sizes, level=level, n_terms=n,
                clients=clients, unit="response", **timed(routes, reps))


def batch_sum_throughput(reps):
    """one batch_sum launch alone: bytes = every input word read once + every output word written once"""
    L = F._capi.lib()
    out = []
    for degree, sizes, count, n in ((1 << 15, [62] * 14, 256, 16), (1 << 15, [62] * 14, 512, 512),
                                    (1 << 13, [62] * 2, 1000, 1000)):
        par = F.BfvParameters(degree, 786433, moduli_sizes=sizes, device=0)
        rng = np.random.default_rng(count)
        X = F.Ciphertext.from_host(par, words(rng, par.moduli(), (1, 2), degree))
        X = F.Ciphertext.from_host(par, np.repeat(X.to_host(), count, axis=0))
        res = F.Ciphertext(par, count // n, 2)
        fn = lambda: L.fhe_b200_batch_sum(X._h, n, 0, res._h, None)   # noqa: E731
        fn()
        torch.cuda.synchronize()
        ms = []
        for _ in range(reps):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(10):
                fn()
            b.record()
            b.synchronize()
            ms.append(a.elapsed_time(b) / 10)
        med = float(np.median(ms))
        nbytes = (count + count // n) * 2 * len(sizes) * degree * 8
        tbs = nbytes / (med * 1e-3) / 1e12
        out.append(dict(workload="batch_sum_%d_to_%d" % (count, count // n), N=degree, moduli_bits=sizes,
                        bytes=nbytes, ms_per_call=med, TB_per_s=tbs, share_of_3_35_TBs=tbs / HBM_TBS))
    return out


def main():
    out = sys.argv[1] if len(sys.argv) > 1 else None
    info = gpu_info()
    print("gpu:", info, flush=True)
    rows = []
    # 128 terms x 16 groups would hold 2048 set-C ciphertexts per operand (15 GB) plus the products: 4 groups instead
    for n, groups in ((16, 1), (16, 16), (128, 1), (128, 4)):
        rows.append(set_c(n, groups, 5 if n * groups <= 256 else 3))
        print(json.dumps(rows[-1]), flush=True)
    rows.append(mulpir_clients(10))
    print(json.dumps(rows[-1]), flush=True)
    for r in batch_sum_throughput(10):
        rows.append(r)
        print(json.dumps(r), flush=True)
    if out:
        with open(out, "w") as f:
            json.dump({"gpu": info, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
