"""Per-ciphertext keys (the fhe_b200_*_keyed entry points): a server answering many clients, each with its own keys,
one call per client against one keyed call for all of them, alternating the routes in one run.
    python profiles/keyed_bench.py [out.json]
Workloads:
  * MulPIR expansion, 16 clients (examples/mulpir.rs: N = 8192, moduli 50/55/55, query at level 1, keys at level 0,
    size 115): 16 fhe_b200_expand calls (Q = 1, own keys) against one fhe_b200_expand_keyed (Q = 16, 16 key sets); the
    shared-key Q = 16 call of profiles/expand_bench.py is the ceiling.
  * Relinearized products, 64 clients: fhe_b200_mul_relin at N = 2^14, 8 x 62-bit, 4 ciphertext pairs per client: 64
    single-key calls against one keyed call.
  * The cost of per-ciphertext key staging: set C (N = 2^15, 14 x 62-bit) keyed mul_relin over 256 pairs with 256
    distinct keys against the shared key on the same inputs.
Keys and ciphertexts are random words (the timing does not depend on them).  Times are wall clock between device
synchronisations after warm-up; launches are counted per call.  Each keyed route is checked word for word against the
per-client route before it is timed."""
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "profiles"))
import fhe_rs_b200 as F  # noqa: E402
from expand_bench import gpu_info  # noqa: E402

L = F._capi.lib()
MULPIR_T = (1 << 20) + (1 << 19) + (1 << 17) + (1 << 16) + (1 << 14) + 1


def sync():
    F._capi.check(L.fhe_b200_sync(None))


def words(rng, moduli, prefix, degree):
    a = np.zeros(tuple(prefix) + (len(moduli), degree), np.uint64)
    for j, q in enumerate(moduli):
        a[..., j, :] = rng.integers(0, q, size=tuple(prefix) + (degree,), dtype=np.uint64)
    return a


def ksk(par, rng, ct_level, key_level):
    m = par.moduli()
    c = words(rng, m[:len(m) - key_level], (2, len(m) - ct_level), par.degree())
    return F.KeySwitchingKey.from_arrays(par, c[0], c[1], ct_level, key_level)


def timed(routes, reps):
    res = {}
    for name, (fn, units) in routes.items():   # warm-up, launch count
        fn()
        sync()
        c0 = L.fhe_b200_launch_count()
        fn()
        sync()
        res[name] = {"launches_per_unit": (L.fhe_b200_launch_count() - c0) / units, "seconds": 0.0}
    for _ in range(reps):
        for name, (fn, _) in routes.items():
            sync()
            t0 = time.perf_counter()
            fn()
            sync()
            res[name]["seconds"] += time.perf_counter() - t0
    for name, (_, units) in routes.items():
        s = res[name].pop("seconds") / reps
        res[name].update(ms_per_call=s * 1e3, ms_per_unit=s * 1e3 / units, units_per_s=units / s)
    return res


def expansion(reps):
    degree, size, clients = 8192, 115, 16
    par = F.BfvParameters(degree, MULPIR_T, moduli_sizes=[50, 55, 55], device=0)
    rng = np.random.default_rng(1)
    level = (size - 1).bit_length()
    eks = []
    for _ in range(clients):
        ek = F.EvaluationKey(par, 1, 0)
        for l in range(level):
            ek.add_galois_key(F.GaloisKey((degree >> l) + 1, ksk(par, rng, 1, 0)))
        eks.append(ek)
    X = F.Ciphertext.from_host(par, words(rng, par.moduli()[:2], (clients, 2), degree), level=1)
    singles = [X.take(c, 1) for c in range(clients)]
    index = list(range(clients))
    keyed = F.expands_batch_keyed(X, eks, index, size).to_host()
    for c in (0, clients - 1):
        one = eks[c].expands_batch(singles[c], size).to_host()
        for i in (0, size - 1):
            assert (keyed[i * clients + c] == one[i]).all(), (c, i)
    del keyed
    routes = {
        "per_client_expand": (lambda: [eks[c].expands_batch(singles[c], size) for c in range(clients)], clients),
        "expand_keyed": (lambda: F.expands_batch_keyed(X, eks, index, size), clients),
        "shared_key_ceiling": (lambda: eks[0].expands_batch(X, size), clients),
    }
    r = timed(routes, reps)
    return dict(workload="mulpir_expansion_16_clients", N=degree, moduli_bits=[50, 55, 55], ct_level=1, key_level=0,
                size=size, clients=clients, unit="expansion", **r)


def products(name, degree, sizes, clients, per_client, reps, shared_route):
    par = F.BfvParameters(degree, 786433, moduli_sizes=sizes, device=0)
    rng = np.random.default_rng(degree + clients)
    # (each key is a device buffer of its own; the words repeat every 8 keys to spare host memory at set C)
    pool = [words(rng, par.moduli(), (2, len(par.moduli())), degree) for _ in range(min(clients, 8))]
    rks = [F.RelinearizationKey(F.KeySwitchingKey.from_arrays(par, pool[c % 8][0], pool[c % 8][1]))
           for c in range(clients)]
    n = clients * per_client
    m = par.moduli()
    A = F.Ciphertext.from_host(par, words(rng, m, (n, 2), degree))
    B = F.Ciphertext.from_host(par, words(rng, m, (n, 2), degree))
    index = [j // per_client for j in range(n)]
    keyed = F.multiply_keyed(A, B, rks, index).to_host()
    mults = [F.Multiplicator.default(rk) for rk in rks]
    As = [A.take(c * per_client, per_client) for c in range(clients)]
    Bs = [B.take(c * per_client, per_client) for c in range(clients)]
    for c in (0, clients - 1):
        assert (mults[c].multiply(As[c], Bs[c]).to_host() == keyed[c * per_client:(c + 1) * per_client]).all(), c
    del keyed
    routes = {"mul_relin_keyed": (lambda: F.multiply_keyed(A, B, rks, index), n)}
    if shared_route:
        routes["shared_key"] = (lambda: mults[0].multiply(A, B), n)
    else:
        routes = dict(per_client_mul_relin=(lambda: [mults[c].multiply(As[c], Bs[c]) for c in range(clients)], n),
                      **routes)
    r = timed(routes, reps)
    return dict(workload=name, N=degree, moduli_bits=sizes, clients=clients, pairs_per_client=per_client,
                unit="product", **r)


def main():
    out = sys.argv[1] if len(sys.argv) > 1 else None
    info = gpu_info()
    print("gpu:", info, flush=True)
    rows = [expansion(20), products("mul_relin_64_clients", 1 << 14, [62] * 8, 64, 4, 10, False),
            products("set_c_key_staging_256_keys", 1 << 15, [62] * 14, 256, 1, 5, True)]
    for r in rows:
        print(json.dumps(r), flush=True)
    if out:
        with open(out, "w") as f:
            json.dump({"gpu": info, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
