"""Run by tests/test_gpu_work_split.py in subprocesses, because the library reads its switches once per process.

    work_split_probe.py sweep OUT.json SHAPES
                                            shapes of work_split_cases ({name: counts} as JSON), every operation: a
                                            digest of every output ciphertext
    work_split_probe.py bench OUT.json [--oracle]
                                            the benchmarked shape (N = 2^15, 14 x 62-bit) on 520 pairs filled in HBM
                                            from a fixed seed: a digest of every mul_relin product and every
                                            exponent-3 rotation; --oracle also checks ciphertexts 0, 259 and 519
    work_split_probe.py threads             four host threads sharing one fresh parameter set, each on its own
                                            stream, against the same calls made one thread at a time
"""
import json
import os
import sys
import threading

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle"), os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)
import fhe_rs_b200 as F  # noqa: E402
import work_split_cases as W  # noqa: E402


def sweep(out, shapes):
    res = {}
    for name, counts in json.loads(shapes).items():
        res[name] = W.device_digests(F, name, counts)
    with open(out, "w") as f:
        json.dump(res, f)


BENCH_COUNT = 4 * 128 + 8


def bench(out, with_oracle):
    import torch
    degree, t, L = 1 << 15, 786433, 14
    gpar = F.BfvParameters(degree, t, moduli_sizes=[62] * L, device=0)
    moduli = gpar.moduli()
    rng = np.random.default_rng(520)
    kc, gc = W._rows(rng, moduli, (2, L), degree), W._rows(rng, moduli, (2, L), degree)
    A = F.Ciphertext(gpar, BENCH_COUNT, 2)
    B = F.Ciphertext(gpar, BENCH_COUNT, 2)
    for ct, seed in ((A, 1), (B, 2)):   # uniform residues written straight into HBM, as bench.py fills its batch
        count, parts, limbs, n = ct.shape()
        ptr = ct.device_ptr()

        class Dev:
            __cuda_array_interface__ = {"shape": (count * parts * limbs * n,), "typestr": "<i8", "data": (ptr, False),
                                        "version": 3}
        view = torch.as_tensor(Dev(), device="cuda").view(count, parts, limbs, n)
        g = torch.Generator(device="cuda")
        g.manual_seed(seed)
        for i, q in enumerate(moduli):
            view[:, :, i, :].copy_(torch.randint(0, q, (count, parts, n), dtype=torch.int64, device="cuda", generator=g))
    torch.cuda.synchronize()
    rk = F.RelinearizationKey.from_arrays(gpar, kc[0], kc[1])
    gk = F.GaloisKey.from_arrays(gpar, 3, gc[0], gc[1])
    P = F.Multiplicator.default(rk).multiply(A, B)
    R = gk.relinearize(A)
    res = {"mul": W.device_batch_digests(P), "rot3": W.device_batch_digests(R)}
    if with_oracle:
        import fhe_oracle as O
        opar = O.BfvParameters(degree, t, moduli_sizes=[62] * L)
        assert opar.moduli == moduli
        om = O.Multiplicator.default(O.RelinearizationKey.from_ksk(O.KeySwitchingKey.from_arrays(opar, kc[0], kc[1])))
        ogk = O.GaloisKey.__new__(O.GaloisKey)
        ogk.exponent, ogk.ksk = 3, O.KeySwitchingKey.from_arrays(opar, gc[0], gc[1])
        one = np.empty((1, 2, L, degree), np.uint64)
        for i in (0, 259, BENCH_COUNT - 1):
            a = O.Ciphertext.from_array(opar, A.to_host(one.copy(), first=i)[0], 0)
            b = O.Ciphertext.from_array(opar, B.to_host(one.copy(), first=i)[0], 0)
            assert W.digest(om.multiply(a, b).to_array()) == res["mul"][i], "product %d differs from the oracle" % i
            assert W.digest(ogk.relinearize(a).to_array()) == res["rot3"][i], "rotation %d differs from the oracle" % i
        res["oracle_checked"] = [0, 259, BENCH_COUNT - 1]
    with open(out, "w") as f:
        json.dump(res, f)


def threads():
    """fhe_b200.h: a parameter set may be shared by host threads.  Each thread takes a different count and level, its
    own stream, a rotation exponent no other call has used, and a 2-level expansion, on a parameter set whose levels,
    gather tables and expansion monomials are all still to be built."""
    import torch
    degree, t = 1 << 13, 786433
    jobs = [(5, 0, 5), (9, 1, 7), (11, 0, 11), (16, 1, 13)]   # (count, level, Galois exponent)

    def setup(gpar):
        moduli = gpar.moduli()
        state = []
        for k, (count, level, e) in enumerate(jobs):
            rng = np.random.default_rng(4000 + k)
            ct_mod = moduli[:len(moduli) - level]
            key = lambda: W._rows(rng, moduli[:len(moduli) - level], (2, len(ct_mod)), degree)   # noqa: E731
            kc, gc = key(), key()
            ek_keys = [(degree >> l) + 1 for l in range(2)]
            ekc = [key() for _ in ek_keys]
            a, b = W._rows(rng, ct_mod, (count, 2), degree), W._rows(rng, ct_mod, (count, 2), degree)
            state.append((count, level, e, kc, gc, ek_keys, ekc, a, b))
        return state

    def run(gpar, job, stream, out, k):
        count, level, e, kc, gc, ek_keys, ekc, a, b = job
        with torch.cuda.stream(stream):
            h = stream.cuda_stream
            rk = F.RelinearizationKey.from_arrays(gpar, kc[0], kc[1], ciphertext_level=level, key_level=level)
            gk = F.GaloisKey.from_arrays(gpar, e, gc[0], gc[1], ciphertext_level=level, key_level=level)
            ek = F.EvaluationKey(gpar, level, level)
            for x, c in zip(ek_keys, ekc):
                ek.add_galois_key(F.GaloisKey.from_arrays(gpar, x, c[0], c[1], ciphertext_level=level, key_level=level))
            A = F.Ciphertext.from_host(gpar, a, level=level, stream=h)
            B = F.Ciphertext.from_host(gpar, b, level=level, stream=h)
            res = [F.Multiplicator.default(rk).multiply(A, B).to_host(), gk.relinearize(A).to_host()]
            res += [x.to_host() for x in ek.expands(A, 4)]
            stream.synchronize()
            out[k] = res

    def fresh():
        return F.BfvParameters(degree, t, moduli_sizes=[62, 62, 62], device=0)

    par = fresh()
    state = setup(par)
    shared = [None] * len(jobs)
    errors = []

    def guarded(k):
        try:
            run(par, state[k], torch.cuda.Stream(), shared, k)
        except Exception as exc:   # reported by the main thread
            errors.append((k, repr(exc)))
    ths = [threading.Thread(target=guarded, args=(k,)) for k in range(len(jobs))]
    for th in ths:
        th.start()
    for th in ths:
        th.join()
    assert not errors, errors
    par1 = fresh()
    alone = [None] * len(jobs)
    for k in range(len(jobs)):
        run(par1, state[k], torch.cuda.Stream(), alone, k)
    names = ["mul_relin", "rotation", "expansion 0", "expansion 1", "expansion 2", "expansion 3"]
    for k in range(len(jobs)):
        for n, x, y in zip(names, shared[k], alone[k]):
            assert x.shape == y.shape and (x == y).all(), "thread %d (%d ciphertexts, level %d): %s differs" % (
                k, jobs[k][0], jobs[k][1], n)
    print("threads probe ok", len(jobs), "threads")


if __name__ == "__main__":
    cmd = sys.argv[1]
    if cmd == "sweep":
        sweep(sys.argv[2], sys.argv[3])
    elif cmd == "bench":
        bench(sys.argv[2], "--oracle" in sys.argv[3:])
    elif cmd == "threads":
        threads()
    else:
        raise SystemExit("unknown command " + cmd)
    print("work split probe ok", cmd)
