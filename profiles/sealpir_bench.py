"""The SealPIR server (examples/sealpir.rs) on the device, per stage, and the reply fold against the host route it
replaces (download, numpy transcode, encode from host values), alternated in one run.
    python profiles/sealpir_bench.py [out.json]
Workloads: the example's default database (65 536 elements of 1 024 bytes, dim1 = dim2 = 81) and a larger one (2^20
elements of 256 bytes, dim1 = dim2 = 162, 1.7 GB of level-1 plaintexts), N = 4096, t = 2056193, moduli 36/36/37,
expansion keys of EvaluationKeyBuilder::new_leveled(&sk, 1, 0) generated on the device.
Reports, from CUDA events after warm-up: ms per query of each server stage (expand, first dimension, switch, fold,
second dimension, switch) and responses per second; the database encode rate (transcode_from_bytes + encode, from a
CUDA tensor); the transcoder's and the fold's achieved bytes per second (bytes read + bytes written, the least traffic
each needs) and their share of the 3.35 TB/s HBM3 bandwidth of the H100 SXM data sheet.  The card's name and power limit
are read in the same run and written beside the numbers.  Checks that the client recovers the element and that the
host route's plaintexts equal the fold's."""
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import fhe_rs_b200 as F  # noqa: E402
import pir_reference as R  # noqa: E402

HBM = 3.35e12
L = F._capi.lib()


def sync():
    F._capi.check(L.fhe_b200_sync(None))


def host_transcode(rows: np.ndarray, in_bits: int, out_bits: int) -> np.ndarray:
    """transcode_bidirectional of every row with numpy, vectorised over the output values"""
    n = rows.shape[1]
    e = -(-n * in_bits // out_bits)
    k = np.arange(e, dtype=np.uint64)
    total = np.uint64(n * in_bits)
    b0 = k * np.uint64(out_bits)
    b1 = np.minimum(b0 + np.uint64(out_bits), total)
    mask_in = np.uint64((1 << in_bits) - 1) if in_bits < 64 else np.uint64(~0 & ((1 << 64) - 1))
    out = np.zeros((rows.shape[0], e), np.uint64)
    first = b0 // np.uint64(in_bits)
    for d in range(-(-out_bits // in_bits) + 1):
        idx = first + np.uint64(d)
        s = idx * np.uint64(in_bits)
        live = s < b1
        w = rows[:, np.minimum(idx, np.uint64(n - 1)).astype(np.int64)] & mask_in
        up = np.where(s >= b0, s - b0, 0).astype(np.uint64)
        down = np.where(s < b0, b0 - s, 0).astype(np.uint64)
        out |= np.where(live, (w >> down) << up, np.uint64(0))
    if out_bits < 64:
        out &= np.uint64((1 << out_bits) - 1)
    return out


def encode_database(par, database, dim1, dim2, epp):
    """encode_database (util.rs:95-145) on the device, the plaintexts transposed for the first dimension: entry
    i * dim1 + k holds row k * dim2 + i.  database: CUDA uint8 tensor [n][elements_size]"""
    n, es = database.shape
    N, nbits = par.degree(), par.plaintext().bit_length() - 1
    flat = torch.zeros((dim1, dim2, epp * es), dtype=torch.uint8, device="cuda")
    flat.view(-1)[: n * es] = database.reshape(-1)
    vals = torch.empty((dim2, dim1, N), dtype=torch.uint64, device="cuda")
    for k in range(dim1):     # rows k * dim2 + i, i < dim2, land at i * dim1 + k: an output row stride of dim1 * N
        F.transcode_from_bytes(par, flat[k], nbits, out_len=N, out=vals[:, k, :])
    return F.PlaintextVec.try_encode(vals.view(-1), F.Encoding.poly_at_level(1), par)


def server(par, ek, query, db, dim1, dim2):
    """sealpir.rs:158-211: expand, first dimension, switch, fold, second dimension, switch"""
    X = ek.expands_batch(query, dim1 + dim2)
    first = F.dot_product_scalar(X.take(0, dim1), db, n_terms=dim1).switch_to_level(par.max_level())
    pts = first.fold(int(par.moduli()[0]).bit_length(), par.plaintext().bit_length() - 1, 1)
    return F.dot_product_scalar(X.take(dim1, dim2), pts, n_terms=dim2).switch_to_level(par.max_level())


def client(par, sk, responses, index, es, epp):
    """sealpir.rs:222-273: decrypt, decode, unfold into a level-2 ciphertext, decrypt, decode, bytes"""
    import ctypes as C
    N, nbits = par.degree(), par.plaintext().bit_length() - 1
    in_bits, lvl = int(par.moduli()[0]).bit_length(), par.max_level()
    dec = torch.empty(responses.count * N, dtype=torch.uint64, device="cuda")
    sk.try_decrypt(responses).try_decode(F.Encoding.poly_at_level(lvl), out=dec)
    E = -(-N * in_bits // nbits)
    ct = F.Ciphertext(par, 1, 2, lvl, F.NTT)
    dptr, nw = C.c_void_p(), C.c_size_t()
    F._capi.check(L.fhe_b200_batch_device_ptr(ct._h, C.byref(dptr), C.byref(nw)))
    F._capi.check(L.fhe_b200_transcode(par._h, dec.data_ptr(), 8, E, E, nbits, dptr, 8, N, N, in_bits, 2, None))
    vals = torch.empty(N, dtype=torch.uint64, device="cuda")
    sk.try_decrypt(ct).try_decode(F.Encoding.poly_at_level(lvl), out=vals)
    plaintext = F.transcode_to_bytes(par, vals, nbits)
    off = index % epp
    return bytes(plaintext[off * es:(off + 1) * es])


def timed(fn, reps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        r = fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / reps, r


def measure(n_el, es, reps):
    N, t = R.SEALPIR_DEGREE, R.SEALPIR_T
    par = F.BfvParameters(N, t, moduli_sizes=R.SEALPIR_SIZES, device=0)
    epp, rows, dim1, dim2 = R.layout(N, t, n_el, es)
    nbits, in_bits = t.bit_length() - 1, int(par.moduli()[0]).bit_length()
    g = torch.Generator(device="cuda").manual_seed(n_el)
    database = torch.randint(0, 256, (n_el, es), dtype=torch.uint8, device="cuda", generator=g)
    encode_database(par, database, dim1, dim2, epp)              # warm-up
    sync()
    t0 = time.perf_counter()
    db = encode_database(par, database, dim1, dim2, epp)
    sync()
    encode_s = time.perf_counter() - t0
    rng = np.random.default_rng(n_el)
    sk = F.SecretKey(par, rng.integers(-1, 2, size=N))
    level = (dim1 + dim2 - 1).bit_length()
    ek = F.EvaluationKey.from_bytes(par, F.EvaluationKeyBuilder.new_leveled(sk, 1, 0).enable_expansion(level)
                                    .build(seed=bytes(32)).to_bytes())
    index = int(rng.integers(0, n_el))
    pts = F.PlaintextVec.try_encode(R.query_values(dim1, dim2, index, epp, t), F.Encoding.poly_at_level(1), par)
    q = sk.try_encrypt(pts, seed=bytes([7]) * 32)
    resp = server(par, ek, q, db, dim1, dim2)
    ok = client(par, sk, resp, index, es, epp) == database[index].cpu().numpy().tobytes()

    # per stage, each stage's inputs made once
    X = ek.expands_batch(q, dim1 + dim2)
    s1, s2 = X.take(0, dim1), X.take(dim1, dim2)
    first = F.dot_product_scalar(s1, db, n_terms=dim1)
    first_sw = first.switch_to_level(par.max_level())
    folded = first_sw.fold(in_bits, nbits, 1)
    second = F.dot_product_scalar(s2, folded, n_terms=dim2)
    stages = {
        "expand": lambda: ek.expands_batch(q, dim1 + dim2),
        "first_dimension": lambda: F.dot_product_scalar(s1, db, n_terms=dim1),
        "switch_first": lambda: first.switch_to_level(par.max_level()),
        "fold": lambda: first_sw.fold(in_bits, nbits, 1),
        "second_dimension": lambda: F.dot_product_scalar(s2, folded, n_terms=dim2),
        "switch_second": lambda: second.switch_to_level(par.max_level()),
    }
    ms = {}
    for name, fn in stages.items():
        fn()
        sync()
        ms[name] = timed(fn, reps)[0]
    total_ms, _ = timed(lambda: server(par, ek, q, db, dim1, dim2), reps)

    # the fold against the host route, alternated; each window holds the call and the release of its result, as the
    # back-to-back stage loop above does (there a result is released when the next call replaces it)
    P = len(folded) // dim2
    fold_bytes = dim2 * 2 * N * 8 + P * dim2 * 2 * N * 8            # ciphertext words read, level-1 plaintexts written

    def host_route():
        words = first_sw.to_host()                                   # [dim2][2][1][N]
        vals = host_transcode(words.reshape(dim2 * 2, N), in_bits, nbits).reshape(dim2, -1)
        lay = np.zeros((P, dim2, N), np.uint64)
        flat = np.zeros((dim2, P * N), np.uint64)
        flat[:, :vals.shape[1]] = vals
        lay[:] = flat.reshape(dim2, P, N).transpose(1, 0, 2)
        return F.PlaintextVec.try_encode(lay.reshape(-1), F.Encoding.poly_at_level(1), par)
    equal = bool((host_route().batch.to_host() == folded.batch.to_host()).all())
    dev_s = host_s = 0.0
    for _ in range(reps):
        for route in ("device", "host"):
            sync()
            t0 = time.perf_counter()
            r = first_sw.fold(in_bits, nbits, 1) if route == "device" else host_route()
            del r
            sync()
            if route == "device":
                dev_s += time.perf_counter() - t0
            else:
                host_s += time.perf_counter() - t0

    # the transcoder alone, device to device: the first dimension's words of 64 queries' worth of rows
    rows_in = torch.randint(0, 1 << 36, (8192, N), dtype=torch.int64, device="cuda", generator=g).view(torch.uint64)
    e = -(-N * in_bits // nbits)
    rows_out = torch.empty((8192, e), dtype=torch.uint64, device="cuda")
    F.transcode_bidirectional(par, rows_in, in_bits, nbits, out=rows_out)
    tr_ms, _ = timed(lambda: L.fhe_b200_transcode(par._h, rows_in.data_ptr(), 8, N, N, in_bits, rows_out.data_ptr(),
                                                  8, e, e, nbits, 8192, None), reps * 4)
    tr_bytes = rows_in.numel() * 8 + rows_out.numel() * 8
    row = dict(elements=n_el, element_bytes=es, dim1=dim1, dim2=dim2, plaintexts_per_ct=P, answer_ok=bool(ok),
               stage_ms_per_query=ms, server_ms_per_query=total_ms, responses_per_s=1e3 / total_ms,
               database_encode=dict(seconds=encode_s, database_bytes_per_s=n_el * es / encode_s),
               fold=dict(ms=dev_s * 1e3 / reps, bytes=fold_bytes, bytes_per_s=fold_bytes / (dev_s / reps),
                         share_of_hbm=fold_bytes / (dev_s / reps) / HBM),
               host_route_fold=dict(ms=host_s * 1e3 / reps, plaintexts_equal=equal, speedup=host_s / dev_s,
                                    speedup_vs_stage_ms=host_s * 1e3 / reps / ms["fold"]),
               transcoder=dict(rows=8192, in_len=N, in_bits=in_bits, out_bits=nbits, ms=tr_ms, bytes=tr_bytes,
                               bytes_per_s=tr_bytes / (tr_ms / 1e3), share_of_hbm=tr_bytes / (tr_ms / 1e3) / HBM))
    print(json.dumps(row), flush=True)
    return row


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader",
                               "-i", os.environ.get("CUDA_VISIBLE_DEVICES", "0").split(",")[0]],
                              capture_output=True, text=True, timeout=60).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return ""


if __name__ == "__main__":
    info = gpu_info()
    print(json.dumps({"gpu": info}), flush=True)
    rows = [measure(65536, 1024, reps=10), measure(1 << 20, 256, reps=5)]
    if len(sys.argv) > 1:
        os.makedirs(os.path.dirname(os.path.abspath(sys.argv[1])), exist_ok=True)
        with open(sys.argv[1], "w") as f:
            json.dump({"gpu": info, "rows": rows}, f, indent=1)
