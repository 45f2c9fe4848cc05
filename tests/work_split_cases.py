"""Shared by tests/test_gpu_work_split.py and tests/work_split_probe.py: the batch shapes and counts that cut the
persistent kernels' work split, their inputs (a pure function of shape, count and ciphertext index, so an oracle
worker can rebuild any one ciphertext without receiving it), the device side of every operation on the whole batch,
and the oracle side of one ciphertext.  Outputs are compared as a SHA-256 digest of every word of each output
ciphertext.  Importing this module touches neither CUDA nor the oracle's library."""
import hashlib

import numpy as np

T = 786433
SHAPES = {
    # 2 x 62-bit, K = 5, n_dig = 2: every count from 1 to 14 crosses items < grid, grid + 1 and the tensor fusion's
    # 3-ciphertext threshold for each kernel (14: the first count above one wave of the 6-CTA-per-SM cols kernel on
    # 132 SMs); 17 / 31 / 64 / 67 cut runs inside the CTA ranges of larger grids
    "n13_2x62": dict(logn=13, sizes=[62, 62], t=T, counts=list(range(1, 15)) + [17, 31, 64, 67]),
    # the reduce-on-load cols kernel, the per-tile scaler for the non-Solinas limbs, and n_dig = 3 (odd)
    "n13_62_40_30": dict(logn=13, sizes=[62, 40, 30], t=65537, counts=[1, 2, 3, 7, 33]),
    "n14_8x62": dict(logn=14, sizes=[62] * 8, t=T, counts=[1, 3, 5, 33]),
    # 259 = chunks of 128, 128 and 3 under the default chunk of 256 over 2 streams
    "n15_14x62": dict(logn=15, sizes=[62] * 14, t=T, counts=[1, 3, 259]),
}
FULL_OPS = ("fwd1", "fwd2", "fwd3", "bwd1", "bwd2", "bwd3", "mul", "mul_ms", "tensor", "relin", "rot3", "rot_row",
            "ks", "l1_mul", "l1_rot", "decrypt")


def ops_for(name, count):
    if name != "n15_14x62":
        return FULL_OPS
    # set C: the product and the rotation over the three-chunk batch; everything else on small batches
    if count > 3:
        return ("mul", "rot3")
    return ("fwd1", "fwd2", "fwd3", "bwd1", "bwd2", "bwd3", "mul", "rot3", "ks", "decrypt")


def digest(words):
    return hashlib.sha256(np.ascontiguousarray(words, dtype=np.uint64).tobytes()).hexdigest()[:32]


def _shape_id(name):
    return list(SHAPES).index(name)


def moduli_of(name):
    """the moduli the oracle's builder generates for the shape (the device takes the same list)"""
    import fhe_oracle as O
    s = SHAPES[name]
    return O.BfvParameters(1 << s["logn"], s["t"], moduli_sizes=s["sizes"]).moduli


def _rows(rng, moduli, prefix, n):
    a = np.zeros(tuple(prefix) + (len(moduli), n), np.uint64)
    for i, q in enumerate(moduli):
        a[..., i, :] = rng.integers(0, q, size=tuple(prefix) + (n,), dtype=np.uint64)
    return a


def ct_words(name, moduli, tag, count, i, level=0):
    """ciphertext i of operand `tag` ('a', 'b') of the count-`count` batch: [2][L_level][N] uniform residues"""
    rng = np.random.default_rng([_shape_id(name), ord(tag), level, count, i])
    return _rows(rng, moduli[:len(moduli) - level], (2,), 1 << SHAPES[name]["logn"])


def batch_words(name, moduli, tag, count, level=0):
    return np.stack([ct_words(name, moduli, tag, count, i, level) for i in range(count)])


def ntt_input(a_i, b_i, parts):
    """the P-part polynomials of the NTT batches: parts of a, then of b"""
    return np.concatenate([a_i, b_i], axis=0)[:parts]


KEYS = {"rk": 0, "g3": 0, "grow": 0, "rk1": 1, "g1": 1}   # the ciphertext level each key serves


def key_arrays(name, moduli, which):
    """random key material (c0, c1) [n_dig][key limbs][N] at key level 0; bit-exactness needs no real keys"""
    ct_level = KEYS[which]
    rng = np.random.default_rng([_shape_id(name), 1000 + list(KEYS).index(which)])
    return _rows(rng, moduli, (2, len(moduli) - ct_level), 1 << SHAPES[name]["logn"])


def exponent(name, which):
    return 2 * (1 << SHAPES[name]["logn"]) - 1 if which == "grow" else 3


def secret_coeffs(name):
    rng = np.random.default_rng([_shape_id(name), 77])
    return rng.integers(-1, 2, size=1 << SHAPES[name]["logn"]).astype(np.int64)


def needed_keys(name):
    ops = set(o for c in SHAPES[name]["counts"] for o in ops_for(name, c))
    need = {"rk"} if ops & {"mul", "mul_ms", "relin", "ks"} else set()
    need |= {"g3"} if "rot3" in ops else set()
    need |= {"grow"} if "rot_row" in ops else set()
    need |= {"rk1"} if "l1_mul" in ops else set()
    need |= {"g1"} if "l1_rot" in ops else set()
    return sorted(need)


# ---------------------------------------------------------------------------------------------------- device side
def device_batch_digests(ct, block=16):
    """digest of every ciphertext of a device batch, downloaded a few at a time"""
    out = []
    shape = ct.shape()
    for first in range(0, shape[0], block):
        n = min(block, shape[0] - first)
        w = ct.to_host(np.empty((n,) + tuple(shape[1:]), np.uint64), first=first)
        out += [digest(w[k]) for k in range(n)]
    return out


def device_digests(F, name, counts=None):
    """{"op@count": [digest of output ciphertext i]} for every operation of the shape on whole batches"""
    s = SHAPES[name]
    moduli = moduli_of(name)
    gpar = F.BfvParameters(1 << s["logn"], s["t"], moduli=moduli, device=0)
    keys = {}
    for k in needed_keys(name):
        c = key_arrays(name, moduli, k)
        lvl = KEYS[k]
        if k.startswith("rk"):
            keys[k] = F.RelinearizationKey.from_arrays(gpar, c[0], c[1], ciphertext_level=lvl, key_level=0)
        else:
            keys[k] = F.GaloisKey.from_arrays(gpar, exponent(name, k), c[0], c[1], ciphertext_level=lvl, key_level=0)
    gsk = F.SecretKey(gpar, secret_coeffs(name))
    res = {}
    for count in counts or s["counts"]:
        ops = ops_for(name, count)
        a, b = batch_words(name, moduli, "a", count), batch_words(name, moduli, "b", count)
        A, B = F.Ciphertext.from_host(gpar, a), F.Ciphertext.from_host(gpar, b)

        def put(op, ct):
            res["%s@%d" % (op, count)] = device_batch_digests(ct)
        for p in (1, 2, 3):
            x = np.concatenate([a, b], axis=1)[:, :p]
            if "fwd%d" % p in ops:
                put("fwd%d" % p, F.Ciphertext.from_host(gpar, x, repr=F.POWER_BASIS).into_ntt())
            if "bwd%d" % p in ops:
                put("bwd%d" % p, F.Ciphertext.from_host(gpar, x, repr=F.NTT).into_power_basis())
        del a, b
        P = None
        if "mul" in ops:
            P = F.Multiplicator.default(keys["rk"]).multiply(A, B)
            put("mul", P)
        if "mul_ms" in ops:
            m = F.Multiplicator.default(keys["rk"])
            m.enable_mod_switching()
            put("mul_ms", m.multiply(A, B))
        if "tensor" in ops or "relin" in ops:
            C3 = A * B
            if "tensor" in ops:
                put("tensor", C3)
            if "relin" in ops:
                put("relin", keys["rk"].relinearizes(C3))
            del C3
        if "rot3" in ops:
            put("rot3", keys["g3"].relinearize(A))
        if "rot_row" in ops:
            put("rot_row", keys["grow"].relinearize(A))
        if "ks" in ops:
            put("ks", keys["rk"].ksk.key_switch(A.clone().into_power_basis(), part=1))
        if "l1_mul" in ops or "l1_rot" in ops:
            LA = F.Ciphertext.from_host(gpar, batch_words(name, moduli, "a", count, 1), level=1)
            LB = F.Ciphertext.from_host(gpar, batch_words(name, moduli, "b", count, 1), level=1)
            if "l1_mul" in ops:
                put("l1_mul", F.Multiplicator.default(keys["rk1"]).multiply(LA, LB))
            if "l1_rot" in ops:
                put("l1_rot", keys["g1"].relinearize(LA))
        if "decrypt" in ops:
            # the TMA scaler's one-output-row launch (polys == cts) on the products
            put("decrypt", gsk.try_decrypt(P).batch)
        del A, B, P
    return res


# ---------------------------------------------------------------------------------------------------- oracle side
_W = {}


def oracle_init(name):
    """pool initializer: the oracle's parameters, keys and multiplicators of one shape, built once per worker"""
    import fhe_oracle as O
    s = SHAPES[name]
    opar = O.BfvParameters(1 << s["logn"], s["t"], moduli_sizes=s["sizes"])
    moduli = opar.moduli
    st = dict(O=O, opar=opar, moduli=moduli, name=name)
    for k in needed_keys(name):
        c = key_arrays(name, moduli, k)
        ksk = O.KeySwitchingKey.from_arrays(opar, c[0], c[1], KEYS[k], 0)
        if k.startswith("rk"):
            st[k] = O.RelinearizationKey.from_ksk(ksk)
        else:
            g = O.GaloisKey.__new__(O.GaloisKey)
            g.exponent, g.ksk = exponent(name, k), ksk
            st[k] = g
    sk = O.SecretKey.__new__(O.SecretKey)
    sk.par, sk.coeffs = opar, secret_coeffs(name)
    st["sk"] = sk
    _W.clear()
    _W.update(st)


def oracle_digests(count, i):
    """{op: digest} of ciphertext i of the count-`count` batch, every operation of ops_for"""
    W = _W
    O, opar, moduli, name = W["O"], W["opar"], W["moduli"], W["name"]
    ops = ops_for(name, count)
    a_i, b_i = ct_words(name, moduli, "a", count, i), ct_words(name, moduli, "b", count, i)
    ctx = opar.context_at_level(0)
    out = {}
    for p in (1, 2, 3):
        for d in ("fwd", "bwd"):
            if "%s%d" % (d, p) in ops:
                x = ntt_input(a_i, b_i, p).copy()
                for r in range(p):
                    for j, op in enumerate(ctx.ops):
                        (op.forward if d == "fwd" else op.backward)(x[r, j])
                out["%s%d" % (d, p)] = digest(x)
    A, B = O.Ciphertext.from_array(opar, a_i, 0), O.Ciphertext.from_array(opar, b_i, 0)
    if "mul" in ops:
        prod = O.Multiplicator.default(W["rk"]).multiply(A, B)
        out["mul"] = digest(prod.to_array())
        if "relin" in ops:
            out["relin"] = out["mul"]   # relinearizes(ct * ct) is Multiplicator::default's product
        if "decrypt" in ops:
            out["decrypt"] = digest(O.Poly.from_u64(ctx, W["sk"].decrypt(prod), O.NTT).c)
    if "mul_ms" in ops:
        m = O.Multiplicator.default(W["rk"])
        m.enable_mod_switching()
        out["mul_ms"] = digest(m.multiply(A, B).to_array())
    if "tensor" in ops:
        out["tensor"] = digest(A.mul(B).to_array())
    if "rot3" in ops:
        out["rot3"] = digest(W["g3"].relinearize(A).to_array())
    if "rot_row" in ops:
        out["rot_row"] = digest(W["grow"].relinearize(A).to_array())
    if "ks" in ops:
        c0, c1 = W["rk"].ksk.key_switch(A.c[1].copy().into_power_basis())
        out["ks"] = digest(np.stack([c0.c, c1.c]))
    if "l1_mul" in ops or "l1_rot" in ops:
        LA = O.Ciphertext.from_array(opar, ct_words(name, moduli, "a", count, i, 1), 1)
        LB = O.Ciphertext.from_array(opar, ct_words(name, moduli, "b", count, i, 1), 1)
        if "l1_mul" in ops:
            out["l1_mul"] = digest(O.Multiplicator.default(W["rk1"]).multiply(LA, LB).to_array())
        if "l1_rot" in ops:
            out["l1_rot"] = digest(W["g1"].relinearize(LA).to_array())
    return count, i, out


def oracle_expected(name, workers):
    """{"op@count": [digest of ciphertext i]} from the oracle, spread over a pool of `spawn` workers"""
    import multiprocessing as mp
    from concurrent.futures import ProcessPoolExecutor
    counts = SHAPES[name]["counts"]
    res = {}
    with ProcessPoolExecutor(max_workers=workers, mp_context=mp.get_context("spawn"), initializer=oracle_init,
                             initargs=(name,)) as pool:
        futs = [pool.submit(oracle_digests, c, i) for c in counts for i in range(c)]
        for f in futs:
            c, i, d = f.result()
            for op, h in d.items():
                res.setdefault("%s@%d" % (op, c), [None] * c)[i] = h
    return res


def compare(got, exp):
    """the (op@count, ciphertext) pairs whose words differ, and the operations the device did not run"""
    bad = []
    for key, want in exp.items():
        have = got.get(key)
        if have is None or len(have) != len(want):
            bad.append((key, "missing"))
            continue
        bad += [(key, i) for i, (h, w) in enumerate(zip(have, want)) if h != w]
    return bad
