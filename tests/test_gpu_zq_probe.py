"""Device probe of the modular-arithmetic primitives of fhe_rs_b200/csrc/zq.cuh at the edges of their stated domains.

tests/cuda/zq_probe.cu wraps each primitive in one element-wise kernel.  It is built here with the flags of
fhe_rs_b200/build.py into a library under a temporary directory (it is never part of libfhe_b200.so), and every result
word is compared with Python integers: lazy results must lie in their stated range and be congruent, canonical results
must be exact.  The CPU part only compiles the probe, so a probe that no longer builds against zq.cuh fails without a
GPU."""
import ctypes as C
import os
import random
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PROBE_SRC = os.path.join(ROOT, "tests", "cuda", "zq_probe.cu")
M64 = (1 << 64) - 1

(MUL_SHOUP_LAZY, MUL_SHOUP, MUL_SOLINAS_LAZY, MUL_SOLINAS_LAZY_V1, FOLD63_SOLINAS, ADDBACK2P, SHOUP_OF,
 BARRETT128_LAZY, BARRETT128, BARRETT64, MULMOD, MUL128_62, FOLD192_SOLINAS, ACC192, ACC_THETA, MULMOD_LIMB_LAZY,
 MULMOD_LIMB, REDUCE128_LIMB, REDUCE94_LIMB) = range(19)

# the three boundary primes of tests/edge_inputs.py, a small-c Solinas prime, a 36-bit prime, a 17-bit plaintext
# modulus, and 2^62 - 1 (no contract below needs a prime)
MODULI = [0x3ffffffff00a0001, 0x3fffffffeff50001, 0x20000000000b0001, (1 << 62) - 57, 0xffffee001, 65537,
          (1 << 62) - 1]


def build_probe(out_dir: str) -> str:
    from fhe_rs_b200 import build as b
    so = os.path.join(out_dir, "libzq_probe.so")
    cmd = [b._nvcc(), *b.NVCC_FLAGS, "-shared", "-cudart", "static", PROBE_SRC, "-o", so]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, "nvcc failed:\n%s\n%s" % (r.stdout, r.stderr)
    return so


def test_probe_compiles_for_sm90a(tmp_path):
    """The probe builds against the current zq.cuh for sm_90a (no GPU needed)."""
    so = build_probe(str(tmp_path))
    assert os.path.getsize(so) > 0


def sol_c(p: int) -> int:
    """the device's Solinas rule (capi.cu): p = 2^62 - c with c < 2^28"""
    return (1 << 62) - p if (p >> 61) == 1 and (1 << 62) - p < (1 << 28) else 0


class Probe:
    def __init__(self, so: str):
        self.lib = C.CDLL(so)
        self.lib.zq_probe_run.restype = C.c_int
        self.lib.zq_probe_run.argtypes = [C.c_int] + [C.c_void_p] * 5 + [C.c_uint64, C.c_void_p]

    def run(self, op, p, a, b=None, c=None, d=None):
        """per element: the 8 result words as Python ints"""
        n = len(a)
        B = (1 << 128) // p
        limb = np.array([p, 2 * p, B >> 64, B & M64, (1 << 128) % p, sol_c(p)], np.uint64)
        arr = [np.array([int(v) & M64 for v in (x if x is not None else [0] * n)], np.uint64) for x in (a, b, c, d)]
        out = np.zeros((n, 8), np.uint64)
        code = self.lib.zq_probe_run(op, limb.ctypes.data, *[x.ctypes.data for x in arr], n, out.ctypes.data)
        assert code == 0, "CUDA error %d" % code
        return [[int(v) for v in row] for row in out]


@pytest.fixture(scope="module")
def probe(tmp_path_factory):
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    return Probe(build_probe(str(tmp_path_factory.mktemp("zq_probe"))))


def operands64(p, rnd):
    """64-bit operands at the edges of the lazy domains"""
    v = [0, 1, 2, p - 1, p, p + 1, 2 * p - 1, 2 * p, 4 * p - 1, (1 << 62) - 1, (1 << 63) - 1, 1 << 63, M64 - 1, M64]
    return [x for x in v if x <= M64] + [rnd.getrandbits(64) for _ in range(8)]


def residues(p, rnd):
    return [0, 1, 2, (p - 1) // 2, (p + 1) // 2, p - 2, p - 1] + [rnd.randrange(p) for _ in range(6)]


@pytest.mark.gpu
@pytest.mark.parametrize("p", MODULI, ids=hex)
def test_shoup_products(probe, p):
    """mul_shoup_lazy: [0, 2p) and congruent for ANY 64-bit operand; mul_shoup canonical; shoup_of == floor(a 2^64 / p)"""
    rnd = random.Random(p)
    pairs = [(a, w) for a in operands64(p, rnd) for w in residues(p, rnd)]
    a, w = [x for x, _ in pairs], [y for _, y in pairs]
    ws = [(y << 64) // p for y in w]
    lazy = probe.run(MUL_SHOUP_LAZY, p, a, w, ws)
    canon = probe.run(MUL_SHOUP, p, a, w, ws)
    for x, y, r, s in zip(a, w, lazy, canon):
        assert r[0] < 2 * p and r[0] % p == x * y % p, (hex(x), hex(y), hex(r[0]))
        assert s[0] == x * y % p
    res = residues(p, rnd)
    for x, r in zip(res, probe.run(SHOUP_OF, p, res)):
        assert r[0] == (x << 64) // p, hex(x)


@pytest.mark.gpu
@pytest.mark.parametrize("p", [q for q in MODULI if sol_c(q)], ids=hex)
def test_solinas_products_and_folds(probe, p):
    """mul_solinas_lazy and its _v1 form: [0, 2p) and congruent for any 64-bit y (w1 = w 2^32 mod p); fold63_solinas
    subtracts 2p exactly when bit 63 is set; fold192_solinas takes hi up to 2^32 - 1"""
    rnd = random.Random(p)
    c = sol_c(p)
    pairs = [(y, w) for y in operands64(p, rnd) for w in residues(p, rnd)]
    y, w0 = [a for a, _ in pairs], [b for _, b in pairs]
    w1 = [(b << 32) % p for b in w0]
    r0 = probe.run(MUL_SOLINAS_LAZY, p, y, w0, w1)
    r1 = probe.run(MUL_SOLINAS_LAZY_V1, p, y, w0, w1)
    for a, b, u, v in zip(y, w0, r0, r1):
        assert u[0] < 2 * p and u[0] % p == a * b % p, (hex(a), hex(b), hex(u[0]))
        assert v[0] == u[0]
    xs = operands64(p, rnd)
    for x, r in zip(xs, probe.run(FOLD63_SOLINAS, p, xs)):
        assert r[0] == (x - 2 * p if x >> 63 else x) and r[0] < (1 << 63) + 2 * c
    his = [0, 1, (1 << 16) - 1, 1 << 16, 1 << 31, (1 << 32) - 1]
    los = [0, M64, rnd.getrandbits(64)]
    cases = [(lo, mid, hi) for hi in his for mid in los for lo in los]
    out = probe.run(FOLD192_SOLINAS, p, *zip(*cases))
    for (lo, mid, hi), r in zip(cases, out):
        v = (hi << 128) | (mid << 64) | lo
        assert r[0] < 2 * p and r[0] % p == v % p, (hex(hi), hex(mid), hex(lo), hex(r[0]))


@pytest.mark.gpu
@pytest.mark.parametrize("p", MODULI, ids=hex)
def test_barrett_and_wide_products(probe, p):
    """barrett128_lazy [0, 2p) for any 128-bit value, barrett128 / barrett64 / mulmod canonical at their maximum
    inputs, mul128_62 exact, addback2p on t in {-2p+1, -1, 0, 2p-1}, reduce128_limb / reduce94_limb canonical"""
    rnd = random.Random(p)
    vals = [0, 1, p - 1, p, (p - 1) ** 2, (4 * p - 1) * (p - 1), (M64 * M64), (1 << 128) - 1, (1 << 127),
            ((1 << 128) // p) * p - 1] + [rnd.getrandbits(128) for _ in range(8)]
    vals = [v for v in vals if v < (1 << 128)]
    lo, hi = [v & M64 for v in vals], [v >> 64 for v in vals]
    for v, r, s, t in zip(vals, probe.run(BARRETT128_LAZY, p, lo, hi), probe.run(BARRETT128, p, lo, hi),
                          probe.run(REDUCE128_LIMB, p, lo, hi)):
        assert r[0] < 2 * p and r[0] % p == v % p, hex(v)
        assert s[0] == v % p and t[0] == v % p
    v94 = [v for v in vals if v < (1 << 94)] + [(1 << 94) - 1, (1 << 70) - 1]
    for v, r in zip(v94, probe.run(REDUCE94_LIMB, p, [v & M64 for v in v94], [v >> 64 for v in v94])):
        assert r[0] == v % p, hex(v)
    xs = operands64(p, rnd)
    for x, r in zip(xs, probe.run(BARRETT64, p, xs)):
        assert r[0] == x % p
    ops = residues(p, rnd) + [M64]
    pairs = [(a, b) for a in ops for b in ops]
    for (a, b), r in zip(pairs, probe.run(MULMOD, p, *zip(*pairs))):
        assert r[0] == a * b % p, (hex(a), hex(b))
    ops62 = [0, 1, (1 << 62) - 1, p - 1 if p < (1 << 62) else 1, rnd.getrandbits(62)]
    pairs = [(a, b) for a in ops62 for b in ops62]
    for (a, b), r in zip(pairs, probe.run(MUL128_62, p, *zip(*pairs))):
        assert r[0] | (r[1] << 64) == a * b
    ts = [-2 * p + 1, -1, 0, 2 * p - 1]
    for t, r in zip(ts, probe.run(ADDBACK2P, p, [t & M64 for t in ts])):
        assert r[0] == (t + 2 * p if t < 0 else t)
    # mulmod_limb[_lazy]: the limb's own mode (Solinas fold or Barrett) on canonical operands
    res = residues(p, rnd)
    pairs = [(a, b) for a in res for b in res]
    for (a, b), r, s in zip(pairs, probe.run(MULMOD_LIMB_LAZY, p, *zip(*pairs)), probe.run(MULMOD_LIMB, p, *zip(*pairs))):
        assert r[0] < 2 * p and r[0] % p == a * b % p and s[0] == a * b % p


@pytest.mark.gpu
@pytest.mark.parametrize("p", MODULI, ids=hex)
def test_lazy_accumulators(probe, p):
    """Acc192: n terms of (4p - 1)(p - 1) (the key-switch digit bound times a canonical key word) and of
    (2^64 - 1)^2, n up to 2^20, plus one add64 of 2^64 - 1: exact merged words, reduce canonical, reduce_lazy in
    [0, 2p).  AccTheta equals repeated mac_theta and the exact sum (mod 2^224) at the largest operands."""
    counts = [1, 2, 63, 64, 1 << 20]
    cases = [(x, y, z, k) for x, y in ((4 * p - 1, p - 1), (M64, M64)) for z in (0, M64) for k in counts
             if x <= M64]
    out = probe.run(ACC192, p, *zip(*cases))
    for (x, y, z, k), r in zip(cases, out):
        v = k * x * y + z
        assert v < (1 << 160)
        assert r[0] | (r[1] << 64) | (r[2] << 128) == v, (hex(x), k)
        assert r[3] == v % p, (hex(x), k)
        assert r[4] < 2 * p and r[4] % p == v % p, (hex(x), k)
    rnd = random.Random(p)
    cases = [(r, t & M64, t >> 64, k) for r in (M64, rnd.getrandbits(64)) for t in ((1 << 128) - 1, rnd.getrandbits(128))
             for k in (1, 64, 1 << 20)]
    out = probe.run(ACC_THETA, p, *zip(*cases))

    def value(words):
        return words[0] | (words[1] << 64) | (words[2] << 128) | ((words[3] & 0xffffffff) << 192)
    for (r, tlo, thi, k), o in zip(cases, out):
        exp = (k * r * ((thi << 64) | tlo)) % (1 << 224)
        assert value(o[:4]) == exp and value(o[4:]) == exp, (hex(r), k)
