"""The three-product accumulator of the exact scaler (AccKara, fhe_rs_b200/csrc/zq.cuh).

Each term r * w with r, w < 2^62 is split at bit 31 and accumulated as three 96-bit column sums
L = sum r0 w0, M = sum (r0 + r1)(w0 + w1), H = sum r1 w1, combined once as L + 2^31 (M - L - H) + 2^62 H.  The CPU
test checks that identity and the stated bounds on exact integers; the GPU tests run tests/cuda/acc_kara_probe.cu
(built here with the flags of fhe_rs_b200/build.py into a temporary directory) and compare the merged 160-bit words
and the canonical reduction with Python integers."""
import ctypes as C
import os
import random
import subprocess

import numpy as np
import pytest

import edge_inputs as E

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PROBE_SRC = os.path.join(ROOT, "tests", "cuda", "acc_kara_probe.cu")
M64 = (1 << 64) - 1
MASK31 = (1 << 31) - 1
TOP = (1 << 62) - 1                      # the largest operand the split admits
MAX_TERMS = 64 + 1                       # the scaler: n_from <= 64 omega terms and the gamma term (plus one add64)
COUNTS = [1, 14, 29, 64, MAX_TERMS]
MODULI = list(E.BOUNDARY_PRIMES.values()) + [(1 << 62) - 57]


def sol_c(p: int) -> int:
    """the device's Solinas rule (capi.cu): p = 2^62 - c with c < 2^28"""
    return (1 << 62) - p if (p >> 61) == 1 and (1 << 62) - p < (1 << 28) else 0


def split31(x: int):
    lo, hi = x & MASK31, x >> 31
    return lo, hi, lo + hi


def column_sums(terms, add=0):
    """the three sums the device keeps (add64 adds its addend to L and M)"""
    L = M = H = 0
    for r, w in terms:
        r0, r1, rs = split31(r)
        w0, w1, ws = split31(w)
        L += r0 * w0
        M += rs * ws
        H += r1 * w1
    return L + add, M + add, H


def merged(L, M, H):
    return L + ((M - L - H) << 31) + (H << 62)


def test_merge_identity_and_bounds():
    """L + 2^31 (M - L - H) + 2^62 H is the exact sum; every product fits its word, every sum its 96 bits, and the
    value stays below 2^160 at the scaler's largest term count with the extreme operands and addend."""
    rnd = random.Random(7)
    for r, w in [(TOP, TOP), (MASK31, 0), (0, MASK31), (MASK31, TOP), (1 << 31, 1 << 31), (TOP, 1)]:
        r0, r1, rs = split31(r)
        w0, w1, ws = split31(w)
        assert max(r0, r1, w0, w1) < (1 << 31) and max(rs, ws) < (1 << 32)
        assert r0 * w0 < (1 << 62) and r1 * w1 < (1 << 62) and rs * ws < (1 << 64)
    for n in COUNTS:
        for terms, add in [([(TOP, TOP)] * n, M64),
                           ([(rnd.getrandbits(62), rnd.getrandbits(62)) for _ in range(n)], rnd.getrandbits(64))]:
            L, M, H = column_sums(terms, add)
            assert max(L, M, H) < (1 << 96)
            assert M - L - H >= 0
            v = merged(L, M, H)
            assert v == sum(r * w for r, w in terms) + add
            assert v < (1 << 160)
    # the 96-bit sums hold 2^32 - 1 maximal terms and addends together
    n = (1 << 32) - 1
    assert n * TOP * TOP < (1 << 160) and n * (2 * MASK31) ** 2 < (1 << 96)


def build_probe(out_dir: str) -> str:
    from fhe_rs_b200 import build as b
    so = os.path.join(out_dir, "libacc_kara_probe.so")
    cmd = [b._nvcc(), *b.NVCC_FLAGS, "-shared", "-cudart", "static", PROBE_SRC, "-o", so]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, "nvcc failed:\n%s\n%s" % (r.stdout, r.stderr)
    return so


def test_probe_compiles_for_sm90a(tmp_path):
    """The probe builds against the current zq.cuh for sm_90a (no GPU needed)."""
    assert os.path.getsize(build_probe(str(tmp_path))) > 0


@pytest.fixture(scope="module")
def probe(tmp_path_factory):
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    lib = C.CDLL(build_probe(str(tmp_path_factory.mktemp("acc_kara_probe"))))
    lib.acc_kara_probe_run.restype = C.c_int
    lib.acc_kara_probe_run.argtypes = [C.c_void_p] * 5 + [C.c_uint32, C.c_void_p]
    return lib


def run(lib, p, cases):
    """cases: (terms, addend) pairs -> per case (merged value, canonical residue)"""
    B = (1 << 128) // p
    limb = np.array([p, 2 * p, B >> 64, B & M64, (1 << 128) % p, sol_c(p)], np.uint64)
    r = np.array([t[0] for terms, _ in cases for t in terms], np.uint64)
    w = np.array([t[1] for terms, _ in cases for t in terms], np.uint64)
    off = np.cumsum([0] + [len(terms) for terms, _ in cases]).astype(np.uint32)
    add = np.array([a for _, a in cases], np.uint64)
    out = np.zeros((len(cases), 4), np.uint64)
    code = lib.acc_kara_probe_run(limb.ctypes.data, r.ctypes.data, w.ctypes.data, off.ctypes.data, add.ctypes.data,
                                  len(cases), out.ctypes.data)
    assert code == 0, "CUDA error %d" % code
    return [(int(o[0]) | (int(o[1]) << 64) | (int(o[2]) << 128), int(o[3])) for o in out]


@pytest.mark.gpu
@pytest.mark.parametrize("p", MODULI, ids=hex)
def test_acc_kara_exact(probe, p):
    """merged() equals the exact sum word for word and reduce() is canonical: all operands 2^62 - 1 or q - 1,
    all-zero halves, one half at 2^31 - 1 and the other zero, random operands below 2^62 and below q, term counts
    up to the scaler's maximum, and add64 of 0 and 2^64 - 1"""
    rnd = random.Random(p)
    edge = [(TOP, TOP), (p - 1, p - 1), (TOP, p - 1), (0, TOP), (0, 0), (MASK31, MASK31), (MASK31 << 31, MASK31),
            (MASK31, MASK31 << 31), (MASK31 << 31, MASK31 << 31), (1 << 31, (1 << 31) - 1)]
    cases = []
    for n in COUNTS:
        for t in edge:
            for add in (0, M64):
                cases.append(([t] * n, add))
        cases.append(([(rnd.getrandbits(62), rnd.getrandbits(62)) for _ in range(n)], rnd.getrandbits(64)))
        cases.append(([(rnd.randrange(p), rnd.randrange(p)) for _ in range(n)], M64))
        cases.append(([rnd.choice(edge) for _ in range(n)], rnd.choice((0, M64))))
    cases.append(([], M64))
    for (terms, add), (v, res) in zip(cases, run(probe, p, cases)):
        exp = sum(r * w for r, w in terms) + add
        assert v == exp, (len(terms), hex(terms[0][0]) if terms else None, hex(add))
        assert res == exp % p, (len(terms), hex(add))
