"""GPU tests of the device plaintext encoders (fhe_b200_encode) and of ct x pt / ct +- pt with device plaintexts
(fhe_b200_mul_plain_batch / fhe_b200_add_plain_batch): bit-exact against the encoders restated in
tests/encode_reference.py on the CPU oracle.  Run with `-m gpu`."""
import os
import subprocess
import sys

import numpy as np
import pytest

import encode_reference as R

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
I64_EDGES = np.array([np.iinfo(np.int64).min, -1, np.iinfo(np.int64).max, -786433, 0], np.int64)


@pytest.fixture(scope="module")
def F():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import fhe_rs_b200
    return fhe_rs_b200


def pair(oracle, F, degree, t, sizes, psi_t=None):
    opar = oracle.BfvParameters(degree, t, moduli_sizes=sizes, psi={t: psi_t} if psi_t else None)
    gpar = F.BfvParameters(degree, t, moduli=opar.moduli, device=0, plaintext_psi=psi_t)
    return opar, gpar


def values(rng, n, t, signed, full_range=False):
    if signed:
        v = rng.integers(np.iinfo(np.int64).min, np.iinfo(np.int64).max, size=n, dtype=np.int64, endpoint=True)
        v[:min(n, len(I64_EDGES))] = I64_EDGES[:min(n, len(I64_EDGES))]
        return v
    hi = np.iinfo(np.uint64).max if full_range else t - 1
    return rng.integers(0, hi, size=n, dtype=np.uint64, endpoint=True)


def check_encode(oracle, F, opar, gpar, level, ns, rng, full_range_poly=False):
    n = opar.degree
    for count in ns:
        for simd in (False, True):
            for signed in (False, True):
                full = full_range_poly and not simd and not signed
                v = values(rng, count, opar.plaintext, signed, full)
                enc = F.Encoding.simd_at_level(level) if simd else F.Encoding.poly_at_level(level)
                got = F.PlaintextVec.try_encode(v, enc, gpar)
                assert len(got) == max(1, -(-count // n)) and got.level == level
                exp = R.try_encode(opar, v, simd, level, signed)
                assert (got.poly_ntt() == exp).all(), (count, simd, signed, level)


CONFIGS = {
    # degree 16 (generic NTT kernels), 3 limbs
    "n16": (16, 1153, [62, 62, 62]),
    # set A
    "setA": (1 << 12, 1032193, [62, 62]),
    # 2^14 x 8 limbs (register-resident kernels below 8 plaintexts, TMA kernels from 8 on)
    "n14": (1 << 14, 786433, [62] * 8),
    # set C
    "setC": (1 << 15, 786433, [62] * 14),
    # mixed sizes with t above 4 * q_min: every lift reduces on load
    "mixed": (1 << 13, None, [62, 30, 50]),
}


def config(oracle, name):
    degree, t, sizes = CONFIGS[name]
    if t is None:
        t = oracle.generate_prime(40, 2 * degree, 1 << 40)
    return degree, t, sizes


@pytest.mark.parametrize("name", list(CONFIGS))
def test_encode_parity_matrix(oracle, F, name):
    degree, t, sizes = config(oracle, name)
    opar, gpar = pair(oracle, F, degree, t, sizes)
    rng = np.random.default_rng(degree + len(sizes))
    n = degree
    check_encode(oracle, F, opar, gpar, 0, [0, 1, n - 1, n, n + 1, 3 * n], rng, full_range_poly=True)
    last = len(sizes) - 1
    for level in sorted({1, last}):
        # single-limb level: parity holds for words below q_0, so no full-range Poly words there
        check_encode(oracle, F, opar, gpar, level, [n - 1, n + 1], rng, full_range_poly=level < last)
    if name == "n14":
        check_encode(oracle, F, opar, gpar, 0, [9 * n], rng, full_range_poly=True)   # 9 plaintexts: TMA kernels


def test_encode_custom_psi_t(oracle, F):
    degree, t = 1 << 13, 786433
    psi_t = pow(oracle.default_psi(t, degree), 5, t)
    opar, gpar = pair(oracle, F, degree, t, [62, 62], psi_t)
    v = np.random.default_rng(3).integers(0, t, size=degree, dtype=np.uint64)
    got = F.Plaintext.try_encode(v, F.Encoding.simd(), gpar).poly_ntt()
    assert (got == R.try_encode(opar, v, True)).all()
    _, gdef = pair(oracle, F, degree, t, [62, 62])
    assert not (F.Plaintext.try_encode(v, F.Encoding.simd(), gdef).poly_ntt() == got).all()


def test_encode_input_sources(oracle, F):
    import torch
    degree, t = 1 << 13, 786433
    opar, gpar = pair(oracle, F, degree, t, [62] * 4)
    v = np.random.default_rng(4).integers(-t, t, size=3 * degree + 5, dtype=np.int64)
    ref = F.PlaintextVec.try_encode(v, F.Encoding.simd(), gpar).poly_ntt()
    assert (ref == R.try_encode(opar, v, True, 0, True)).all()
    tv = torch.from_numpy(v)
    for src in (tv, tv.pin_memory(), tv.cuda()):
        assert (F.PlaintextVec.try_encode(src, F.Encoding.simd(), gpar).poly_ntt() == ref).all()
    u = np.random.default_rng(5).integers(0, 1 << 64, size=2 * degree, dtype=np.uint64, endpoint=False)
    ref_u = F.PlaintextVec.try_encode(u, F.Encoding.poly(), gpar).poly_ntt()
    for src in (torch.from_numpy(u).pin_memory(), torch.from_numpy(u).cuda()):
        assert (F.PlaintextVec.try_encode(src, F.Encoding.poly(), gpar).poly_ntt() == ref_u).all()


def test_encode_chunk_boundary():
    """more plaintexts than one chunk (FHE_B200_CHUNK=2, dealt over the side streams) equal one-plaintext calls"""
    env = dict(os.environ, FHE_B200_CHUNK="2")
    out = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "encode_chunk_probe.py")], env=env,
                         capture_output=True, text=True, timeout=600)
    assert out.returncode == 0 and "encode chunk probe ok" in out.stdout, out.stdout + out.stderr


def _ct(opar, rng, count, level=0):
    ctx = opar.context_at_level(level)
    arr = np.zeros((count, 2, len(ctx.moduli), opar.degree), np.uint64)
    for i, q in enumerate(ctx.moduli):
        arr[:, :, i] = rng.integers(0, q, size=(count, 2, opar.degree), dtype=np.uint64)
    return arr


@pytest.mark.parametrize("degree,t,sizes,level", [(64, 1153, [62, 62, 62], 0), (64, 1153, [62, 62, 62], 2),
                                                  (1 << 14, 786433, [62] * 6, 1), (1 << 13, None, [62, 30, 50], 0)])
def test_plain_batch_ops_match_word_forms(oracle, F, degree, t, sizes, level):
    if t is None:
        t = oracle.generate_prime(40, 2 * degree, 1 << 40)
    opar, gpar = pair(oracle, F, degree, t, sizes)
    rng = np.random.default_rng(degree + level)
    cts = 9
    x = _ct(opar, rng, cts, level)
    for n_pt in (1, cts):
        v = rng.integers(0, t, size=n_pt * degree, dtype=np.uint64)
        P = F.PlaintextVec.try_encode(v, F.Encoding.simd_at_level(level), gpar)
        words = P.poly_ntt()
        assert (words == R.try_encode(opar, v, True, level)).all()
        tp = np.stack([R.to_poly(opar, w, level) for w in words])
        arg = words[0] if n_pt == 1 else words
        targ = tp[0] if n_pt == 1 else tp
        a, b = F.Ciphertext.from_host(gpar, x, level), F.Ciphertext.from_host(gpar, x, level)
        assert (a.mul_plain(P).to_host() == b.mul_plain(arg).to_host()).all()
        for sub in (False, True):
            a, b = F.Ciphertext.from_host(gpar, x, level), F.Ciphertext.from_host(gpar, x, level)
            assert (a.add_plain(P, subtract=sub).to_host() == b.add_plain(targ, subtract=sub).to_host()).all()
    # dot_product_scalar over encoded plaintexts equals the uploaded-words call
    P = F.PlaintextVec.try_encode(rng.integers(0, t, size=cts * degree, dtype=np.uint64),
                                  F.Encoding.poly_at_level(level), gpar)
    A = F.Ciphertext.from_host(gpar, x, level)
    assert (F.dot_product_scalar(A, P, 3).to_host() == F.dot_product_scalar(A, P.poly_ntt(), 3).to_host()).all()


@pytest.mark.parametrize("degree,t,sizes", [(1 << 12, 1032193, [62, 62]), (1 << 15, 786433, [62] * 14)])
def test_decrypt_after_plain_ops(oracle, F, degree, t, sizes):
    opar, gpar = pair(oracle, F, degree, t, sizes)
    rng = np.random.default_rng(11)
    sk = oracle.SecretKey(opar, rng)
    m1, m2 = rng.integers(0, t, size=degree, dtype=np.uint64), rng.integers(0, t, size=degree, dtype=np.uint64)
    oct_ = sk.encrypt(oracle.simd_encode(opar, m1), 0, rng)
    P = F.Plaintext.try_encode(m2, F.Encoding.simd(), gpar)
    a1, a2 = m1.astype(object), m2.astype(object)
    cases = {"mul": (lambda c: c.mul_plain(P), a1 * a2 % t), "add": (lambda c: c.add_plain(P), (a1 + a2) % t),
             "sub": (lambda c: c.add_plain(P, subtract=True), (a1 - a2) % t)}
    for name, (op, want) in cases.items():
        ct = op(F.Ciphertext.from_host(gpar, oct_.to_array()[None]))
        dec = sk.decrypt(oracle.Ciphertext.from_array(opar, ct.to_host()[0], 0))
        assert (oracle.simd_decode(opar, dec).astype(object) == want).all(), name


def test_errors(oracle, F):
    from fhe_rs_b200 import _capi
    lib = _capi.lib()
    degree = 1 << 12
    opar, gpar = pair(oracle, F, degree, 1153, [62, 62])   # 1153 has no NTT at N = 2^12
    v = np.arange(degree, dtype=np.uint64)

    def code_of(fn):
        with pytest.raises(F.FheError) as e:
            fn()
        return e.value.code

    assert code_of(lambda: F.Plaintext.try_encode(v, F.Encoding.simd(), gpar)) == _capi.NTT_UNAVAILABLE
    assert (F.Plaintext.try_encode(v, F.Encoding.poly(), gpar).poly_ntt() == R.try_encode(opar, v, False)).all()
    assert code_of(lambda: F.Plaintext.try_encode(v, F.Encoding.poly_at_level(2), gpar)) == _capi.INVALID_LEVEL
    assert code_of(lambda: F.Plaintext.try_encode(np.zeros(degree + 1, np.uint64), F.Encoding.poly(), gpar)) \
        == _capi.INVALID_ARGUMENT
    enc = gpar.encoder()
    two = F.Ciphertext(gpar, 1, 2)
    assert lib.fhe_b200_encode(enc, 0, 0, v.ctypes.data, degree, two._h, None) == _capi.BAD_POLY_COUNT
    wrong = F.Ciphertext(gpar, 2, 1)
    assert lib.fhe_b200_encode(enc, 0, 0, v.ctypes.data, degree, wrong._h, None) == _capi.INVALID_ARGUMENT
    one = F.Ciphertext(gpar, 1, 1)
    assert lib.fhe_b200_encode(enc, 0, 0, None, degree, one._h, None) == _capi.INVALID_ARGUMENT
    assert lib.fhe_b200_encode(enc, 7, 0, v.ctypes.data, degree, one._h, None) == _capi.INVALID_ARGUMENT
    # t beyond a u64 Modulus
    big_t = (1 << 70) + 1
    obig = oracle.BfvParameters(degree, 1153, moduli_sizes=[62, 62])
    gbig = F.BfvParameters(degree, big_t, moduli=obig.moduli, device=0)
    assert code_of(lambda: F.Plaintext.try_encode(v, F.Encoding.poly(), gbig)) == _capi.UNSUPPORTED
    # plaintext batches in ct x pt / ct +- pt
    ct = F.Ciphertext.from_host(gpar, _ct(opar, np.random.default_rng(1), 3))
    P = F.Plaintext.try_encode(v, F.Encoding.poly(), gpar)
    P2 = F.PlaintextVec.try_encode(np.zeros(2 * degree, np.uint64), F.Encoding.poly(), gpar)
    P1 = F.Plaintext.try_encode(v, F.Encoding.poly_at_level(1), gpar)
    for op in (lambda p: ct.mul_plain(p), lambda p: ct.add_plain(p), lambda p: ct.add_plain(p, subtract=True)):
        assert code_of(lambda: op(P2)) == _capi.INVALID_ARGUMENT
        assert code_of(lambda: op(P1)) == _capi.INVALID_LEVEL
        assert code_of(lambda: op(F.PlaintextVec(two, F.Encoding.poly()))) == _capi.BAD_POLY_COUNT
        pb = F.Ciphertext(gpar, 1, 1, repr=F.POWER_BASIS)
        assert code_of(lambda: op(F.PlaintextVec(pb, F.Encoding.poly()))) == _capi.INVALID_REPRESENTATION
        other = F.BfvParameters(degree, 1153, moduli=opar.moduli, device=0)
        assert code_of(lambda: op(F.Plaintext.try_encode(v, F.Encoding.poly(), other))) == _capi.CONTEXT_MISMATCH
    # to_poly needs t < q_0
    omix = oracle.BfvParameters(degree, 1153, moduli_sizes=[30, 62])
    t_big = oracle.generate_prime(40, 2 * degree, 1 << 40)
    gmix = F.BfvParameters(degree, t_big, moduli=omix.moduli, device=0)
    cm = F.Ciphertext(gmix, 1, 2)
    Pm = F.Plaintext.try_encode(np.arange(degree, dtype=np.uint64), F.Encoding.simd(), gmix)
    assert code_of(lambda: cm.add_plain(Pm)) == _capi.UNSUPPORTED
    cm.mul_plain(Pm)


def test_cpp_encode(tmp_path, oracle, F):
    """tests/cpp/encode_test.cpp encodes through include/fhe_b200.hpp and must give the oracle's words"""
    degree, t = 1 << 13, 786433
    opar, _ = pair(oracle, F, degree, t, [62, 62, 62])
    rng = np.random.default_rng(21)
    u = rng.integers(0, t, size=degree, dtype=np.uint64)
    s = rng.integers(-(1 << 40), 1 << 40, size=degree + 3, dtype=np.int64)
    u.tofile(str(tmp_path / "u64.bin"))
    s.tofile(str(tmp_path / "i64.bin"))
    np.array(opar.moduli, np.uint64).tofile(str(tmp_path / "moduli.bin"))
    exe = str(tmp_path / "encode_test")
    lib_dir = os.path.join(ROOT, "fhe_rs_b200")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "cpp", "encode_test.cpp"), "-o", exe,
                           "-L", lib_dir, "-lfhe_b200", "-Wl,-rpath," + lib_dir])
    out = subprocess.run([exe, str(degree), str(t), str(tmp_path)], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0 and out.stdout.startswith("OK"), out.stdout + out.stderr
    simd = np.fromfile(str(tmp_path / "simd.bin"), dtype=np.uint64)
    poly = np.fromfile(str(tmp_path / "poly_l1.bin"), dtype=np.uint64)
    assert (simd == R.try_encode(opar, u, True).ravel()).all()
    assert (poly == R.try_encode(opar, s, False, 1, True).ravel()).all()
