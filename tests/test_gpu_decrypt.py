"""GPU tests of decryption, decoding and noise measurement on the device (fhe_b200_decrypt, fhe_b200_decode,
fhe_b200_measure_noise): bit-exact against the oracle's SecretKey.decrypt / measure_noise and simd_decode, with the
oracle's key coefficients given to the device key.  Run with `-m gpu`."""
import os
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
I64 = np.iinfo(np.int64)


@pytest.fixture(scope="module")
def F():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import fhe_rs_b200
    return fhe_rs_b200


CONFIGS = {
    "n16": (16, 1153, [62, 62, 62]),                 # degree 16, 3 limbs
    "setA": (1 << 12, 1032193, [62, 62]),
    "n14": (1 << 14, 786433, [62] * 8),
    "setC": (1 << 15, 786433, [62] * 14),
    "mixed": (1 << 13, None, [62, 30, 50]),         # 40-bit t: the plaintext context is wider than the last levels
}


def setup(oracle, F, name, seed=0):
    degree, t, sizes = CONFIGS[name]
    if t is None:
        t = oracle.generate_prime(40, 2 * degree, 1 << 40)
    opar = oracle.BfvParameters(degree, t, moduli_sizes=sizes)
    gpar = F.BfvParameters(degree, t, moduli=opar.moduli, device=0)
    rng = np.random.default_rng(degree + len(sizes) + seed)
    osk = oracle.SecretKey(opar, rng)
    return opar, gpar, rng, osk, F.SecretKey(gpar, osk.coeffs)


def has_simd(oracle, opar):
    t, m = opar.plaintext, 2 * opar.degree
    return t % m == 1 and oracle.is_prime(t)


def fresh(oracle, opar, osk, rng, count, level):
    return np.stack([osk.encrypt(rng.integers(0, opar.plaintext, size=opar.degree), level, rng).to_array()
                     for _ in range(count)])


def check_parity(oracle, F, opar, gpar, osk, gsk, words, level, noise=True):
    """device decrypt / decode / measure_noise of the ciphertexts `words` against the oracle, entry by entry"""
    n = opar.degree
    ct = F.Ciphertext.from_host(gpar, words, level)
    pts = gsk.try_decrypt(ct)
    assert pts.encoding is None and len(pts) == len(words) and pts.level == level
    got = pts.poly_ntt()
    ctx = opar.context_at_level(level)
    poly = pts.try_decode(F.Encoding.poly_at_level(level))
    simd = pts.try_decode(F.Encoding.simd_at_level(level)) if has_simd(oracle, opar) else None
    got_noise = gsk.measure_noise(ct) if noise else None
    for k in range(len(words)):
        oc = oracle.Ciphertext.from_array(opar, words[k], level)
        w = osk.decrypt(oc)
        assert (got[k] == oracle.Poly.from_u64(ctx, w, oracle.NTT).c).all(), (level, k)
        assert (poly[k * n:(k + 1) * n] == w).all(), (level, k)
        if simd is not None:
            assert (simd[k * n:(k + 1) * n] == oracle.simd_decode(opar, w)).all(), (level, k)
        if noise:
            assert int(got_noise[k]) == osk.measure_noise(oc), (level, k)
    return got


def _keys(oracle, F, opar, gpar, osk, rng, level=0):
    ork = oracle.RelinearizationKey(osk, rng, level, level)
    grk = F.RelinearizationKey.from_arrays(gpar, *ork.ksk.arrays(), ciphertext_level=level, key_level=level)
    e = oracle.rotation_exponent(opar, 1)
    ogk = oracle.GaloisKey(osk, e, rng, level, level)
    ggk = F.GaloisKey.from_arrays(gpar, e, *ogk.ksk.arrays(), ciphertext_level=level, key_level=level)
    return grk, ggk


@pytest.mark.parametrize("name", list(CONFIGS))
def test_decrypt_parity(oracle, F, name):
    opar, gpar, rng, osk, gsk = setup(oracle, F, name)
    big = opar.degree >= 1 << 14
    count = 2 if big else 3
    last = len(opar.moduli) - 1
    # fresh ciphertexts at every level (the first, the second and the last at the large sets)
    levels = sorted({0, 1, last}) if big else range(last + 1)
    for level in levels:
        check_parity(oracle, F, opar, gpar, osk, gsk, fresh(oracle, opar, osk, rng, count, level), level)
    grk, ggk = _keys(oracle, F, opar, gpar, osk, rng)
    A = F.Ciphertext.from_host(gpar, fresh(oracle, opar, osk, rng, count, 0))
    B = F.Ciphertext.from_host(gpar, fresh(oracle, opar, osk, rng, count, 0))
    # after mul_relin, after a column rotation
    prod = F.Multiplicator.default(grk).multiply(A, B)
    check_parity(oracle, F, opar, gpar, osk, gsk, prod.to_host(), 0)
    check_parity(oracle, F, opar, gpar, osk, gsk, ggk.relinearize(A).to_host(), 0)
    # 3-part products and a 3 x 2 -> 4-part product
    C3 = A * B
    check_parity(oracle, F, opar, gpar, osk, gsk, C3.to_host(), 0)
    C4 = C3 * A
    assert len(C4) == 4
    check_parity(oracle, F, opar, gpar, osk, gsk, C4.to_host(), 0, noise=not big)
    # switched down to the last level (L = 1)
    low = prod.clone()
    low.switch_to_level(last)
    check_parity(oracle, F, opar, gpar, osk, gsk, low.to_host(), last)


def test_decrypt_with_t_above_q0(oracle, F):
    """t >= q_0: decryption stays bit-exact, decoding and measure_noise are UNSUPPORTED"""
    from fhe_rs_b200 import _capi
    degree = 1 << 12
    t = oracle.generate_prime(40, 2 * degree, 1 << 40)
    opar = oracle.BfvParameters(degree, t, moduli_sizes=[30, 62])
    gpar = F.BfvParameters(degree, t, moduli=opar.moduli, device=0)
    rng = np.random.default_rng(5)
    osk = oracle.SecretKey(opar, rng)
    gsk = F.SecretKey(gpar, osk.coeffs)
    for level in (0, 1):
        words = fresh(oracle, opar, osk, rng, 3, level)
        ct = F.Ciphertext.from_host(gpar, words, level)
        pts = gsk.try_decrypt(ct)
        got = pts.poly_ntt()
        ctx = opar.context_at_level(level)
        for k in range(3):
            w = osk.decrypt(oracle.Ciphertext.from_array(opar, words[k], level))
            assert (got[k] == oracle.Poly.from_u64(ctx, w, oracle.NTT).c).all()
        for fn in (lambda: pts.try_decode(F.Encoding.poly_at_level(level)), lambda: gsk.measure_noise(ct)):
            with pytest.raises(F.FheError) as e:
                fn()
            assert e.value.code == _capi.UNSUPPORTED


def _centre(v, t):
    r = np.array([int(x) % t for x in v], dtype=object)
    return np.array([x - t if x >= t >> 1 else x for x in r], dtype=np.int64)


@pytest.mark.parametrize("name", ["n16", "setA", "setC", "mixed"])
def test_decode_round_trip(oracle, F, name):
    import torch
    opar, gpar, rng, _, _ = setup(oracle, F, name)
    n, t = opar.degree, opar.plaintext
    simd_ok = has_simd(oracle, opar)
    h = t >> 1
    edges = np.array([I64.min, -1, I64.max, 0, h, h - 1, -h, -(h - 1), h + 1, t - 1, -786433], np.int64)
    for level in sorted({0, len(opar.moduli) - 1}):
        for simd in ((False, True) if simd_ok else (False,)):
            enc = F.Encoding.simd_at_level(level) if simd else F.Encoding.poly_at_level(level)
            u = rng.integers(0, t, size=2 * n, dtype=np.uint64)
            u[:4] = [0, h, h - 1, t - 1]
            P = F.PlaintextVec.try_encode(u, enc, gpar)
            assert (P.try_decode() == u).all() and (P.try_decode(enc) == u).all()
            s = rng.integers(I64.min, I64.max, size=2 * n, dtype=np.int64, endpoint=True)
            s[:len(edges)] = edges[:min(len(edges), 2 * n)]
            S = F.PlaintextVec.try_encode(s, enc, gpar)
            want = _centre(s, t)
            assert (S.try_decode(signed=True) == want).all()
            # into a CUDA tensor and a pinned host tensor
            for out in (torch.empty(2 * n, dtype=torch.int64, device="cuda"),
                        torch.empty(2 * n, dtype=torch.int64).pin_memory()):
                S.try_decode(signed=True, out=out)
                assert (out.cpu().numpy() == want).all()
    # resolve_encoding (plaintext.rs:137-153)
    P = F.Plaintext.try_encode(np.arange(4, dtype=np.uint64), F.Encoding.poly(), gpar)
    with pytest.raises(F.FheError, match="Mismatch"):
        P.try_decode(F.Encoding.poly_at_level(1))
    if simd_ok:
        with pytest.raises(F.FheError, match="Mismatch"):
            P.try_decode(F.Encoding.simd())
    none = F.PlaintextVec(P.batch, None)
    with pytest.raises(F.FheError, match="MissingEncoding"):
        none.try_decode()
    assert (none.try_decode(F.Encoding.poly())[:4] == np.arange(4)).all()


def _one_coefficient_ct(oracle, opar, level, x, pos):
    """c1 = 0 and c0 = NTT of the polynomial whose coefficient `pos` is x (CRT residues) and all others 0"""
    ctx = opar.context_at_level(level)
    p = oracle.Poly(ctx, oracle.POWER_BASIS)
    for i, q in enumerate(ctx.moduli):
        p.c[i, pos] = x % q
    c0 = p.into_ntt().c
    return np.stack([c0, np.zeros_like(c0)])


@pytest.mark.parametrize("name", ["n16", "setA", "mixed"])
def test_measure_noise_boundaries(oracle, F, name):
    """hand-made c1 = 0 ciphertexts whose phase has one coefficient at 0, 1, Q/2 rounded both ways, Q - 1 and
    2^k +- 1; whatever decryption removes, the oracle gives the expected value"""
    opar, gpar, rng, osk, gsk = setup(oracle, F, name, seed=1)
    for level in range(len(opar.moduli)):
        Q = opar.context_at_level(level).modulus()
        xs = [0, 1, Q // 2, (Q + 1) // 2, Q - 1, Q - 2]
        for k in (1, 20, 62, 63, 64, 65, Q.bit_length() - 2, Q.bit_length() - 1):
            xs += [(1 << k) - 1, 1 << k, (1 << k) + 1]
        xs = [x for x in xs if 0 <= x < Q]
        words = np.stack([_one_coefficient_ct(oracle, opar, level, x, (3 * i) % opar.degree)
                          for i, x in enumerate(xs)])
        got = gsk.measure_noise(F.Ciphertext.from_host(gpar, words, level))
        for i in range(len(xs)):
            assert int(got[i]) == osk.measure_noise(oracle.Ciphertext.from_array(opar, words[i], level)), (level, xs[i])


def test_errors(oracle, F):
    from fhe_rs_b200 import _capi
    lib = _capi.lib()
    degree = 1 << 12
    opar = oracle.BfvParameters(degree, 1153, moduli_sizes=[62, 62])   # 1153 has no NTT at N = 2^12
    gpar = F.BfvParameters(degree, 1153, moduli=opar.moduli, device=0)
    rng = np.random.default_rng(2)
    osk = oracle.SecretKey(opar, rng)
    gsk = F.SecretKey(gpar, osk.coeffs)
    words = fresh(oracle, opar, osk, rng, 2, 0)
    ct = F.Ciphertext.from_host(gpar, words)
    out = np.zeros(2 * degree, np.uint64)
    noise = np.zeros(2, np.uint32)

    def code_of(fn):
        with pytest.raises(F.FheError) as e:
            fn()
        return e.value.code

    # power basis input
    pb = F.Ciphertext.from_host(gpar, words, repr=F.POWER_BASIS)
    assert code_of(lambda: gsk.try_decrypt(pb)) == _capi.INVALID_REPRESENTATION
    assert code_of(lambda: gsk.measure_noise(pb)) == _capi.INVALID_REPRESENTATION
    pts = gsk.try_decrypt(ct)
    pts_pb = F.Ciphertext(gpar, 2, 1, repr=F.POWER_BASIS)
    assert lib.fhe_b200_decode(gpar.encoder(), 0, 0, pts_pb._h, out.ctypes.data, out.size, None) \
        == _capi.INVALID_REPRESENTATION
    # wrong out shape
    for shape in ((2, 2, 0), (3, 1, 0), (2, 1, 1)):
        bad = F.Ciphertext(gpar, *shape)
        assert lib.fhe_b200_decrypt(gsk._h, ct._h, bad._h, None) == _capi.INVALID_ARGUMENT
    assert lib.fhe_b200_decode(gpar.encoder(), 0, 0, pts.batch._h, out.ctypes.data, out.size - 1, None) \
        == _capi.INVALID_ARGUMENT
    assert lib.fhe_b200_decode(gpar.encoder(), 0, 0, ct._h, out.ctypes.data, out.size, None) == _capi.BAD_POLY_COUNT
    # a batch of another parameter set, or over the multiplication basis
    other = F.BfvParameters(degree, 1153, moduli=opar.moduli, device=0)
    ct_other = F.Ciphertext.from_host(other, words)
    assert code_of(lambda: gsk.try_decrypt(ct_other)) == _capi.CONTEXT_MISMATCH
    assert code_of(lambda: gsk.measure_noise(ct_other)) == _capi.CONTEXT_MISMATCH
    out_other = F.Ciphertext(other, 2, 1)
    assert lib.fhe_b200_decrypt(gsk._h, ct._h, out_other._h, None) == _capi.CONTEXT_MISMATCH
    assert lib.fhe_b200_decode(other.encoder(), 0, 0, pts.batch._h, out.ctypes.data, out.size, None) \
        == _capi.CONTEXT_MISMATCH
    mb = F.Ciphertext(gpar, 2, 2, mul_basis=True)
    assert lib.fhe_b200_measure_noise(gsk._h, mb._h, noise.ctypes.data, None) == _capi.CONTEXT_MISMATCH
    # SIMD without an NTT for t
    assert code_of(lambda: pts.try_decode(F.Encoding.simd())) == _capi.NTT_UNAVAILABLE
    assert (pts.try_decode(F.Encoding.poly())[:degree] == osk.decrypt(oracle.Ciphertext.from_array(opar, words[0], 0))).all()
    # a key needs N coefficients
    assert code_of(lambda: F.SecretKey(gpar, osk.coeffs[:-1])) == _capi.INVALID_ARGUMENT


def test_decrypt_chunking():
    """a batch over several chunks on three side streams equals one-ciphertext calls"""
    env = dict(os.environ, FHE_B200_CHUNK="4", FHE_B200_STREAMS="3")
    out = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "decrypt_chunk_probe.py")], env=env,
                         capture_output=True, text=True, timeout=600)
    assert out.returncode == 0 and "decrypt chunk probe ok" in out.stdout, out.stdout + out.stderr


def test_secret_key_bytes_round_trip(oracle, F):
    opar, gpar, rng, osk, gsk = setup(oracle, F, "setA")
    data = gsk.to_bytes()
    again = F.SecretKey.from_bytes(gpar, data)
    words = fresh(oracle, opar, osk, rng, 2, 0)
    ct = F.Ciphertext.from_host(gpar, words)
    assert (again.try_decrypt(ct).poly_ntt() == gsk.try_decrypt(ct).poly_ntt()).all()


def test_cpp_decrypt(tmp_path, oracle, F):
    """tests/cpp/decrypt_test.cpp: from the SecretKey message of an oracle key to decrypted, decoded values and noise,
    through include/fhe_b200.hpp and include/fhe_b200_wire.hpp"""
    from fhe_rs_b200 import wire
    opar, gpar, rng, osk, _ = setup(oracle, F, "setA", seed=3)
    words = fresh(oracle, opar, osk, rng, 3, 0)
    (tmp_path / "sk.bin").write_bytes(wire.encode_secret_key([int(c) for c in osk.coeffs]))
    words.tofile(str(tmp_path / "ct.bin"))
    np.array(opar.moduli, np.uint64).tofile(str(tmp_path / "moduli.bin"))
    exe = str(tmp_path / "decrypt_test")
    lib_dir = os.path.join(ROOT, "fhe_rs_b200")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "cpp", "decrypt_test.cpp"), "-o", exe,
                           "-L", lib_dir, "-lfhe_b200", "-Wl,-rpath," + lib_dir])
    out = subprocess.run([exe, str(opar.degree), str(opar.plaintext), "3", str(tmp_path)], capture_output=True,
                         text=True, timeout=300)
    assert out.returncode == 0 and out.stdout.startswith("OK"), out.stdout + out.stderr
    simd = np.fromfile(str(tmp_path / "simd.bin"), np.uint64)
    signed = np.fromfile(str(tmp_path / "poly_i64.bin"), np.int64)
    noise = np.fromfile(str(tmp_path / "noise.bin"), np.uint32)
    n = opar.degree
    for k in range(3):
        oc = oracle.Ciphertext.from_array(opar, words[k], 0)
        w = osk.decrypt(oc)
        assert (simd[k * n:(k + 1) * n] == oracle.simd_decode(opar, w)).all()
        assert (signed[k * n:(k + 1) * n] == _centre(w, opar.plaintext)).all()
        assert int(noise[k]) == osk.measure_noise(oc)
