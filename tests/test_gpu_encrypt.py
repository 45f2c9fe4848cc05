"""GPU tests of encryption on the device (fhe_b200_encrypt_sk, fhe_b200_encrypt_pk): for the same seed the device
words equal tests/encrypt_reference.py's restatement of the stream on the oracle, word for word; the ciphertexts
decrypt to the values; fresh noise matches the oracle's measurement; the errors follow the stated distributions.
Run with `-m gpu`."""
import os
import subprocess
import sys

import numpy as np
import pytest

import edge_inputs as E
import encrypt_reference as R

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def F():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import fhe_rs_b200
    return fhe_rs_b200


# name -> (degree, t or None for a 40-bit prime, moduli sizes or an edge_inputs.CLIENT_SHAPES name)
SHAPES = {
    "n16": (16, 1153, [62, 62, 62]),
    "setA": (1 << 12, 1032193, [62, 62]),
    "n14": (1 << 14, 786433, [62] * 8),
    "setC": (1 << 15, 786433, [62] * 14),
    "mixed": (1 << 13, None, [62, 30, 50]),
    "q0_barrett": (1 << 13, 786433, "q0_barrett"),
    "q0_above_2_61": (1 << 13, 786433, "q0_above_2_61"),
    "q0_solinas_max_c": (1 << 13, 786433, "q0_solinas_max_c"),
    "q1_barrett": (1 << 13, 786433, "q1_barrett"),
    "l31": (1 << 13, 786433, "l31"),
    "n2_16": (1 << 16, 786433, [62] * 3),
}
BIG = {"n14", "setC", "l31", "n2_16"}


def setup(oracle, F, name, seed=0):
    degree, t, spec = SHAPES[name]
    if t is None:
        t = oracle.generate_prime(40, 2 * degree, 1 << 40)
    moduli = E.client_moduli(spec) if isinstance(spec, str) else oracle.BfvParameters.generate_moduli(spec, degree)
    opar = oracle.BfvParameters(degree, t, moduli=moduli)
    gpar = F.BfvParameters(degree, t, moduli=moduli, device=0)
    rng = np.random.default_rng(degree + len(moduli) + seed)
    osk = oracle.SecretKey(opar, rng)
    return opar, gpar, rng, osk, F.SecretKey(gpar, osk.coeffs)


def seed_of(rng):
    return rng.integers(0, 256, size=32, dtype=np.uint8).tobytes()


def plaintexts(oracle, F, opar, gpar, rng, kind, count, level):
    """(device plaintexts or None, oracle to_poly of each, the values, the encoding)"""
    n, t = opar.degree, opar.plaintext
    if kind == "none":
        return None, None, np.zeros(count * n, np.uint64), F.Encoding.poly_at_level(level)
    values = rng.integers(0, t, size=count * n, dtype=np.uint64)
    if kind == "simd":
        enc = F.Encoding.simd_at_level(level)
        coeffs = [oracle.simd_encode(opar, values[k * n:(k + 1) * n]) for k in range(count)]
    else:
        enc = F.Encoding.poly_at_level(level)
        coeffs = [values[k * n:(k + 1) * n] for k in range(count)]
    ms = [R.to_poly(opar, c, level) for c in coeffs]
    return F.PlaintextVec.try_encode(values, enc, gpar), ms, values, enc


def encrypt_raw(F, fn, key, gpar, pts, variance, seed, count, level):
    """the C ABI call with an explicit variance"""
    from fhe_rs_b200 import _capi
    b = pts.batch if pts is not None else None
    out = F.Ciphertext(gpar, b.count if b else count, 2, b.level if b else level)
    _capi.check(getattr(_capi.lib(), fn)(key, b._h if b else None, variance, seed, out._h, None))
    return out


def check_decrypts(F, gsk, ct, values, enc, oracle=None, osk=None, exp=None):
    pts = gsk.try_decrypt(ct)
    assert (pts.try_decode(enc) == values).all()
    if exp is not None:
        noise = gsk.measure_noise(ct)
        for k, c in enumerate(exp):
            assert int(noise[k]) == osk.measure_noise(c), k


@pytest.mark.parametrize("name", list(SHAPES))
def test_encrypt_parity(oracle, F, name):
    opar, gpar, rng, osk, gsk = setup(oracle, F, name)
    big = name in BIG
    count = 1 if big else 2
    last = len(opar.moduli) - 1
    simd_ok = opar.plaintext % (2 * opar.degree) == 1 and oracle.is_prime(opar.plaintext)
    kinds = ["poly", "simd", "none"] if simd_ok else ["poly", "none"]
    variances = [10, 1, 32]
    # public keys: made on the device (checked against the stream) and made by the oracle's own encryption of zero
    seed_pk = seed_of(rng)
    gpk = F.PublicKey.new(gsk, seed_pk)
    opk_dev = R.encrypt_sk(osk, seed_pk, 1, 0, 10)[0]
    assert (gpk.c.to_host()[0] == opk_dev.to_array()).all()
    ctx0 = opar.context_at_level(0)
    opk_orc = osk.encrypt_poly(oracle.Poly(ctx0, oracle.NTT), 0, rng)
    gpk_orc = F.PublicKey(gpar, F.Ciphertext.from_host(gpar, opk_orc.to_array()[None]))
    levels = sorted({0, 1, last}) if name == "l31" else range(last + 1)
    for i, level in enumerate(levels):
        kind = kinds[i % len(kinds)]
        var = variances[i % len(variances)]
        P, ms, values, enc = plaintexts(oracle, F, opar, gpar, rng, kind, count, level)
        noise = not big or level in (0, last)
        # secret-key encryption
        seed = seed_of(rng)
        got = encrypt_raw(F, "fhe_b200_encrypt_sk", gsk._h, gpar, P, var, seed, count, level)
        exp = R.encrypt_sk(osk, seed, count, level, var, ms)
        words = got.to_host()
        for k in range(count):
            assert (words[k] == exp[k].to_array()).all(), (level, kind, var, k)
        check_decrypts(F, gsk, got, values, enc, oracle, osk, exp if noise else None)
        # public-key encryption with both keys
        for pk, opk in ((gpk, opk_dev), (gpk_orc, opk_orc)):
            seed = seed_of(rng)
            got = encrypt_raw(F, "fhe_b200_encrypt_pk", pk.c._h, gpar, P, var, seed, count, level)
            exp = R.encrypt_pk(opar, opk, seed, count, level, var, ms)
            words = got.to_host()
            for k in range(count):
                assert (words[k] == exp[k].to_array()).all(), (level, kind, var, k, pk is gpk)
            check_decrypts(F, gsk, got, values, enc, oracle, osk, exp if noise and pk is gpk else None)


def test_python_api_and_default_variance(oracle, F):
    """SecretKey.try_encrypt / PublicKey.try_encrypt with the parameter set's variance, a fresh seed per call"""
    opar, gpar, rng, osk, gsk = setup(oracle, F, "setA", seed=1)
    assert gpar.variance == 10
    P, ms, values, enc = plaintexts(oracle, F, opar, gpar, rng, "simd", 3, 0)
    seed = seed_of(rng)
    ct = gsk.try_encrypt(P, seed)
    assert ct.count == 3 and len(ct) == 2 and ct.level == 0
    exp = R.encrypt_sk(osk, seed, 3, 0, 10, ms)
    assert (ct.to_host() == np.stack([c.to_array() for c in exp])).all()
    a, b = gsk.try_encrypt(P).to_host(), gsk.try_encrypt(P).to_host()   # os.urandom seeds
    assert not (a[:, 1] == b[:, 1]).all()
    check_decrypts(F, gsk, gsk.try_encrypt(P), values, enc)
    pk = F.PublicKey.new(gsk)
    check_decrypts(F, gsk, pk.try_encrypt(P), values, enc)
    zeros = gsk.try_encrypt(None, count=4, level=1)
    assert zeros.count == 4 and zeros.level == 1
    check_decrypts(F, gsk, zeros, np.zeros(4 * opar.degree, np.uint64), F.Encoding.poly_at_level(1))
    # another variance through the builder
    g32 = F.BfvParametersBuilder().set_degree(opar.degree).set_plaintext_modulus(opar.plaintext) \
        .set_moduli(opar.moduli).set_variance(32).build()
    sk32 = F.SecretKey(g32, osk.coeffs)
    seed = seed_of(rng)
    got = sk32.try_encrypt(None, seed, count=2).to_host()
    assert (got == np.stack([c.to_array() for c in R.encrypt_sk(osk, seed, 2, 0, 32)])).all()
    # the public key travels as a PublicKey message with both parts
    again = F.PublicKey.from_bytes(gpar, pk.to_bytes())
    assert (again.c.to_host() == pk.c.to_host()).all()


def test_end_to_end_product(oracle, F):
    """public-key-encrypt SIMD vectors, mul_relin, decrypt: the slot-wise product"""
    opar, gpar, rng, osk, gsk = setup(oracle, F, "setA", seed=2)
    n, t = opar.degree, opar.plaintext
    ork = oracle.RelinearizationKey(osk, rng)
    grk = F.RelinearizationKey.from_arrays(gpar, *ork.ksk.arrays())
    pk = F.PublicKey.new(gsk, seed_of(rng))
    x = rng.integers(0, t, size=4 * n, dtype=np.uint64)
    y = rng.integers(0, t, size=4 * n, dtype=np.uint64)
    A = pk.try_encrypt(F.PlaintextVec.try_encode(x, F.Encoding.simd(), gpar), seed_of(rng))
    B = pk.try_encrypt(F.PlaintextVec.try_encode(y, F.Encoding.simd(), gpar), seed_of(rng))
    prod = F.Multiplicator.default(grk).multiply(A, B)
    got = gsk.try_decrypt(prod).try_decode(F.Encoding.simd())
    want = (x.astype(object) * y.astype(object)) % t
    assert (got.astype(object) == want).all()


def _chi2_p(observed, expected):
    from scipy import stats
    return stats.chisquare(observed, expected).pvalue


def test_statistics(oracle, F):
    """set C, fixed seeds: the top bits of a are uniform in every limb; e = b + a s, recovered with the oracle,
    follows the centred binomial distribution of the variance"""
    from scipy import stats
    opar, gpar, rng, osk, gsk = setup(oracle, F, "setC", seed=3)
    n = opar.degree
    ctx = opar.context_at_level(0)
    s = osk.s_ntt(ctx)
    for var in (1, 10, 32):
        seed = bytes(range(var, var + 32))
        ct = encrypt_raw(F, "fhe_b200_encrypt_sk", gsk._h, gpar, None, var, seed, 2, 0).to_host()
        for k in range(2):
            b, a = (oracle.Poly(ctx, oracle.NTT, ct[k, i].copy()) for i in (0, 1))
            if var == 10:
                for j, q in enumerate(ctx.moduli):
                    top = (a.c[j].astype(object) * 64 // q).astype(np.int64)
                    assert _chi2_p(np.bincount(top, minlength=64), np.full(64, n / 64)) > 1e-4, (k, j)
            e = b.iadd(a.mul(s)).into_power_basis()
            q0 = ctx.moduli[0]
            x = np.array([int(v) - q0 if int(v) > q0 // 2 else int(v) for v in e.c[0]], np.int64)
            assert (x == R.cbd(seed, k, R.ROLE_E, var, n)).all()
            assert (np.abs(x) <= 2 * var).all()
            for j, q in enumerate(ctx.moduli):   # the same signed value in every limb
                assert (e.c[j] == np.where(x < 0, q + x, x).astype(np.uint64)).all()
            # x + 2 var ~ Binomial(4 var, 1/2); bins with a small expectation merged into the tails
            support = np.arange(4 * var + 1)
            pmf = stats.binom.pmf(support, 4 * var, 0.5) * n
            keep = pmf >= 5
            lo, hi = support[keep][0], support[keep][-1]
            obs = np.bincount(np.clip(x + 2 * var, lo, hi) - lo, minlength=hi - lo + 1)
            exp = pmf[lo:hi + 1].copy()
            exp[0] += pmf[:lo].sum()
            exp[-1] += pmf[hi + 1:].sum()
            assert _chi2_p(obs, exp * obs.sum() / exp.sum()) > 1e-4, (var, k)


def test_determinism(oracle, F):
    opar, gpar, rng, osk, gsk = setup(oracle, F, "setA", seed=4)
    P, _, _, _ = plaintexts(oracle, F, opar, gpar, rng, "poly", 2, 0)
    seed = seed_of(rng)
    pk = F.PublicKey.new(gsk, seed_of(rng))
    assert (gsk.try_encrypt(P, seed).to_host() == gsk.try_encrypt(P, seed).to_host()).all()
    assert (pk.try_encrypt(P, seed).to_host() == pk.try_encrypt(P, seed).to_host()).all()
    other = bytearray(seed)
    other[31] ^= 1
    a, b = gsk.try_encrypt(P, seed).to_host(), gsk.try_encrypt(P, bytes(other)).to_host()
    for k in range(2):
        assert (a[k, 1] != b[k, 1]).mean() > 0.99
    assert (a[0, 1] != a[1, 1]).mean() > 0.99   # the ciphertext index is part of the address


@pytest.mark.parametrize("streams", ["1", "2", "4"])
def test_encrypt_chunking(streams):
    """a batch over several chunks on 1, 2 and 4 streams equals the stream's definition"""
    env = dict(os.environ, FHE_B200_CHUNK="4", FHE_B200_STREAMS=streams)
    out = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "encrypt_chunk_probe.py")], env=env,
                         capture_output=True, text=True, timeout=600)
    assert out.returncode == 0 and "encrypt chunk probe ok" in out.stdout, out.stdout + out.stderr


def test_errors(oracle, F):
    from fhe_rs_b200 import _capi
    lib = _capi.lib()
    degree = 1 << 12
    opar = oracle.BfvParameters(degree, 1032193, moduli_sizes=[62, 62])
    gpar = F.BfvParameters(degree, 1032193, moduli=opar.moduli, device=0)
    rng = np.random.default_rng(9)
    osk = oracle.SecretKey(opar, rng)
    gsk = F.SecretKey(gpar, osk.coeffs)
    pk = F.PublicKey.new(gsk, seed_of(rng))
    seed = seed_of(rng)
    P = F.PlaintextVec.try_encode(np.arange(2 * degree, dtype=np.uint64), F.Encoding.poly(), gpar)
    out = F.Ciphertext(gpar, 2, 2)
    other = F.BfvParameters(degree, 1032193, moduli=opar.moduli, device=0)
    P_other = F.PlaintextVec.try_encode(np.arange(2 * degree, dtype=np.uint64), F.Encoding.poly(), other)
    P_mb = F.Ciphertext(gpar, 2, 1, mul_basis=True)
    def sk_fn(p, v=10, s=seed, o=out, k=gsk):
        return lib.fhe_b200_encrypt_sk(k._h if k else None, p, v, s, o._h if o else None, None)

    def pk_fn(p, v=10, s=seed, o=out, k=pk.c):
        return lib.fhe_b200_encrypt_pk(k._h if k else None, p, v, s, o._h if o else None, None)
    for fn in (sk_fn, pk_fn):
        assert fn(P.batch._h) == _capi.OK
        # InvalidVariance, NULL arguments, shapes
        for v in (0, 33):
            assert fn(P.batch._h, v=v) == _capi.INVALID_ARGUMENT
            assert b"InvalidVariance" in lib.fhe_b200_last_error()
        assert fn(P.batch._h, s=None) == _capi.INVALID_ARGUMENT
        assert fn(P.batch._h, o=None) == _capi.INVALID_ARGUMENT
        assert fn(P.batch._h, k=None) == _capi.INVALID_ARGUMENT
        assert fn(P.batch._h, o=F.Ciphertext(gpar, 2, 3)) == _capi.INVALID_ARGUMENT
        assert fn(P.batch._h, o=F.Ciphertext(gpar, 3, 2)) == _capi.INVALID_ARGUMENT
        assert fn(out._h) == _capi.INVALID_ARGUMENT                                   # a 2-part "plaintext" batch
        # level, representation, parameter set, multiplication basis
        assert fn(P.batch._h, o=F.Ciphertext(gpar, 2, 2, 1)) == _capi.INVALID_LEVEL
        Ppb = F.Ciphertext(gpar, 2, 1, repr=F.POWER_BASIS)
        assert fn(Ppb._h) == _capi.INVALID_REPRESENTATION
        assert fn(P.batch._h, o=F.Ciphertext(other, 2, 2)) == _capi.CONTEXT_MISMATCH
        assert fn(P_other.batch._h) == _capi.CONTEXT_MISMATCH
        assert fn(P.batch._h, o=F.Ciphertext(gpar, 2, 2, mul_basis=True)) == _capi.CONTEXT_MISMATCH
        assert fn(P_mb._h) == _capi.CONTEXT_MISMATCH
    # the public key: level 0, one 2-part NTT ciphertext
    low = pk.c.clone()
    low.switch_down()
    P1 = F.PlaintextVec.try_encode(np.arange(2 * degree, dtype=np.uint64), F.Encoding.poly_at_level(1), gpar)
    o1 = F.Ciphertext(gpar, 2, 2, 1)
    assert lib.fhe_b200_encrypt_pk(low._h, P1.batch._h, 10, seed, o1._h, None) == _capi.INVALID_LEVEL
    assert b"InvalidPublicKeyLevel" in lib.fhe_b200_last_error()
    with pytest.raises(F.FheError) as e:
        F.PublicKey(gpar, low)
    assert e.value.code == _capi.INVALID_LEVEL
    assert pk_fn(P.batch._h, k=F.Ciphertext(gpar, 2, 2)) == _capi.INVALID_ARGUMENT
    assert pk_fn(P.batch._h, k=F.Ciphertext(gpar, 1, 3)) == _capi.INVALID_ARGUMENT
    assert pk_fn(P.batch._h, k=F.Ciphertext(gpar, 1, 2, repr=F.POWER_BASIS)) == _capi.INVALID_REPRESENTATION
    assert pk_fn(P.batch._h, k=F.Ciphertext(other, 1, 2)) == _capi.CONTEXT_MISMATCH
    assert pk_fn(P.batch._h, k=F.Ciphertext(gpar, 1, 2, mul_basis=True)) == _capi.CONTEXT_MISMATCH
    # a seed of another length through the Python API
    with pytest.raises(F.FheError) as e:
        gsk.try_encrypt(P, b"short")
    assert e.value.code == _capi.INVALID_ARGUMENT
    # t >= q_0
    t40 = oracle.generate_prime(40, 2 * degree, 1 << 40)
    omix = oracle.BfvParameters(degree, t40, moduli_sizes=[30, 62])
    gmix = F.BfvParameters(degree, t40, moduli=omix.moduli, device=0)
    skm = F.SecretKey(gmix, oracle.SecretKey(omix, rng).coeffs)
    om = F.Ciphertext(gmix, 1, 2)
    assert lib.fhe_b200_encrypt_sk(skm._h, None, 10, seed, om._h, None) == _capi.UNSUPPORTED
    with pytest.raises(F.FheError) as e:
        F.PublicKey.new(skm)
    assert e.value.code == _capi.UNSUPPORTED


def test_public_key_from_reference_message(oracle, F):
    """a compact PublicKey message (c0 and the seed of c1, as the reference writes it) decodes with the expanded c1"""
    from fhe_rs_b200 import wire
    opar, gpar, rng, osk, gsk = setup(oracle, F, "setA", seed=5)
    ctx = opar.context_at_level(0)
    opk = osk.encrypt_poly(oracle.Poly(ctx, oracle.NTT), 0, rng)
    pb0 = opk.c[0].copy().into_power_basis()
    rq0 = wire.encode_rq(wire.REP_NTT, opar.degree, oracle.poly_to_rq_coefficients(pb0))
    msg = wire.encode_public_key(wire.encode_ciphertext([rq0], bytes(32), 0))
    with pytest.raises(F.WireError) as e:
        F.PublicKey.from_bytes(gpar, msg)
    assert e.value.variant == "SeedExpansion"
    pk = F.PublicKey.from_bytes(gpar, msg, seeded_c1=opk.c[1].c)
    assert (pk.c.to_host()[0] == opk.to_array()).all()
    P, ms, values, enc = plaintexts(oracle, F, opar, gpar, rng, "simd", 2, 0)
    seed = seed_of(rng)
    got = pk.try_encrypt(P, seed).to_host()
    assert (got == np.stack([c.to_array() for c in R.encrypt_pk(opar, opk, seed, 2, 0, 10, ms)])).all()


def test_cpp_encrypt(tmp_path, oracle, F):
    """tests/cpp/encrypt_test.cpp: secret-key and public-key encryption through include/fhe_b200.hpp, the public key
    through its message in include/fhe_b200_wire.hpp, equal to the stream's definition"""
    from fhe_rs_b200 import wire
    opar, gpar, rng, osk, _ = setup(oracle, F, "setA", seed=6)
    n, count = opar.degree, 3
    values = rng.integers(0, opar.plaintext, size=count * n, dtype=np.uint64)
    seeds = [seed_of(rng) for _ in range(3)]
    (tmp_path / "sk.bin").write_bytes(wire.encode_secret_key([int(c) for c in osk.coeffs]))
    (tmp_path / "seeds.bin").write_bytes(b"".join(seeds))
    values.tofile(str(tmp_path / "values.bin"))
    np.array(opar.moduli, np.uint64).tofile(str(tmp_path / "moduli.bin"))
    exe = str(tmp_path / "encrypt_test")
    lib_dir = os.path.join(ROOT, "fhe_rs_b200")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "cpp", "encrypt_test.cpp"), "-o", exe,
                           "-L", lib_dir, "-lfhe_b200", "-Wl,-rpath," + lib_dir])
    out = subprocess.run([exe, str(n), str(opar.plaintext), str(count), str(tmp_path)], capture_output=True,
                         text=True, timeout=300)
    assert out.returncode == 0 and out.stdout.startswith("OK"), out.stdout + out.stderr
    ms = [R.to_poly(opar, oracle.simd_encode(opar, values[k * n:(k + 1) * n]), 0) for k in range(count)]
    pk = R.encrypt_sk(osk, seeds[0], 1, 0, 10)[0]
    want_sk = np.stack([c.to_array() for c in R.encrypt_sk(osk, seeds[1], count, 0, 10, ms)])
    want_pk = np.stack([c.to_array() for c in R.encrypt_pk(opar, pk, seeds[2], count, 0, 10, ms)])
    shape = want_sk.shape
    assert (np.fromfile(str(tmp_path / "ct_sk.bin"), np.uint64).reshape(shape) == want_sk).all()
    assert (np.fromfile(str(tmp_path / "ct_pk.bin"), np.uint64).reshape(shape) == want_pk).all()
    assert (tmp_path / "pk.bin").read_bytes() == F.PublicKey(gpar, F.Ciphertext.from_host(gpar, pk.to_array()[None])).to_bytes()


@pytest.mark.parametrize("env", [{"FHE_B200_NTT": "fast"}, {"FHE_B200_NTT": "tma"}, {"FHE_B200_GENERIC_NTT": "1"},
                                 {"FHE_B200_NO_SOLINAS": "1"}, {"FHE_B200_SOLINAS_NTT": "1"}],
                         ids=lambda e: ",".join("%s=%s" % kv for kv in e.items()))
def test_alternate_code_paths(F, env):
    """every NTT variant gives the same words: rerun the parity tests of this module under each switch"""
    out = subprocess.run([sys.executable, "-m", "pytest", "-q", "-x", "-m", "gpu", "tests/test_gpu_encrypt.py",
                          "-k", "test_encrypt_parity or test_end_to_end_product", "-p", "no:cacheprovider"],
                         cwd=ROOT, env=dict(os.environ, **env), capture_output=True, text=True, timeout=1800)
    assert out.returncode == 0, out.stdout[-2000:] + out.stderr[-2000:]
