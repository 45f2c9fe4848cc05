"""GPU tests of key generation on the device (fhe_b200_relin_key_generate, fhe_b200_galois_keys_generate,
fhe_b200_rgsw_encrypt, fhe_b200_ksk_download): for the same seed the downloaded words equal tests/keygen_reference.py's
restatement word for word; keys made on the device alone relinearize, rotate, expand and take external products
correctly; the words follow the stated distributions.  Run with `-m gpu`."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

import edge_inputs as E
import keygen_reference as K

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MULPIR_T = (1 << 20) + (1 << 19) + (1 << 17) + (1 << 16) + (1 << 14) + 1   # examples/mulpir.rs:36


@pytest.fixture(scope="module")
def F():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import fhe_rs_b200
    return fhe_rs_b200


# the shapes of tests/test_gpu_encrypt.py: name -> (degree, t or None for a 40-bit prime, moduli sizes or an
# edge_inputs.CLIENT_SHAPES name)
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


def check_key(osk, ksk, frm, seed, key, variance, big, what):
    """the downloaded words of `ksk` equal the restatement: every digit, or the first, a middle and the last one"""
    c0, c1 = ksk.arrays()
    n = c0.shape[0]
    assert n == len(K.gadget(osk.par, ksk.ciphertext_level, ksk.ksk_level)), what
    for i in sorted({0, n // 2, n - 1}) if big else range(n):
        w0, w1 = K.key_digit(osk, frm, ksk.ciphertext_level, ksk.ksk_level, seed, key, i, variance)
        assert (c1[i] == w1).all(), (what, "c1", i)
        assert (c0[i] == w0).all(), (what, "c0", i)


@pytest.mark.parametrize("name", list(SHAPES))
def test_keygen_parity(oracle, F, name):
    opar, gpar, rng, osk, gsk = setup(oracle, F, name)
    big = name in BIG
    n, last, var = opar.degree, len(opar.moduli) - 1, opar.variance
    # relinearization keys
    for c, k in sorted({(0, 0), (1, 0), (max(last - 1, 0), 0)}):
        seed = seed_of(rng)
        rk = F.RelinearizationKey.new_leveled(gsk, c, k, seed)
        check_key(osk, rk.ksk, K.relin_from(osk, c, k), seed, 0, var, big, ("relin", c, k))
    # Galois keys: one call for several exponents, leveled keys, the decomposition variant at the last level
    exps = [3, pow(3, 2, 2 * n), 2 * n - 1, (n >> 1) + 1]
    cases = [(exps, 0, 0), ([3, 2 * n - 1], 1, 0), ([2 * n - 1], last, last)]
    if last >= 2:
        cases.append(([(n >> 2) + 1], last, last - 1))
    for es, c, k in cases:
        if big and len(es) > 2:
            es = es[:1] + es[-1:]
        seed = seed_of(rng)
        gks = F.bfv._galois_keys(gsk, es, c, k, seed)
        for key, (e, gk) in enumerate(zip(es, gks)):
            assert gk.exponent == e % (2 * n)
            check_key(osk, gk.ksk, K.galois_from(osk, e, c, k), seed, key, var, big, ("galois", e, c, k))
    # RGSW of Poly and SIMD plaintexts at several levels
    simd_ok = opar.plaintext % (2 * n) == 1 and oracle.is_prime(opar.plaintext)
    for level, kind in ((0, "poly"), (last, "simd" if simd_ok else "poly"), (min(1, last), "poly")):
        count = 1 if big else 2
        values = rng.integers(0, opar.plaintext, size=count * n, dtype=np.uint64)
        enc = F.Encoding.simd_at_level(level) if kind == "simd" else F.Encoding.poly_at_level(level)
        P = F.PlaintextVec.try_encode(values, enc, gpar)
        ms = [oracle.Poly(opar.context_at_level(level), oracle.NTT, w.copy()) for w in P.batch.to_host()[:, 0]]
        seed = seed_of(rng)
        rg = gsk.try_encrypt_rgsw(P, seed)
        assert len(rg) == count
        for p, r in enumerate(rg):
            for which, ksk in enumerate((r.ksk0, r.ksk1)):
                check_key(osk, ksk, K.rgsw_from(osk, ms[p], level, bool(which)), seed, 2 * p + which, var, big,
                          ("rgsw", level, kind, p, which))


def _negacyclic(x, y, t):
    n = len(x)
    out = np.zeros(n, dtype=object)
    for i in range(n):
        out[i:] += int(x[i]) * y[:n - i].astype(object)
        out[:i] -= int(x[i]) * y[n - i:].astype(object)
    return out % t


def test_device_keys_compute(oracle, F):
    """keys made on the device alone: mul_relin, rotations, the inner sum and RGSW external products decrypt to the
    expected values; the device measures the product's noise as the oracle does"""
    opar, gpar, rng, osk, gsk = setup(oracle, F, "setA", seed=1)
    n, t = opar.degree, opar.plaintext
    rk = F.RelinearizationKey.new(gsk, seed_of(rng))
    x = rng.integers(0, t, size=2 * n, dtype=np.uint64)
    y = rng.integers(0, t, size=2 * n, dtype=np.uint64)
    A = gsk.try_encrypt(F.PlaintextVec.try_encode(x, F.Encoding.simd(), gpar), seed_of(rng))
    B = gsk.try_encrypt(F.PlaintextVec.try_encode(y, F.Encoding.simd(), gpar), seed_of(rng))
    prod = F.Multiplicator.default(rk).multiply(A, B)
    got = gsk.try_decrypt(prod).try_decode(F.Encoding.simd())
    assert (got.astype(object) == (x.astype(object) * y.astype(object)) % t).all()
    noise = gsk.measure_noise(prod)
    words = prod.to_host()
    for k in range(2):
        assert int(noise[k]) == osk.measure_noise(oracle.Ciphertext.from_array(opar, words[k], 0))
    # rotations and the inner sum from one EvaluationKeyBuilder call
    ek = F.EvaluationKeyBuilder(gsk).enable_inner_sum().enable_column_rotation(5).build(seed_of(rng))
    assert sorted(ek.gk) == K.evaluation_key_exponents(n, inner_sum=True, column_rotation=(5,))
    half = n // 2
    xs = x[:n].reshape(2, half)
    rows = ek.rotates_rows(A.take(0, 1))
    got = gsk.try_decrypt(rows).try_decode(F.Encoding.simd()).reshape(2, half)
    assert (got == xs[::-1]).all()
    cols = ek.rotates_columns_by(A.take(0, 1), 5)
    got = gsk.try_decrypt(cols).try_decode(F.Encoding.simd()).reshape(2, half)
    assert (got == np.roll(xs, -5, axis=1)).all()
    s = ek.computes_inner_sum(A.take(0, 1))
    got = gsk.try_decrypt(s).try_decode(F.Encoding.simd())
    assert (got == int(x[:n].astype(object).sum() % t)).all()
    # RGSW external product (the decomposition variant's words are pinned by test_keygen_parity; at one 62-bit
    # modulus its noise leaves too little room for a 20-bit t to decrypt a product)
    for level in (0,):
        m = rng.integers(0, t, size=n, dtype=np.uint64)
        m[8:] = 0                                              # a small product keeps the check cheap
        yy = rng.integers(0, t, size=n, dtype=np.uint64)
        enc = F.Encoding.poly_at_level(level)
        r = gsk.try_encrypt_rgsw(F.PlaintextVec.try_encode(m, enc, gpar), seed_of(rng))[0]
        ct = gsk.try_encrypt(F.PlaintextVec.try_encode(yy, enc, gpar), seed_of(rng))
        got = gsk.try_decrypt(r.external_product(ct)).try_decode(enc)
        assert (got.astype(object) == _negacyclic(m, yy, t)).all(), level


def test_key_switch_error_bound(oracle, F):
    """key_switching_key.rs:531-559 at N = 16: c0 + c1 s - input from, the key-switch error of a device key, stays
    within 70 bits for random inputs"""
    opar, gpar, rng, osk, gsk = setup(oracle, F, "n16", seed=7)
    ctx = opar.context_at_level(0)
    s, Q = osk.s_ntt(ctx), ctx.modulus()
    keys = [(F.RelinearizationKey.new(gsk, seed_of(rng)).ksk, K.relin_from(osk, 0, 0)),
            (F.GaloisKey.new(gsk, 3, seed=seed_of(rng)).ksk, K.galois_from(osk, 3, 0, 0))]
    for ksk, frm in keys:
        frm_ntt = frm.copy().into_ntt()
        for _ in range(20):
            inp = oracle.Poly.random(ctx, oracle.POWER_BASIS, rng)
            X = F.Ciphertext.from_host(gpar, inp.c[None, None].copy(), 0, F.POWER_BASIS)
            c0, c1 = (oracle.Poly(ctx, oracle.NTT, w.copy()) for w in ksk.key_switch(X, 0).to_host()[0])
            d = c0.iadd(c1.mul(s)).isub(inp.copy().into_ntt().mul(frm_ntt)).into_power_basis()
            assert max(min(v.bit_length(), (Q - v).bit_length()) for v in d.to_bigints()) <= 70


def test_mulpir_shape_expansion(oracle, F):
    """examples/mulpir.rs: keys of EvaluationKeyBuilder.new_leveled(sk, 1, 0) made on the device expand a level-1
    query encrypted on the device: output k decrypts to 1 at the two chosen indices and to 0 elsewhere"""
    size, level = 115, 7
    opar = oracle.BfvParameters(8192, MULPIR_T, moduli_sizes=[50, 55, 55])
    gpar = F.BfvParameters(8192, MULPIR_T, moduli=opar.moduli, device=0)
    rng = np.random.default_rng(8192)
    osk = oracle.SecretKey(opar, rng)
    gsk = F.SecretKey(gpar, osk.coeffs)
    ek = F.EvaluationKeyBuilder.new_leveled(gsk, 1, 0).enable_expansion(level).build(seed_of(rng))
    assert sorted(ek.gk) == sorted((8192 >> l) + 1 for l in range(level))
    pt = np.zeros(size, np.uint64)
    chosen = (17, 98)
    pt[list(chosen)] = pow(1 << level, -1, MULPIR_T)
    query = gsk.try_encrypt(F.PlaintextVec.try_encode(pt, F.Encoding.poly_at_level(1), gpar), seed_of(rng))
    assert query.level == 1
    out = ek.expands_batch(query, size)
    dec = gsk.try_decrypt(out).try_decode(F.Encoding.poly_at_level(1)).reshape(size, -1)
    for k in range(size):
        assert int(dec[k, 0]) == (1 if k in chosen else 0) and not dec[k, 1:].any(), k


def test_statistics(oracle, F):
    """set C, fixed seeds: the top bits of c1 are uniform in every key limb; c0 + c1 s - g from, recovered with the
    oracle, is the centred binomial sample of the stream"""
    from scipy import stats
    opar, gpar, rng, osk, gsk = setup(oracle, F, "setC", seed=3)
    n = opar.degree
    seed = bytes(range(40, 72))
    rk = F.RelinearizationKey.new(gsk, seed)
    c0, c1 = rk.ksk.arrays()
    ctx = opar.context_at_level(0)
    for i in (0, 13):
        for j, q in enumerate(ctx.moduli):
            top = (c1[i, j].astype(object) * 64 // q).astype(np.int64)
            assert stats.chisquare(np.bincount(top, minlength=64), np.full(64, n / 64)).pvalue > 1e-4, (i, j)
    s = osk.s_ntt(ctx)
    frm = K.relin_from(osk, 0, 0)
    g = K.gadget(opar, 0, 0)
    for i in (0, 7):
        e = oracle.Poly(ctx, oracle.NTT, c0[i].copy()).iadd(oracle.Poly(ctx, oracle.NTT, c1[i].copy()).mul(s))
        e = e.into_power_basis().isub(frm.mul_scalar_big(g[i]))
        q0 = ctx.moduli[0]
        x = np.array([int(v) - q0 if int(v) > q0 // 2 else int(v) for v in e.c[0]], np.int64)
        assert (x == K.error(seed, 0, i, 10, n)).all()
        var = 10
        support = np.arange(4 * var + 1)
        pmf = stats.binom.pmf(support, 4 * var, 0.5) * n
        keep = pmf >= 5
        lo, hi = support[keep][0], support[keep][-1]
        obs = np.bincount(np.clip(x + 2 * var, lo, hi) - lo, minlength=hi - lo + 1)
        exp = pmf[lo:hi + 1].copy()
        exp[0] += pmf[:lo].sum()
        exp[-1] += pmf[hi + 1:].sum()
        assert stats.chisquare(obs, exp * obs.sum() / exp.sum()).pvalue > 1e-4, i


def test_determinism_and_addressing(oracle, F):
    opar, gpar, rng, osk, gsk = setup(oracle, F, "setA", seed=4)
    n = opar.degree
    seed = seed_of(rng)
    a = F.RelinearizationKey.new(gsk, seed).ksk.arrays()
    b = F.RelinearizationKey.new(gsk, seed).ksk.arrays()
    assert (a[0] == b[0]).all() and (a[1] == b[1]).all()
    other = bytearray(seed)
    other[0] ^= 1
    c = F.RelinearizationKey.new(gsk, bytes(other)).ksk.arrays()
    assert (a[1] != c[1]).mean() > 0.99
    assert (a[1][0] != a[1][1]).mean() > 0.99                  # digits
    g = F.bfv._galois_keys(gsk, [3, 3], 0, 0, seed)             # the key index is part of the address
    assert (g[0].ksk.arrays()[1] != g[1].ksk.arrays()[1]).mean() > 0.99
    # build() orders the exponents, so the same seed gives each exponent the same key
    e1 = F.EvaluationKeyBuilder(gsk).enable_column_rotation(1).enable_row_rotation().build(seed)
    e2 = F.EvaluationKeyBuilder(gsk).enable_row_rotation().enable_column_rotation(1).build(seed)
    for e in e1.gk:
        assert (e1.gk[e].ksk.arrays()[0] == e2.gk[e].ksk.arrays()[0]).all()


def test_wire_and_upload_round_trips(oracle, F):
    """to_bytes -> from_bytes gives the same words (uncompact messages: no seed, both rows); upload -> download is
    the identity for both key variants"""
    from fhe_rs_b200 import wire
    opar, gpar, rng, osk, gsk = setup(oracle, F, "n16", seed=5)
    last = len(opar.moduli) - 1
    rk = F.RelinearizationKey.new_leveled(gsk, 1, 0, seed_of(rng))
    again = F.RelinearizationKey.from_bytes(gpar, rk.to_bytes())
    for u, v in zip(rk.ksk.arrays(), again.ksk.arrays()):
        assert (u == v).all()
    assert wire.decode_ksk(wire.decode_relinearization_key(rk.to_bytes()))["seed"] == b""
    for c, k in ((0, 0), (last, last)):
        gk = F.GaloisKey.new(gsk, 5, c, k, seed_of(rng))
        back = F.GaloisKey.from_bytes(gpar, gk.to_bytes())
        assert back.exponent == 5 and back.ksk.log_base == gk.ksk.log_base and (gk.ksk.log_base != 0) == (k == last)
        for u, v in zip(gk.ksk.arrays(), back.ksk.arrays()):
            assert (u == v).all()
        # the oracle reads the same words
        ok = oracle.KeySwitchingKey.from_arrays(opar, *gk.ksk.arrays(), c, k)
        assert ok.log_base == gk.ksk.log_base
        up = F.KeySwitchingKey(gpar, *gk.ksk.arrays(), c, k)
        for u, v in zip(gk.ksk.arrays(), up.arrays()):
            assert (u == v).all()
    P = F.PlaintextVec.try_encode(np.arange(16, dtype=np.uint64), F.Encoding.poly(), gpar)
    r = gsk.try_encrypt_rgsw(P, seed_of(rng))[0]
    back = F.RGSWCiphertext.from_bytes(gpar, r.to_bytes())
    for a, b in ((r.ksk0, back.ksk0), (r.ksk1, back.ksk1)):
        for u, v in zip(a.arrays(), b.arrays()):
            assert (u == v).all()


def test_errors(oracle, F):
    from fhe_rs_b200 import _capi
    lib = _capi.lib()
    opar, gpar, rng, osk, gsk = setup(oracle, F, "n16", seed=6)
    n, last = opar.degree, len(opar.moduli) - 1
    seed = seed_of(rng)
    out = C.c_void_p()
    outs = (C.c_void_p * 4)()
    pp = C.cast(outs, C.POINTER(C.c_void_p))

    def relin(c=0, k=0, v=10, s=seed, sk=gsk):
        out.value = None
        r = lib.fhe_b200_relin_key_generate(sk._h if sk else None, c, k, v, s, C.byref(out), None)
        if r != _capi.OK:
            assert out.value is None
        return r

    def galois(es, c=0, k=0, v=10):
        for i in range(4):
            outs[i] = None
        arr = (C.c_uint32 * len(es))(*es)
        r = lib.fhe_b200_galois_keys_generate(gsk._h, arr, len(es), c, k, v, seed, pp, None)
        if r != _capi.OK:
            assert all(outs[i] is None for i in range(4))
        return r

    assert relin() == _capi.OK
    lib.fhe_b200_ksk_free(out)
    assert relin(v=0) == _capi.INVALID_ARGUMENT and b"InvalidVariance" in lib.fhe_b200_last_error()
    assert relin(v=33) == _capi.INVALID_ARGUMENT
    assert relin(s=None) == _capi.INVALID_ARGUMENT
    assert relin(sk=None) == _capi.INVALID_ARGUMENT
    assert relin(0, 1) == _capi.INVALID_LEVEL
    assert relin(last + 1, 0) == _capi.INVALID_LEVEL
    assert relin(last, last) == _capi.UNSUPPORTED and b"KeySwitchingNotSupported" in lib.fhe_b200_last_error()
    assert galois([3, 4]) == _capi.INVALID_EXPONENT
    assert galois([3, 2 * n + 2]) == _capi.INVALID_EXPONENT
    assert galois([3], 0, 1) == _capi.INVALID_LEVEL
    assert galois([3], last, 0) == _capi.OK                   # a single-modulus ciphertext level under a wide key
    lib.fhe_b200_ksk_free(outs[0])
    assert galois([3, 5, 7, 2 * n + 9]) == _capi.OK
    for i in range(4):
        lib.fhe_b200_ksk_free(outs[i])
    P = F.PlaintextVec.try_encode(np.arange(n, dtype=np.uint64), F.Encoding.poly(), gpar)
    other = F.BfvParameters(n, opar.plaintext, moduli=opar.moduli, device=0)
    Po = F.PlaintextVec.try_encode(np.arange(n, dtype=np.uint64), F.Encoding.poly(), other)
    for b, code in ((None, _capi.INVALID_ARGUMENT), (F.Ciphertext(gpar, 1, 2), _capi.INVALID_ARGUMENT),
                    (F.Ciphertext(gpar, 1, 1, repr=F.POWER_BASIS), _capi.INVALID_REPRESENTATION),
                    (Po.batch, _capi.CONTEXT_MISMATCH), (F.Ciphertext(gpar, 1, 1, mul_basis=True), _capi.CONTEXT_MISMATCH)):
        outs[0] = outs[1] = None
        assert lib.fhe_b200_rgsw_encrypt(gsk._h, b._h if b else None, 10, seed, pp, None) == code
        assert outs[0] is None and outs[1] is None
    assert lib.fhe_b200_rgsw_encrypt(gsk._h, P.batch._h, 0, seed, pp, None) == _capi.INVALID_ARGUMENT
    buf = np.zeros(16, np.uint64)
    assert lib.fhe_b200_ksk_download(None, buf.ctypes.data, buf.ctypes.data, None) == _capi.INVALID_ARGUMENT
    with pytest.raises(F.FheError) as e:
        F.GaloisKey.new(gsk, 4)
    assert e.value.code == _capi.INVALID_EXPONENT


def test_no_device_memory_kept(oracle, F):
    """generated keys are the only device memory a call keeps: freeing them gives back what they took, and refused
    calls (levels, exponents, variance) keep nothing.  2^14 x 8 moduli: every key holds 16.8 MB, so one kept key
    would show far above the 8 MB the comparison allows for the driver's own bookkeeping"""
    import torch
    from fhe_rs_b200 import _capi
    lib = _capi.lib()
    opar, gpar, rng, osk, gsk = setup(oracle, F, "n14", seed=8)
    n, last = opar.degree, len(opar.moduli) - 1
    seed = seed_of(rng)
    outs = (C.c_void_p * 8)()
    pp = C.cast(outs, C.POINTER(C.c_void_p))
    exps = (C.c_uint32 * 8)(*[pow(3, i, 2 * n) for i in range(1, 8)], 2 * n - 1)
    P = F.PlaintextVec.try_encode(np.arange(4 * n, dtype=np.uint64), F.Encoding.poly(), gpar)
    bad = (C.c_uint32 * 8)(*[pow(3, i, 2 * n) for i in range(1, 8)], 4)

    def cycle():
        assert lib.fhe_b200_galois_keys_generate(gsk._h, exps, 8, 0, 0, 10, seed, pp, None) == _capi.OK
        for i in range(8):
            lib.fhe_b200_ksk_free(outs[i])
        assert lib.fhe_b200_rgsw_encrypt(gsk._h, P.batch._h, 10, seed, pp, None) == _capi.OK
        for i in range(8):
            lib.fhe_b200_ksk_free(outs[i])
        assert lib.fhe_b200_galois_keys_generate(gsk._h, bad, 8, 0, 0, 10, seed, pp, None) == _capi.INVALID_EXPONENT
        assert lib.fhe_b200_galois_keys_generate(gsk._h, exps, 8, 0, 1, 10, seed, pp, None) == _capi.INVALID_LEVEL
        assert lib.fhe_b200_galois_keys_generate(gsk._h, exps, 8, 0, 0, 0, seed, pp, None) == _capi.INVALID_ARGUMENT
        out = C.c_void_p()
        assert lib.fhe_b200_relin_key_generate(gsk._h, last, last, 10, seed, C.byref(out), None) == _capi.UNSUPPORTED
        assert out.value is None
        assert lib.fhe_b200_sync(None) == _capi.OK
    cycle()                                   # the parameter set's tables and scratch pool are built on first use
    free0 = torch.cuda.mem_get_info()[0]
    for _ in range(5):
        cycle()
    assert abs(torch.cuda.mem_get_info()[0] - free0) < 8 << 20


@pytest.mark.parametrize("streams", ["1", "2", "4"])
def test_keygen_chunking(streams):
    """keys over several chunks on 1, 2 and 4 streams equal the stream's definition"""
    # 20 error rows per chunk: 5 (key, digit) items of the probe's 4-limb keys, so chunks start and end inside keys
    env = dict(os.environ, FHE_B200_CHUNK="20", FHE_B200_STREAMS=streams)
    out = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "keygen_chunk_probe.py")], env=env,
                         capture_output=True, text=True, timeout=600)
    assert out.returncode == 0 and "keygen chunk probe ok" in out.stdout, out.stdout + out.stderr


def test_cpp_keygen(tmp_path, oracle, F):
    """tests/cpp/keygen_test.cpp: keys generated through include/fhe_b200.hpp and serialized through
    include/fhe_b200_wire.hpp are byte for byte the messages of the Python mirror for the same seeds"""
    from fhe_rs_b200 import wire
    opar, gpar, rng, osk, gsk = setup(oracle, F, "setA", seed=9)
    n, t, last = opar.degree, opar.plaintext, len(opar.moduli) - 1
    values = rng.integers(0, t, size=n, dtype=np.uint64)
    seeds = [seed_of(rng) for _ in range(4)]
    (tmp_path / "sk.bin").write_bytes(wire.encode_secret_key([int(c) for c in osk.coeffs]))
    (tmp_path / "seeds.bin").write_bytes(b"".join(seeds))
    values.tofile(str(tmp_path / "values.bin"))
    np.array(opar.moduli, np.uint64).tofile(str(tmp_path / "moduli.bin"))
    exe = str(tmp_path / "keygen_test")
    lib_dir = os.path.join(ROOT, "fhe_rs_b200")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "cpp", "keygen_test.cpp"), "-o", exe,
                           "-L", lib_dir, "-lfhe_b200", "-Wl,-rpath," + lib_dir])
    out = subprocess.run([exe, str(n), str(t), str(tmp_path)], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0 and out.stdout.startswith("OK"), out.stdout + out.stderr
    got = lambda name: (tmp_path / name).read_bytes()  # noqa: E731
    assert got("rk.bin") == F.RelinearizationKey.new(gsk, seeds[0]).to_bytes()
    g3, grow = F.bfv._galois_keys(gsk, [3, 2 * n - 1], 0, 0, seeds[1])
    assert got("gk3.bin") == g3.to_bytes() and got("gk_row.bin") == grow.to_bytes()
    assert got("gk_last.bin") == F.GaloisKey.new(gsk, 2 * n - 1, last, last, seeds[2]).to_bytes()
    P = F.PlaintextVec.try_encode(values, F.Encoding.poly(), gpar)
    assert got("rgsw.bin") == gsk.try_encrypt_rgsw(P, seeds[3])[0].to_bytes()
    # and the messages carry the restated words
    rk = F.RelinearizationKey.from_bytes(gpar, got("rk.bin"))
    check_key(osk, rk.ksk, K.relin_from(osk, 0, 0), seeds[0], 0, 10, False, "cpp relin")


@pytest.mark.parametrize("env", [{"FHE_B200_NTT": "fast"}, {"FHE_B200_GENERIC_NTT": "1"}],
                         ids=lambda e: ",".join("%s=%s" % kv for kv in e.items()))
def test_alternate_code_paths(F, env):
    """the same words under the other NTT implementations"""
    out = subprocess.run([sys.executable, "-m", "pytest", "-q", "-x", "-m", "gpu", "tests/test_gpu_keygen.py",
                          "-k", "test_keygen_parity and (n16 or setA or mixed or q0_barrett) or test_device_keys_compute",
                          "-p", "no:cacheprovider"],
                         cwd=ROOT, env=dict(os.environ, **env), capture_output=True, text=True, timeout=1800)
    assert out.returncode == 0, out.stdout[-2000:] + out.stderr[-2000:]
