"""The server path at large plaintext moduli, device against oracle word for word (bigt_reference.BIGT_SETS): t of 62 to
807 bits, t in the library's own range [2^62, 2^64), a u64 t above q_0, and the levels where Q_l < t, at which the
down scaler's factor t / Q_l is one or more.  The client entry points refuse such a t, so every key comes from the
oracle through from_arrays, and tests/bigt_reference.py (the reference's large-t client) encrypts and decrypts:
  * ct x ct, relinearizes, Multiplicator::default with and without modulus switching, and the fused product with a
    leveled key, at every level (levels 0, 1 and the last at N = 2^15);
  * Multiplicator::new with post factor t / P;
  * the down scaler on crafted ties, sign boundary and wide w sums at level 0 and at the levels with t > Q_l;
  * device products that decrypt to the negacyclic product mod t (biguint.rs: 10 * (t - 20) = t - 200);
  * a set read from a plaintext_big Parameters message;
  * UNSUPPORTED, with device memory unchanged, from every entry point that reads t without a key, and the same words
    as at a small t from those that do not read it.
test_alternate_code_paths reruns the kernel tests under each kernel-selection switch.  Run with `-m gpu`."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

import bigt_reference as R
import edge_inputs as E

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def F():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import fhe_rs_b200
    return fhe_rs_b200


def make(oracle, F, name):
    degree, t, moduli = R.bigt_set(name)
    opar = oracle.BfvParameters(degree, t, moduli=moduli)
    gpar = F.BfvParameters(degree, t, moduli=moduli, device=0)
    assert gpar.mul_basis(0) == opar.level(0).mul_params.to.moduli
    return opar, gpar


def rand_rows(rng, moduli, prefix, degree):
    a = np.zeros(tuple(prefix) + (len(moduli), degree), np.uint64)
    for i, q in enumerate(moduli):
        a[..., i, :] = rng.integers(0, q, size=tuple(prefix) + (degree,), dtype=np.uint64)
    return a


def levels_of(name, n_moduli):
    """every level; at N = 2^15 the first two and the last"""
    return [0, 1, n_moduli - 1] if name == "set_c_near_q" else list(range(n_moduli))


def _products(oracle, F, opar, gpar, level, rng):
    """A * B, rk.relinearizes, Multiplicator::default (with modulus switching when a level is left) with a key at the
    ciphertext's level (when it has two moduli or more) and with a key at level 0, against the oracle"""
    N, L0 = opar.degree, len(opar.moduli)
    mods = opar.context_at_level(level).moduli
    L = len(mods)
    a, b = rand_rows(rng, mods, (1, 2), N), rand_rows(rng, mods, (1, 2), N)
    A, B = F.Ciphertext.from_host(gpar, a, level=level), F.Ciphertext.from_host(gpar, b, level=level)
    oa, ob = oracle.Ciphertext.from_array(opar, a[0], level), oracle.Ciphertext.from_array(opar, b[0], level)
    C3 = A * B
    exp3 = oa.mul(ob)
    assert (C3.to_host()[0] == exp3.to_array()).all(), ("A * B", level)
    for key_level in ([level] if L >= 2 else []) + ([0] if level > 0 else []):
        kc = rand_rows(rng, opar.moduli[:L0 - key_level], (2, L), N)
        ork = oracle.RelinearizationKey.from_ksk(oracle.KeySwitchingKey.from_arrays(opar, kc[0], kc[1], level, key_level))
        grk = F.RelinearizationKey.from_arrays(gpar, kc[0], kc[1], ciphertext_level=level, key_level=key_level)
        assert (grk.relinearizes(C3).to_host()[0] == ork.relinearizes(exp3).to_array()).all(), ("relin", level, key_level)
        for ms in (False, True) if level < L0 - 1 else (False,):
            om, gm = oracle.Multiplicator.default(ork), F.Multiplicator.default(grk)
            if ms:
                om.enable_mod_switching()
                gm.enable_mod_switching()
            got = gm.multiply(A, B).to_host()[0]
            assert (got == om.multiply(oa, ob).to_array()).all(), ("default", level, key_level, ms)


@pytest.mark.parametrize("name", list(R.BIGT_SETS))
def test_products(oracle, F, name):
    opar, gpar = make(oracle, F, name)
    rng = np.random.default_rng(len(name))
    for level in levels_of(name, len(opar.moduli)):
        _products(oracle, F, opar, gpar, level, rng)


@pytest.mark.parametrize("name", ["m127", "tma_200"])
def test_custom_multiplicator(oracle, F, name):
    """Multiplicator::new (mul.rs:37-75) with lhs factor one, rhs factor P / Q and post factor t / P over the moduli
    followed by L extra primes, with and without relinearization and modulus switching"""
    opar, gpar = make(oracle, F, name)
    N, t, mods = opar.degree, opar.plaintext, opar.moduli
    L = len(mods)
    extra, ub = [], 1 << 62
    while len(extra) < L:
        ub = oracle.generate_prime(62, 2 * N, ub)
        if ub not in mods:
            extra.append(ub)
    basis, P, Q = mods + extra, E.product(extra), E.product(mods)
    rng = np.random.default_rng(N)
    a, b = rand_rows(rng, mods, (2, 2), N), rand_rows(rng, mods, (2, 2), N)
    kc = rand_rows(rng, mods, (2, L), N)
    A, B = F.Ciphertext.from_host(gpar, a), F.Ciphertext.from_host(gpar, b)
    ork = oracle.RelinearizationKey.from_ksk(oracle.KeySwitchingKey.from_arrays(opar, kc[0], kc[1]))
    grk = F.RelinearizationKey.from_arrays(gpar, kc[0], kc[1])
    om = oracle.Multiplicator(opar, oracle.ScalingFactor.one(), oracle.ScalingFactor(P, Q), basis,
                              oracle.ScalingFactor(t, P))
    gm = F.Multiplicator.new(F.ScalingFactor.one(), F.ScalingFactor(P, Q), basis, F.ScalingFactor(t, P), gpar)
    for step in ("plain", "relin", "mod_switch"):
        if step == "relin":
            om.enable_relinearization(ork)
            gm.enable_relinearization(grk)
        elif step == "mod_switch":
            om.enable_mod_switching()
            gm.enable_mod_switching()
        got = gm.multiply(A, B).to_host()
        for i in range(2):
            exp = om.multiply(oracle.Ciphertext.from_array(opar, a[i], 0), oracle.Ciphertext.from_array(opar, b[i], 0))
            assert (got[i] == exp.to_array()).all(), (step, i)


@pytest.mark.parametrize("name", list(R.BIGT_SETS))
def test_scaler_edges(oracle, F, name):
    """the down scaler (scale(1)) of level 0 and of every level with t > Q_l on the rounding ties of t x / Q_l, the
    sign boundary QP / 2 and the w sums whose sign sits at bit 191, as test_gpu_edges.test_scaler_edges"""
    opar, gpar = make(oracle, F, name)
    N, t = opar.degree, opar.plaintext
    above = R.levels_t_above_q(t, opar.moduli)
    assert above
    levels = [0] + ([1, len(opar.moduli) - 1] if name == "set_c_near_q" else above)
    for level in levels:
        rng = np.random.default_rng(level + N)
        mp = opar.level(level).mul_params
        Q, QP = mp.frm.modulus(), mp.to.modulus()
        y = E.polys_from_values(E.scaler_near_ties(QP, t, Q, rng, max(4, N // 64)) + E.sign_boundary(QP),
                                mp.to.moduli, N)
        wide = E.wide_w_sums(mp.down_scaler.scaler, mp.to.moduli, rng, 16)
        if wide:
            y = np.concatenate([y, E.polys_from_residues(wide, N)])
        got = F.Ciphertext.from_host(gpar, y[:, None], level=level, repr=F.POWER_BASIS, mul_basis=True)
        got = got.into_ntt().scale(1).into_power_basis().to_host()
        for c in range(len(y)):
            exp = mp.down_scaler.scale(oracle.Poly(mp.to, oracle.POWER_BASIS, y[c].copy())).c
            assert (got[c, 0] == exp).all(), ("down scaler", level, c)


@pytest.mark.parametrize("name", ["m127", "tma_200"])
def test_products_decrypt(oracle, F, name):
    """device products of ciphertexts the big-integer client encrypted decrypt, with that client, to the negacyclic
    product mod t: A * B, relinearized, and Multiplicator::default.  Pair 1 is biguint.rs's 10 * (t - 20) = t - 200."""
    opar, gpar = make(oracle, F, name)
    N, t = opar.degree, opar.plaintext
    rng = np.random.default_rng(t % 1000)
    sk = oracle.SecretKey(opar, rng)
    ork = oracle.RelinearizationKey(sk, rng)
    grk = F.RelinearizationKey.from_arrays(gpar, *ork.ksk.arrays())
    nz = min(N, 16)
    rand = lambda: [int(rng.integers(0, 1 << 62)) * t >> 62 for _ in range(nz)]   # noqa: E731
    msgs = [(rand(), [0] * (N - nz) + rand()), ([10], [t - 20])]
    msgs = [(a + [0] * (N - len(a)), b + [0] * (N - len(b))) for a, b in msgs]
    cts = [(R.encrypt(sk, R.encode(opar, a), 0, rng), R.encrypt(sk, R.encode(opar, b), 0, rng)) for a, b in msgs]
    A = F.Ciphertext.from_host(gpar, np.stack([ca.to_array() for ca, _ in cts]))
    B = F.Ciphertext.from_host(gpar, np.stack([cb.to_array() for _, cb in cts]))
    C3 = A * B
    outs = {"A * B": C3.to_host(), "relinearized": grk.relinearizes(C3).to_host(),
            "default": F.Multiplicator.default(grk).multiply(A, B).to_host()}
    for what, got in outs.items():
        for i, (a, b) in enumerate(msgs):
            dec = R.decode(opar, R.decrypt(sk, oracle.Ciphertext.from_array(opar, got[i], 0)))
            assert dec == R.negacyclic(a, b, t), (what, i)
        assert R.decode(opar, R.decrypt(sk, oracle.Ciphertext.from_array(opar, got[1], 0)))[0] == t - 200


@pytest.mark.parametrize("name", ["m127", "wide_2_62"])
def test_parameters_message(oracle, F, name):
    """a set read from its Parameters message (plaintext_big, bfv.proto:40-48) gives the products of the set built
    directly"""
    from fhe_rs_b200 import wire
    opar, gpar = make(oracle, F, name)
    assert not wire.plaintext_is_small(opar.plaintext)
    back = F.BfvParameters.from_bytes(gpar.to_bytes(), device=0)
    assert back.plaintext() == opar.plaintext and back.moduli() == opar.moduli
    for level in range(len(opar.moduli)):
        _products(oracle, F, opar, back, level, np.random.default_rng(level))


@pytest.mark.parametrize("name", ["m127", "wide_2_62"])
def test_refusals_and_memory(oracle, F, name):
    """Every entry point that reads t and needs no key refuses a t that is not a u64 Modulus with UNSUPPORTED and keeps
    no device memory: secret_key_create and secret_keys_random (so encryption, decryption, measure_noise, key
    generation and the multiparty shares have no key to run with), encode (Poly and SIMD), decode, add_plain_batch,
    encrypt_pk (with and without plaintexts) and decryption_aggregate.  encoder_create runs (its tables are t's only
    when t has an NTT).  fold, mul_plain, mul_plain_batch and add_plain of delta-scaled words do not read t: they give
    the words they give at t = 1153 over the same moduli."""
    import torch
    from fhe_rs_b200 import _capi
    lib = _capi.lib()
    opar, gpar = make(oracle, F, name)
    N = opar.degree
    enc = gpar.encoder()
    seed = bytes(32)
    coeffs = np.zeros(N, np.int64)
    vals = np.zeros(2 * N, np.uint64)
    ct, ct1 = F.Ciphertext(gpar, 2, 2, 0), F.Ciphertext(gpar, 1, 2, 0)
    pt, one = F.Ciphertext(gpar, 2, 1, 0), F.Ciphertext(gpar, 1, 1, 0)
    pk = F.Ciphertext(gpar, 1, 2, 0)
    h, keys = C.c_void_p(), (C.c_void_p * 2)()
    shares = (C.c_void_p * 1)(one._h)

    def refusals():
        return [
            ("secret_key_create", lib.fhe_b200_secret_key_create(gpar._h, coeffs.ctypes.data, C.byref(h))),
            ("secret_keys_random", lib.fhe_b200_secret_keys_random(gpar._h, 2, 10, seed, keys, None)),
            ("encode poly", lib.fhe_b200_encode(enc, _capi.ENCODING_POLY, 0, vals.ctypes.data, 2 * N, pt._h, None)),
            ("encode simd", lib.fhe_b200_encode(enc, _capi.ENCODING_SIMD, 0, vals.ctypes.data, 2 * N, pt._h, None)),
            ("encode signed", lib.fhe_b200_encode(enc, _capi.ENCODING_POLY, 1, vals.ctypes.data, 2 * N, pt._h, None)),
            ("decode", lib.fhe_b200_decode(enc, _capi.ENCODING_POLY, 0, pt._h, vals.ctypes.data, 2 * N, None)),
            ("decode signed", lib.fhe_b200_decode(enc, _capi.ENCODING_POLY, 1, pt._h, vals.ctypes.data, 2 * N, None)),
            ("add_plain_batch", lib.fhe_b200_add_plain_batch(ct._h, pt._h, 0, None)),
            ("sub_plain_batch", lib.fhe_b200_add_plain_batch(ct._h, one._h, 1, None)),
            ("encrypt_pk", lib.fhe_b200_encrypt_pk(pk._h, None, 10, seed, ct._h, None)),
            ("encrypt_pk pts", lib.fhe_b200_encrypt_pk(pk._h, pt._h, 10, seed, ct._h, None)),
            ("decryption_aggregate", lib.fhe_b200_decryption_aggregate(enc, ct1._h, shares, 1, one._h, None)),
        ]
    for what, code in refusals():
        assert code == _capi.UNSUPPORTED, (what, code, lib.fhe_b200_last_error())
    assert h.value is None and keys[0] is None
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    for _ in range(5):
        assert all(code == _capi.UNSUPPORTED for _, code in refusals())
    torch.cuda.synchronize()
    assert abs(torch.cuda.mem_get_info()[0] - free0) < 4 << 20
    # the entry points that do not read t: the same words at t = 1153
    rng = np.random.default_rng(7)
    x, w = rand_rows(rng, opar.moduli, (2, 2), N), rand_rows(rng, opar.moduli, (2,), N)

    def t_free(par):
        X = F.Ciphertext.from_host(par, x)
        pts = F.PlaintextVec(F.Ciphertext.from_host(par, w[:, None]), F.Encoding.poly())
        return [X.fold(62, 40, 0).poly_ntt(), X.clone().mul_plain(w).to_host(), X.clone().add_plain(w).to_host(),
                X.clone().mul_plain(pts).to_host()]
    small = F.BfvParameters(N, 1153, moduli=opar.moduli, device=0)
    for got, exp in zip(t_free(gpar), t_free(small)):
        assert (got == exp).all()


SWITCHES = [{"FHE_B200_KSMAC": "tma"}, {"FHE_B200_KSMAC": "classic"}, {"FHE_B200_SCALER": "classic"},
            {"FHE_B200_NO_SOLINAS": "1"}, {"FHE_B200_SOLINAS_NTT": "1"}, {"FHE_B200_NTT": "fast"}, {"FHE_B200_NTT": "tma"},
            {"FHE_B200_GENERIC_NTT": "1"}]


def test_alternate_code_paths(F):
    """every kernel variant gives the same words at large t: the products, the custom multiplicator and the scaler
    edges rerun under each switch (a switch is read once per process, so each takes a process of its own; the eight
    run side by side).  The N = 2^15 set is left out: test_gpu_edges reruns its kernels at set C's shape."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    cmd = [sys.executable, "-m", "pytest", "-q", "-x", "-m", "gpu", "tests/test_gpu_bigt.py", "-p", "no:cacheprovider",
           "-k", "(test_products or test_custom_multiplicator or test_scaler_edges) and not set_c_near_q"]
    runs = [(env, subprocess.Popen(cmd, cwd=root, env=dict(os.environ, **env), stdout=subprocess.PIPE,
                                   stderr=subprocess.STDOUT, text=True)) for env in SWITCHES]
    failed = []
    try:
        for env, p in runs:
            out = p.communicate(timeout=800)[0]
            if p.returncode != 0:
                failed.append((env, out[-2000:]))
    finally:   # a timeout leaves no process behind
        for _, p in runs:
            if p.poll() is None:
                p.kill()
                p.wait()
    assert not failed, failed
