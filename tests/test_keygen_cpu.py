"""CPU tests of key generation's host side: the stream's key rows, the device's closed form of the switch-up and of
the gadget table against the oracle's Switcher and Garner coefficients, the restated keys' algebra and function, the
EvaluationKeyBuilder index sets and the refusals that need no device."""
import ctypes as C
import os
import re
import types

import numpy as np
import pytest

import encrypt_reference as R
import keygen_reference as K

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def F():
    import fhe_rs_b200
    return fhe_rs_b200


def test_key_rows_use_words_13_to_15():
    """block b of the row (key k, role, limb j, digit i) is the block of (b, k, role << 8 | j, i)"""
    seed = bytes(range(7, 39))
    for role in (K.ROLE_C1, K.ROLE_KEY_E):
        lo, hi = K.row_values(seed, 3, role, [0, 2], 5, 64)
        for b in (0, 9, 15):
            for r, j in enumerate((0, 2)):
                words = np.frombuffer(R.chacha20_block(seed, b, 3, (role << 8) | j, 5), "<u8")
                for m in range(4):
                    assert lo[r, 4 * b + m] == words[2 * m] and hi[r, 4 * b + m] == words[2 * m + 1]
    # digit 0 of a key row is the encryption row of the same (index, role, limb): word 15 = 0 leaves roles 0-4 as they
    # were, and distinct digits give distinct rows
    assert (K.row_values(seed, 4, 1, [0], 0, 64)[0] == R.row_values(seed, 4, 1, [0], 64)[0]).all()
    assert (K.row_values(seed, 4, K.ROLE_C1, [0], 1, 64)[0] != K.row_values(seed, 4, K.ROLE_C1, [0], 0, 64)[0]).all()


def test_encryption_rows_unchanged():
    """RFC 8439 words of an encryption row do not depend on the key roles: word 15 is 0"""
    seed = bytes(range(32))
    a = R.row_values(seed, 2, R.ROLE_A, [1], 32)
    blk = np.frombuffer(R.chacha20_block(seed, 3, 2, (R.ROLE_A << 8) | 1, 0), "<u8")
    assert a[0][0, 12] == blk[0] and a[1][0, 12] == blk[1]


# the shapes of tests/test_gpu_keygen.py: (degree, moduli sizes or an edge_inputs.CLIENT_SHAPES name)
SHAPES = {
    "n16": (16, [62, 62, 62]),
    "setA": (16, [62, 62]),
    "n14": (16, [62] * 8),
    "setC": (16, [62] * 14),
    "mixed": (16, [62, 30, 50]),
    "q0_barrett": (16, "q0_barrett"),
    "q0_above_2_61": (16, "q0_above_2_61"),
    "q0_solinas_max_c": (16, "q0_solinas_max_c"),
    "q1_barrett": (16, "q1_barrett"),
    "l31": (16, "l31"),
}


def shape_params(oracle, name):
    import edge_inputs as E
    degree, spec = SHAPES[name]
    moduli = E.client_moduli(spec) if isinstance(spec, str) else oracle.BfvParameters.generate_moduli(spec, 1 << 13)
    # the moduli of the GPU shapes (degree 2^13 or above) are NTT-friendly for every smaller power of two
    return oracle.BfvParameters(degree, 1153 if degree == 16 else 786433, moduli=moduli)


@pytest.mark.parametrize("name", list(SHAPES))
def test_switch_up_closed_form(oracle, name):
    """Switcher(ctx_ct, ctx_key).switch(x) equals x (Q_key / Q_ct) on the ciphertext limbs and 0 on the others, for
    every level pair, random rows and the rows around floor(Q_ct / 2)"""
    par = shape_params(oracle, name)
    rng = np.random.default_rng(len(par.moduli))
    last = len(par.moduli) - 1
    pairs = [(c, k) for c in range(last + 1) for k in range(c + 1)]
    if len(pairs) > 40:
        pairs = [(c, k) for (c, k) in pairs if c in (0, 1, 2, last - 1, last) or k in (0, c)]
    for c, k in pairs:
        ctx_ct, ctx_key = par.context_at_level(c), par.context_at_level(k)
        Q = ctx_ct.modulus()
        specials = [Q // 2, Q // 2 + 1, Q // 2 - 1, 0, 1, Q - 1]
        vals = [int(v) for v in rng.integers(0, 1 << 62, par.degree - len(specials), dtype=np.uint64)] + specials
        vals = [v % Q for v in vals]
        x = oracle.Poly(ctx_ct, oracle.POWER_BASIS)
        for j, q in enumerate(ctx_ct.moduli):
            x.c[j] = np.array([v % q for v in vals], dtype=np.uint64)
        want = oracle.Switcher(ctx_ct, ctx_key).switch(x.copy()).into_ntt()
        got = K.switch_up_closed_form(x.copy().into_ntt(), ctx_key)
        assert (got.c == want.c).all(), (name, c, k)


@pytest.mark.parametrize("name", ["n16", "mixed", "l31"])
def test_gadget_table(oracle, name):
    """g_i mod q_j is δ_ij on the ciphertext limbs (so G[i][j] = δ_ij P mod q_j with the switched-up x); the
    decomposition digits are powers of two"""
    par = shape_params(oracle, name)
    last = len(par.moduli) - 1
    for c in range(last):
        g = K.gadget(par, c, 0)
        for i, gi in enumerate(g):
            for j, q in enumerate(par.context_at_level(c).moduli):
                assert gi % q == (1 if i == j else 0)
    log_base, n_dec = oracle._ksk_log_base(par.context_at_level(last))
    assert K.gadget(par, last, last) == [1 << (i * log_base) for i in range(n_dec)]
    assert log_base * n_dec >= (par.moduli[0] - 1).bit_length() and n_dec in (2, 3)


def _algebra(oracle, osk, ksk, frm):
    """c0_i + c1_i s = e_i + g_i from, e_i small"""
    par = osk.par
    s = osk.s_ntt(ksk.ctx_ksk)
    for i, g in enumerate(K.gadget(par, ksk.ciphertext_level, ksk.ksk_level)):
        e = ksk.c0[i].copy()
        e.rep = oracle.NTT
        e.iadd(oracle.Poly(ksk.ctx_ksk, oracle.NTT, ksk.c1[i].c.copy()).mul(s))
        e = e.into_power_basis().isub(frm.mul_scalar_big(g))
        q0 = ksk.ctx_ksk.moduli[0]
        x = np.array([int(v) - q0 if int(v) > q0 // 2 else int(v) for v in e.c[0]], np.int64)
        assert np.abs(x).max() <= 2 * par.variance


def test_restated_keys(oracle):
    """the restated relinearization, Galois and RGSW keys satisfy the key equation and work on oracle ciphertexts"""
    par = oracle.BfvParameters(16, 1153, moduli_sizes=[62, 62, 62])
    rng = np.random.default_rng(5)
    osk = oracle.SecretKey(par, rng)
    seed = bytes(range(32))
    t, n = par.plaintext, par.degree
    for c, k in ((0, 0), (1, 0), (1, 1)):
        rk = K.relinearization_key(osk, seed, c, k, 10)
        ctx_ct, ctx_rk = par.context_at_level(c), par.context_at_level(k)
        s = osk.s_ntt(ctx_ct)
        _algebra(oracle, osk, rk.ksk, oracle.Switcher(ctx_ct, ctx_rk).switch(s.mul(s).into_power_basis()))
        x, y = rng.integers(0, t, n), rng.integers(0, t, n)
        a, b = osk.encrypt(x, c, rng), osk.encrypt(y, c, rng)
        prod = rk.relinearizes(a.mul(b))
        want = np.zeros(n, dtype=object)
        for i in range(n):
            for j in range(n):
                sgn = 1 if i + j < n else -1
                want[(i + j) % n] += sgn * int(x[i]) * int(y[j])
        assert (osk.decrypt(prod).astype(object) == want % t).all()
    last = len(par.moduli) - 1
    for c, k in ((0, 0), (2, 1), (last, last)):
        gk = K.galois_keys(osk, [2 * n - 1], seed, c, k, 10)[0]
        x = rng.integers(0, t, n)
        rot = gk.relinearize(osk.encrypt(x, c, rng))
        want = oracle.Poly.from_i64(oracle.Context([t], n), np.array([int(v) for v in x], np.int64)).substitute(2 * n - 1)
        assert (osk.decrypt(rot) == want.c[0]).all()
    for level in (0, last):
        m = rng.integers(0, t, n)
        mp = oracle.Poly.from_u64(par.context_at_level(level), m.astype(np.uint64), oracle.NTT)
        r = K.rgsw(osk, [mp], level, seed, 10)[0]
        y = rng.integers(0, t, n)
        got = osk.decrypt(r.external_product(osk.encrypt(y, level, rng))).astype(object)
        want = np.zeros(n, dtype=object)
        for i in range(n):
            for j in range(n):
                want[(i + j) % n] += (1 if i + j < n else -1) * int(m[i]) * int(y[j])
        assert (got == want % t).all()


def test_evaluation_key_builder_index_sets(F, oracle):
    """EvaluationKeyBuilder's exponents (evaluation_key.rs:439-463) and its refusals, on host-only parameters"""
    from fhe_rs_b200 import _capi
    n = 16
    gpar = F.BfvParameters(n, 1153, moduli=oracle.BfvParameters(n, 1153, moduli_sizes=[62, 62]).moduli, device=-1)
    sk = types.SimpleNamespace(par=gpar)          # the builder reads only the parameters until build()
    b = F.EvaluationKeyBuilder(sk)
    assert b.exponents() == []
    assert b.enable_inner_sum().exponents() == K.evaluation_key_exponents(n, inner_sum=True) == sorted({31, 3, 9, 81 % 32})
    assert F.EvaluationKeyBuilder(sk).enable_row_rotation().exponents() == [2 * n - 1]
    assert F.EvaluationKeyBuilder(sk).enable_expansion(4).exponents() == [3, 5, 9, 17]
    b = F.EvaluationKeyBuilder(sk).enable_column_rotation(1).enable_column_rotation(7).enable_expansion(2)
    assert b.exponents() == K.evaluation_key_exponents(n, expansion_level=2, column_rotation=(1, 7))
    for bad in (0, n // 2):
        with pytest.raises(F.FheError) as e:
            F.EvaluationKeyBuilder(sk).enable_column_rotation(bad)
        assert e.value.code == _capi.INVALID_ARGUMENT
    with pytest.raises(F.FheError) as e:
        F.EvaluationKeyBuilder(sk).enable_expansion(5)
    assert e.value.code == _capi.INVALID_LEVEL
    for c, k in ((2, 0), (0, 1)):
        with pytest.raises(F.FheError) as e:
            F.EvaluationKeyBuilder.new_leveled(sk, c, k)
        assert e.value.code == _capi.INVALID_LEVEL
    assert F.EvaluationKeyBuilder.new_leveled(sk, 1, 0).ciphertext_level == 1


def test_refusals_without_a_device(F, oracle):
    from fhe_rs_b200 import _capi
    lib = _capi.lib()
    seed = bytes(32)
    out = C.c_void_p()
    outs = (C.c_void_p * 2)()
    pp = C.cast(outs, C.POINTER(C.c_void_p))
    exps = (C.c_uint32 * 2)(3, 5)
    for v in (0, 33):
        assert lib.fhe_b200_relin_key_generate(None, 0, 0, v, seed, C.byref(out), None) == _capi.INVALID_ARGUMENT
        assert b"InvalidVariance" in lib.fhe_b200_last_error()
        assert lib.fhe_b200_galois_keys_generate(None, exps, 2, 0, 0, v, seed, pp, None) == _capi.INVALID_ARGUMENT
        assert lib.fhe_b200_rgsw_encrypt(None, None, v, seed, pp, None) == _capi.INVALID_ARGUMENT
    assert lib.fhe_b200_relin_key_generate(None, 0, 0, 10, seed, C.byref(out), None) == _capi.INVALID_ARGUMENT
    assert lib.fhe_b200_galois_keys_generate(None, exps, 2, 0, 0, 10, seed, pp, None) == _capi.INVALID_ARGUMENT
    assert lib.fhe_b200_rgsw_encrypt(None, None, 10, seed, pp, None) == _capi.INVALID_ARGUMENT
    buf = np.zeros(16, np.uint64)
    assert lib.fhe_b200_ksk_download(None, buf.ctypes.data, buf.ctypes.data, None) == _capi.INVALID_ARGUMENT
    # a seed of another length through the Python API
    gpar = F.BfvParameters(16, 1153, moduli=oracle.BfvParameters(16, 1153, moduli_sizes=[62, 62]).moduli, device=-1)
    with pytest.raises(F.FheError) as e:
        F.RelinearizationKey.new(types.SimpleNamespace(par=gpar, _h=None), b"short")
    assert e.value.code == _capi.INVALID_ARGUMENT


def test_symbols_declared_and_bound():
    """the four new entry points are in the header, in the ctypes table and exported by the library"""
    from fhe_rs_b200 import _capi
    header = open(os.path.join(ROOT, "include", "fhe_b200.h")).read()
    names = ["fhe_b200_relin_key_generate", "fhe_b200_galois_keys_generate", "fhe_b200_rgsw_encrypt",
             "fhe_b200_ksk_download"]
    for name in names:
        assert re.search(r"\bint %s\(" % name, header), name
        assert name in _capi.SYMBOLS
        assert hasattr(_capi.lib(), name)
    argc = {n: len(re.search(r"\bint %s\(([^)]*)\)" % n, header).group(1).split(",")) for n in names}
    for n in names:
        assert argc[n] == len(_capi.SYMBOLS[n][1]), n
