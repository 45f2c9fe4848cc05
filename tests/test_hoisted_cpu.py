"""Hoisted rotations without a device: the identity of tests/hoisting_reference.py against the oracle's
GaloisKey.relinearize word for word (every modulus width set, the lazy-bound bases, a leveled key, every odd exponent
at N = 16), the zero predicate that sends an output back to the unhoisted path, and the C ABI symbol, argtypes,
mirrors and argument checks that need no device."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TESTS = os.path.join(ROOT, "tests")
if TESTS not in sys.path:
    sys.path.insert(0, TESTS)

import edge_inputs   # noqa: E402


@pytest.fixture(scope="module")
def H(oracle):
    import hoisting_reference
    return hoisting_reference


def _random_key(O, par, rng, level, key_level):
    ct_mod = par.moduli[:len(par.moduli) - level]
    key_mod = par.moduli[:len(par.moduli) - key_level]
    c = np.zeros((2, len(ct_mod), len(key_mod), par.degree), np.uint64)
    for j, q in enumerate(key_mod):
        c[:, :, j] = rng.integers(0, q, size=(2, len(ct_mod), par.degree), dtype=np.uint64)
    return O.KeySwitchingKey.from_arrays(par, c[0], c[1], level, key_level)


def _galois_key(O, ksk, e):
    g = O.GaloisKey.__new__(O.GaloisKey)
    g.exponent, g.ksk = e % (2 * ksk.par.degree), ksk
    return g


def _ct(O, par, rng, level, c1_power=None):
    """a random 2-part NTT ciphertext; c1 given in power basis when c1_power is not None"""
    ctx = par.context_at_level(level)
    c0 = O.Poly.random(ctx, O.NTT, rng)
    c1 = O.Poly.random(ctx, O.NTT, rng) if c1_power is None else O.Poly(ctx, O.POWER_BASIS, c1_power).into_ntt()
    return O.Ciphertext(par, [c0, c1], level)


def _check(O, H, par, exponents, level=0, key_level=0, seed=1, c1_power=None):
    """every exponent: hoisted == GaloisKey.relinearize, from one digit decomposition; returns the exponents whose
    outputs differ"""
    rng = np.random.default_rng(seed)
    ksk = _random_key(O, par, rng, level, key_level)
    ct = _ct(O, par, rng, level, c1_power)
    D = H.digits(ksk, ct.c[1].copy().into_power_basis())
    differ = []
    for e in exponents:
        g = _galois_key(O, ksk, e)
        if not (H.hoisted_relinearize(g, ct, D).to_array() == g.relinearize(ct).to_array()).all():
            differ.append(e)
    return differ


def _some_exponents(degree):
    return [3, 5, 7, 9, degree + 1, 2 * degree - 1, pow(3, 5, 2 * degree)]


@pytest.mark.parametrize("degree,sizes", [(16, [62, 62, 62]), (64, [62, 62, 62]), (16, [62, 40, 30]),
                                          (64, [62, 40, 30])])
def test_identity_equals_relinearize(oracle, H, degree, sizes):
    par = oracle.BfvParameters(degree, 1153 if degree == 16 else 257, moduli_sizes=sizes)
    assert _check(oracle, H, par, _some_exponents(degree), seed=degree) == []


@pytest.mark.parametrize("name", sorted(n for n in edge_inputs.WIDTH_SETS if edge_inputs.WIDTH_SETS[n][0] == 64))
def test_identity_at_every_width(oracle, H, name):
    degree, t, sizes = edge_inputs.WIDTH_SETS[name]
    par = oracle.BfvParameters(degree, t, moduli_sizes=sizes)
    assert _check(oracle, H, par, [3, 2 * degree - 1, degree + 1], seed=len(sizes)) == []


@pytest.mark.parametrize("name", ["unreduced", "reduced", "reduced_8x"])
def test_identity_at_the_lazy_bounds(oracle, H, name):
    """digits that reach (or pass) 4 q_j go through the transform unreduced or reduced as in the reference"""
    degree = 16
    moduli = edge_inputs.lazy_bound_bases(degree)[name]
    par = oracle.BfvParameters(degree, 257, moduli=moduli)
    top = np.array([[q - 1] * degree for q in moduli], np.uint64)   # all-(q_i - 1) digits
    assert _check(oracle, H, par, [3, 2 * degree - 1], c1_power=top) == []
    assert _check(oracle, H, par, [3, 2 * degree - 1], seed=2) == []


def test_identity_with_a_leveled_key(oracle, H):
    """ciphertext level 1, key level 0: Lk = L + 1 limbs, then the reference's switch down"""
    for degree in (16, 32):
        par = oracle.BfvParameters(degree, 257, moduli_sizes=[62, 62, 62])
        assert _check(oracle, H, par, _some_exponents(degree), level=1, key_level=0, seed=degree) == []


def test_identity_for_every_odd_exponent(oracle, H):
    degree = 16
    par = oracle.BfvParameters(degree, 1153, moduli_sizes=[62, 62, 62])
    assert _check(oracle, H, par, range(1, 2 * degree, 2), seed=3) == []


def test_zero_predicate(oracle, H):
    """zeros at s = 0 never send an output back; a zero at s sends back exactly the exponents that negate s, and the
    identity fails for exactly those; c1 = 0 sends back every exponent but 1"""
    degree = 16
    par = oracle.BfvParameters(degree, 1153, moduli_sizes=[62, 62, 62])
    rng = np.random.default_rng(5)
    odd = list(range(1, 2 * degree, 2))
    rows = np.stack([rng.integers(1, q, degree, dtype=np.uint64) for q in par.moduli])
    assert not any(H.needs_fallback(rows, e) for e in odd)
    r0 = rows.copy()
    r0[:, 0] = 0
    assert not any(H.needs_fallback(r0, e) for e in odd)
    assert _check(oracle, H, par, odd, c1_power=r0) == []
    for s, k in ((5, 1), (1, 0), (degree - 1, 2)):
        rs = rows.copy()
        rs[k, s] = 0
        want = [e for e in odd if H.negates(degree, e, s)]
        assert [e for e in odd if H.needs_fallback(rs, e)] == want
        assert 0 < len(want) < len(odd)
        assert _check(oracle, H, par, odd, c1_power=rs) == want, s
    zero = np.zeros_like(rows)
    assert [e for e in odd if H.needs_fallback(zero, e)] == odd[1:]
    assert H.hoisted_count([rows, zero], [3, 5, 1, 3], [0, 0, 1, 1]) == 3
    assert H.hoisted_count([rows, zero], [3, 5, 3], [0, 1, 1]) == 0


@pytest.fixture(scope="module")
def F():
    from fhe_rs_b200 import build
    build.build()
    import fhe_rs_b200
    return fhe_rs_b200


def test_symbol_and_argtypes(F):
    from fhe_rs_b200 import _capi
    lib = _capi.lib()
    u32, pu32, pp, vp = C.c_uint32, C.POINTER(C.c_uint32), C.POINTER(C.c_void_p), C.c_void_p
    f = lib.fhe_b200_galois_many_hoisted
    assert f.restype is C.c_int and list(f.argtypes) == [vp, pu32, pp, pu32, u32, pu32, vp, pu32, vp]
    assert callable(F.galois_many_hoisted) and "galois_many_hoisted" in F.bfv.__all__
    assert callable(F.EvaluationKey.rotates_columns_by_many_hoisted)


def test_argument_checks(F):
    """NULL batches, key lists, exponent lists and indices and no keys: INVALID_ARGUMENT, n_hoisted left as it was"""
    from fhe_rs_b200 import _capi
    lib, bad = _capi.lib(), _capi.INVALID_ARGUMENT
    one = (C.c_uint32 * 1)(0)
    three = (C.c_uint32 * 1)(3)
    keys = (C.c_void_p * 1)(None)
    kp = C.cast(keys, C.POINTER(C.c_void_p))
    n_h = C.c_uint32(77)
    for n_keys, k, ex, ix in ((1, None, three, one), (0, kp, three, one), (1, kp, None, one), (1, kp, three, None),
                              (1, kp, three, one)):
        for src in (None, one):
            for nh in (None, C.byref(n_h)):
                assert lib.fhe_b200_galois_many_hoisted(None, src, k, ex, n_keys, ix, None, nh, None) == bad
    assert n_h.value == 77
    assert b"null" in lib.fhe_b200_last_error()


class _Batch:
    """what the mirrors read of a batch before they reach the device"""

    def __init__(self, par, count):
        self.par, self.count, self.level, self.stream = par, count, 0, 0

    def __len__(self):
        return 2


def test_mirrors_check_lengths_and_keys(F):
    """one key index per output, sources in range, and an EvaluationKey that supports every rotation, checked before
    the library is called"""
    from fhe_rs_b200 import _capi
    par = F.BfvParameters(16, 1153, moduli_sizes=[62, 62], device=-1)
    ct = _Batch(par, 3)
    ek = F.EvaluationKey(par)
    for call in (lambda: F.galois_many_hoisted(ct, [], [0, 0]),
                 lambda: F.galois_many_hoisted(ct, [], [0, 0, 0], [0, 1]),
                 lambda: F.galois_many_hoisted(ct, [], [0], [-1]),
                 lambda: ek.rotates_columns_by_many_hoisted(ct, [1, 2])):
        with pytest.raises(F.FheError) as e:
            call()
        assert e.value.code == _capi.INVALID_ARGUMENT
