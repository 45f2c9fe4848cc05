"""CPU checks behind tests/test_gpu_client_edges.py: the oracle's decryption rounds the crafted phases exactly except
inside the reference's two 2^-40 windows (and the crafted phases do reach both windows), the plain-integer noise rule
used for single-coefficient phases equals the oracle's measure_noise, and the generators of tests/edge_inputs.py
produce the points they promise."""
import numpy as np
import pytest

import edge_inputs as E


def client_levels(name, L):
    return (0, 15, 30) if name == "l31" else range(L)


def phase_words(oracle, par, level, polys):
    """[count][2][L][N] NTT words of the ciphertexts c1 = 0, c0 = NTT(polys[k]): the phase is polys[k]"""
    ctx = par.context_at_level(level)
    c0 = np.stack([oracle.Poly(ctx, oracle.POWER_BASIS, p.copy()).into_ntt().c for p in polys])
    return np.stack([c0, np.zeros_like(c0)], axis=1)


def _scale(x, Q, t, Qp, negative):
    """rns/scaler.rs:397-414 (exact centred rounding of t x / Q into [0, Qp)) with the sign branch given"""
    if negative:
        r = ((Q - x) * t + ((Q >> 1) - 1 if Q % 2 == 0 else Q >> 1)) // Q
        return (Qp - r % Qp) % Qp
    return ((x * t + (Q >> 1)) // Q) % Qp


@pytest.mark.parametrize("shape", list(E.CLIENT_SHAPES))
def test_decrypt_rounding_envelope(oracle, shape):
    """SecretKey::decrypt of c1 = 0 ciphertexts whose phase sits at the ties of t x / Q, at Q / 2 and at
    Delta m +/- Q / 2t: ((v + t) mod q_0) mod t with v = round(t x / Q), except inside the two windows of the fixed-point
    scaler -- t x / Q within 2^-40 of a half-integer (v may be one larger) and x within 2^-40 Q of Q / 2 (v may come
    from the other sign branch, possibly plus one).  Every (t, level) whose Q is large enough for the windows to hold
    an integer reaches both, so the device test on the same phases checks the decisions themselves."""
    degree, _ = E.CLIENT_SHAPES[shape]
    moduli = E.client_moduli(shape)
    q0 = moduli[0]
    for tname, t in E.client_plaintexts(degree, moduli).items():
        par = oracle.BfvParameters(degree, t, moduli=moduli)
        Qp = par.plaintext_context.modulus()
        sk = oracle.SecretKey(par, np.random.default_rng(0))
        rng = np.random.default_rng(degree + t % 1000)

        def epilogue(v):
            return ((v % Qp % q0) + t) % q0 % t
        for level in client_levels(shape, len(moduli)):
            ctx = par.context_at_level(level)
            Q = ctx.modulus()
            xs = E.decrypt_phases(Q, t, rng, 4 if degree < 1 << 12 else 64)
            polys = E.polys_from_values(xs, ctx.moduli, degree)
            words = phase_words(oracle, par, level, polys)
            got = np.concatenate([sk.decrypt(oracle.Ciphertext.from_array(par, w, level)) for w in words])
            reached = {"tie": 0, "sign": 0}
            for i, x in enumerate(xs):
                g = int(got[i])
                assert g == E.decrypt_one(par, level, x), (tname, level, x)
                negative = x >= Q >> 1
                near_tie, near_sign = E.decrypt_windows(x, Q, t)
                reached["tie"] += near_tie
                reached["sign"] += near_sign
                exp = _scale(x, Q, t, Qp, negative)
                if g == epilogue(exp):
                    continue
                if near_tie and g == epilogue(exp + 1):
                    continue
                other = _scale(x, Q, t, Qp, not negative)
                assert near_sign and g in (epilogue(other), epilogue(other + 1)), (tname, level, x)
            if t << 42 < Q:
                assert reached["tie"] > 0 and reached["sign"] > 0, (tname, level, reached)


@pytest.mark.parametrize("shape", ["n16_l5", "ten_bit"])
def test_single_coefficient_noise_rule(oracle, shape):
    """E.noise_one (plain integers around the oracle's scaler) equals SecretKey::measure_noise on c1 = 0 ciphertexts
    whose phase has one nonzero coefficient: the word boundaries of Q, Q / 2 both ways and decryption-boundary
    phases"""
    degree, _ = E.CLIENT_SHAPES[shape]
    moduli = E.client_moduli(shape)
    par = oracle.BfvParameters(degree, 1153, moduli=moduli)
    sk = oracle.SecretKey(par, np.random.default_rng(1))
    rng = np.random.default_rng(2)
    for level in range(len(moduli)):
        ctx = par.context_at_level(level)
        Q = ctx.modulus()
        xs = E.noise_points(Q) + E.decrypt_phases(Q, 1153, rng)[::5]
        for i, x in enumerate(xs):
            poly = np.zeros((len(ctx.moduli), degree), np.uint64)
            poly[:, (7 * i) % degree] = [x % q for q in ctx.moduli]
            w = phase_words(oracle, par, level, poly[None])[0]
            assert E.noise_one(par, level, x) == sk.measure_noise(oracle.Ciphertext.from_array(par, w, level)), x


def test_generators():
    """the edge generators give what their docstrings promise"""
    Q = (1 << 129) + 51
    pts = E.noise_points(Q)
    for k in (64, 128):
        assert {(1 << k) - 1, 1 << k, (1 << k) + 1, Q - (1 << k)} <= set(pts)
    assert Q // 2 in pts and (Q + 1) // 2 in pts and all(0 <= x < Q for x in pts)
    t = 1153
    xs = E.decrypt_phases(Q, t, np.random.default_rng(0))
    delta, half = Q // t, Q // (2 * t)
    for m in (0, 1, t // 2, t - 1):
        assert (delta * m + half) % Q in xs and (delta * m - half) % Q in xs
    keys = E.key_extremes(64, (1 << 62) - 57, np.random.default_rng(0))
    assert keys["minus_one"][0] == -1 and not keys["minus_one"][1:].any()
    ex = set(keys["extremes"].tolist())
    assert {np.iinfo(np.int64).min, np.iinfo(np.int64).max, (1 << 62) - 58, -((1 << 62) - 57)} <= ex
    moduli = [(1 << 62) - 57, 786433]
    ts = E.client_plaintexts(1 << 12, moduli)
    assert ts["below_q0"] < moduli[0] <= ts["max"] < 1 << 62
