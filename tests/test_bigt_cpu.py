"""The plaintext-modulus axis on the CPU: the reference's large-t client (tests/bigt_reference.py) against the oracle and
against the literal decryption formula, the exact scaler's rounding envelope at numerators of 63 to 807 bits and at
factors t / Q_l >= 1, and the t-dependent host tables of the parameter builder against the oracle on host-only
parameter sets (device = -1), at every set of bigt_reference.BIGT_SETS and every level."""
import ctypes as C

import numpy as np
import pytest

import bigt_reference as R
import edge_inputs as E
from test_oracle_pinning import _expected_scale, _scale_branch, _windows

M127 = (1 << 127) - 1


@pytest.fixture(scope="module")
def F():
    from fhe_rs_b200 import build
    build.build()
    import fhe_rs_b200
    return fhe_rs_b200


def _m127(oracle):
    """parameters() of biguint.rs:11-23: N = 16, t = 2^127 - 1, five 60-bit moduli"""
    return oracle.BfvParameters(16, M127, moduli_sizes=[60] * 5)


def _one(par, v):
    vals = [0] * par.degree
    vals[0] = v
    return vals


# ----------------------------------------------------------------------------------------------- biguint.rs

def test_biguint_encryption_decryption(oracle):
    """biguint.rs:26-52: 123456789, t - 1 and t / 2 survive encrypt / decrypt / decode"""
    par = _m127(oracle)
    rng = np.random.default_rng(1)
    sk = oracle.SecretKey(par, rng)
    vals = [0] * par.degree
    vals[:3] = [123456789, M127 - 1, M127 // 2]
    ct = R.encrypt(sk, R.encode(par, vals), 0, rng)
    assert R.decode(par, R.decrypt(sk, ct)) == vals


def test_biguint_homomorphic_addition(oracle):
    """biguint.rs:54-88: 10 + (t - 50) = t - 40"""
    par = _m127(oracle)
    rng = np.random.default_rng(2)
    sk = oracle.SecretKey(par, rng)
    c1 = R.encrypt(sk, R.encode(par, _one(par, 10)), 0, rng)
    c2 = R.encrypt(sk, R.encode(par, _one(par, M127 - 50)), 0, rng)
    assert R.decode(par, R.decrypt(sk, c1.add(c2)))[0] == M127 - 40


def test_biguint_multiplication_without_relin(oracle):
    """biguint.rs:90-125: 10 * (t - 20) = t - 200 from the 3-part product"""
    par = _m127(oracle)
    rng = np.random.default_rng(3)
    sk = oracle.SecretKey(par, rng)
    c1 = R.encrypt(sk, R.encode(par, _one(par, 10)), 0, rng)
    c2 = R.encrypt(sk, R.encode(par, _one(par, M127 - 20)), 0, rng)
    prod = c1.mul(c2)
    assert len(prod.c) == 3
    assert R.decode(par, R.decrypt(sk, prod)) == _one(par, M127 - 200)


def test_biguint_multiplication_with_relin(oracle):
    """biguint.rs:127-166: t = 1153, three 62-bit moduli, BigUint inputs 10 and t - 20, relinearized: t - 200.  The
    client takes the small-t branches here, so its ciphertexts and decryptions equal the oracle's own."""
    par = oracle.BfvParameters(16, 1153, moduli_sizes=[62] * 3)
    rng = np.random.default_rng(4)
    sk = oracle.SecretKey(par, rng)
    rk = oracle.RelinearizationKey(sk, rng)
    c1 = R.encrypt(sk, R.encode(par, _one(par, 10)), 0, rng)
    c2 = R.encrypt(sk, R.encode(par, _one(par, 1153 - 20)), 0, rng)
    res = rk.relinearizes(c1.mul(c2))
    assert len(res.c) == 2
    assert R.decode(par, R.decrypt(sk, res))[0] == 1153 - 200
    assert R.decrypt_values(sk, res) == [int(v) for v in sk.decrypt(res)]
    # the restated encryption is the oracle's for a small t (same random stream)
    ra, rb = np.random.default_rng(9), np.random.default_rng(9)
    vals = list(range(16))
    assert (R.encrypt(sk, R.encode(par, vals), 1, ra).to_array() == sk.encrypt(vals, 1, rb).to_array()).all()


def test_small_modulus_with_biguint_input(oracle):
    """biguint.rs:168-195: t = 1153, one 62-bit modulus, the BigUint t + 5 decodes to 5"""
    par = oracle.BfvParameters(16, 1153, moduli_sizes=[62])
    rng = np.random.default_rng(5)
    sk = oracle.SecretKey(par, rng)
    ct = R.encrypt(sk, R.encode(par, _one(par, 1153 + 5)), 0, rng)
    assert R.decode(par, R.decrypt(sk, ct))[0] == 5


def test_signed_encoding(oracle):
    """plaintext.rs:351-372: -1 and -(t - 1) / 2 encode as t - 1 and (t + 1) / 2"""
    par = _m127(oracle)
    pt = R.encode_signed(par, [-1, -(M127 - 1) // 2, 7])
    assert R.decode(par, pt)[:3] == [M127 - 1, (M127 + 1) // 2, 7]


# ------------------------------------------------------------------------------------- two decryptions agree

def _params(oracle, name):
    degree, t, moduli = R.bigt_set(name)
    return oracle.BfvParameters(degree, t, moduli=moduli)


# N = 2^15 costs the oracle seconds per ciphertext: that set is left to the envelope and table tests
@pytest.mark.parametrize("name", [n for n in R.BIGT_SETS if n != "set_c_near_q"])
def test_decryptions_agree(oracle, name):
    """try_decrypt as restated and round(t * phase / Q_l) mod t agree on every coefficient of fresh ciphertexts at
    every level and of products at level 0 (except with a u64 t above q_0, where the reference's decryption departs).  Where Q_l leaves room for the noise, the fresh ciphertexts also decode to
    their messages, and at level 0 of the two sets whose Q exceeds t^2 N 2^10 the product decodes to the negacyclic
    product mod t."""
    par = _params(oracle, name)
    t, N = par.plaintext, par.degree
    rng = np.random.default_rng(N + len(par.moduli))
    sk = oracle.SecretKey(par, rng)
    nz = min(N, 16)
    if R.is_small(t) and t > par.moduli[0]:
        # the `Some` branch keeps limb 0 of the scaled phase only (secret_key.rs:229-238), which loses v >= q_0: the
        # reference's decryption is not round(t phase / Q) there, and this library's client refuses such a t
        ct = R.encrypt(sk, R.encode(par, [t - 1 - k for k in range(N)]), 0, rng)
        assert R.decrypt_values(sk, ct) != R.decrypt_literal(sk, ct)
        return
    for level in range(len(par.moduli)):
        msg = [int(rng.integers(0, 1 << 62)) * t >> 62 for _ in range(nz)] + [0] * (N - nz)
        ct = R.encrypt(sk, R.encode(par, msg, level), level, rng)
        got = R.decrypt_values(sk, ct)
        assert got == R.decrypt_literal(sk, ct), (name, level)
        Q = par.context_at_level(level).modulus()
        if Q > t << 40:
            assert got == msg, (name, level)
    a = [int(rng.integers(0, 1 << 62)) * t >> 62 for _ in range(nz)] + [0] * (N - nz)
    b = [10, t - 20] + [0] * (N - 2)
    ca = R.encrypt(sk, R.encode(par, a), 0, rng)
    cb = R.encrypt(sk, R.encode(par, b), 0, rng)
    prod = ca.mul(cb)
    got = R.decrypt_values(sk, prod)
    assert got == R.decrypt_literal(sk, prod)
    roomy = par.context_at_level(0).modulus() > t * t * N << 10
    assert roomy or name not in ("m127", "tma_200")
    if roomy:
        assert got == R.negacyclic(a, b, t)


# ------------------------------------------------------------------------------------------ rounding envelope

# name -> (parameters, levels): the numerator t has 63 (wide_2_62), 64, 127, 200 and 807 bits; the levels are level 0
# and every level with t > Q_l
def _envelope_cases(oracle):
    out = {}
    for name in R.BIGT_SETS:
        par = _params(oracle, name)
        lv = R.levels_t_above_q(par.plaintext, par.moduli)
        out[name] = (par, [0] + (lv if name != "set_c_near_q" else [1, 7, 13]))
    t64 = R.prime_below(1 << 64)
    par = oracle.BfvParameters(16, t64, moduli_sizes=[62] * 3)
    out["t64"] = (par, [0] + R.levels_t_above_q(t64, par.moduli))
    return out


def test_down_scaler_envelope_at_large_numerators(oracle):
    """The down scaler t / Q_l of the multiplication basis keeps the envelope of test_scaler_rounding_envelope (exact
    centred rounding outside the 2^-40 windows around a tie and around F / 2) at numerators of 63 to 807 bits,
    including every level where t > Q_l, on the crafted ties, sign boundary and wide w sums."""
    seen = {"exact": 0, "tie_plus_one": 0, "other_branch": 0}
    bits = set()
    for name, (par, levels) in _envelope_cases(oracle).items():
        t = par.plaintext
        bits.add(t.bit_length())
        for level in levels:
            mp = par.level(level).mul_params
            sc, frm, to = mp.down_scaler.scaler, mp.to.rns, mp.frm.rns
            QP, Q = frm.product, to.product
            rng = np.random.default_rng(level + t.bit_length())
            xs = E.scaler_near_ties(QP, t, Q, rng) + E.sign_boundary(QP)
            xs += [frm.lift(r) for r in E.wide_w_sums(sc, frm.moduli_u64, rng, 8)]
            for x in xs:
                got = sc.scale_one(frm.project(x), len(to.moduli))
                exp = _expected_scale(x, QP, t, Q, Q)
                if got == to.project(exp % Q):
                    seen["exact"] += 1
                    continue
                near_tie, near_sign = _windows(x, QP, t, Q)
                if near_tie and got == to.project((exp + 1) % Q):
                    seen["tie_plus_one"] += 1
                    continue
                other = _scale_branch(x, QP, t, Q, Q, x < QP // 2)
                assert near_sign and got in (to.project(other % Q), to.project((other + 1) % Q)), \
                    (name, level, x, near_tie, near_sign)
                seen["other_branch"] += 1
    assert bits == {63, 64, 127, 200, 807, 62}
    assert min(seen.values()) > 0, seen   # the crafted inputs reach both departures


# ---------------------------------------------------------------------------------------------- host tables

def _same_tables(tb, sc):
    assert tb["n_from"] == len(sc.frm.moduli) and tb["n_to"] == len(sc.to.moduli)
    assert tb["shift"] == sc.theta_garner_shift
    assert (tb["gamma"] == sc.gamma).all() and (tb["omega"] == sc.omega).all()
    assert (tb["theta_omega_lo"] == sc.theta_omega_lo).all() and (tb["theta_omega_hi"] == sc.theta_omega_hi).all()
    assert (tb["theta_omega_sign"] == sc.theta_omega_sign).all()
    assert (tb["theta_garner_lo"] == sc.theta_garner_lo).all() and (tb["theta_garner_hi"] == sc.theta_garner_hi).all()
    assert [int(x) for x in tb["theta_gamma"]] == [sc.theta_gamma_lo, sc.theta_gamma_hi, int(sc.theta_gamma_sign)]


@pytest.mark.parametrize("name", list(R.BIGT_SETS))
def test_host_tables_match_oracle(oracle, F, name):
    """On a host-only parameter set, at every level: the down scaler t / Q_l (which = 1), the decryption scaler t / Q_l
    into the plaintext context (which = 2, whose n_to is the plaintext context's modulus count) and the delta residues
    (-t)^-1 mod q_i equal the oracle's word for word; q_mod_t is refused where t is not a u64 Modulus."""
    from fhe_rs_b200 import _capi
    lib = _capi.lib()
    degree, t, moduli = R.bigt_set(name)
    opar = oracle.BfvParameters(degree, t, moduli=moduli)
    gpar = F.BfvParameters(degree, t, moduli=moduli, device=-1)
    n_plain = len(opar.plaintext_context.moduli)
    if name in ("m127", "set_c_near_q"):   # bits(t) + 60 spans several moduli
        assert n_plain == {"m127": 4, "set_c_near_q": 14}[name]
    enc = gpar.encoder()
    for level in range(len(moduli)):
        lvl = opar.level(level)
        _same_tables(gpar.scaler_tables(level, 1), lvl.mul_params.down_scaler.scaler)
        plain = gpar.scaler_tables(level, 2)
        assert plain["n_to"] == n_plain
        _same_tables(plain, lvl.scaler.scaler)
        delta = np.zeros(len(moduli) - level, np.uint64)
        assert lib.fhe_b200_debug_encoder_tables(enc, level, None, None, None, None, delta.ctypes.data) == _capi.OK
        assert [int(d) for d in delta] == lvl.delta_rests
        qmt = C.c_uint64()
        code = lib.fhe_b200_debug_encoder_tables(enc, level, None, None, None, C.byref(qmt), None)
        if R.is_small(t):
            assert code == _capi.OK and qmt.value == lvl.q_mod_t
        else:
            assert code == _capi.UNSUPPORTED
    assert lib.fhe_b200_debug_scaler_tables(gpar._h, 0, 3, *([None] * 11)) == _capi.INVALID_ARGUMENT
