"""Device against oracle at the edges of the arithmetic, word for word, through the C ABI.

The parity suite (test_gpu_parity.py) feeds uniform random residues or fresh encryptions; these tests feed the inputs
where fixed-point and lazy arithmetic make their decisions (tests/edge_inputs.py):
  * the exact scaler's rounding ties and sign boundary, on every scaler kernel (scale_small_kernel for N < 128,
    scale_tma_kernel when every output limb is a Solinas prime, scale_kernel otherwise), and switch_down's ties;
  * extreme residues (all q - 1 and friends) through the NTT families, the key switch, the tensor product, the dot
    product and the plaintext operations, which drive every lazy sum to its maximum;
  * boundary primes: the Solinas prime with the largest c, the smallest 62-bit prime that is not Solinas (a Barrett
    limb next to Solinas limbs), a prime just above 2^61, and a 10-bit modulus;
  * the largest shapes: 31 moduli (63-limb multiplication basis, theta_garner_shift 123), a 64-limb custom basis, and
    N = 2^16.
test_alternate_code_paths reruns the module under each kernel-selection switch.  Run with `-m gpu`."""
import os
import subprocess
import sys

import numpy as np
import pytest

import edge_inputs as E

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def F():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import fhe_rs_b200
    return fhe_rs_b200


def make(oracle, F, degree, t, sizes=None, moduli=None):
    opar = oracle.BfvParameters(degree, t, moduli=moduli, moduli_sizes=sizes)
    gpar = F.BfvParameters(degree, t, moduli=opar.moduli, device=0)
    assert gpar.mul_basis(0) == opar.level(0).mul_params.to.moduli
    return opar, gpar


def rand_rows(rng, moduli, prefix, degree):
    a = np.zeros(tuple(prefix) + (len(moduli), degree), np.uint64)
    for i, q in enumerate(moduli):
        a[..., i, :] = rng.integers(0, q, size=tuple(prefix) + (degree,), dtype=np.uint64)
    return a


def max_rows(moduli, prefix, degree):
    """every word q - 1"""
    q = np.array(moduli, dtype=np.uint64)[:, None] - np.uint64(1)
    return np.ascontiguousarray(np.broadcast_to(q, tuple(prefix) + (len(moduli), degree)))


def gen62(degree, k, skip=()):
    """the k-th 62-bit NTT-friendly prime below 2^62 (the generator's order), skipping `skip`"""
    import fhe_oracle as O
    out, ub = [], 1 << 62
    while len(out) <= k:
        ub = O.generate_prime(62, 2 * degree, ub)
        if ub not in skip:
            out.append(ub)
    return out[k]


# -------------------------------------------------------------------------------------------------------- scalers

# name -> (degree, t, moduli sizes or explicit moduli)
SCALER_SETS = {
    "n16_l5": (16, 1153, [62] * 5),                       # scale_small_kernel
    "set_a": (1 << 12, 1032193, [62] * 2),                # TMA scaler
    "set_c": (1 << 15, 786433, [62] * 14),                # TMA scaler, extension 14 -> 15, down 29 -> 14
    "mixed_13": (1 << 13, 786433, [62, 40, 30]),          # down scaler -> scale_kernel (outputs not all Solinas)
    "l31_13": (1 << 13, 786433, [62] * 31),               # down 63 -> 31, theta_garner_shift 123
    "bp_13": (1 << 13, 786433, "boundary"),               # Barrett 62-bit limb next to Solinas limbs
    "bp_sol_15": (1 << 15, 786433, "boundary_solinas"),   # the largest-c Solinas prime, TMA scaler
    "bp_wide_13": (1 << 13, 786433, "boundary_wide"),     # scale_kernel with 45 source limbs: w sums past 2^190
    "ten_bit_64": (64, 17, [62, 62, 10]),                 # a 10-bit modulus
}


def boundary_moduli(kind, degree):
    bp = [E.BOUNDARY_PRIMES[k] for k in ("solinas_max_c", "non_solinas_min", "above_2_61")]
    if kind == "boundary":
        return [gen62(degree, 0)] + bp
    if kind == "boundary_wide":   # 22 moduli
        return [gen62(degree, 0)] + bp + [gen62(degree, k) for k in range(1, 19)]
    return [E.BOUNDARY_PRIMES["solinas_max_c"], gen62(degree, 0), gen62(degree, 1)]


def make_set(oracle, F, name):
    degree, t, spec = SCALER_SETS[name]
    if isinstance(spec, str):
        return make(oracle, F, degree, t, moduli=boundary_moduli(spec, degree))
    return make(oracle, F, degree, t, sizes=spec)


@pytest.mark.parametrize("name", list(SCALER_SETS))
def test_scaler_edges(oracle, F, name):
    """Extender (scale(0)) and down scaler (scale(1)) of the multiplication basis on crafted power-basis inputs --
    rounding ties of t x / Q, the sign boundary QP / 2, the extender's (Q +/- 1) / 2 -- transformed on the device,
    scaled, transformed back: equal to the oracle's Scaler on the same polynomials."""
    opar, gpar = make_set(oracle, F, name)
    rng = np.random.default_rng(len(name))
    mp = opar.level(0).mul_params
    N, t = opar.degree, opar.plaintext
    Q, QP = mp.frm.modulus(), mp.to.modulus()
    n_m = max(4, N // 7)
    # down scaler: inputs in the multiplication basis
    down = E.scaler_near_ties(QP, t, Q, rng, n_m) + E.sign_boundary(QP)
    y = E.polys_from_values(down, mp.to.moduli, N)
    wide = E.wide_w_sums(mp.down_scaler.scaler, mp.to.moduli, rng, 64)   # w's sign test at bit 191
    if wide:
        y = np.concatenate([y, E.polys_from_residues(wide, N)])
    if name in ("l31_13", "bp_wide_13"):
        assert len(wide) == 64
    got = F.Ciphertext.from_host(gpar, y[:, None], repr=F.POWER_BASIS, mul_basis=True).into_ntt().scale(1)
    got = got.into_power_basis().to_host()
    for c in range(len(y)):
        exp = mp.down_scaler.scale(oracle.Poly(mp.to, oracle.POWER_BASIS, y[c].copy())).c
        assert (got[c, 0] == exp).all(), "down scaler, polynomial %d" % c
    # extender: inputs in the ciphertext basis
    ext = E.extender_edges(Q) + E.sign_boundary(Q)
    ext += [int(rng.integers(0, 1 << 62)) * Q // (1 << 62) for _ in range(max(1, N - len(ext)))]
    x = E.polys_from_values(ext, mp.frm.moduli, N)
    got = F.Ciphertext.from_host(gpar, x[:, None], repr=F.POWER_BASIS).into_ntt().scale(0).into_power_basis().to_host()
    for c in range(len(x)):
        exp = mp.extender.scale(oracle.Poly(mp.frm, oracle.POWER_BASIS, x[c].copy())).c
        assert (got[c, 0] == exp).all(), "extender, polynomial %d" % c


@pytest.mark.parametrize("degree,sizes", [(16, [62] * 5), (1 << 13, [62, 40, 30]), (1 << 15, [62] * 14)])
def test_switch_down_ties(oracle, F, degree, sizes):
    """Ciphertext::switch_down at x mod q_last in {(q_last -/+ 1) / 2, 0, q_last - 1}: equal to the oracle, and to
    the exact rule round(x / q_last) that rq/mod.rs:456-478 computes."""
    opar, gpar = make(oracle, F, degree, 1153, sizes=sizes)
    ctx = opar.context_at_level(0)
    Q, q_last = ctx.modulus(), ctx.moduli[-1]
    vals = E.switch_down_ties(Q, q_last, np.random.default_rng(degree), max(8, degree // 4))
    x = E.polys_from_values(vals, ctx.moduli, degree)
    X = F.Ciphertext.from_host(gpar, x[:, None], repr=F.POWER_BASIS).into_ntt()
    got = X.switch_down().into_power_basis().to_host()
    nxt = ctx.next_context
    for c in range(len(x)):
        exp = oracle.Poly(ctx, oracle.POWER_BASIS, x[c].copy()).switch_down()
        assert (got[c, 0] == exp.c).all()
        for j in range(0, degree, max(1, degree // 256)):
            big = ctx.rns.lift([int(v) for v in x[c, :, j]])
            assert nxt.rns.lift([int(v) for v in got[c, 0, :, j]]) == ((big + (q_last >> 1)) // q_last) % nxt.modulus()


# ----------------------------------------------------------------------------------------------- extreme residues

@pytest.mark.parametrize("degree,moduli", [(16, "62x3"), (4096, "62x2"), (1 << 13, "boundary"), (1 << 14, "62x2"),
                                           (1 << 15, "boundary_solinas"), (1 << 16, "62x2")])
def test_ntt_extreme_residues(oracle, F, degree, moduli):
    """Forward and backward transforms of all-0, all-(q - 1), alternating, (q -/+ 1) / 2 and unit rows (8 polynomials
    per limb, enough for the TMA kernels) against the oracle."""
    mods = boundary_moduli(moduli, degree) if moduli.startswith("boundary") else \
        oracle.BfvParameters.generate_moduli([62] * int(moduli[-1]), degree)
    opar, gpar = make(oracle, F, degree, 1153 if degree < 4096 else 786433, moduli=mods)
    ctx = opar.context_at_level(0)
    rows = list(E.residue_rows(ctx.moduli, degree).values())
    rows.append(rand_rows(np.random.default_rng(degree), ctx.moduli, (), degree))
    x = np.stack(rows)[:, None]
    got = F.Ciphertext.from_host(gpar, x, repr=F.POWER_BASIS).into_ntt().to_host()
    back = F.Ciphertext.from_host(gpar, x, repr=F.NTT).into_power_basis().to_host()
    for c in range(len(rows)):
        for i, op in enumerate(ctx.ops):
            f = x[c, 0, i].copy()
            op.forward(f)
            assert (got[c, 0, i] == f).all(), (c, i)
            b = x[c, 0, i].copy()
            op.backward(b)
            assert (back[c, 0, i] == b).all(), (c, i)


def _mul_rot_parity(oracle, F, opar, gpar, a, b, kc, gc, idx, level=0, mod_switch=(False, True)):
    """default product (with / without modulus switching) and the rotation by exponent 3, at ciphertexts idx"""
    ork = oracle.RelinearizationKey.from_ksk(oracle.KeySwitchingKey.from_arrays(opar, kc[0], kc[1], level, level))
    grk = F.RelinearizationKey.from_arrays(gpar, kc[0], kc[1], ciphertext_level=level, key_level=level)
    A, B = F.Ciphertext.from_host(gpar, a, level=level), F.Ciphertext.from_host(gpar, b, level=level)
    for ms in mod_switch:
        om, gm = oracle.Multiplicator.default(ork), F.Multiplicator.default(grk)
        if ms:
            om.enable_mod_switching()
            gm.enable_mod_switching()
        got = gm.multiply(A, B).to_host()
        for i in idx:
            exp = om.multiply(oracle.Ciphertext.from_array(opar, a[i], level), oracle.Ciphertext.from_array(opar, b[i], level))
            assert (got[i] == exp.to_array()).all(), ("product", ms, i)
    if gc is not None:
        ogk = oracle.GaloisKey.__new__(oracle.GaloisKey)
        ogk.exponent, ogk.ksk = 3, oracle.KeySwitchingKey.from_arrays(opar, gc[0], gc[1], level, level)
        got = F.GaloisKey.from_arrays(gpar, 3, gc[0], gc[1], ciphertext_level=level, key_level=level).relinearize(A).to_host()
        for i in idx:
            assert (got[i] == ogk.relinearize(oracle.Ciphertext.from_array(opar, a[i], level)).to_array()).all(), ("rotation", i)


def _dot_parity(oracle, F, opar, gpar, carr, parr):
    ctx = opar.context_at_level(0)
    got = F.dot_product_scalar(F.Ciphertext.from_host(gpar, carr), parr).to_host()
    exp = oracle.dot_product_scalar([oracle.Ciphertext.from_array(opar, c, 0) for c in carr],
                                    [oracle.Poly(ctx, oracle.NTT, p.copy()) for p in parr])
    assert (got[0] == exp.to_array()).all()


@pytest.mark.parametrize("degree,sizes", [(16, [62] * 3), (4096, [62] * 2), (1 << 13, "boundary")])
def test_all_max_keys_and_ciphertexts(oracle, F, degree, sizes):
    """Products (with and without modulus switching) and a rotation with keys and ciphertexts of all q - 1: the
    key-switch inner products and the tensor sums reach their largest values."""
    if sizes == "boundary":
        opar, gpar = make(oracle, F, degree, 786433, moduli=boundary_moduli(sizes, degree))
    else:
        opar, gpar = make(oracle, F, degree, 1153 if degree < 4096 else 1032193, sizes=sizes)
    mods = opar.context_at_level(0).moduli
    L = len(mods)
    k = max_rows(mods, (2, L), degree)
    a = max_rows(mods, (2, 2), degree)
    a[1] = rand_rows(np.random.default_rng(degree), mods, (2,), degree)   # one extreme, one random ciphertext
    _mul_rot_parity(oracle, F, opar, gpar, a, a.copy(), k, k, (0, 1))
    # n x m tensor products of extreme operands
    for na, nb in [(3, 2), (2, 3), (3, 3)]:
        x, y = max_rows(mods, (1, na), degree), max_rows(mods, (1, nb), degree)
        got = (F.Ciphertext.from_host(gpar, x) * F.Ciphertext.from_host(gpar, y)).to_host()
        exp = oracle.Ciphertext.from_array(opar, x[0], 0).mul(oracle.Ciphertext.from_array(opar, y[0], 0))
        assert (got[0] == exp.to_array()).all(), (na, nb)


def test_power_basis_key_switch_extremes(oracle, F):
    """A raw key switch of all-(q - 1) power-basis polynomials with an all-(q - 1) key at [62, 40, 30] (the
    reduce-on-load digit path: digits of a 62-bit limb taken to 40- and 30-bit limbs)."""
    degree = 1 << 13
    opar, gpar = make(oracle, F, degree, 786433, sizes=[62, 40, 30])
    ctx = opar.context_at_level(0)
    mods = ctx.moduli
    k = max_rows(mods, (2, 3), degree)
    ok = oracle.KeySwitchingKey.from_arrays(opar, k[0], k[1])
    gk = F.KeySwitchingKey.from_arrays(gpar, k[0], k[1])
    x = np.concatenate([max_rows(mods, (1, 1), degree), rand_rows(np.random.default_rng(3), mods, (1, 1), degree)])
    got = gk.key_switch(F.Ciphertext.from_host(gpar, x, repr=F.POWER_BASIS), 0).to_host()
    for i in range(2):
        c0, c1 = ok.key_switch(oracle.Poly(ctx, oracle.POWER_BASIS, x[i, 0].copy()))
        assert (got[i, 0] == c0.c).all() and (got[i, 1] == c1.c).all()


@pytest.mark.parametrize("degree", [16, 4096])
def test_dot_product_extremes(oracle, F, degree):
    """dot_product_scalar over 1 024 terms whose operands are all q - 1: the wide accumulator's largest sum."""
    opar, gpar = make(oracle, F, degree, 1153, sizes=[62, 62])
    mods = opar.context_at_level(0).moduli
    n = 1024
    c, p = max_rows(mods, (n, 2), degree), max_rows(mods, (n,), degree)
    if degree <= 16:
        _dot_parity(oracle, F, opar, gpar, c, p)
    else:   # (q - 1)^2 == 1: the sum is n mod q in every word
        got = F.dot_product_scalar(F.Ciphertext.from_host(gpar, c), p).to_host()
        assert (got[0] == np.array([n % q for q in mods], np.uint64)[None, :, None]).all()
    # 3-part ciphertexts and a mixed extreme / random batch through the oracle
    rng = np.random.default_rng(degree)
    c3 = max_rows(mods, (64, 3), degree)
    c3[::2] = rand_rows(rng, mods, (32, 3), degree)
    _dot_parity(oracle, F, opar, gpar, c3, max_rows(mods, (64,), degree))


@pytest.mark.parametrize("degree", [16, 1 << 13])
def test_plaintext_ops_extremes(oracle, F, degree):
    """mul_plain and add_plain / sub_plain with plaintext words 0, q - 1 and (q -/+ 1) / 2 on extreme ciphertexts."""
    opar, gpar = make(oracle, F, degree, 786433, sizes=[62, 62, 62])
    ctx = opar.context_at_level(0)
    rows = E.residue_rows(ctx.moduli, degree)
    x = np.stack([max_rows(ctx.moduli, (2,), degree), np.stack([rows["half_up"], rows["alternating"]])])
    for name, w in rows.items():
        pw = oracle.Poly(ctx, oracle.NTT, w.copy())
        got_m = F.Ciphertext.from_host(gpar, x).mul_plain(w).to_host()
        got_a = F.Ciphertext.from_host(gpar, x).add_plain(w).to_host()
        got_s = F.Ciphertext.from_host(gpar, x).sub_plain(w).to_host()
        for i in range(len(x)):
            parts = [oracle.Poly(ctx, oracle.NTT, x[i, p].copy()) for p in range(2)]
            assert (got_m[i] == np.stack([p.mul(pw).c for p in parts])).all(), name
            assert (got_a[i, 0] == parts[0].copy().iadd(pw).c).all() and (got_a[i, 1] == x[i, 1]).all(), name
            assert (got_s[i, 0] == parts[0].copy().isub(pw).c).all() and (got_s[i, 1] == x[i, 1]).all(), name


# --------------------------------------------------------------------------------------------- boundary primes

@pytest.mark.parametrize("degree,kind", [(1 << 13, "boundary"), (1 << 13, "boundary_solinas"), (1 << 15, "boundary"),
                                         (64, "ten_bit")])
def test_boundary_prime_sets(oracle, F, degree, kind):
    """Sets mixing the boundary primes with generated ones (and a 10-bit modulus at N = 64): products with and without
    modulus switching, a rotation and a dot product on random words, against the oracle."""
    if kind == "ten_bit":
        opar, gpar = make(oracle, F, degree, 17, sizes=[62, 62, 10])
    else:
        opar, gpar = make(oracle, F, degree, 786433, moduli=boundary_moduli(kind, degree))
    mods = opar.context_at_level(0).moduli
    L = len(mods)
    rng = np.random.default_rng(degree + L)
    kc, gc = rand_rows(rng, mods, (2, L), degree), rand_rows(rng, mods, (2, L), degree)
    a, b = rand_rows(rng, mods, (2, 2), degree), rand_rows(rng, mods, (2, 2), degree)
    _mul_rot_parity(oracle, F, opar, gpar, a, b, kc, gc, (0, 1))
    _dot_parity(oracle, F, opar, gpar, rand_rows(rng, mods, (5, 2), degree), rand_rows(rng, mods, (5,), degree))


# ------------------------------------------------------------------------------------------------ largest shapes

def test_31_moduli(oracle, F):
    """L = 31 at N = 2^13: 63-limb multiplication basis (K = 63 of 64 positions, 31 digits in the fused key switch,
    theta_garner_shift 123).  Eight ciphertexts: a product, a rotation and a product with modulus switching."""
    degree, L = 1 << 13, 31
    opar, gpar = make(oracle, F, degree, 786433, sizes=[62] * L)
    assert len(opar.level(0).mul_params.to.moduli) == 63
    assert opar.level(0).mul_params.down_scaler.scaler.theta_garner_shift == 123
    mods = opar.context_at_level(0).moduli
    rng = np.random.default_rng(31)
    kc, gc = rand_rows(rng, mods, (2, L), degree), rand_rows(rng, mods, (2, L), degree)
    a, b = rand_rows(rng, mods, (8, 2), degree), rand_rows(rng, mods, (8, 2), degree)
    _mul_rot_parity(oracle, F, opar, gpar, a, b, kc, gc, (0, 7))


def test_64_limb_custom_basis(oracle, F):
    """Multiplicator::new with a basis of exactly 64 limbs (the device's limit) matches the oracle; 65 limbs are
    refused with UNSUPPORTED."""
    degree, L, t = 1 << 13, 31, 786433
    opar, gpar = make(oracle, F, degree, t, sizes=[62] * L)
    base = list(opar.moduli)
    basis = list(base)
    ub = 1 << 62
    while len(basis) < 65:
        ub = oracle.generate_prime(62, 2 * degree, ub)
        if ub not in basis:
            basis.append(ub)
    Q = opar.context_at_level(0).modulus()
    P = 1
    for q in basis[L:64]:
        P *= q
    rng = np.random.default_rng(64)
    a, b = rand_rows(rng, base, (1, 2), degree), rand_rows(rng, base, (1, 2), degree)
    om = oracle.Multiplicator(opar, oracle.ScalingFactor.one(), oracle.ScalingFactor(P, Q), basis[:64],
                              oracle.ScalingFactor(t, P))
    gm = F.Multiplicator.new(F.ScalingFactor.one(), F.ScalingFactor(P, Q), basis[:64], F.ScalingFactor(t, P), gpar)
    got = gm.multiply(F.Ciphertext.from_host(gpar, a), F.Ciphertext.from_host(gpar, b)).to_host()
    exp = om.multiply(oracle.Ciphertext.from_array(opar, a[0], 0), oracle.Ciphertext.from_array(opar, b[0], 0))
    assert (got[0] == exp.to_array()).all()
    with pytest.raises(F.FheError) as e:
        F.Multiplicator.new(F.ScalingFactor.one(), F.ScalingFactor.one(), basis, F.ScalingFactor(t, Q), gpar)
    assert e.value.code == -11


def test_degree_2_16(oracle, F):
    """N = 2^16 with 3 moduli (the non-TMA key switch): a product, a rotation and a raw key switch."""
    degree, L = 1 << 16, 3
    opar, gpar = make(oracle, F, degree, 65537, sizes=[62] * L)
    ctx = opar.context_at_level(0)
    mods = ctx.moduli
    rng = np.random.default_rng(16)
    kc, gc = rand_rows(rng, mods, (2, L), degree), rand_rows(rng, mods, (2, L), degree)
    a, b = rand_rows(rng, mods, (1, 2), degree), rand_rows(rng, mods, (1, 2), degree)
    _mul_rot_parity(oracle, F, opar, gpar, a, b, kc, gc, (0,), mod_switch=(False,))
    ok = oracle.KeySwitchingKey.from_arrays(opar, kc[0], kc[1])
    got = F.KeySwitchingKey.from_arrays(gpar, kc[0], kc[1]).key_switch(
        F.Ciphertext.from_host(gpar, a, repr=F.POWER_BASIS), 1).to_host()
    c0, c1 = ok.key_switch(oracle.Poly(ctx, oracle.POWER_BASIS, a[0, 1].copy()))
    assert (got[0, 0] == c0.c).all() and (got[0, 1] == c1.c).all()


# -------------------------------------------------------------------------------------------------- code paths

@pytest.mark.parametrize("env", [{"FHE_B200_KSMAC": "tma"}, {"FHE_B200_KSMAC": "classic"}, {"FHE_B200_SCALER": "classic"},
                                 {"FHE_B200_NO_SOLINAS": "1"}, {"FHE_B200_SOLINAS_NTT": "1"}, {"FHE_B200_NTT": "fast"},
                                 {"FHE_B200_NTT": "tma"}, {"FHE_B200_GENERIC_NTT": "1"}],
                         ids=lambda e: ",".join("%s=%s" % kv for kv in e.items()))
def test_alternate_code_paths(F, env):
    """every kernel variant must be bit-identical at the edges too: rerun this module (but this test) under each
    switch"""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    out = subprocess.run([sys.executable, "-m", "pytest", "-q", "-x", "-m", "gpu", "tests/test_gpu_edges.py", "-k",
                          "not test_alternate_code_paths"],
                         cwd=root, env=dict(os.environ, **env), capture_output=True, text=True, timeout=900)
    assert out.returncode == 0, out.stdout[-2000:] + out.stderr[-2000:]
