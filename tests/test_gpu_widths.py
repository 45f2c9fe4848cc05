"""Device against oracle across modulus widths, word for word.

Almost every other test runs 62-bit moduli.  These feed the places where the code decides from a modulus's width:
  * the single-modulus decomposition key switch at every q_0 width from 10 to 62 (3 digits at odd widths, log_base
    other than 31): decompose_kernel, the gadget 2^(i log_base) mod q_0 of device key generation, the inner product
    with 3 digits at one key limb, the RGSW external product, and the key messages through both host codecs; at
    N = 2^12 and 2^15 as well;
  * the wire bit packer at every field width from 10 to 62, with 65537 (a 17-bit field), mixed widths at N = 8 and
    16 (per-limb offsets of a few bytes), fields in [q, 2^nbits) that only a message can carry, and 31 limbs at
    N = 2^16;
  * the RNS-digit transform next to its reduce-on-load decision: all-(q_i - 1) digits just under 4 q_j (taken
    unreduced), just above it and near 8 q_j (reduced), through relinearize, a Galois key switch and a raw key
    switch, with the fused TMA kernel;
  * whole pipelines on bases that sweep 10 to 62 bits, with q_0 narrow and wide.
Every comparison is bit-exact against the oracle or its restatements (tests/keygen_reference.py,
tests/encrypt_reference.py).  test_alternate_code_paths reruns the module under each kernel-selection switch.
Run with `-m gpu`."""
import os
import subprocess
import sys

import numpy as np
import pytest

import edge_inputs as E
import encrypt_reference as R
import keygen_reference as K
from test_widths_cpu import WIDTHS, ksk_codec, pack_words

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def F():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import fhe_rs_b200
    return fhe_rs_b200


@pytest.fixture(scope="module")
def ow(oracle):
    import fhe_wire
    return fhe_wire


@pytest.fixture(scope="module")
def codec(tmp_path_factory, F):
    return ksk_codec(tmp_path_factory.mktemp("ksk_wire"))


def make(oracle, F, degree, t, moduli):
    opar = oracle.BfvParameters(degree, t, moduli=moduli)
    return opar, F.BfvParameters(degree, t, moduli=opar.moduli, device=0)


def seed_of(rng):
    return rng.integers(0, 256, size=32, dtype=np.uint8).tobytes()


def rand_rows(rng, moduli, prefix, degree):
    a = np.zeros(tuple(prefix) + (len(moduli), degree), np.uint64)
    for i, q in enumerate(moduli):
        a[..., i, :] = rng.integers(0, q, size=tuple(prefix) + (degree,), dtype=np.uint64)
    return a


def max_rows(moduli, prefix, degree):
    q = np.array(moduli, dtype=np.uint64)[:, None] - np.uint64(1)
    return np.ascontiguousarray(np.broadcast_to(q, tuple(prefix) + (len(moduli), degree)))


def check_key(osk, ksk, frm, seed, key, what):
    """the downloaded words of a device-generated key equal the restatement, every digit"""
    c0, c1 = ksk.arrays()
    assert c0.shape[0] == len(K.gadget(osk.par, ksk.ciphertext_level, ksk.ksk_level)), what
    for i in range(c0.shape[0]):
        w0, w1 = K.key_digit(osk, frm, ksk.ciphertext_level, ksk.ksk_level, seed, key, i, osk.par.variance)
        assert (c1[i] == w1).all(), (what, "c1", i)
        assert (c0[i] == w0).all(), (what, "c0", i)


def has_simd(oracle, opar):
    t = opar.plaintext
    return t < opar.moduli[0] and t % (2 * opar.degree) == 1 and oracle.is_prime(t)


# ------------------------------------------------------------------------------------------------- decomposition

def check_decomposition(oracle, F, ow, codec, degree, bits, rng, n_inputs):
    """the single-modulus key switch at the last level of [q_0 (bits), 62, 62]"""
    moduli = E.decomposition_moduli(bits, degree)
    t = 97 if degree == 16 else 786433
    opar, gpar = make(oracle, F, degree, t, moduli)
    last = len(moduli) - 1
    ctx = opar.context_at_level(last)
    q = moduli[0]
    n_dig = 3 if bits % 2 else 2
    osk = oracle.SecretKey(opar, rng)
    gsk = F.SecretKey(gpar, osk.coeffs)
    # raw key switch of an oracle key: random inputs, all q - 1, and the residue_rows extremes
    ok = oracle.KeySwitchingKey(sk=osk, frm=oracle.Poly.random(ctx, oracle.POWER_BASIS, rng), ciphertext_level=last,
                                ksk_level=last, rng=rng)
    assert len(ok.c0) == n_dig and ok.log_base == bits // 2
    gk = F.KeySwitchingKey.from_arrays(gpar, *ok.arrays(), ciphertext_level=last, key_level=last)
    assert gk.n_digits == n_dig and gk.log_base == ok.log_base
    rows = [r for r in E.residue_rows([q], degree).values()] + [rand_rows(rng, [q], (), degree) for _ in range(n_inputs)]
    x = np.stack(rows)[:, None]
    got = gk.key_switch(F.Ciphertext.from_host(gpar, x, level=last, repr=F.POWER_BASIS), 0).to_host()
    for i in range(len(x)):
        c0, c1 = ok.key_switch(oracle.Poly(ctx, oracle.POWER_BASIS, x[i, 0].copy()))
        assert (got[i, 0] == c0.c).all() and (got[i, 1] == c1.c).all(), (bits, i)
    # Galois key generated on the device at the last level: its words, a rotation with it against the oracle
    seed = seed_of(rng)
    ggk = F.GaloisKey.new(gsk, 3, last, last, seed)
    check_key(osk, ggk.ksk, K.galois_from(osk, 3, last, last), seed, 0, ("galois", bits))
    ogk = oracle.GaloisKey.__new__(oracle.GaloisKey)
    ogk.exponent, ogk.ksk = 3, oracle.KeySwitchingKey.from_arrays(opar, *ggk.ksk.arrays(), last, last)
    m = rng.integers(0, t, size=(2, degree))
    cts = [osk.encrypt(v, last, rng) for v in m]
    A = F.Ciphertext.from_host(gpar, np.stack([c.to_array() for c in cts]), level=last)
    rot = ggk.relinearize(A).to_host()
    for i, c in enumerate(cts):
        assert (rot[i] == ogk.relinearize(c).to_array()).all(), (bits, "rotation", i)
    # RGSW: device-generated keys against the restatement, external products of device and oracle RGSW ciphertexts
    values = rng.integers(0, t, size=degree, dtype=np.uint64)
    P = F.PlaintextVec.try_encode(values, F.Encoding.poly_at_level(last), gpar)
    mp = oracle.Poly(ctx, oracle.NTT, P.batch.to_host()[0, 0].copy())
    seed = seed_of(rng)
    grg = gsk.try_encrypt_rgsw(P, seed)[0]
    for which, ksk in enumerate((grg.ksk0, grg.ksk1)):
        check_key(osk, ksk, K.rgsw_from(osk, mp, last, bool(which)), seed, which, ("rgsw", bits, which))
    org = oracle.RGSWCiphertext.__new__(oracle.RGSWCiphertext)
    org.level = last
    org.ksk0 = oracle.KeySwitchingKey.from_arrays(opar, *grg.ksk0.arrays(), last, last)
    org.ksk1 = oracle.KeySwitchingKey.from_arrays(opar, *grg.ksk1.arrays(), last, last)
    org2 = oracle.RGSWCiphertext(osk, oracle.Poly.random(ctx, oracle.NTT, rng), last, rng)
    grg2 = F.RGSWCiphertext.from_arrays(gpar, *org2.ksk0.arrays(), *org2.ksk1.arrays(), level=last)
    ext = max_rows([q], (2,), degree)[None]
    words = np.concatenate([A.to_host(), ext])
    W = F.Ciphertext.from_host(gpar, words, level=last)
    for r_dev, r_orc in ((grg, org), (grg2, org2)):
        got = r_dev.external_product(W).to_host()
        for i, w in enumerate(words):
            exp = r_orc.external_product(oracle.Ciphertext.from_array(opar, w, last))
            assert (got[i] == exp.to_array()).all(), (bits, "external product", i)
    # key messages: the device's bytes are the oracle's; back through the Python mirror and the C++ host
    msgs = [ggk.ksk.to_bytes(), gk.to_bytes()]
    assert msgs[0] == ow.ksk_to_bytes(ogk.ksk) and msgs[1] == ow.ksk_to_bytes(ok)
    assert ow.rgsw_to_bytes(org) == grg.to_bytes()
    for msg, key in zip(msgs, (ggk.ksk, gk)):
        back = F.KeySwitchingKey.from_bytes(gpar, msg)
        assert back.n_digits == n_dig and back.log_base == bits // 2
        assert all((u == v).all() for u, v in zip(back.arrays(), key.arrays()))
    back = F.RGSWCiphertext.from_bytes(gpar, grg.to_bytes())
    assert all((u == v).all() for a, b in ((grg.ksk0, back.ksk0), (grg.ksk1, back.ksk1))
               for u, v in zip(a.arrays(), b.arrays()))
    assert codec(degree, t, moduli, 0, msgs) == [("k", m) for m in msgs]


@pytest.mark.parametrize("bits", WIDTHS)
def test_decomposition_every_width(oracle, F, ow, codec, bits):
    """N = 16, q_0 of every width from 10 to 62: the device key switch of an oracle key on random, all-(q - 1) and
    extreme power-basis rows; a Galois key and an RGSW ciphertext generated on the device at the last level, word for
    word against tests/keygen_reference.py, a rotation with that key and external products of both RGSW ciphertexts
    (one of them all q - 1) against the oracle; the key messages equal the oracle's bytes and come back unchanged
    through the Python mirror and the C++ host codec."""
    check_decomposition(oracle, F, ow, codec, 16, bits, np.random.default_rng(bits), 2)


@pytest.mark.parametrize("degree,bits", [(1 << 12, 61), (1 << 12, 31), (1 << 15, 61), (1 << 15, 31)])
def test_decomposition_large_degree(oracle, F, ow, codec, degree, bits):
    """the same at N = 2^12 (register-resident transforms) and 2^15 (the TMA transforms; 3 digits of one limb are
    three rows), with a 61-bit (3 digits of 30 bits) and a 31-bit q_0 (3 digits of 15 bits)"""
    check_decomposition(oracle, F, ow, codec, degree, bits, np.random.default_rng(degree + bits), 1)


# ---------------------------------------------------------------------------------------------------- bit packer

def check_packer(oracle, F, opar, gpar, x_pb):
    """to_packed / from_packed of power-basis words x_pb [count][parts][L][N] (fields may lie in [q, 2^nbits)), in
    both representations, against poly_to_rq_coefficients / poly_from_rq_coefficients; at N = 2^16 against
    test_widths_cpu.pack_words and the oracle's transform of the reduced words (the same, pinned on the CPU)"""
    ctx = opar.context_at_level(0)
    small = opar.degree <= 64
    count, parts = x_pb.shape[:2]
    reduced = (x_pb % np.array(ctx.moduli, np.uint64)[:, None]).astype(np.uint64)
    blobs = pack_words(x_pb, ctx.moduli)
    if small:
        for c in range(count):
            for p in range(parts):
                assert blobs[c, p].tobytes() == b"".join(oracle.transcode_to_bytes(x_pb[c, p, i], (q - 1).bit_length())
                                                         for i, q in enumerate(ctx.moduli))
    # power basis: fields kept as they are; packing the words gives the same bytes back
    Z = F.Ciphertext.from_packed(gpar, blobs, repr=F.POWER_BASIS)
    assert (Z.to_host() == x_pb).all()
    assert (Z.to_packed() == blobs).all()
    # NTT: the transform of the fields; packing an NTT batch packs its (canonical) power basis
    got = F.Ciphertext.from_packed(gpar, blobs, repr=F.NTT).to_host()
    for c in range(count):
        for p in range(parts):
            if small:
                exp = oracle.poly_from_rq_coefficients(ctx, blobs[c, p].tobytes(), oracle.NTT).c
            else:
                exp = oracle.Poly(ctx, oracle.POWER_BASIS, reduced[c, p].copy()).into_ntt().c
            assert (got[c, p] == exp).all(), (c, p)
    packed = F.Ciphertext.from_host(gpar, got, repr=F.NTT).to_packed()
    assert (packed == pack_words(reduced, ctx.moduli)).all()
    if small:
        for c in range(count):
            for p in range(parts):
                assert packed[c, p].tobytes() == oracle.poly_to_rq_coefficients(oracle.Poly(ctx, oracle.NTT, got[c, p].copy()))


def pack_batch(moduli, degree, rng):
    """[rows][1][L][N]: one polynomial per E.pack_rows kind, each limb its own modulus's row of that kind"""
    per_limb = [E.pack_rows(q, degree, rng) for q in moduli]
    return np.stack([np.stack([r[name] for r in per_limb]) for name in per_limb[0]])[:, None]


@pytest.mark.parametrize("bits", WIDTHS)
def test_packer_every_width(oracle, F, bits):
    """N = 16 and 64, [q (bits), 62-bit]: 0, q - 1, alternating, random and field-overflow rows, plus random batches
    in the NTT representation, packed and unpacked against the oracle"""
    for degree in (16, 64):
        moduli = oracle.BfvParameters.generate_moduli([bits, 62], degree)
        opar, gpar = make(oracle, F, degree, 2, moduli)
        rng = np.random.default_rng(degree + bits)
        check_packer(oracle, F, opar, gpar, pack_batch(moduli, degree, rng))
        check_packer(oracle, F, opar, gpar, rand_rows(rng, moduli, (3, 2), degree))


@pytest.mark.parametrize("degree,moduli", [(16, "65537_last"), (64, "65537_first"), (8, [62, 17, 40, 10, 33, 55]),
                                           (16, [10, 62, 23, 31, 47, 11, 58]), (8, [61, 13, 29]),
                                           (16, [41, 27, 19, 52])])
def test_packer_mixed_widths(oracle, F, degree, moduli):
    """a parameter set holding 65537 = 2^16 + 1 (a 17-bit field), and mixed widths at N = 8 and 16, where a limb's
    bytes start nbits (N = 8) or 2 nbits (N = 16) bytes after the previous limb's"""
    if moduli == "65537_last":
        moduli = [E.prime_of_width(62, degree), 65537]
    elif moduli == "65537_first":
        moduli = [65537] + oracle.BfvParameters.generate_moduli([62, 40], degree)
    else:
        moduli = oracle.BfvParameters.generate_moduli(moduli, degree)
    opar, gpar = make(oracle, F, degree, 3, moduli)
    rng = np.random.default_rng(degree + len(moduli))
    check_packer(oracle, F, opar, gpar, pack_batch(moduli, degree, rng))
    check_packer(oracle, F, opar, gpar, rand_rows(rng, moduli, (5, 3), degree))


def test_packer_n2_16_l31(oracle, F):
    """N = 2^16 and 31 limbs of widths 24 to 62 (offsets up to 12 MiB into a 12.6 MiB polynomial): a batch of two
    2-part ciphertexts with random, all-(q - 1) and overflow fields, checked against the oracle in full"""
    degree = 1 << 16
    sizes = [62 - (13 * k) % 39 for k in range(31)]
    moduli = oracle.BfvParameters.generate_moduli(sizes, degree)
    opar, gpar = make(oracle, F, degree, 3, moduli)
    rng = np.random.default_rng(16)
    rows = [E.pack_rows(q, degree, rng) for q in moduli]
    x = np.stack([np.stack([np.stack([r["random"] for r in rows]), np.stack([r["max"] for r in rows])]),
                  np.stack([np.stack([r["field_random"] for r in rows]), np.stack([r["field_alternating"] for r in rows])])])
    check_packer(oracle, F, opar, gpar, x)


# --------------------------------------------------------------------------------------- digits at the lazy bound

def lazy_inputs(oracle, opar, count):
    """[count][3][L][N] NTT ciphertexts whose c2 is all q - 1 in the power basis (c0, c1 all q - 1 in NTT words),
    and [count][2][L][N] ones whose Galois key-switch input substitute(c1, 3) is all q - 1 in the power basis"""
    degree = opar.degree
    ctx = opar.context_at_level(0)
    mx = max_rows(ctx.moduli, (), degree).copy()
    mx_ntt = oracle.Poly(ctx, oracle.POWER_BASIS, mx.copy()).into_ntt().c
    three = np.stack([np.stack([mx, mx, mx_ntt])] * count)
    inv = pow(3, -1, 2 * degree)
    pre = oracle.Poly(ctx, oracle.POWER_BASIS, mx.copy()).substitute(inv)
    assert (pre.copy().substitute(3).c == mx).all()
    two = np.stack([np.stack([mx, pre.copy().into_ntt().c])] * count)
    return three, two


@pytest.mark.parametrize("base", ["unreduced", "reduced", "reduced_8x"])
def test_digit_transform_lazy_bound(oracle, F, base):
    """N = 2^13, bases of tests/edge_inputs.lazy_bound_bases: every digit of modulus q_i is q_i - 1, a hair under
    4 q_j (transformed unreduced), at / above it, or near 8 q_j (reduced on load).  relinearize (c2 all q - 1), a Galois key
    switch (substitute(c1) all q - 1) and a raw key switch (all q - 1 power-basis input) of 8 ciphertexts -- so the
    digit transform takes the TMA path and the fused key-switch kernel -- with all-(q - 1) and random keys, against
    the oracle."""
    degree, t = 1 << 13, 786433
    moduli = E.lazy_bound_bases(degree)[base]
    opar, gpar = make(oracle, F, degree, t, moduli)
    ctx = opar.context_at_level(0)
    L, count = len(moduli), 8
    rng = np.random.default_rng(13 + len(base))
    three, two = lazy_inputs(oracle, opar, count)
    for kname, k in (("max", max_rows(moduli, (2, L), degree)), ("random", rand_rows(rng, moduli, (2, L), degree))):
        oksk = oracle.KeySwitchingKey.from_arrays(opar, k[0], k[1])
        # relinearize
        ork = oracle.RelinearizationKey.from_ksk(oksk)
        got = F.RelinearizationKey.from_arrays(gpar, k[0], k[1]).relinearizes(F.Ciphertext.from_host(gpar, three)).to_host()
        exp = ork.relinearizes(oracle.Ciphertext.from_array(opar, three[0], 0)).to_array()
        for i in range(count):
            assert (got[i] == exp).all(), (base, kname, "relinearize", i)
        # Galois key switch
        ogk = oracle.GaloisKey.__new__(oracle.GaloisKey)
        ogk.exponent, ogk.ksk = 3, oksk
        got = F.GaloisKey.from_arrays(gpar, 3, k[0], k[1]).relinearize(F.Ciphertext.from_host(gpar, two)).to_host()
        exp = ogk.relinearize(oracle.Ciphertext.from_array(opar, two[0], 0)).to_array()
        for i in range(count):
            assert (got[i] == exp).all(), (base, kname, "galois", i)
        # raw key switch of all-(q - 1) power-basis polynomials
        x = max_rows(moduli, (count, 1), degree)
        got = F.KeySwitchingKey.from_arrays(gpar, k[0], k[1]).key_switch(
            F.Ciphertext.from_host(gpar, x, repr=F.POWER_BASIS), 0).to_host()
        c0, c1 = oksk.key_switch(oracle.Poly(ctx, oracle.POWER_BASIS, x[0, 0].copy()))
        for i in range(count):
            assert (got[i, 0] == c0.c).all() and (got[i, 1] == c1.c).all(), (base, kname, "key switch", i)


# ------------------------------------------------------------------------------------------------- width sweep

@pytest.mark.parametrize("name", list(E.WIDTH_SETS))
def test_width_sweep(oracle, F, name):
    """Bases sweeping 10 to 62 bits (tests/edge_inputs.WIDTH_SETS), q_0 narrow or wide: NTT round trip; mul_relin
    with and without modulus switching and a rotation; switch-down through every level; encrypt_sk / encrypt_pk at
    every level (tests/encrypt_reference.py); decryption, Poly / SIMD decoding and measure_noise; relinearization keys
    generated on the device (tests/keygen_reference.py) -- all against the oracle."""
    degree, t, sizes = E.WIDTH_SETS[name]
    moduli = oracle.BfvParameters.generate_moduli(sizes, degree)
    opar, gpar = make(oracle, F, degree, t, moduli)
    ctx = opar.context_at_level(0)
    L, last = len(moduli), len(moduli) - 1
    rng = np.random.default_rng(degree + sizes[0])
    osk = oracle.SecretKey(opar, rng)
    gsk = F.SecretKey(gpar, osk.coeffs)
    # NTT round trip on random and extreme rows
    x = np.stack([rand_rows(rng, moduli, (2,), degree), max_rows(moduli, (2,), degree)])
    X = F.Ciphertext.from_host(gpar, x, repr=F.POWER_BASIS)
    got = X.into_ntt().to_host()
    for c in range(2):
        for p in range(2):
            for i, op in enumerate(ctx.ops):
                f = x[c, p, i].copy()
                op.forward(f)
                assert (got[c, p, i] == f).all(), (name, "ntt", c, p, i)
    assert (X.into_power_basis().to_host() == x).all()
    # products and a rotation with oracle keys on fresh encryptions
    ork = oracle.RelinearizationKey(osk, rng)
    grk = F.RelinearizationKey.from_arrays(gpar, *ork.ksk.arrays())
    ogk = oracle.GaloisKey(osk, 3, rng)
    ggk = F.GaloisKey.from_arrays(gpar, 3, *ogk.ksk.arrays())
    ma, mb = rng.integers(0, t, size=(2, 2, degree))
    octa, octb = [osk.encrypt(m, 0, rng) for m in ma], [osk.encrypt(m, 0, rng) for m in mb]
    A = F.Ciphertext.from_host(gpar, np.stack([c.to_array() for c in octa]))
    B = F.Ciphertext.from_host(gpar, np.stack([c.to_array() for c in octb]))
    for ms in (False, True):
        om, gm = oracle.Multiplicator.default(ork), F.Multiplicator.default(grk)
        if ms:
            om.enable_mod_switching()
            gm.enable_mod_switching()
        got = gm.multiply(A, B).to_host()
        for i in range(2):
            assert (got[i] == om.multiply(octa[i], octb[i]).to_array()).all(), (name, "product", ms, i)
    got = ggk.relinearize(A).to_host()
    for i in range(2):
        assert (got[i] == ogk.relinearize(octa[i]).to_array()).all(), (name, "rotation", i)
    # switch down through every level
    cur, ocur = A.clone(), [c.copy() for c in octa]
    for level in range(1, L):
        cur = cur.switch_down()
        ocur = [c.switch_to_level(level) for c in ocur]
        assert cur.level == level
        got = cur.to_host()
        for i in range(2):
            assert (got[i] == ocur[i].to_array()).all(), (name, "switch_down", level, i)
    # encryption at every level (sk and pk), decryption, decoding and noise
    seed_pk = seed_of(rng)
    gpk = F.PublicKey.new(gsk, seed_pk)
    opk = R.encrypt_sk(osk, seed_pk, 1, 0, 10)[0]
    assert (gpk.c.to_host()[0] == opk.to_array()).all(), name
    simd = has_simd(oracle, opar)
    levels = range(L) if degree <= 64 else (0, 1, last // 2, last)
    for level in levels:
        lctx = opar.context_at_level(level)
        values = rng.integers(0, t, size=2 * degree, dtype=np.uint64)
        values[:degree:2] = t - 1
        enc = F.Encoding.simd_at_level(level) if simd and level % 2 else F.Encoding.poly_at_level(level)
        coeffs = [values[k * degree:(k + 1) * degree] for k in range(2)]
        if simd and level % 2:
            coeffs = [oracle.simd_encode(opar, c) for c in coeffs]
        ms = [R.to_poly(opar, c, level) for c in coeffs]
        P = F.PlaintextVec.try_encode(values, enc, gpar)
        for which in ("sk", "pk"):
            seed = seed_of(rng)
            if which == "sk":
                ct = gsk.try_encrypt(P, seed)
                exp = R.encrypt_sk(osk, seed, 2, level, 10, ms)
            else:
                ct = gpk.try_encrypt(P, seed)
                exp = R.encrypt_pk(opar, opk, seed, 2, level, 10, ms)
            assert ct.level == level
            words = ct.to_host()
            pts = gsk.try_decrypt(ct)
            dec = pts.poly_ntt()
            noise = gsk.measure_noise(ct)
            decoded = pts.try_decode(enc)
            for k in range(2):
                assert (words[k] == exp[k].to_array()).all(), (name, which, level, k)
                w = osk.decrypt(exp[k])
                assert (dec[k] == oracle.Poly.from_u64(lctx, w, oracle.NTT).c).all(), (name, which, level, k)
                want = oracle.simd_decode(opar, w) if simd and level % 2 else w
                assert (decoded[k * degree:(k + 1) * degree] == want).all(), (name, which, level, k)
                assert int(noise[k]) == osk.measure_noise(exp[k]), (name, which, level, k)
            # fresh noise is below 2^12 at these sizes: with room for it the messages come back
            if (lctx.modulus() // t).bit_length() > 16:
                assert (decoded == values).all(), (name, which, level)
    # relinearization keys generated on the device, leveled ones included
    for c, k in sorted({(0, 0), (1, 0), (last - 1, 0), (last - 1, last - 2)}):
        seed = seed_of(rng)
        rk = F.RelinearizationKey.new_leveled(gsk, c, k, seed)
        check_key(osk, rk.ksk, K.relin_from(osk, c, k), seed, 0, (name, "relin", c, k))


# -------------------------------------------------------------------------------------------------- code paths

@pytest.mark.parametrize("env", [{"FHE_B200_NTT": "fast"}, {"FHE_B200_NTT": "tma"}, {"FHE_B200_GENERIC_NTT": "1"},
                                 {"FHE_B200_NO_SOLINAS": "1"}, {"FHE_B200_SOLINAS_NTT": "1"},
                                 {"FHE_B200_KSMAC": "tma"}, {"FHE_B200_KSMAC": "classic"}],
                         ids=lambda e: ",".join("%s=%s" % kv for kv in e.items()))
def test_alternate_code_paths(F, env):
    """every kernel variant must be bit-identical across the widths too: rerun this module (but this test) under
    each switch"""
    out = subprocess.run([sys.executable, "-m", "pytest", "-q", "-x", "-m", "gpu", "tests/test_gpu_widths.py",
                          "-k", "not test_alternate_code_paths", "-p", "no:cacheprovider"],
                         cwd=ROOT, env=dict(os.environ, **env), capture_output=True, text=True, timeout=1800)
    assert out.returncode == 0, out.stdout[-2000:] + out.stderr[-2000:]
