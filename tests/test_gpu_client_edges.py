"""Device against oracle at the edges of the client side -- decryption, noise measurement, decoding, the plaintext
lift and oblivious expansion -- word for word (or against plain integers), through the Python mirror.

The decryption suite (test_gpu_decrypt.py) uses fresh encryptions, whose phase sits about Q / 2t away from every
decision.  These tests feed the phases where the code decides something (tests/edge_inputs.py):
  * the decryption scaler (t / Q, one output row) at the ties of t x / Q, at Q / 2 and at Delta m +/- Q / 2t, on
    scale_small_kernel, scale_tma_kernel and scale_kernel, with t from 2 to the largest the library takes;
  * the phase at its extremes: keys whose NTT words are all q - 1, i64 extremes in the key, 1 to 8 parts;
  * the lift of plaintext words below t into limbs smaller than t (left unreduced up to 4 q_min - 1);
  * measure_noise's multi-word arithmetic: 31 limbs, N = 2^16, Q at a word boundary, one atomic per block;
  * centring at t = 2, 3, 4 and near 2^62, and the expansion butterfly on all-(q - 1) words and keys.
test_alternate_code_paths reruns the module under each kernel-selection switch.  Run with `-m gpu`."""
import os
import subprocess
import sys

import numpy as np
import pytest

import edge_inputs as E
import encode_reference as R

pytestmark = pytest.mark.gpu
I64 = np.iinfo(np.int64)


@pytest.fixture(scope="module")
def F():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import fhe_rs_b200
    return fhe_rs_b200


def make(oracle, F, degree, t, moduli):
    opar = oracle.BfvParameters(degree, t, moduli=moduli)
    return opar, F.BfvParameters(degree, t, moduli=opar.moduli, device=0)


def keys(oracle, F, opar, gpar, rng, coeffs=None):
    osk = oracle.SecretKey(opar, rng)
    if coeffs is not None:
        osk.coeffs = np.array(coeffs, np.int64)
    return osk, F.SecretKey(gpar, osk.coeffs)


def has_simd(oracle, opar):
    t = opar.plaintext
    return t < opar.moduli[0] and t % (2 * opar.degree) == 1 and oracle.is_prime(t)


def phase_words(oracle, opar, level, polys, parts=2):
    """[count][parts][L][N] NTT words with c0 = NTT(polys[k]) and every other part 0: the phase is polys[k]"""
    ctx = opar.context_at_level(level)
    c0 = np.stack([oracle.Poly(ctx, oracle.POWER_BASIS, p.copy()).into_ntt().c for p in polys])
    out = np.zeros((len(polys), parts) + c0.shape[1:], np.uint64)
    out[:, 0] = c0
    return out


def centre(v, t):
    """Modulus::center as test_gpu_decrypt._centre: a - t when a >= t >> 1"""
    r = [int(x) % t for x in v]
    return np.array([x - t if x >= t >> 1 else x for x in r], dtype=np.int64)


def check_decrypt(oracle, F, opar, gpar, osk, gsk, words, level, decode=True, noise=True):
    """decrypt (and, for t < q_0, Poly / signed / SIMD decode and measure_noise) of `words` against the oracle"""
    n, t = opar.degree, opar.plaintext
    ctx = opar.context_at_level(level)
    ct = F.Ciphertext.from_host(gpar, words, level)
    pts = gsk.try_decrypt(ct)
    got = pts.poly_ntt()
    exp = [osk.decrypt(oracle.Ciphertext.from_array(opar, w, level)) for w in words]
    for k, w in enumerate(exp):
        assert (got[k] == oracle.Poly.from_u64(ctx, w, oracle.NTT).c).all(), ("decrypt", level, k)
    if t >= opar.moduli[0]:
        return
    if decode:
        poly = pts.try_decode(F.Encoding.poly_at_level(level))
        signed = pts.try_decode(F.Encoding.poly_at_level(level), signed=True)
        simd = pts.try_decode(F.Encoding.simd_at_level(level)) if has_simd(oracle, opar) else None
        for k, w in enumerate(exp):
            assert (poly[k * n:(k + 1) * n] == w).all(), ("poly", level, k)
            assert (signed[k * n:(k + 1) * n] == centre(w, t)).all(), ("signed", level, k)
            if simd is not None:
                assert (simd[k * n:(k + 1) * n] == oracle.simd_decode(opar, w)).all(), ("simd", level, k)
    if noise:
        got_noise = gsk.measure_noise(ct)
        for k, w in enumerate(words):
            assert int(got_noise[k]) == osk.measure_noise(oracle.Ciphertext.from_array(opar, w, level)), ("noise", k)


# ---------------------------------------------------------------------------------------------- decryption scaler

@pytest.mark.parametrize("tname", ["t2", "t1153", "t40", "below_q0", "max"])
@pytest.mark.parametrize("shape", list(E.CLIENT_SHAPES))
def test_decrypt_scaler_edges(oracle, F, shape, tname):
    """Decryption of c1 = 0 ciphertexts whose phase sits at the ties of t x / Q, at Q / 2 and at Delta m +/- Q / 2t
    (the inputs test_client_edges_cpu.py shows to reach both windows of the reference's scaler), at every level (0, 15
    and 30 of 31 moduli); for t < q_0 also Poly, signed and SIMD decoding and measure_noise (at the first and last
    level of the N >= 2^14 shapes)."""
    degree, _ = E.CLIENT_SHAPES[shape]
    moduli = E.client_moduli(shape)
    t = E.client_plaintexts(degree, moduli)[tname]
    opar, gpar = make(oracle, F, degree, t, moduli)
    rng = np.random.default_rng(degree + len(moduli) + t % 4093)
    osk, gsk = keys(oracle, F, opar, gpar, rng)
    L = len(moduli)
    levels = (0, 15, 30) if shape == "l31" else range(L)
    for level in levels:
        ctx = opar.context_at_level(level)
        xs = E.decrypt_phases(ctx.modulus(), t, rng, 4 if degree < 1 << 12 else 64)
        words = phase_words(oracle, opar, level, E.polys_from_values(xs, ctx.moduli, degree))
        noise = degree < 1 << 14 or level in (0, L - 1)
        check_decrypt(oracle, F, opar, gpar, osk, gsk, words, level, noise=noise)


# ------------------------------------------------------------------------------------------------ phase extremes

def phase_set(oracle, name):
    if name == "n16":
        return 16, 1153, oracle.BfvParameters.generate_moduli([62] * 3, 16)
    degree = 1 << 13
    return degree, 786433, [E.gen62(degree, 0)] + [E.BOUNDARY_PRIMES[k] for k in
                                                   ("solinas_max_c", "non_solinas_min", "above_2_61")]


@pytest.mark.parametrize("name", ["n16", "boundary"])
def test_phase_extremes(oracle, F, name):
    """c0 + c1 s + ... + c_k s^k with s = -1 (every NTT word q - 1), s = 1, and s holding i64 min / max, +/-(q_0 - 1)
    and +/-q_0 (the host's signed reduction), on ciphertexts of 1, 2, 3, 5 and 8 parts whose words are all q - 1,
    alternating 0 / q - 1, or random: decryption and measure_noise against the oracle, at the first and last level."""
    degree, t, moduli = phase_set(oracle, name)
    opar, gpar = make(oracle, F, degree, t, moduli)
    rng = np.random.default_rng(degree)
    for kname, coeffs in E.key_extremes(degree, moduli[0], rng).items():
        osk, gsk = keys(oracle, F, opar, gpar, rng, coeffs)
        for level in (0, len(moduli) - 1):
            ctx = opar.context_at_level(level)
            rows = E.residue_rows(ctx.moduli, degree)
            for parts in (1, 2, 3, 5, 8):
                rnd = np.stack([np.stack([rng.integers(0, q, size=degree, dtype=np.uint64) for q in ctx.moduli])
                                for _ in range(parts)])
                mixed = np.stack([[rows["max"], rows["alternating"], rnd[p]][p % 3] for p in range(parts)])
                words = np.stack([np.stack([rows["max"]] * parts), np.stack([rows["alternating"]] * parts), mixed])
                ct = F.Ciphertext.from_host(gpar, words, level)
                got, noise = gsk.try_decrypt(ct).poly_ntt(), gsk.measure_noise(ct)
                for k in range(len(words)):
                    oc = oracle.Ciphertext.from_array(opar, words[k], level)
                    w = osk.decrypt(oc)
                    assert (got[k] == oracle.Poly.from_u64(ctx, w, oracle.NTT).c).all(), (kname, level, parts, k)
                    assert int(noise[k]) == osk.measure_noise(oc), (kname, level, parts, k)


# --------------------------------------------------------------------------------------------- the unreduced lift

def lift_set(oracle, degree, qmin_bits):
    """two generated 62-bit moduli (Solinas limbs) and a small last modulus q_min (a Barrett limb); 193 is below 2^8"""
    qmin = 193 if qmin_bits == 8 else oracle.generate_prime(qmin_bits, 2 * degree, 1 << qmin_bits)
    return [E.gen62(degree, 0), E.gen62(degree, 1), qmin]


def lift_plaintexts(oracle, degree, qmin):
    """t on both sides of the switch at 4 q_min - 1 (4 q_min itself shares a factor with q_min), q_min + 1, and the
    largest prime t < 4 q_min with t = 1 mod 2N (SIMD)"""
    m = 2 * degree
    simd = (4 * qmin - 2) // m * m + 1
    while not oracle.is_prime(simd):
        simd -= m
    assert 2 * qmin < simd < 4 * qmin
    return {"4q-1": 4 * qmin - 1, "4q+1": 4 * qmin + 1, "q+1": qmin + 1, "simd": simd}


@pytest.mark.parametrize("degree,qmin_bits", [(16, 20), (1 << 12, 20), (1 << 13, 20), (1 << 14, 20), (16, 8)])
def test_unreduced_lift(oracle, F, degree, qmin_bits):
    """Words below t go into the forward NTT of a limb q_min < t without a reduction when t <= 4 q_min - 1 (decrypt,
    encode, to_poly): decryption of c1 = 0 ciphertexts whose phase is to_poly(m) for m all t - 1 and alternating
    0 / t - 1, measure_noise, SIMD and signed Poly encoding, and add_plain / sub_plain with such plaintexts -- against
    the oracle and tests/encode_reference.py, at N = 16 (generic kernels), 2^12 and 2^13 (register-resident) and 2^14
    with 8 plaintexts (TMA), and with q_min = 193 < 2^8.  t = 4 q_min is refused (not coprime with q_min)."""
    from fhe_rs_b200 import _capi
    moduli = lift_set(oracle, degree, qmin_bits)
    qmin = moduli[-1]
    with pytest.raises(F.FheError) as e:
        F.BfvParameters(degree, 4 * qmin, moduli=moduli, device=0)
    assert e.value.code == _capi.INVALID_MODULUS
    count = 8
    for tname, t in lift_plaintexts(oracle, degree, qmin).items():
        opar, gpar = make(oracle, F, degree, t, moduli)
        rng = np.random.default_rng(degree + t)
        osk, gsk = keys(oracle, F, opar, gpar, rng)
        ctx = opar.context_at_level(0)
        msgs = np.zeros((count, degree), np.uint64)
        msgs[0::2] = t - 1
        msgs[1::2, 1::2] = t - 1
        c0 = np.stack([oracle.plaintext_to_poly(opar, m, 0).c for m in msgs])
        words = np.zeros((count, 2) + c0.shape[1:], np.uint64)
        words[:, 0] = c0
        check_decrypt(oracle, F, opar, gpar, osk, gsk, words, 0)
        dec = gsk.try_decrypt(F.Ciphertext.from_host(gpar, words)).try_decode(F.Encoding.poly())
        assert (dec == msgs.ravel()).all(), tname
        # encoders: signed Poly (-1 -> t - 1) and SIMD
        signed = np.where(msgs.ravel() == t - 1, -1, 0).astype(np.int64)
        plains = {"signed": (F.PlaintextVec.try_encode(signed, F.Encoding.poly(), gpar),
                             R.try_encode(opar, signed, False, 0, True))}
        if has_simd(oracle, opar):
            u = rng.integers(0, t, size=count * degree, dtype=np.uint64)
            u[::3] = t - 1
            plains["simd"] = (F.PlaintextVec.try_encode(u, F.Encoding.simd(), gpar), R.try_encode(opar, u, True))
        x = np.stack([np.stack([np.stack([rng.integers(0, q, size=degree, dtype=np.uint64) for q in ctx.moduli])
                                for _ in range(2)]) for _ in range(count)])
        for pname, (P, exp) in plains.items():
            assert (P.poly_ntt() == exp).all(), (tname, pname)
            for sub in (False, True):
                got = F.Ciphertext.from_host(gpar, x).add_plain(P, subtract=sub).to_host()
                for k in range(count):
                    a = oracle.Poly(ctx, oracle.NTT, x[k, 0].copy())
                    m = oracle.Poly(ctx, oracle.NTT, R.to_poly(opar, exp[k], 0))
                    want = a.isub(m) if sub else a.iadd(m)
                    assert (got[k, 0] == want.c).all() and (got[k, 1] == x[k, 1]).all(), (tname, pname, sub, k)


# --------------------------------------------------------------------------------------------------- noise kernel

NOISE_SETS = {
    "l31": (1 << 13, [62] * 31),      # L = W = 31, the kernel's largest local arrays
    "n2_16": (1 << 16, [62] * 3),     # 256 blocks per ciphertext
    "ten_bit": (64, [62, 62, 10]),
    "boundary": (1 << 13, None),
    "q128": (16, [62, 40, 26]),       # bits(Q) = 128: Q fills two words
    "q129": (16, [62, 40, 27]),       # bits(Q) = 129: one bit in a third word
}


def noise_set(oracle, name):
    degree, sizes = NOISE_SETS[name]
    if sizes is None:
        return degree, phase_set(oracle, "boundary")[2]
    moduli = oracle.BfvParameters.generate_moduli(sizes, degree)
    if name.startswith("q12"):
        assert E.product(moduli).bit_length() == int(name[1:])
    return degree, moduli


def single_coefficient_phases(oracle, opar, xs, positions):
    """1-part ciphertexts, the k-th with phase xs[k] at coefficient positions[k] and 0 elsewhere"""
    ctx = opar.context_at_level(0)
    polys = np.zeros((len(xs), len(ctx.moduli), opar.degree), np.uint64)
    for k, (x, p) in enumerate(zip(xs, positions)):
        polys[k, :, p] = [x % q for q in ctx.moduli]
    return phase_words(oracle, opar, 0, polys, parts=1)


@pytest.mark.parametrize("name", list(NOISE_SETS))
def test_noise_kernel_limits(oracle, F, name):
    """measure_noise of single-coefficient phases 2^k - 1, 2^k, 2^k + 1 and Q - 2^k at every 64-bit word boundary k
    below bits(Q), floor(Q / 2) and ceil(Q / 2), at coefficients 0, 255, 256, N - 256 and N - 1, against the same
    rule in plain integers (E.noise_one, pinned to the oracle by test_client_edges_cpu.py) and, at the small shapes,
    the oracle itself.  Then one batch whose ciphertexts have different maxima -- one of them 0, the largest in the
    last coefficient of the last ciphertext -- each in its own slot."""
    degree, moduli = noise_set(oracle, name)
    opar, gpar = make(oracle, F, degree, 1153, moduli)
    rng = np.random.default_rng(degree + len(moduli))
    osk, gsk = keys(oracle, F, opar, gpar, rng)
    Q = opar.context_at_level(0).modulus()
    pos = sorted({p % degree for p in (0, 255, 256, degree - 256, degree - 1)})
    xs = E.noise_points(Q) + E.decrypt_phases(Q, 1153, rng, 1)[::4]
    exp = [E.noise_one(opar, 0, x) for x in xs]
    small = degree * len(moduli) <= 1 << 14
    for first in range(0, len(xs), 32):
        sl = slice(first, first + 32)
        words = single_coefficient_phases(oracle, opar, xs[sl], [pos[k % len(pos)] for k in range(first, len(xs))])
        got = gsk.measure_noise(F.Ciphertext.from_host(gpar, words))
        for k, w in enumerate(words):
            assert int(got[k]) == exp[first + k], (xs[first + k], pos[(first + k) % len(pos)])
            if small:
                assert exp[first + k] == osk.measure_noise(oracle.Ciphertext.from_array(opar, w, 0))
    # one batch, five maxima: small, 0, Q/2 at coefficient 0, 2^70 at N - 256, and Q/2 at N - 1 of the last ciphertext
    # next to a small value at coefficient 0
    batch = [[(5, 300 % degree)], [], [(Q // 2, 0)], [(1 << 70, (degree - 256) % degree)], [(3, 0), (Q // 2, degree - 1)]]
    polys = np.zeros((len(batch), len(moduli), degree), np.uint64)
    for k, coeffs in enumerate(batch):
        for x, p in coeffs:
            polys[k, :, p] = [x % q for q in moduli]
    got = gsk.measure_noise(F.Ciphertext.from_host(gpar, phase_words(oracle, opar, 0, polys, parts=1)))
    want = [max([E.noise_one(opar, 0, x) for x, _ in coeffs], default=0) for coeffs in batch]
    assert len(set(want)) >= 4 and want[1] == 0
    assert [int(v) for v in got] == want


# ------------------------------------------------------------------------------------------ decoding and centring

def decode_plaintexts(oracle, degree, moduli):
    """t = 2, 3, 4, the largest t below q_0, and the largest prime t = 1 mod 2N below q_0 (SIMD)"""
    ub = moduli[0]
    while True:
        ub = oracle.generate_prime(62, 2 * degree, ub)
        if ub not in moduli:
            break
    return {"t2": 2, "t3": 3, "t4": 4, "below_q0": E.coprime_below(moduli[0], moduli), "simd_max": ub}


@pytest.mark.parametrize("degree", [16, 1 << 12])
def test_decode_edges(oracle, F, degree):
    """encode -> decode and decrypt -> decode where centring decides something: t >> 1 = 1 at t = 2 and 3, and
    a - t across the i64 range at t near 2^62 (signed encoding of i64 min / max); signed results against
    test_gpu_decrypt._centre's rule, SIMD against oracle.simd_decode"""
    moduli = oracle.BfvParameters.generate_moduli([62] * 3, degree)
    for tname, t in decode_plaintexts(oracle, degree, moduli).items():
        opar, gpar = make(oracle, F, degree, t, moduli)
        rng = np.random.default_rng(degree + t % 1000)
        h = t >> 1
        u = rng.integers(0, t, size=2 * degree, dtype=np.uint64)
        u[:6] = [0, h, max(h - 1, 0), t - 1, min(h + 1, t - 1), 1]
        s = rng.integers(I64.min, I64.max, size=2 * degree, dtype=np.int64, endpoint=True)
        s[:10] = [I64.min, I64.max, I64.min + 1, I64.max - 1, -1, 0, h, -h, t - 1, -(t - 1)]
        encs = [F.Encoding.poly()] + ([F.Encoding.simd()] if has_simd(oracle, opar) else [])
        for enc in encs:
            P = F.PlaintextVec.try_encode(u, enc, gpar)
            assert (P.try_decode() == u).all() and (P.try_decode(signed=True) == centre(u, t)).all(), (tname, enc)
            S = F.PlaintextVec.try_encode(s, enc, gpar)
            assert (S.try_decode(signed=True) == centre(s, t)).all(), (tname, enc)
            assert (S.try_decode() == np.array([int(v) % t for v in s], np.uint64)).all(), (tname, enc)
        # decrypt -> decode on fresh encryptions of the edge values
        osk, gsk = keys(oracle, F, opar, gpar, rng)
        words = np.stack([osk.encrypt(u[k * degree:(k + 1) * degree], 0, rng).to_array() for k in range(2)])
        check_decrypt(oracle, F, opar, gpar, osk, gsk, words, 0)
        # the messages come back while 2t <= q_0; above, the reference's ((v + t) mod q_0) mod t wraps every
        # v >= q_0 - t to v - 1, and the device follows it word for word (check_decrypt)
        if 2 * t <= moduli[0]:
            assert (gsk.try_decrypt(F.Ciphertext.from_host(gpar, words)).try_decode(F.Encoding.poly(), signed=True)
                    == centre(u, t)).all(), tname


# ---------------------------------------------------------------------------------------------------- expansion

def max_rows(moduli, prefix, degree):
    q = np.array(moduli, dtype=np.uint64)[:, None] - np.uint64(1)
    return np.ascontiguousarray(np.broadcast_to(q, tuple(prefix) + (len(moduli), degree)))


def expansion_moduli(kind, degree):
    bp = [E.BOUNDARY_PRIMES[k] for k in ("solinas_max_c", "non_solinas_min", "above_2_61")]
    if kind == "boundary":
        return [E.gen62(degree, 0)] + bp
    return [E.BOUNDARY_PRIMES["solinas_max_c"], E.gen62(degree, 0), E.gen62(degree, 1)]


@pytest.mark.parametrize("degree,kind,size", [(16, "boundary", 16), (16, "boundary", 13), (16, "boundary_solinas", 16),
                                              (16, "boundary_solinas", 11), (1 << 13, "boundary", 1000),
                                              (1 << 13, "boundary_solinas", 600)])
def test_expand_extremes(oracle, F, degree, kind, size):
    """fhe_b200_expand with all-(q - 1) Galois keys on an all-(q - 1) ciphertext (and, at N = 16, an alternating
    0 / q - 1 one): every output against oracle.expands.  At N = 2^13 the sizes stay below N: the oracle runs one key
    switch per output."""
    moduli = expansion_moduli(kind, degree)
    opar, gpar = make(oracle, F, degree, 786433 if degree > 16 else 1153, moduli)
    L = len(moduli)
    k = max_rows(moduli, (2, L), degree)
    ogk, ek = {}, F.EvaluationKey(gpar)
    for l in range((size - 1).bit_length()):
        e = (degree >> l) + 1
        g = oracle.GaloisKey.__new__(oracle.GaloisKey)
        g.exponent, g.ksk = e, oracle.KeySwitchingKey.from_arrays(opar, k[0], k[1])
        ogk[e] = g
        ek.add_galois_key(F.GaloisKey.from_arrays(gpar, e, k[0], k[1]))
    rows = E.residue_rows(moduli, degree)
    cts = np.stack([max_rows(moduli, (2,), degree), np.stack([rows["alternating"], rows["max"]])])[:2 if degree == 16 else 1]
    got = ek.expands_batch(F.Ciphertext.from_host(gpar, cts), size).to_host()
    for q in range(len(cts)):
        exp = oracle.expands(opar, ogk, oracle.Ciphertext.from_array(opar, cts[q], 0), size)
        for i in range(size):
            assert (got[i * len(cts) + q] == exp[i].to_array()).all(), (q, i)


# -------------------------------------------------------------------------------------------------- code paths

@pytest.mark.parametrize("env", [{"FHE_B200_SCALER": "classic"}, {"FHE_B200_NTT": "fast"}, {"FHE_B200_NTT": "tma"},
                                 {"FHE_B200_GENERIC_NTT": "1"}, {"FHE_B200_NO_SOLINAS": "1"},
                                 {"FHE_B200_SOLINAS_NTT": "1"}],
                         ids=lambda e: ",".join("%s=%s" % kv for kv in e.items()))
def test_alternate_code_paths(F, env):
    """every kernel variant must be bit-identical at the client-side edges too: rerun this module (but this test)
    under each switch"""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    out = subprocess.run([sys.executable, "-m", "pytest", "-q", "-x", "-m", "gpu", "tests/test_gpu_client_edges.py",
                          "-k", "not test_alternate_code_paths", "-p", "no:cacheprovider"],
                         cwd=root, env=dict(os.environ, **env), capture_output=True, text=True, timeout=1800)
    assert out.returncode == 0, out.stdout[-2000:] + out.stderr[-2000:]
