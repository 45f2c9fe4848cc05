"""CPU-side tests of the product: the C-ABI library loads and exports every symbol of
include/fhe_b200.h, the host precompute (parameter builder, NTT / scaler tables) equals the
oracle's, error codes mirror the reference, and compute entry points refuse to run without a
CUDA device (there is no CPU fallback)."""
import os
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def F():
    from fhe_rs_b200 import build
    build.build()
    import fhe_rs_b200
    return fhe_rs_b200


def test_library_exports_every_declared_symbol(F):
    from fhe_rs_b200 import _capi
    hdr = open(os.path.join(ROOT, "include", "fhe_b200.h")).read()
    declared = set(re.findall(r"\b(fhe_b200_[a-z0-9_]+)\s*\(", hdr))
    lib = _capi.lib()
    for name in sorted(declared):
        assert hasattr(lib, name), "missing symbol " + name
    assert declared == set(_capi.SYMBOLS), declared ^ set(_capi.SYMBOLS)
    assert b"sm_90a" in lib.fhe_b200_version()


def test_ctypes_signatures_match_the_header(F):
    """the hand-written ctypes table must agree with the prototypes of include/fhe_b200.h: argument count, and
    pointer-vs-integer kind of every argument (a mismatch corrupts the call silently)"""
    import ctypes as C
    from fhe_rs_b200 import _capi
    hdr = open(os.path.join(ROOT, "include", "fhe_b200.h")).read()
    hdr = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    protos = re.findall(r"\b[a-z_0-9]+\s*\*?\s*(fhe_b200_[a-z0-9_]+)\s*\(([^;{]*)\)\s*;", hdr)
    assert len(protos) == len(_capi.SYMBOLS)
    for name, args in protos:
        params = [a.strip() for a in args.split(",")]
        if params == ["void"]:
            params = []
        restype, argtypes = _capi.SYMBOLS[name]
        assert len(params) == len(argtypes), (name, params, argtypes)
        for decl, ct in zip(params, argtypes):
            is_ptr = "*" in decl
            ct_ptr = ct in (C.c_void_p, C.c_char_p) or hasattr(ct, "contents") or getattr(ct, "_type_", None) == "P"
            assert is_ptr == bool(ct_ptr), (name, decl, ct)


def test_cubin_is_sm_90a(F):
    import subprocess
    from fhe_rs_b200 import _capi
    out = subprocess.run(["cuobjdump", "-lelf", _capi.LIB_PATH], capture_output=True, text=True).stdout
    assert "sm_90a" in out


@pytest.mark.parametrize("degree,sizes,t", [(16, [62, 62, 62], 1153), (4096, [62, 62], 1032193),
                                            (1024, [50, 40, 30], 65537)])
def test_host_precompute_matches_oracle(F, oracle, degree, sizes, t):
    gpar = F.BfvParameters(degree, t, moduli_sizes=sizes, device=-1)
    opar = oracle.BfvParameters(degree, t, moduli_sizes=sizes)
    assert gpar.moduli() == opar.moduli
    for level in range(len(sizes)):
        mp = opar.level(level).mul_params
        assert gpar.mul_basis(level) == mp.to.moduli
        for which, sc in ((0, mp.extender.scaler), (1, mp.down_scaler.scaler)):
            tb = gpar.scaler_tables(level, which)
            assert tb["shift"] == sc.theta_garner_shift
            assert (tb["gamma"] == sc.gamma).all() and (tb["omega"] == sc.omega).all()
            assert (tb["theta_omega_lo"] == sc.theta_omega_lo).all()
            assert (tb["theta_omega_hi"] == sc.theta_omega_hi).all()
            assert (tb["theta_omega_sign"] == sc.theta_omega_sign).all()
            assert (tb["theta_garner_lo"] == sc.theta_garner_lo).all()
            assert (tb["theta_garner_hi"] == sc.theta_garner_hi).all()
            assert [int(x) for x in tb["theta_gamma"]] == [sc.theta_gamma_lo, sc.theta_gamma_hi,
                                                           int(sc.theta_gamma_sign)]
    for q in gpar.mul_basis(0):
        nt = gpar.ntt_tables(q)
        op = oracle._ntt_op(q, degree, None)
        assert gpar.psi(q) == op.psi and nt["size_inv"] == op.size_inv
        assert (nt["omegas"] == op.omegas).all() and (nt["omegas_shoup"] == op.omegas_shoup).all()
        assert (nt["zetas_inv"] == op.zetas_inv).all() and (nt["zetas_inv_shoup"] == op.zetas_inv_shoup).all()


def test_custom_psi_is_honoured(F, oracle):
    opar = oracle.BfvParameters(16, 1153, moduli_sizes=[62, 62])
    primes = opar.moduli + opar.extended_basis
    psi = [pow(oracle.default_psi(q, 16), 3, q) for q in primes]   # another primitive 32nd root
    gpar = F.BfvParameters(16, 1153, moduli=opar.moduli, psi=psi, device=-1)
    for q, r in zip(primes, psi):
        assert gpar.psi(q) == r
        op = oracle.NttOperator(oracle.Modulus(q), 16, r)
        assert (gpar.ntt_tables(q)["omegas"] == op.omegas).all()
    bad = list(psi)
    bad[0] = 1
    with pytest.raises(F.FheError) as e:
        F.BfvParameters(16, 1153, moduli=opar.moduli, psi=bad, device=-1)
    assert e.value.code == -4


def test_error_codes_mirror_reference(F):
    cases = [
        (dict(degree=12, moduli_sizes=[62]), -3),                    # InvalidPolynomialDegree
        (dict(degree=16, moduli=[1 << 62]), -2),                     # InvalidModulus
        (dict(degree=16, moduli=[4611686018427387617] * 2), -2),     # DuplicateModuli
        (dict(degree=16, moduli=[1153 * 5]), -4),                    # not NTT friendly / not prime
        (dict(degree=16, moduli_sizes=[9]), -2),                     # InvalidModulusSize
    ]
    for kw, code in cases:
        with pytest.raises(F.FheError) as e:
            F.BfvParameters(plaintext_modulus=1153 if "moduli" not in kw or kw["moduli"] != [1153 * 5] else 7,
                            device=-1, **kw)
        assert e.value.code == code, (kw, e.value)
    with pytest.raises(F.FheError):
        F.BfvParameters(16, 1153, device=-1)                         # neither moduli nor sizes


def test_no_cpu_fallback(F):
    """compute entry points must fail loudly without a device"""
    gpar = F.BfvParameters(16, 1153, moduli_sizes=[62, 62], device=-1)
    with pytest.raises(F.FheError) as e:
        F.Ciphertext(gpar, 1)
    assert e.value.code == -22
    with pytest.raises(F.FheError) as e:
        F.KeySwitchingKey(gpar, np.zeros((2, 2, 16), np.uint64), np.zeros((2, 2, 16), np.uint64))
    assert e.value.code == -22


def test_golden_fixture_matches_oracle(oracle):
    """the committed fixture is what the (pinned) oracle produces: regression pin for both"""
    g = np.load(os.path.join(ROOT, "tests", "golden", "golden_n16_l3.npz"))
    par = oracle.BfvParameters(int(g["degree"]), int(g["t"]), moduli=[int(x) for x in g["moduli"]])
    a = [oracle.Ciphertext.from_array(par, x, 0) for x in g["a"]]
    b = [oracle.Ciphertext.from_array(par, x, 0) for x in g["b"]]
    assert (np.stack([x.mul(y).to_array() for x, y in zip(a, b)]) == g["mul3"]).all()
    assert (np.stack([x.add(y).to_array() for x, y in zip(a, b)]) == g["add"]).all()
    # decrypt with the stored secret key
    rng = np.random.default_rng(0)
    sk = oracle.SecretKey(par, rng)
    sk.coeffs = g["sk"]
    res = oracle.Ciphertext.from_array(par, g["mul_relin"][0], 0)
    ma, mb = sk.decrypt(a[0]), sk.decrypt(b[0])
    exp = np.zeros(16, dtype=object)
    for i in range(16):
        for j in range(16):
            k, v = i + j, int(ma[i]) * int(mb[j])
            exp[k % 16] = (exp[k % 16] + (v if k < 16 else -v)) % 1153
    assert (sk.decrypt(res).astype(object) == exp).all()


def test_wide_golden_fixture_matches_oracle(oracle):
    """tests/golden/golden_n16_l3_wide.npz (operations around the core): the oracle reproduces the stored outputs
    from the stored inputs, and the stored results decrypt to what the operations mean"""
    g = np.load(os.path.join(ROOT, "tests", "golden", "golden_n16_l3_wide.npz"))
    t, degree = int(g["t"]), int(g["degree"])
    par = oracle.BfvParameters(degree, t, moduli=[int(x) for x in g["moduli"]])
    ctx = par.context_at_level(0)
    a = [oracle.Ciphertext.from_array(par, x, 0) for x in g["a"]]
    b = [oracle.Ciphertext.from_array(par, x, 0) for x in g["b"]]
    assert (np.stack([x.sub(y).to_array() for x, y in zip(a, b)]) == g["sub"]).all()
    assert (np.stack([x.copy().switch_to_level(2).to_array() for x in a]) == g["switch_to_2"]).all()
    pts = [oracle.Poly(ctx, oracle.NTT, x.copy()) for x in g["dot_pts"]]
    for grp in range(2):
        assert (oracle.dot_product_scalar(a[2 * grp:2 * grp + 2], pts[2 * grp:2 * grp + 2]).to_array() == g["dot"][grp]).all()
    basis = [int(x) for x in g["basis"]]
    P = 1
    for q in basis[3:]:
        P *= q
    m2 = oracle.Multiplicator(par, oracle.ScalingFactor.one(), oracle.ScalingFactor(P, ctx.modulus()), basis,
                              oracle.ScalingFactor(t, P))
    assert (np.stack([m2.multiply(x, y).to_array() for x, y in zip(a, b)]) == g["strategy2"]).all()
    k2 = oracle.KeySwitchingKey.from_arrays(par, g["k2_c0"], g["k2_c1"], 2, 2)
    ctx2 = par.context_at_level(2)
    for x, exp in zip(g["k2_in"], g["k2_out"]):
        c0, c1 = k2.key_switch(oracle.Poly(ctx2, oracle.POWER_BASIS, x.copy()))
        assert (c0.c == exp[0]).all() and (c1.c == exp[1]).all()
    # meaning: decrypt with the stored secret key
    sk = oracle.SecretKey(par, np.random.default_rng(0))
    sk.coeffs = g["sk"]
    ma = oracle.simd_decode(par, sk.decrypt(a[0])).astype(np.int64)
    mb = oracle.simd_decode(par, sk.decrypt(b[0])).astype(np.int64)
    dec = lambda arr, lvl=0: oracle.simd_decode(par, sk.decrypt(oracle.Ciphertext.from_array(par, arr, lvl))).astype(np.int64)
    assert (dec(g["sub"][0]) == (ma - mb) % t).all() and (dec(g["neg"][0]) == (-ma) % t).all()
    assert (dec(g["switch_to_2"][0], 2) == ma).all()
    assert (dec(g["strategy2"][0]) == (ma * mb) % t).all() and (dec(g["strategy2_relin"][0]) == (ma * mb) % t).all()
    assert (dec(g["mul_3x2"][0]) == (ma * mb * mb) % t).all()


def test_environment_switches_are_documented_and_tested():
    """The engine reads its FHE_B200_* switches in one place (switches(), ntt.cu): no other source under csrc/ calls
    getenv, the names it reads are exactly the ones the appendix of DESIGN.md lists, and every one of them is set by at
    least one test's environment parametrization, so every variant they select is parity-tested."""
    csrc = os.path.join(ROOT, "fhe_rs_b200", "csrc")
    callers, body = [], None
    for d, _, files in os.walk(csrc):
        for f in files:
            src = open(os.path.join(d, f)).read()
            if "getenv" in src:
                callers.append(os.path.relpath(os.path.join(d, f), csrc))
            m = re.search(r"^const Switches& switches\(\) \{\n(.*?)^\}\n", src, flags=re.S | re.M)
            if m:
                body = m.group(1)
                assert src.count("getenv") == body.count("getenv"), "getenv outside switches() in " + f
    assert callers == ["ntt.cu"], callers
    assert body is not None and "getenv" in body
    read = set(re.findall(r'"(FHE_B200_[A-Z_]+)"', body))
    design = open(os.path.join(ROOT, "DESIGN.md")).read()
    table = design.split("## Appendix — environment switches", 1)[1]
    documented = set()
    for line in table.splitlines()[1:]:
        if line.startswith("## "):
            break
        if line.startswith("| `"):
            documented |= set(re.findall(r"FHE_B200_[A-Z_]+", line.split("|")[1]))
    documented.discard("FHE_B200_LIB")   # read by the Python loader, not by the engine
    assert read == documented, read ^ documented
    tested = set()
    for f in os.listdir(os.path.join(ROOT, "tests")):
        if f.endswith(".py"):
            tested |= set(re.findall(r'"(FHE_B200_[A-Z_]+)"\s*:', open(os.path.join(ROOT, "tests", f)).read()))
    assert read <= tested, read - tested
