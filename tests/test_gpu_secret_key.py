"""GPU tests of SecretKey::random on the device (fhe_b200_secret_keys_random, fhe_b200_secret_key_coeffs) and of the
Parameters message on the product path: for the same seed every key's coefficients equal
tests/secret_key_reference.py's restatement; a device-born key behaves word for word as the key SecretKey(par, coeffs)
makes from its coefficients; the keys follow the binomial law and are independent; a client built from parameter bytes
and a random key computes what numpy does; and every refusal keeps no memory.  Run with `-m gpu`."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

import edge_inputs as E
import secret_key_reference as S
from test_secret_key_cpu import _binomial_chi2

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def F():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import fhe_rs_b200
    return fhe_rs_b200


# name -> (degree, t, moduli sizes or an edge_inputs.CLIENT_SHAPES name)
SHAPES = {
    "n16": (16, 1153, [62, 62, 62]),
    "setC": (1 << 15, 786433, [62] * 14),
    "n2_16": (1 << 16, 786433, [62] * 3),
    "l31": (1 << 13, 786433, "l31"),
    "q0_barrett": (1 << 13, 786433, "q0_barrett"),
    "q0_above_2_61": (1 << 13, 786433, "q0_above_2_61"),
    "q0_solinas_max_c": (1 << 13, 786433, "q0_solinas_max_c"),
    "q1_barrett": (1 << 13, 786433, "q1_barrett"),
}


def params(oracle, F, name, variance=10):
    degree, t, spec = SHAPES[name]
    moduli = E.client_moduli(spec) if isinstance(spec, str) else oracle.BfvParameters.generate_moduli(spec, degree)
    return F.BfvParameters(degree, t, moduli=moduli, device=0, variance=variance)


def seed_of(i):
    return np.random.default_rng(i).integers(0, 256, 32, dtype=np.uint8).tobytes()


@pytest.mark.parametrize("name", list(SHAPES))
def test_same_seed_same_coefficients(oracle, F, name):
    par = params(oracle, F, name)
    seed = seed_of(len(name))
    n = 3
    keys = F.SecretKey.random_vec(par, n, seed)
    for k, sk in enumerate(keys):
        want = S.secret_key_coeffs(seed, k, par.variance, par.degree())
        assert (sk._download_coeffs() == want).all(), k
    assert (F.SecretKey.random(par, seed)._download_coeffs() == keys[0]._download_coeffs()).all()


@pytest.mark.parametrize("name", ["n16", "setC", "q0_solinas_max_c", "l31"])
def test_identical_to_a_host_made_key(oracle, F, name):
    """encryption, decryption, noise, relinearization and Galois keys of a device-born key equal those of
    SecretKey(par, coeffs) of its downloaded coefficients, word for word"""
    par = params(oracle, F, name, variance=7)
    dev = F.SecretKey.random(par, seed_of(5))
    host = F.SecretKey(par, dev._download_coeffs())
    s1, s2 = seed_of(6), seed_of(7)
    levels = (0, par.max_level()) if par.max_level() else (0,)
    for level in levels:
        a = dev.try_encrypt(seed=s1, count=3, level=level)
        b = host.try_encrypt(seed=s1, count=3, level=level)
        assert (a.to_host() == b.to_host()).all(), level
        assert (dev.try_decrypt(a).batch.to_host() == host.try_decrypt(a).batch.to_host()).all(), level
        assert (dev.measure_noise(a) == host.measure_noise(a)).all(), level
    if len(par.moduli()) > 1:
        for x, y in zip(F.RelinearizationKey.new(dev, s2).ksk.arrays(), F.RelinearizationKey.new(host, s2).ksk.arrays()):
            assert (x == y).all()
    for x, y in zip(F.GaloisKey.new(dev, 3, seed=s2).ksk.arrays(), F.GaloisKey.new(host, 3, seed=s2).ksk.arrays()):
        assert (x == y).all()


def test_distribution_and_independence(oracle, F):
    par = params(oracle, F, "setC")
    seed = seed_of(64)
    keys = F.SecretKey.random_vec(par, 64, seed)
    c = np.stack([k._download_coeffs() for k in keys])
    assert _binomial_chi2(c.ravel(), par.variance) > 1e-3
    assert abs(c.var() / par.variance - 1) < 0.02
    for i in range(1, 64):
        assert (c[i] != c[i - 1]).any() and (c[i] != c[0]).any()
    again = F.SecretKey.random_vec(par, 64, seed)
    assert all((k._download_coeffs() == c[i]).all() for i, k in enumerate(again))
    other = F.SecretKey.random_vec(par, 2, seed_of(65))
    assert (other[0]._download_coeffs() != c[0]).any()
    for v in (1, 32):   # the variance of the parameter set is the variance of the keys
        pv = F.BfvParameters(par.degree(), 786433, moduli=par.moduli(), device=0, variance=v)
        x = np.concatenate([k._download_coeffs() for k in F.SecretKey.random_vec(pv, 4, seed)])
        assert (x == np.concatenate([S.secret_key_coeffs(seed, k, v, par.degree()) for k in range(4)])).all()
        assert _binomial_chi2(x, v) > 1e-3


@pytest.mark.parametrize("chunk,streams", [(6, 1), (6, 2), (24, 4), (24, 2)])
def test_secret_key_chunking(chunk, streams):
    env = dict(os.environ, FHE_B200_CHUNK=str(chunk), FHE_B200_STREAMS=str(streams))
    out = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "secret_key_chunk_probe.py")], env=env,
                         capture_output=True, text=True, timeout=600)
    assert out.returncode == 0 and "secret key chunk probe ok" in out.stdout, out.stdout + out.stderr


def test_client_from_bytes_end_to_end(F):
    """parameters from bytes, a random key, keygen, SIMD encryption, mul_relin, a column rotation, decryption and
    decoding, with no oracle object on the path; the values equal numpy's"""
    degree, t = 1 << 13, 786433
    server = F.BfvParametersBuilder().set_degree(degree).set_plaintext_modulus(t).set_moduli_sizes([62] * 4) \
        .set_variance(10).build()
    par = F.BfvParameters.from_bytes(server.to_bytes())
    assert par.to_bytes() == server.to_bytes() and par.moduli() == server.moduli()
    sk = F.SecretKey.random(par)
    rk = F.RelinearizationKey.new(sk)
    ek = F.EvaluationKeyBuilder.new(sk).enable_column_rotation(1).build()
    rng = np.random.default_rng(3)
    a, b = (rng.integers(0, t, size=(2, degree), dtype=np.uint64) for _ in range(2))
    enc = F.Encoding.simd()
    A = sk.try_encrypt(F.PlaintextVec.try_encode(a.ravel(), enc, par))
    B = sk.try_encrypt(F.PlaintextVec.try_encode(b.ravel(), enc, par))
    prod = F.Multiplicator.default(rk).multiply(A, B)
    rot = ek.rotates_columns_by(prod, 1)
    got = sk.try_decrypt(rot).try_decode(enc).reshape(2, degree)
    want = (a.astype(object) * b.astype(object) % t).astype(np.uint64)
    half = degree // 2
    want = np.concatenate([np.roll(want[:, :half], -1, axis=1), np.roll(want[:, half:], -1, axis=1)], axis=1)
    assert (got == want).all()
    assert (sk.try_decrypt(prod).try_decode(enc).reshape(2, degree) == (a * b) % t).all()


def test_voting_with_random_party_keys(F):
    """examples/voting.rs with the 10 party keys from one random_vec call: 1000 votes under the collective key, the
    collective decryption of the tally is the number of yes votes"""
    degree, t, moduli = 4096, 4096, [0xffffee001, 0xffffc4001, 0x1ffffe0001]
    par = F.BfvParameters(degree, t, moduli=moduli, device=0)
    sks = F.SecretKey.random_vec(par, 10)
    crp = F.mbfv.CommonRandomPoly.new(par)
    pk = F.mbfv.aggregate([F.mbfv.PublicKeyShare(s, crp) for s in sks])
    rng = np.random.default_rng(1000)
    votes = rng.integers(0, 2, size=1000, dtype=np.uint64)
    values = np.zeros(1000 * degree, np.uint64)
    values[::degree] = votes
    ballots = pk.try_encrypt(F.PlaintextVec.try_encode(values, F.Encoding.poly(), par))
    tally = _tally(F, par, ballots)
    pt = F.mbfv.aggregate([F.mbfv.DecryptionShare(s, tally) for s in sks])
    got = pt.try_decode(F.Encoding.poly())
    assert int(got[0]) == int(votes.sum()) and not got[1:].any()


def _tally(F, par, ballots):
    """the sum of every ciphertext of the batch, by halving (an odd remainder is added to the first half's sum)"""
    batch = ballots
    while batch.count > 1:
        h = batch.count // 2
        a = batch.take(0, h)
        a += batch.take(h, h)
        if batch.count % 2:
            first = a.take(0, 1)
            first += batch.take(2 * h, 1)
            rest = a.take(1, h - 1) if h > 1 else None
            a = first if rest is None else F.Ciphertext.from_host(
                par, np.concatenate([first.to_host(), rest.to_host()]), 0)
        batch = a
    return batch


def test_messages_of_a_device_born_key(oracle, F, tmp_path):
    """to_bytes of a device-born key, decoded by wire.decode_secret_key and by the C++ mirror, gives the coefficients
    fhe_b200_secret_key_coeffs returns; the rebuilt key encrypts the same words; the C++ mirror's keys, parameters and
    encryptions equal the Python mirror's"""
    from fhe_rs_b200 import build, wire
    par = params(oracle, F, "l31")
    seed = seed_of(31)
    keys = F.SecretKey.random_vec(par, 3, seed)
    msgs = [k.to_bytes() for k in keys]
    for k, m in zip(keys, msgs):
        assert wire.decode_secret_key(m, par.degree()) == k._download_coeffs().tolist()
    rebuilt = F.SecretKey.from_bytes(par, msgs[0])
    ct = keys[0].try_encrypt(seed=seed, count=2)
    assert (rebuilt.try_encrypt(seed=seed, count=2).to_host() == ct.to_host()).all()
    assert (rebuilt.try_decrypt(ct).batch.to_host() == keys[0].try_decrypt(ct).batch.to_host()).all()
    build.build()
    exe = str(tmp_path / "secret_key_random_test")
    lib_dir = os.path.join(ROOT, "fhe_rs_b200")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "cpp", "secret_key_random_test.cpp"), "-o", exe,
                           "-L", lib_dir, "-lfhe_b200", "-Wl,-rpath," + lib_dir])
    (tmp_path / "par_in.bin").write_bytes(par.to_bytes())
    (tmp_path / "seed.bin").write_bytes(seed)
    out = subprocess.run([exe, str(tmp_path / "par_in.bin"), str(tmp_path / "seed.bin"), "3", str(tmp_path)],
                         capture_output=True, text=True, timeout=600)
    assert out.returncode == 0 and out.stdout.startswith("OK"), out.stdout + out.stderr
    assert (tmp_path / "par.bin").read_bytes() == par.to_bytes()
    for k in range(3):
        assert (tmp_path / ("sk%d.bin" % k)).read_bytes() == msgs[k], k
    assert (tmp_path / "one.bin").read_bytes() == msgs[0]
    want = ct.to_host().ravel()
    assert (np.fromfile(str(tmp_path / "ct.bin"), np.uint64) == want).all()
    assert (np.fromfile(str(tmp_path / "rebuilt.bin"), np.uint64) == want).all()


def test_errors_and_memory(oracle, F):
    """every refusal returns its code, no handle and no memory; freed keys give their memory back"""
    import torch
    from fhe_rs_b200 import _capi
    lib = _capi.lib()
    par = params(oracle, F, "setC")
    big = F.BfvParameters(1 << 15, 340282366920938463463374607431768211507, moduli=par.moduli(), device=0)
    seed = seed_of(1)
    hs = (C.c_void_p * 8)()
    out = C.cast(hs, C.POINTER(C.c_void_p))

    def call(p=par._h, n=8, v=10, s=seed, o=out):
        code = lib.fhe_b200_secret_keys_random(p, n, v, s, o, None)
        if code != _capi.OK:
            assert not any(hs), code
        return code

    def refusals():
        assert call(v=0) == _capi.INVALID_ARGUMENT
        assert call(v=33) == _capi.INVALID_ARGUMENT
        assert call(n=0) == _capi.INVALID_ARGUMENT
        assert call(s=None) == _capi.INVALID_ARGUMENT
        assert call(o=None) == _capi.INVALID_ARGUMENT
        assert call(p=None) == _capi.INVALID_ARGUMENT
        assert call(p=big._h) == _capi.UNSUPPORTED
        assert lib.fhe_b200_secret_key_coeffs(None, np.zeros(4, np.int64).ctypes.data, None) == _capi.INVALID_ARGUMENT

    def cycle():
        assert call() == _capi.OK
        first = np.zeros(par.degree(), np.int64)
        assert lib.fhe_b200_secret_key_coeffs(hs[0], first.ctypes.data, None) == _capi.OK
        assert lib.fhe_b200_secret_key_coeffs(hs[0], None, None) == _capi.INVALID_ARGUMENT
        for i in range(8):
            assert lib.fhe_b200_secret_key_free(hs[i]) == _capi.OK
            hs[i] = None
        refusals()
        assert lib.fhe_b200_sync(None) == _capi.OK
    cycle()
    free0 = torch.cuda.mem_get_info()[0]
    for _ in range(3):
        cycle()
    assert abs(torch.cuda.mem_get_info()[0] - free0) < 4 << 20
    # a host-only parameter set
    host = F.BfvParameters(16, 1153, moduli=oracle.BfvParameters.generate_moduli([62], 16), device=-1)
    assert call(p=host._h) == _capi.NO_DEVICE
