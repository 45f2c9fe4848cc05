"""CPU tests of encryption's host side: the ChaCha20 stream restated in tests/encrypt_reference.py against RFC 8439 and
an independent implementation, the centred binomial sampler against the binomial distribution, the PublicKey message
codec against the google.protobuf runtime, and the refusals that need no device."""
import ctypes as C
import os
import struct

import numpy as np
import pytest
from google.protobuf import descriptor_pb2, descriptor_pool, message_factory

import encrypt_reference as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def F():
    import fhe_rs_b200
    return fhe_rs_b200


def test_chacha20_block_rfc8439():
    """RFC 8439 section 2.3.2: key 00..1f, block count 1, nonce 00:00:00:09:00:00:00:4a:00:00:00:00"""
    got = R.chacha20_block(bytes(range(32)), 1, 0x09000000, 0x4A000000, 0)
    assert got.hex() == ("10f1e7e4d13b5915500fdd1fa32071c4c7d1f4c733c068030422aa9ac3d46c4e"
                         "d2826446079faa0914c2d705d98b02a2b5129cd1de164eb9cbd083e8a2503c4e")


def test_chacha20_matches_an_independent_implementation():
    """the `cryptography` package's ChaCha20 takes a 16-byte nonce: state words 12..15, little endian"""
    pytest.importorskip("cryptography")
    from cryptography.hazmat.primitives.ciphers import Cipher, algorithms
    rng = np.random.default_rng(11)
    for _ in range(8):
        key = rng.integers(0, 256, 32, dtype=np.uint8).tobytes()
        w12, w13 = (int(x) for x in rng.integers(0, 1 << 32, 2, dtype=np.uint64))
        w12 = min(w12, (1 << 32) - 4)                      # the 32-bit block counter must not wrap in 4 blocks
        w14 = (int(rng.integers(0, 5)) << 8) | int(rng.integers(0, 32))
        nonce16 = struct.pack("<4I", w12, w13, w14, 0)
        want = Cipher(algorithms.ChaCha20(key, nonce16), mode=None).encryptor().update(bytes(4 * 64))
        got = R.chacha20_blocks(key, np.arange(w12, w12 + 4, dtype=np.uint64), w13, w14).astype("<u4").tobytes()
        assert got == want


def test_row_layout():
    """coefficient 4b + m takes value m of block b; value m is u64 words 2m (low) and 2m + 1 (high)"""
    seed = bytes(range(100, 132))
    lo, hi = R.row_values(seed, 5, R.ROLE_U, [3], 64)
    for b in (0, 7, 15):
        words = np.frombuffer(R.chacha20_block(seed, b, 5, (R.ROLE_U << 8) | 3), "<u8")
        for m in range(4):
            assert lo[0, 4 * b + m] == words[2 * m] and hi[0, 4 * b + m] == words[2 * m + 1]


def test_uniform_sampler_reduces_the_whole_128_bits(oracle):
    ctx = oracle.BfvParameters(16, 1153, moduli_sizes=[62, 60]).context_at_level(0)
    seed = bytes(32)
    a = R.uniform_ntt(seed, 2, ctx)
    lo, hi = R.row_values(seed, 2, R.ROLE_A, [0, 1], 16)
    for j, q in enumerate(ctx.moduli):
        assert [int(x) for x in a.c[j]] == [((int(h) << 64) | int(l)) % q for l, h in zip(lo[j], hi[j])]


@pytest.mark.parametrize("variance", [1, 10, 16, 17, 32])
def test_cbd_matches_the_binomial_distribution(variance):
    """x + 2 variance ~ Binomial(4 variance, 1/2), the distribution of sample_vec_cbd (fhe-util/src/lib.rs:22-67)"""
    from scipy import stats
    n = 1 << 14
    x = np.concatenate([R.cbd(bytes([variance] * 32), ct, R.ROLE_E, variance, n) for ct in range(4)])
    assert np.abs(x).max() <= 2 * variance
    support = np.arange(4 * variance + 1)
    pmf = stats.binom.pmf(support, 4 * variance, 0.5) * x.size
    keep = np.nonzero(pmf >= 5)[0]
    lo, hi = keep[0], keep[-1]
    obs = np.bincount(np.clip(x + 2 * variance, lo, hi) - lo, minlength=hi - lo + 1)
    exp = pmf[lo:hi + 1].copy()
    exp[0] += pmf[:lo].sum()
    exp[-1] += pmf[hi + 1:].sum()
    assert stats.chisquare(obs, exp * obs.sum() / exp.sum()).pvalue > 1e-4
    assert abs(x.mean()) < 0.05 * np.sqrt(variance) and abs(x.var() / variance - 1) < 0.05


def test_cbd_masks():
    for v in (1, 10, 16, 17, 31, 32):
        (alo, ahi), (slo, shi) = R.cbd_masks(v)
        add, sub = (int(ahi) << 64) | int(alo), (int(shi) << 64) | int(slo)
        assert add == (1 << (2 * v)) - 1 and sub == add << (2 * v) and add & sub == 0


def _public_key_classes():
    """bfv.proto:5-9 and :50-52 as descriptors of the google.protobuf runtime"""
    T = descriptor_pb2.FieldDescriptorProto
    pool = descriptor_pool.DescriptorPool()
    f = descriptor_pb2.FileDescriptorProto(name="test_pk.proto", package="fhers.bfv", syntax="proto3")
    ct = f.message_type.add(name="Ciphertext")
    ct.field.add(name="c", number=1, type=T.TYPE_BYTES, label=T.LABEL_REPEATED)
    ct.field.add(name="seed", number=2, type=T.TYPE_BYTES, label=T.LABEL_OPTIONAL)
    ct.field.add(name="level", number=3, type=T.TYPE_UINT32, label=T.LABEL_OPTIONAL)
    pk = f.message_type.add(name="PublicKey")
    pk.field.add(name="c", number=1, type=T.TYPE_MESSAGE, label=T.LABEL_OPTIONAL, type_name=".fhers.bfv.Ciphertext")
    pool.Add(f)
    get = lambda n: message_factory.GetMessageClass(pool.FindMessageTypeByName("fhers.bfv." + n))
    return get("Ciphertext"), get("PublicKey")


CT, PK = _public_key_classes()


@pytest.mark.parametrize("seeded", [False, True])
def test_public_key_codec_matches_protobuf(F, seeded):
    from fhe_rs_b200 import wire
    rng = np.random.default_rng(3)
    polys = [rng.integers(0, 256, 300, dtype=np.uint8).tobytes() for _ in range(1 if seeded else 2)]
    seed = bytes(range(32)) if seeded else b""
    ct = wire.encode_ciphertext(polys, seed, 0)
    msg = wire.encode_public_key(ct)
    want = PK(c=CT(c=polys, seed=seed, level=0)).SerializeToString()
    assert msg == want
    assert bytes(wire.decode_public_key(want)) == ct
    parsed = PK()
    parsed.ParseFromString(msg)
    assert list(parsed.c.c) == polys and parsed.c.seed == seed


def test_public_key_refusals(F, oracle):
    """InvalidPublicKeyLevel, a compact message without its expanded c1, a missing ciphertext; host-only parameters
    reach the device (NO_DEVICE) only for a well-formed message"""
    from fhe_rs_b200 import _capi, wire
    degree = 16
    opar = oracle.BfvParameters(degree, 1153, moduli_sizes=[62, 62])
    gpar = F.BfvParameters(degree, 1153, moduli=opar.moduli, device=-1)
    rq = wire.encode_rq(wire.REP_NTT, degree, bytes(2 * 62 * degree // 8))
    level1 = PK(c=CT(c=[rq, rq], level=1)).SerializeToString()
    with pytest.raises(F.WireError) as e:
        F.PublicKey.from_bytes(gpar, level1)
    assert e.value.variant == "InvalidPublicKeyLevel" and e.value.code == _capi.INVALID_LEVEL
    compact = PK(c=CT(c=[rq], seed=bytes(32))).SerializeToString()
    with pytest.raises(F.WireError) as e:
        F.PublicKey.from_bytes(gpar, compact)
    assert e.value.variant == "SeedExpansion" and e.value.code == _capi.UNSUPPORTED
    with pytest.raises(F.WireError) as e:
        F.PublicKey.from_bytes(gpar, b"")
    assert e.value.variant == "MissingField"
    with pytest.raises(F.FheError) as e:
        F.PublicKey.from_bytes(gpar, PK(c=CT(c=[rq, rq])).SerializeToString())
    assert e.value.code == _capi.NO_DEVICE


def test_encryption_refusals_without_a_device(F, oracle):
    from fhe_rs_b200 import _capi
    lib = _capi.lib()
    degree = 1 << 12
    opar = oracle.BfvParameters(degree, 1032193, moduli_sizes=[62, 62])
    for v in (0, 33):
        with pytest.raises(F.FheError) as e:
            F.BfvParametersBuilder().set_degree(degree).set_plaintext_modulus(1032193).set_moduli(opar.moduli) \
                .set_variance(v).build(device=-1)
        assert e.value.code == _capi.INVALID_ARGUMENT and "InvalidVariance" in str(e.value)
        assert lib.fhe_b200_encrypt_sk(None, None, v, bytes(32), None, None) == _capi.INVALID_ARGUMENT
        assert b"InvalidVariance" in lib.fhe_b200_last_error()
        assert lib.fhe_b200_encrypt_pk(None, None, v, bytes(32), None, None) == _capi.INVALID_ARGUMENT
        assert b"InvalidVariance" in lib.fhe_b200_last_error()
    assert lib.fhe_b200_encrypt_sk(None, None, 10, bytes(32), None, None) == _capi.INVALID_ARGUMENT
    assert lib.fhe_b200_encrypt_pk(None, None, 10, bytes(32), None, None) == _capi.INVALID_ARGUMENT
    gpar = F.BfvParametersBuilder().set_degree(degree).set_plaintext_modulus(1032193).set_moduli(opar.moduli) \
        .set_variance(32).build(device=-1)
    assert gpar.variance == 32
    # host-only parameters hold no key and no batch: the key that would encrypt is refused with NO_DEVICE
    h = C.c_void_p()
    assert lib.fhe_b200_secret_key_create(gpar._h, np.zeros(degree, np.int64).ctypes.data, C.byref(h)) == _capi.NO_DEVICE
    with pytest.raises(F.FheError) as e:
        F.SecretKey(gpar, np.zeros(degree, np.int64))
    assert e.value.code == _capi.NO_DEVICE
