"""CPU tests of decryption's host side: the SecretKey message codecs (fhe_rs_b200/wire.py and include/fhe_b200_wire.hpp)
against the google.protobuf runtime, and the refusals of the decryption entry points that need no device."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest
from google.protobuf import descriptor_pb2, descriptor_pool, message_factory

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
I64 = np.iinfo(np.int64)
EXTREMES = [I64.min, -1, I64.max, 0, 1, I64.min + 1, I64.max - 1]


@pytest.fixture(scope="module")
def F():
    import fhe_rs_b200
    return fhe_rs_b200


def _secret_key_class():
    """bfv.proto:54-56 (`message SecretKey { repeated sint64 coeffs = 1; }`, packed by default in proto3) as a
    descriptor of the google.protobuf runtime, independent of both hand-written codecs"""
    T = descriptor_pb2.FieldDescriptorProto
    pool = descriptor_pool.DescriptorPool()
    f = descriptor_pb2.FileDescriptorProto(name="test_sk.proto", package="fhers.bfv", syntax="proto3")
    m = f.message_type.add(name="SecretKey")
    m.field.add(name="coeffs", number=1, type=T.TYPE_SINT64, label=T.LABEL_REPEATED)
    pool.Add(f)
    return message_factory.GetMessageClass(pool.FindMessageTypeByName("fhers.bfv.SecretKey"))


SK = _secret_key_class()


def _proto_bytes(coeffs):
    return SK(coeffs=[int(c) for c in coeffs]).SerializeToString()


def _cases():
    rng = np.random.default_rng(7)
    cbd = rng.integers(-10, 11, size=64).tolist()
    wide = rng.integers(I64.min, I64.max, size=64, dtype=np.int64, endpoint=True).tolist()
    return {"cbd": cbd, "wide": wide, "extremes": (EXTREMES * 10)[:64], "zeros": [0] * 64}


@pytest.mark.parametrize("case", list(_cases()))
def test_python_secret_key_codec_matches_protobuf(F, case):
    from fhe_rs_b200 import wire
    coeffs = _cases()[case]
    msg = wire.encode_secret_key(coeffs)
    assert msg == _proto_bytes(coeffs)
    assert wire.decode_secret_key(msg, len(coeffs)) == coeffs
    # unpacked encoding (what a proto2 writer emits) is accepted too, as prost does
    unpacked = b"".join(b"\x08" + wire._varint(wire._zigzag(c)) for c in coeffs)
    assert wire.decode_secret_key(unpacked, len(coeffs)) == coeffs
    parsed = SK()
    parsed.ParseFromString(msg)
    assert list(parsed.coeffs) == coeffs


def test_python_secret_key_codec_rejects_a_wrong_count(F):
    from fhe_rs_b200 import wire
    msg = wire.encode_secret_key([1, -1, 0])
    for degree in (2, 4, 16):
        with pytest.raises(wire.WireError) as e:
            wire.decode_secret_key(msg, degree)
        assert e.value.variant == "InvalidSecretKeyCoefficientCount"
    with pytest.raises(wire.WireError) as e:
        wire.decode_secret_key(b"", 16)
    assert e.value.variant == "InvalidSecretKeyCoefficientCount"
    with pytest.raises(wire.WireError) as e:
        wire.decode_secret_key(b"\x0a\x02\xff", 1)      # truncated packed varint
    assert e.value.variant == "Decode"


def test_cpp_secret_key_codec_matches_protobuf(F, tmp_path):
    from fhe_rs_b200 import build
    build.build()                               # the header links against the C ABI library (no-op when it is current)
    exe = str(tmp_path / "secret_key_wire_test")
    lib_dir = os.path.join(ROOT, "fhe_rs_b200")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "cpp", "secret_key_wire_test.cpp"), "-o", exe,
                           "-L", lib_dir, "-lfhe_b200", "-Wl,-rpath," + lib_dir])
    for name, coeffs in _cases().items():
        np.array(coeffs, np.int64).tofile(str(tmp_path / "c.i64"))
        subprocess.check_call([exe, "e", str(tmp_path / "c.i64"), str(tmp_path / "m.bin")])
        msg = (tmp_path / "m.bin").read_bytes()
        assert msg == _proto_bytes(coeffs), name
        out = subprocess.run([exe, "d", str(tmp_path / "m.bin"), str(len(coeffs)), str(tmp_path / "d.i64")],
                             capture_output=True, text=True)
        assert out.returncode == 0, out.stdout + out.stderr
        assert np.fromfile(str(tmp_path / "d.i64"), np.int64).tolist() == coeffs, name
        out = subprocess.run([exe, "d", str(tmp_path / "m.bin"), str(len(coeffs) + 1), str(tmp_path / "d.i64")],
                             capture_output=True, text=True)
        assert out.returncode == 3 and out.stdout.strip() == "InvalidSecretKeyCoefficientCount", name


def test_decryption_entry_points_need_a_device(F, oracle):
    from fhe_rs_b200 import _capi
    lib = _capi.lib()
    degree = 1 << 12
    opar = oracle.BfvParameters(degree, 1032193, moduli_sizes=[62, 62])
    gpar = F.BfvParameters(degree, 1032193, moduli=opar.moduli, device=-1)
    coeffs = np.zeros(degree, np.int64)
    h = C.c_void_p()
    assert lib.fhe_b200_secret_key_create(gpar._h, coeffs.ctypes.data, C.byref(h)) == _capi.NO_DEVICE
    assert not h.value
    with pytest.raises(F.FheError) as e:
        F.SecretKey(gpar, coeffs)
    assert e.value.code == _capi.NO_DEVICE
    out = np.zeros(degree, np.uint64)
    for enc in (_capi.ENCODING_POLY, _capi.ENCODING_SIMD):
        assert lib.fhe_b200_decode(gpar.encoder(), enc, 0, None, out.ctypes.data, degree, None) == _capi.NO_DEVICE
    # without a key (which host-only parameters cannot have) decrypt and measure_noise refuse their arguments
    assert lib.fhe_b200_decrypt(None, None, None, None) == _capi.INVALID_ARGUMENT
    assert lib.fhe_b200_measure_noise(None, None, out.ctypes.data, None) == _capi.INVALID_ARGUMENT


def test_large_plaintext_modulus_is_unsupported(F, oracle):
    from fhe_rs_b200 import _capi
    lib = _capi.lib()
    degree = 1 << 12
    opar = oracle.BfvParameters(degree, 1032193, moduli_sizes=[62, 62])
    coeffs = np.zeros(degree, np.int64)
    out = np.zeros(degree, np.uint64)
    # t beyond a u64 Modulus: the large-t branch of try_decrypt is not implemented
    gbig = F.BfvParameters(degree, (1 << 70) + 1, moduli=opar.moduli, device=-1)
    h = C.c_void_p()
    assert lib.fhe_b200_secret_key_create(gbig._h, coeffs.ctypes.data, C.byref(h)) == _capi.UNSUPPORTED
    assert lib.fhe_b200_decode(gbig.encoder(), 0, 0, None, out.ctypes.data, degree, None) == _capi.UNSUPPORTED
    # t >= q_0: decoding would need the CRT lift of every limb
    omix = oracle.BfvParameters(degree, 1032193, moduli_sizes=[30, 62])
    t40 = oracle.generate_prime(40, 2 * degree, 1 << 40)
    gmix = F.BfvParameters(degree, t40, moduli=omix.moduli, device=-1)
    for enc in (0, 1):
        assert lib.fhe_b200_decode(gmix.encoder(), enc, 0, None, out.ctypes.data, degree, None) == _capi.UNSUPPORTED
