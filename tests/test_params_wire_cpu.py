"""CPU tests of the Parameters message (bfv.proto:40-48, BfvParameters::to_bytes / try_deserialize at
parameters.rs:741-789) in both host codecs: fhe_rs_b200/wire.py and include/fhe_b200_wire.hpp (through
tests/cpp/params_wire_test.cpp) against the google.protobuf runtime, the reference's `serialize` and
`big_plaintext_modulus` cases restated, and the refusals of the decoder.

prost writes a oneof at the position of its lowest field number, so a message with `plaintext_big` (5) has it before
`variance` (4), where the runtime, which writes field-number order, puts it after.  The codecs' bytes are therefore
pinned to the runtime's own encoding of each field, concatenated in prost's order; for `plaintext` (3) both orders are
the same and the bytes equal the runtime's whole message."""
import os
import subprocess

import pytest
from google.protobuf import descriptor_pb2, descriptor_pool, message_factory

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BIG_PRIME = 340282366920938463463374607431768211507    # parameters.rs:876-930
SERIALIZE_MODULI = [4611686018427387617, 4611686018427387329, 4611686018427387073, 2305843009213693921,
                    1152921504606845473, 2017]          # set_moduli_sizes(&[62, 62, 62, 61, 60, 11]) at degree 16


def _parameters_class():
    """bfv.proto:40-48 as a descriptor of the google.protobuf runtime, independent of both hand-written codecs"""
    T = descriptor_pb2.FieldDescriptorProto
    pool = descriptor_pool.DescriptorPool()
    f = descriptor_pb2.FileDescriptorProto(name="test_params.proto", package="fhers.bfv", syntax="proto3")
    m = f.message_type.add(name="Parameters")
    m.oneof_decl.add(name="plaintext_modulus")
    m.field.add(name="degree", number=1, type=T.TYPE_UINT32, label=T.LABEL_OPTIONAL)
    m.field.add(name="moduli", number=2, type=T.TYPE_UINT64, label=T.LABEL_REPEATED)
    m.field.add(name="plaintext", number=3, type=T.TYPE_UINT64, label=T.LABEL_OPTIONAL, oneof_index=0)
    m.field.add(name="variance", number=4, type=T.TYPE_UINT32, label=T.LABEL_OPTIONAL)
    m.field.add(name="plaintext_big", number=5, type=T.TYPE_BYTES, label=T.LABEL_OPTIONAL, oneof_index=0)
    pool.Add(f)
    return message_factory.GetMessageClass(pool.FindMessageTypeByName("fhers.bfv.Parameters"))


P = _parameters_class()


def _le(t: int) -> bytes:
    return t.to_bytes(max(1, (t.bit_length() + 7) // 8), "little")


def prost_bytes(degree, moduli, t, variance) -> bytes:
    """what prost emits: degree, moduli, the oneof member, variance, each field as the runtime encodes it"""
    member = P(plaintext=t) if 2 <= t < 1 << 62 else P(plaintext_big=_le(t))
    return (P(degree=degree, moduli=moduli).SerializeToString() + member.SerializeToString()
            + P(variance=variance).SerializeToString())


CASES = {
    "serialize_small": (16, SERIALIZE_MODULI, 2, 4),
    "serialize_big": (16, SERIALIZE_MODULI[:3], BIG_PRIME, 4),
    "set_c": (1 << 15, [(1 << 62) - 57 - 2 * k for k in range(14)], 786433, 10),
    "t_2_62_minus_1": (1 << 12, [(1 << 62) - 1], (1 << 62) - 1, 32),
    "t_2_62": (1 << 12, [(1 << 63) + 1], 1 << 62, 1),          # a wide modulus: plaintext_big
    "t_2_64_minus_1": (8, [3], (1 << 64) - 1, 10),
    "t_1": (8, [17], 1, 10),
    "defaults": (0, [], 2, 0),
    "max_words": (0xFFFFFFFF, [(1 << 64) - 1, 0], 3, 0xFFFFFFFF),
}


@pytest.mark.parametrize("case", list(CASES))
def test_python_codec_matches_runtime(case):
    from fhe_rs_b200 import wire
    degree, moduli, t, variance = CASES[case]
    msg = wire.encode_parameters(degree, moduli, t, variance)
    assert msg == prost_bytes(degree, moduli, t, variance)
    if wire.plaintext_is_small(t):
        assert msg == P(degree=degree, moduli=moduli, plaintext=t, variance=variance).SerializeToString()
    parsed = P()
    parsed.ParseFromString(msg)
    assert parsed.WhichOneof("plaintext_modulus") == ("plaintext" if wire.plaintext_is_small(t) else "plaintext_big")
    assert (parsed.degree, list(parsed.moduli), parsed.variance) == (degree, moduli, variance)
    assert wire.decode_parameters(msg) == (degree, moduli, t, variance)
    # the runtime's field-number order reads back the same
    full = P(degree=degree, moduli=moduli, variance=variance)
    if wire.plaintext_is_small(t):
        full.plaintext = t
    else:
        full.plaintext_big = _le(t)
    assert wire.decode_parameters(full.SerializeToString()) == (degree, moduli, t, variance)


def _unpacked(degree, moduli, t, variance) -> bytes:
    from fhe_rs_b200 import wire
    body = b"".join(b"\x10" + wire._varint(q) for q in moduli)
    return P(degree=degree).SerializeToString() + body + P(plaintext=t, variance=variance).SerializeToString()


def test_python_decoder_edges():
    from fhe_rs_b200 import wire
    assert wire.decode_parameters(_unpacked(16, [97, 193], 5, 3)) == (16, [97, 193], 5, 3)
    # unknown fields (every wire type) are skipped
    extra = b"\x30\x07" + b"\x3a\x02ab" + b"\x41" + bytes(8) + b"\x4d" + bytes(4) + b"\x53\x08\x01\x54"
    msg = wire.encode_parameters(16, [97], 5, 3)
    assert wire.decode_parameters(extra + msg + extra) == (16, [97], 5, 3)
    # the last oneof member wins, either way round
    assert wire.decode_parameters(msg + P(plaintext_big=_le(BIG_PRIME)).SerializeToString())[2] == BIG_PRIME
    assert wire.decode_parameters(P(plaintext_big=b"\x07").SerializeToString() + msg)[2] == 5
    # a zero plaintext is still a present member
    assert wire.decode_parameters(b"\x18\x00")[2] == 0
    assert wire.decode_parameters(P(plaintext_big=b"").SerializeToString() + b"\x2a\x00")[2] == 0
    for bad in (P(degree=16, moduli=[97], variance=3).SerializeToString(), b""):
        with pytest.raises(wire.WireError) as e:
            wire.decode_parameters(bad)
        assert e.value.variant == "MissingField" and "ParametersPlaintextModulus" in str(e.value)
    for n in (1, 3, 4, len(msg) - 1):           # cut inside a field: truncated key, length, payload or value
        with pytest.raises(wire.WireError) as e:
            wire.decode_parameters(msg[:n])
        assert e.value.variant == "Decode", n
    for bad in (b"\x08", b"\x12\x05\x01", b"\x1a\x00", b"\x2d\x00\x00\x00\x00", b"\x12\x01\xff" + msg, b"\x0f"):
        with pytest.raises(wire.WireError) as e:
            wire.decode_parameters(bad)
        assert e.value.variant == "Decode", bad


@pytest.fixture(scope="module")
def F():
    import fhe_rs_b200
    return fhe_rs_b200


def test_reference_serialize(F):
    """parameters.rs `serialize`: the small variant carries plaintext = 2 and the big one the prime's
    little-endian bytes; both decode to equal parameters"""
    par = F.BfvParameters(16, 2, moduli_sizes=[62, 62, 62, 61, 60, 11], device=-1, variance=4)
    assert par.moduli() == SERIALIZE_MODULI
    data = par.to_bytes()
    m = P()
    m.ParseFromString(data)
    assert m.WhichOneof("plaintext_modulus") == "plaintext" and m.plaintext == 2
    back = F.BfvParameters.from_bytes(data, device=-1)
    assert (back.degree(), back.moduli(), back.plaintext(), back.variance) == (16, SERIALIZE_MODULI, 2, 4)
    assert back.to_bytes() == data

    par = F.BfvParameters(16, BIG_PRIME, moduli_sizes=[62] * 5, device=-1, variance=4)
    data = par.to_bytes()
    m.ParseFromString(data)
    assert m.WhichOneof("plaintext_modulus") == "plaintext_big" and m.plaintext_big == _le(BIG_PRIME)
    back = F.BfvParameters.from_bytes(data, device=-1)
    assert (back.degree(), back.moduli(), back.plaintext(), back.variance) == (16, par.moduli(), BIG_PRIME, 4)
    assert back.to_bytes() == data


def test_reference_big_plaintext_modulus(F):
    """parameters.rs `big_plaintext_modulus`: a 128-bit prime builds; as_u64 is None, so the message is plaintext_big"""
    from fhe_rs_b200 import wire
    par = F.BfvParameters(16, BIG_PRIME, moduli_sizes=[62] * 5, device=-1)
    assert par.plaintext() == BIG_PRIME and not wire.plaintext_is_small(par.plaintext())


def test_decoder_builds_through_the_constructor(F):
    from fhe_rs_b200 import _capi, wire
    moduli = SERIALIZE_MODULI[:2]
    cases = {
        "variance 0": (wire.encode_parameters(16, moduli, 2, 0), _capi.INVALID_ARGUMENT, "InvalidVariance"),
        "variance 33": (wire.encode_parameters(16, moduli, 2, 33), _capi.INVALID_ARGUMENT, "InvalidVariance"),
        "degree 12": (wire.encode_parameters(12, moduli, 2, 4), _capi.INVALID_DEGREE, "InvalidPolynomialDegree"),
        "no moduli": (wire.encode_parameters(16, [], 2, 4), _capi.INVALID_ARGUMENT, None),
        "t 0": (b"\x08\x10\x18\x00\x20\x04", _capi.INVALID_ARGUMENT, None),
        "t not coprime": (wire.encode_parameters(16, moduli, moduli[0], 4), _capi.INVALID_MODULUS, None),
        "duplicate": (wire.encode_parameters(16, moduli[:1] * 2, 2, 4), _capi.INVALID_MODULUS, "DuplicateModuli"),
    }
    for name, (data, code, text) in cases.items():
        with pytest.raises(F.FheError) as e:
            F.BfvParameters.from_bytes(data, device=-1)
        assert e.value.code == code, name
        assert text is None or text in str(e.value), name
    # t in [2^62, 2^64): the reference's builder refuses it; this constructor takes it as a wide modulus
    par = F.BfvParameters(1 << 4, (1 << 62) + 135, moduli_sizes=[62] * 3, device=-1, variance=7)
    m = P()
    m.ParseFromString(par.to_bytes())
    assert m.WhichOneof("plaintext_modulus") == "plaintext_big"
    assert F.BfvParameters.from_bytes(par.to_bytes(), device=-1).plaintext() == (1 << 62) + 135


@pytest.fixture(scope="module")
def cpp(tmp_path_factory):
    from fhe_rs_b200 import build
    build.build()                               # the header links against the C ABI library (no-op when it is current)
    d = tmp_path_factory.mktemp("params_wire")
    exe = str(d / "params_wire_test")
    lib_dir = os.path.join(ROOT, "fhe_rs_b200")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-I", os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "cpp", "params_wire_test.cpp"), "-o", exe,
                           "-L", lib_dir, "-lfhe_b200", "-Wl,-rpath," + lib_dir])

    def run(*args):
        return subprocess.run([exe, *map(str, args)], capture_output=True, text=True, timeout=300)
    return run, d


def test_cpp_codec_matches_runtime(cpp):
    run, d = cpp
    msg_path = d / "m.bin"
    for name, (degree, moduli, t, variance) in CASES.items():
        out = run("e", degree, variance, _le(t).hex(), ",".join(map(str, moduli)), msg_path)
        assert out.returncode == 0, out.stdout + out.stderr
        assert msg_path.read_bytes() == prost_bytes(degree, moduli, t, variance), name
        out = run("d", msg_path)
        assert out.returncode == 0, out.stdout + out.stderr
        deg, var, t_hex, mods = out.stdout.split(" ")
        assert (int(deg), int(var), int.from_bytes(bytes.fromhex(t_hex), "little")) == (degree, variance, t), name
        assert [int(q) for q in mods.split(",") if q.strip()] == moduli, name
    msg_path.write_bytes(_unpacked(16, [97, 193], 5, 3))
    assert run("d", msg_path).stdout.split() == ["16", "3", "0500000000000000", "97,193"]
    msg_path.write_bytes(P(degree=16).SerializeToString() + b"\x3a\x02ab" + P(plaintext=5).SerializeToString())
    assert run("d", msg_path).stdout.split() == ["16", "0", "0500000000000000"]
    for bad, variant in ((P(degree=16, moduli=[97]).SerializeToString(), "MissingField"), (b"\x08", "Decode"),
                         (b"\x12\x05\x01", "Decode"), (b"\x1a\x00", "Decode")):
        msg_path.write_bytes(bad)
        out = run("d", msg_path)
        assert out.returncode == 3 and out.stdout.strip() == variant, bad


def test_cpp_round_trip_through_the_constructor(cpp, F):
    from fhe_rs_b200 import _capi
    run, d = cpp
    src, dst = d / "src.bin", d / "dst.bin"
    for t, sizes in ((2, [62, 62, 62, 61, 60, 11]), (BIG_PRIME, [62] * 5), ((1 << 62) + 135, [62] * 3)):
        data = F.BfvParameters(16, t, moduli_sizes=sizes, device=-1, variance=4).to_bytes()
        src.write_bytes(data)
        out = run("r", src, dst)
        assert out.returncode == 0, out.stdout + out.stderr
        assert dst.read_bytes() == data
    src.write_bytes(prost_bytes(16, SERIALIZE_MODULI[:2], 2, 0))
    out = run("r", src, dst)
    assert out.returncode == 4 and int(out.stdout) == _capi.INVALID_ARGUMENT
