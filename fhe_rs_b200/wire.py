"""Protobuf framing of the messages either side of the accelerated path (SURVEY section 8f row 1).

The reference serialises polynomials, ciphertexts and key-switching keys with prost:

    fhers.rq.Rq                  fhe-math/src/proto/rq.proto:12-17   (written by rq/convert.rs:17-44)
    fhers.bfv.Ciphertext         fhe/src/proto/bfv.proto:5-9         (bfv/ciphertext.rs:230-257)
    fhers.bfv.KeySwitchingKey    bfv.proto:16-23                     (keys/key_switching_key.rs:365-385)
    fhers.bfv.RelinearizationKey bfv.proto:25-27, GaloisKey :29-32, RGSWCiphertext :11-14
    fhers.bfv.EvaluationKey      bfv.proto:34-38                     (keys/evaluation_key.rs:293-310, :494-550)
    fhers.bfv.SecretKey          bfv.proto:54-56                     (keys/secret_key.rs:142-175)
    fhers.bfv.Parameters         bfv.proto:40-48                     (bfv/parameters.rs:741-789)

The heavy part of every one of them -- `Rq.coefficients`, the bit-packed power-basis words -- is produced and consumed
on the device (fhe_b200_batch_pack / fhe_b200_batch_unpack).  This module is the few bytes around it: a hand-written
proto3 wire codec for exactly these messages, emitting what prost emits (fields in field-number order, a oneof at its lowest field number, zero scalars
and empty singular `bytes` omitted, every element of a repeated `bytes` present, a present sub-message always
written) and accepting what prost accepts (any field order, unknown fields skipped, last scalar wins).  It depends on
nothing but the standard library; the tests compare it byte for byte with the google.protobuf runtime.

Seeded messages carry a 32-byte ChaCha8 seed instead of the last polynomial; expanding it is the Rust host's job
(include/fhe_b200.h) -- the decoders return the seed and the callers in bfv.py take the expanded half as an argument.
"""
from __future__ import annotations

from typing import Dict, Iterator, List, Optional, Sequence, Tuple, Union

from . import _capi
from ._capi import FheError

Bytes = Union[bytes, bytearray, memoryview]

# Representation enum, rq.proto:5-10
REP_UNKNOWN, REP_POWERBASIS, REP_NTT, REP_NTTSHOUP = 0, 1, 2, 3

_VARINT, _I64, _LEN, _I32 = 0, 1, 2, 5


class WireError(FheError):
    """PolynomialSerializationError (fhe-math/src/errors.rs) / SerializationError (fhe/src/errors.rs): `variant` is the
    reference's variant name, `code` the C-ABI status a host would map it to."""

    def __init__(self, variant: str, code: int = _capi.INVALID_ARGUMENT, detail: str = ""):
        super().__init__(code, variant + (": " + detail if detail else ""))
        self.variant = variant


# ------------------------------------------------------------------------------------------ primitives
def _varint(n: int) -> bytes:
    out = bytearray()
    while True:
        b = n & 0x7F
        n >>= 7
        if n:
            out.append(b | 0x80)
        else:
            out.append(b)
            return bytes(out)


def _key(field: int, wire_type: int) -> bytes:
    return _varint((field << 3) | wire_type)


def _put_uint(out: List[Bytes], field: int, value: int) -> None:
    if value:                                   # proto3: default values are not written
        out.append(_key(field, _VARINT) + _varint(value))


def _put_len(out: List[Bytes], field: int, payload: Bytes) -> None:
    out.append(_key(field, _LEN) + _varint(len(payload)))
    out.append(payload)


_START_GROUP, _END_GROUP = 3, 4


def _fields(buf: Bytes) -> Iterator[Tuple[int, int, Union[int, memoryview]]]:
    """(field number, wire type, value) of one message; raises WireError("Decode") on malformed input.  Follows prost's
    decoder: keys are 32-bit with a field number >= 1, varints are at most ten bytes, unknown groups are skipped whole
    (they never occur in these messages), an unmatched end-group or wire types 6 / 7 are errors."""
    mv = memoryview(buf).cast("B") if not isinstance(buf, memoryview) else buf.cast("B")
    pos, end = 0, len(mv)

    def varint() -> int:
        nonlocal pos
        shift = value = 0
        while True:
            if pos >= end:
                raise WireError("Decode", detail="truncated varint")
            b = mv[pos]
            pos += 1
            if shift == 63 and b > 1:
                raise WireError("Decode", detail="varint overflows 64 bits")
            value |= (b & 0x7F) << shift
            if not b & 0x80:
                return value
            shift += 7

    def key() -> Tuple[int, int]:
        k = varint()
        if k > 0xFFFFFFFF:
            raise WireError("Decode", detail="key does not fit 32 bits")
        if k >> 3 == 0:
            raise WireError("Decode", detail="field number 0")
        return k >> 3, k & 7

    def value(field: int, wt: int, depth: int):
        nonlocal pos
        if wt == _VARINT:
            return varint()
        if wt == _LEN:
            n = varint()
            if n > end - pos:
                raise WireError("Decode", detail="length-delimited field overruns the buffer")
            pos += n
            return mv[pos - n:pos]
        if wt == _I64 or wt == _I32:
            n = 8 if wt == _I64 else 4
            if n > end - pos:
                raise WireError("Decode", detail="truncated fixed-width field")
            pos += n
            return int.from_bytes(mv[pos - n:pos], "little")
        if wt == _START_GROUP:
            if depth >= 100:
                raise WireError("Decode", detail="recursion limit")
            while True:
                if pos >= end:
                    raise WireError("Decode", detail="unterminated group")
                f, w = key()
                if w == _END_GROUP:
                    if f != field:
                        raise WireError("Decode", detail="mismatched end of group")
                    return None
                value(f, w, depth + 1)
        raise WireError("Decode", detail="unsupported wire type %d" % wt)

    while pos < end:
        field, wt = key()
        v = value(field, wt, 0)
        if wt != _START_GROUP:
            yield field, wt, v
        else:
            yield field, wt, 0


def _expect(wt: int, want: int) -> None:
    if wt != want:
        raise WireError("Decode", detail="wire type %d where %d was expected" % (wt, want))


def _join(parts: Sequence[Bytes]) -> bytes:
    return b"".join(bytes(p) if isinstance(p, memoryview) else p for p in parts)


# ------------------------------------------------------------------------------------------ Rq
def encode_rq(representation: int, degree: int, coefficients: Bytes) -> bytes:
    """Rq::from(&poly).encode_to_vec(): allow_variable_time is always false on the wire (rq/convert.rs:39-41)"""
    out: List[Bytes] = []
    _put_uint(out, 1, representation)
    _put_uint(out, 2, degree)
    if len(coefficients):
        _put_len(out, 3, coefficients)
    return _join(out)


def rq_overhead(degree: int, n_coefficient_bytes: int, representation: int = REP_NTT) -> int:
    """bytes encode_rq adds around the coefficients"""
    return len(encode_rq(representation, degree, b"")) + (len(_key(3, _LEN) + _varint(n_coefficient_bytes))
                                                          if n_coefficient_bytes else 0)


def decode_rq(data: Bytes) -> Tuple[int, int, memoryview]:
    """-> (representation, degree, coefficients); the checks of parse_proto (rq/convert.rs:46-98) that need the context
    are the caller's"""
    rep, degree, coeffs = 0, 0, memoryview(b"")
    for field, wt, v in _fields(data):
        if field == 1:
            _expect(wt, _VARINT)
            rep = v & 0xFFFFFFFF
            rep = rep - (1 << 32) if rep >> 31 else rep          # enum fields are int32
        elif field == 2:
            _expect(wt, _VARINT)
            degree = v & 0xFFFFFFFF
        elif field == 3:
            _expect(wt, _LEN)
            coeffs = v
        elif field == 4:
            _expect(wt, _VARINT)                                  # the timing flag never grants anything (convert.rs:39-41)
    if rep not in (REP_UNKNOWN, REP_POWERBASIS, REP_NTT, REP_NTTSHOUP):
        raise WireError("InvalidRepresentation", _capi.INVALID_REPRESENTATION, str(rep))
    if rep == REP_UNKNOWN:
        raise WireError("UnknownRepresentation", _capi.INVALID_REPRESENTATION)
    if degree % 8 != 0 or degree < 8:
        raise WireError("InvalidDegree", _capi.INVALID_DEGREE, str(degree))
    return rep, degree, coeffs


# ------------------------------------------------------------------------------------------ Ciphertext
def encode_ciphertext(polys: Sequence[Bytes], seed: Bytes = b"", level: int = 0) -> bytes:
    """CiphertextProto::from(&ct).encode_to_vec() (bfv/ciphertext.rs:230-257): `polys` are encoded Rq messages --
    every part, or every part but the last when `seed` is the seed the last one was drawn from"""
    out: List[Bytes] = []
    for p in polys:
        _put_len(out, 1, p)
    if len(seed):
        _put_len(out, 2, seed)
    _put_uint(out, 3, level)
    return _join(out)


def decode_ciphertext(data: Bytes) -> Tuple[List[memoryview], bytes, int]:
    """-> (Rq messages, seed, level) with the count check of ciphertext.rs:261-269"""
    c: List[memoryview] = []
    seed, level = b"", 0
    for field, wt, v in _fields(data):
        if field == 1:
            _expect(wt, _LEN)
            c.append(v)
        elif field == 2:
            _expect(wt, _LEN)
            seed = bytes(v)
        elif field == 3:
            _expect(wt, _VARINT)
            level = v & 0xFFFFFFFF
    if not c or (len(c) == 1 and not seed):
        raise WireError("InvalidCiphertextPolynomialCount", _capi.BAD_POLY_COUNT,
                        "%d polynomials, seed %s" % (len(c), "present" if seed else "absent"))
    return c, seed, level


# ------------------------------------------------------------------------------------------ keys
def encode_ksk(c0: Sequence[Bytes], c1: Sequence[Bytes], seed: Bytes, ciphertext_level: int, ksk_level: int,
               log_base: int) -> bytes:
    """KeySwitchingKeyProto::from(&ksk).encode_to_vec() (key_switching_key.rs:365-385)"""
    out: List[Bytes] = []
    for p in c0:
        _put_len(out, 1, p)
    for p in c1:
        _put_len(out, 2, p)
    if len(seed):
        _put_len(out, 3, seed)
    _put_uint(out, 4, ciphertext_level)
    _put_uint(out, 5, ksk_level)
    _put_uint(out, 6, log_base)
    return _join(out)


def decode_ksk(data: Bytes) -> Dict[str, object]:
    k: Dict[str, object] = {"c0": [], "c1": [], "seed": b"", "ciphertext_level": 0, "ksk_level": 0, "log_base": 0}
    names = {4: "ciphertext_level", 5: "ksk_level", 6: "log_base"}
    for field, wt, v in _fields(data):
        if field in (1, 2):
            _expect(wt, _LEN)
            k["c0" if field == 1 else "c1"].append(v)
        elif field == 3:
            _expect(wt, _LEN)
            k["seed"] = bytes(v)
        elif field in names:
            _expect(wt, _VARINT)
            k[names[field]] = v & 0xFFFFFFFF
    return k


def _sub_messages(data: Bytes, wanted: Sequence[int]) -> Dict[int, Optional[memoryview]]:
    found: Dict[int, Optional[memoryview]] = {f: None for f in wanted}
    scalars: Dict[int, int] = {}
    for field, wt, v in _fields(data):
        if field in found:
            _expect(wt, _LEN)
            found[field] = v                   # (prost would merge a repeated occurrence; writers emit one)
        elif wt == _VARINT:
            scalars[field] = v
    found[-1] = scalars                        # type: ignore[assignment]
    return found


def encode_relinearization_key(ksk: Bytes) -> bytes:        # relinearization_key.rs:113-119
    out: List[Bytes] = []
    _put_len(out, 1, ksk)
    return _join(out)


def decode_relinearization_key(data: Bytes) -> memoryview:  # relinearization_key.rs:121-135
    f = _sub_messages(data, (1,))
    if f[1] is None:
        raise WireError("MissingField", detail="RelinearizationKeySwitchingKey")
    return f[1]


def encode_galois_key(ksk: Bytes, exponent: int) -> bytes:  # galois_key.rs:146-153
    out: List[Bytes] = []
    _put_len(out, 1, ksk)
    _put_uint(out, 2, exponent)
    return _join(out)


def decode_galois_key(data: Bytes) -> Tuple[memoryview, int]:   # galois_key.rs:155-173
    f = _sub_messages(data, (1,))
    if f[1] is None:
        raise WireError("MissingField", detail="GaloisKeySwitchingKey")
    return f[1], f[-1].get(2, 0) & 0xFFFFFFFF   # type: ignore[union-attr]


def encode_evaluation_key(galois_keys: Sequence[Bytes], ciphertext_level: int, evaluation_key_level: int) -> bytes:
    """EvaluationKeyProto::from(&ek).encode_to_vec() (evaluation_key.rs:494-505): the GaloisKey messages in the order
    given (the reference writes HashMap order, so a reader may depend on none), then the two levels"""
    out: List[Bytes] = []
    for gk in galois_keys:
        _put_len(out, 2, gk)
    _put_uint(out, 3, ciphertext_level)
    _put_uint(out, 4, evaluation_key_level)
    return _join(out)


def decode_evaluation_key(data: Bytes) -> Tuple[List[memoryview], int, int]:
    """(GaloisKey messages in wire order, ciphertext_level, evaluation_key_level) of an EvaluationKey message"""
    gks: List[memoryview] = []
    levels = {3: 0, 4: 0}
    for field, wt, v in _fields(data):
        if field == 2:
            _expect(wt, _LEN)
            gks.append(v)
        elif field in levels:
            _expect(wt, _VARINT)
            levels[field] = v & 0xFFFFFFFF
    return gks, levels[3], levels[4]


def encode_rgsw(ksk0: Bytes, ksk1: Bytes) -> bytes:         # rgsw_ciphertext.rs:30-37
    out: List[Bytes] = []
    _put_len(out, 1, ksk0)
    _put_len(out, 2, ksk1)
    return _join(out)


def decode_rgsw(data: Bytes) -> Tuple[memoryview, memoryview]:  # rgsw_ciphertext.rs:39-59
    f = _sub_messages(data, (1, 2))
    if f[1] is None:
        raise WireError("MissingField", detail="RgswKeySwitchingKey0")
    if f[2] is None:
        raise WireError("MissingField", detail="RgswKeySwitchingKey1")
    return f[1], f[2]


def encode_public_key(ciphertext: Bytes) -> bytes:         # public_key.rs:95-107, bfv.proto:50-52
    out: List[Bytes] = []
    _put_len(out, 1, ciphertext)
    return _join(out)


def decode_public_key(data: Bytes) -> memoryview:           # public_key.rs:109-149
    """the encoded Ciphertext inside a PublicKey message"""
    f = _sub_messages(data, (1,))
    if f[1] is None:
        raise WireError("MissingField", detail="PublicKeyCiphertext")
    return f[1]


# ------------------------------------------------------------------------------------------ SecretKey
def _zigzag(n: int) -> int:
    return ((n << 1) ^ (n >> 63)) & 0xFFFFFFFFFFFFFFFF


def _unzigzag(n: int) -> int:
    return (n >> 1) ^ -(n & 1)


def encode_secret_key(coeffs: Sequence[int]) -> bytes:   # secret_key.rs:142-148, bfv.proto:54-56
    """`repeated sint64 coeffs = 1`: one packed field of zig-zag varints (absent when there are no coefficients)"""
    out: List[Bytes] = []
    if len(coeffs):
        _put_len(out, 1, b"".join(_varint(_zigzag(int(c))) for c in coeffs))
    return _join(out)


def decode_secret_key(data: Bytes, degree: int) -> List[int]:   # secret_key.rs:151-175
    """the coefficients of a SecretKey message; packed and unpacked encodings are both accepted (as prost does).
    A count other than `degree` is InvalidSecretKeyCoefficientCount."""
    coeffs: List[int] = []
    for field, wt, v in _fields(data):
        if field != 1:
            continue
        if wt == _VARINT:
            coeffs.append(_unzigzag(v))
        elif wt == _LEN:
            coeffs.extend(_unzigzag(x) for x in _packed_varints(v))
        else:
            raise WireError("Decode", detail="wire type %d for a sint64 field" % wt)
    if len(coeffs) != degree:
        raise WireError("InvalidSecretKeyCoefficientCount", detail="%d coefficients, expected %d" % (len(coeffs), degree))
    return coeffs


# ------------------------------------------------------------------------------------------ Parameters
def plaintext_is_small(t: int) -> bool:
    """t is a zq::Modulus (2 <= t < 2^62): where PlaintextModulus::as_u64 is Some and the message carries `plaintext`"""
    return 2 <= t < 1 << 62


def encode_parameters(degree: int, moduli: Sequence[int], plaintext: int, variance: int) -> bytes:
    """BfvParameters::to_bytes (parameters.rs:741-759), bfv.proto:40-48: degree = 1, moduli = 2 (packed), the oneof
    plaintext = 3 (uint64) / plaintext_big = 5 (little-endian bytes), variance = 4.  prost writes a oneof at the
    position of its lowest field number, so plaintext_big goes before variance, as plaintext does."""
    out: List[Bytes] = []
    _put_uint(out, 1, degree)
    if len(moduli):
        _put_len(out, 2, b"".join(_varint(int(q)) for q in moduli))
    t = int(plaintext)
    if plaintext_is_small(t):
        out.append(_key(3, _VARINT) + _varint(t))         # a set oneof member is written even when it is zero
    else:
        _put_len(out, 5, t.to_bytes(max(1, (t.bit_length() + 7) // 8), "little"))   # BigUint::to_bytes_le
    _put_uint(out, 4, variance)
    return _join(out)


def decode_parameters(data: Bytes) -> Tuple[int, List[int], int, int]:
    """(degree, moduli, plaintext modulus, variance) of a Parameters message (parameters.rs:762-781): packed and
    unpacked moduli are both accepted, the last oneof member wins; malformed bytes are Decode, a message without
    either member is MissingField (ParametersPlaintextModulus)."""
    degree = variance = 0
    moduli: List[int] = []
    plaintext: Optional[int] = None
    for field, wt, v in _fields(data):
        if field in (1, 4):
            _expect(wt, _VARINT)
            if field == 1:
                degree = v & 0xFFFFFFFF
            else:
                variance = v & 0xFFFFFFFF
        elif field == 2:
            if wt == _VARINT:
                moduli.append(v)
            else:
                _expect(wt, _LEN)
                moduli.extend(_packed_varints(v))
        elif field == 3:
            _expect(wt, _VARINT)
            plaintext = v
        elif field == 5:
            _expect(wt, _LEN)
            plaintext = int.from_bytes(bytes(v), "little")
    if plaintext is None:
        raise WireError("MissingField", detail="ParametersPlaintextModulus")
    return degree, moduli, plaintext, variance


def _packed_varints(buf: memoryview) -> Iterator[int]:
    pos, end = 0, len(buf)
    while pos < end:
        shift = value = 0
        while True:
            if pos >= end:
                raise WireError("Decode", detail="truncated varint")
            b = buf[pos]
            pos += 1
            if shift == 63 and b > 1:
                raise WireError("Decode", detail="varint overflows 64 bits")
            value |= (b & 0x7F) << shift
            if not b & 0x80:
                break
            shift += 7
        yield value
