"""CPU restatement, on the oracle (oracle/fhe_oracle.py, oracle/fhe_wire.py), of what the PIR tests compare the device
with:
  - fhe_util::transcode_bidirectional (fhe-util/src/lib.rs:148-187), the sibling of the oracle's transcode_to_bytes /
    transcode_from_bytes, and an independent bit-stream statement of all three;
  - the EvaluationKey message (fhe/src/proto/bfv.proto:34-38, keys/evaluation_key.rs:293-310, :494-550) as a
    descriptor of the google.protobuf runtime, and its conversions;
  - the SealPIR example (fhe/examples/sealpir.rs, examples/util.rs:80-145): database encoding, the query, the server's
    response and the client's answer."""
from __future__ import annotations

import math
from typing import Dict, List, Optional, Sequence

import numpy as np
from google.protobuf import descriptor_pb2, descriptor_pool, message_factory

import encode_reference as ER
import fhe_oracle as O
import fhe_wire as W


# ------------------------------------------------------------------------------------------ transcoders
def transcode_bidirectional(a: Sequence[int], input_nbits: int, output_nbits: int) -> List[int]:
    """fhe_util::transcode_bidirectional, lib.rs:148-187: the reference's loop (words masked to input_nbits)"""
    assert 0 < input_nbits <= 64 and 0 < output_nbits <= 64
    in_mask, out_mask = (1 << input_nbits) - 1, (1 << output_nbits) - 1
    out: List[int] = []
    cur = have = idx = 0
    while idx < len(a):
        if have < output_nbits:
            cur |= (int(a[idx]) & in_mask) << have
            have += input_nbits
            idx += 1
        while have >= output_nbits:
            out.append(cur & out_mask)
            cur >>= output_nbits
            have -= output_nbits
    if have > 0:
        out.append(cur)
    assert len(out) == -(-len(a) * input_nbits // output_nbits)
    return out


def bitstream(a: Sequence[int], input_nbits: int, output_nbits: int) -> List[int]:
    """the same map stated on the row's LSB-first bit stream held as one integer"""
    x = 0
    for k, v in enumerate(a):
        x |= (int(v) & ((1 << input_nbits) - 1)) << (k * input_nbits)
    n = -(-len(a) * input_nbits // output_nbits)
    return [(x >> (k * output_nbits)) & ((1 << output_nbits) - 1) for k in range(n)]


def rows_reference(rows: Sequence[Sequence[int]], in_bits: int, out_bits: int, out_len: int) -> np.ndarray:
    """what fhe_b200_transcode writes for these rows: the first out_len values of each, zero-padded"""
    out = np.zeros((len(rows), out_len), np.uint64)
    for r, row in enumerate(rows):
        v = transcode_bidirectional(row, in_bits, out_bits)[:out_len]
        out[r, :len(v)] = np.array(v, dtype=np.uint64)
    return out


# ------------------------------------------------------------------------------------------ EvaluationKey message
def _evaluation_key_class():
    """EvaluationKey (bfv.proto:34-38) in a pool of its own, holding copies of the oracle's rq / bfv descriptors, so the
    oracle's pool is left as it is"""
    pool = descriptor_pool.DescriptorPool()
    for name in ("oracle_rq.proto", "oracle_bfv.proto"):
        f = descriptor_pb2.FileDescriptorProto()
        W._POOL.FindFileByName(name).CopyToProto(f)
        pool.Add(f)
    f = descriptor_pb2.FileDescriptorProto(name="oracle_bfv_ek.proto", package="fhers.bfv", syntax="proto3",
                                           dependency=["oracle_bfv.proto"])
    m = f.message_type.add(name="EvaluationKey")
    T = descriptor_pb2.FieldDescriptorProto
    m.field.add(name="gk", number=2, type=T.TYPE_MESSAGE, type_name=".fhers.bfv.GaloisKey", label=T.LABEL_REPEATED)
    m.field.add(name="ciphertext_level", number=3, type=T.TYPE_UINT32, label=T.LABEL_OPTIONAL)
    m.field.add(name="evaluation_key_level", number=4, type=T.TYPE_UINT32, label=T.LABEL_OPTIONAL)
    pool.Add(f)
    return message_factory.GetMessageClass(pool.FindMessageTypeByName("fhers.bfv.EvaluationKey"))


EvaluationKeyProto = _evaluation_key_class()


class EvaluationKeyError(ValueError):
    def __init__(self, variant: str):
        super().__init__(variant)
        self.variant = variant


def evaluation_key_to_bytes(gks: Dict[int, "O.GaloisKey"], ciphertext_level: int, evaluation_key_level: int,
                            order: Optional[Sequence[int]] = None) -> bytes:
    """From<&EvaluationKey> for EvaluationKeyProto (evaluation_key.rs:494-505), the keys in `order` (default
    ascending exponents; the reference's HashMap order is unspecified)"""
    m = EvaluationKeyProto()
    for e in (sorted(gks) if order is None else order):
        m.gk.add().ParseFromString(W.galois_key_to_bytes(gks[e]))
    m.ciphertext_level, m.evaluation_key_level = ciphertext_level, evaluation_key_level
    return m.SerializeToString()


def evaluation_key_from_bytes(par: "O.BfvParameters", data: bytes):
    """TryConvertFrom<&EvaluationKeyProto> (evaluation_key.rs:507-550): (exponent -> GaloisKey, levels)"""
    m = EvaluationKeyProto()
    m.ParseFromString(data)
    gks: Dict[int, "O.GaloisKey"] = {}
    for g in m.gk:
        key = W.galois_key_from_bytes(par, g.SerializeToString())
        if key.ksk.ciphertext_level != m.ciphertext_level or key.ksk.ksk_level != m.evaluation_key_level:
            raise EvaluationKeyError("InvalidLevel")
        gks[key.exponent] = key                                        # HashMap::insert: the later key wins
    if m.ciphertext_level > par.max_level():                           # par.context_at_level(ciphertext_level)?
        raise EvaluationKeyError("InvalidLevel")
    return gks, m.ciphertext_level, m.evaluation_key_level


def builder_exponents(degree: int, row_rotation=False, inner_sum=False, expansion=0) -> List[int]:
    """the exponents EvaluationKeyBuilder::build (evaluation_key.rs:429-491) generates keys for"""
    idx = set()
    if row_rotation or inner_sum:
        idx.add(2 * degree - 1)
    if inner_sum:
        i = 1
        while i < degree // 2:
            idx.add(pow(3, i, 2 * degree))
            i *= 2
    for l in range(expansion):
        idx.add((degree >> l) + 1)
    return sorted(idx)


# ------------------------------------------------------------------------------------------ SealPIR
SEALPIR_DEGREE, SEALPIR_T, SEALPIR_SIZES = 4096, 2056193, [36, 36, 37]   # sealpir.rs:38-40


def number_elements_per_plaintext(degree: int, plaintext_nbits: int, elements_size: int) -> int:   # util.rs:84-91
    return (plaintext_nbits * degree) // (elements_size * 8)


def layout(degree: int, t: int, n_elements: int, elements_size: int):
    """(elements per plaintext, rows, dim1, dim2) of encode_database (util.rs:95-115)"""
    epp = number_elements_per_plaintext(degree, t.bit_length() - 1, elements_size)
    rows = -(-n_elements // epp)
    dim1 = math.ceil(math.sqrt(rows))
    return epp, rows, dim1, -(-rows // dim1)


def database_values(database: np.ndarray, degree: int, t: int) -> np.ndarray:
    """the u64 values of every row of encode_database (util.rs:117-143) before encoding: [dim1 * dim2][<= N]"""
    n, es = database.shape
    epp, rows, dim1, dim2 = layout(degree, t, n, es)
    nbits = t.bit_length() - 1
    flat = np.zeros(dim1 * dim2 * epp * es, np.uint8)
    flat[: n * es] = database.reshape(-1)
    vals = np.zeros((dim1 * dim2, degree), np.uint64)
    for i in range(rows):
        v = O.transcode_from_bytes(flat[i * epp * es: (i + 1) * epp * es].tobytes(), nbits)
        vals[i, : len(v)] = np.array(v[:degree], dtype=np.uint64)
    return vals


def query_values(dim1: int, dim2: int, index: int, epp: int, t: int) -> np.ndarray:
    """sealpir.rs:126-141: the selection vector of the row holding `index`"""
    level = (dim1 + dim2 - 1).bit_length()                              # next_power_of_two().ilog2()
    qi = index // epp
    inv = pow(1 << level, -1, t)
    pt = np.zeros(dim1 + dim2, np.uint64)
    pt[qi // dim2] = inv
    pt[dim1 + qi % dim2] = inv
    return pt


def server_response(par: "O.BfvParameters", gks: dict, db_ntt: np.ndarray, query: "O.Ciphertext", dim1: int,
                    dim2: int) -> List["O.Ciphertext"]:
    """sealpir.rs:158-211 on the oracle.  db_ntt: poly_ntt words [dim1 * dim2][limbs][N] of the level-1 database"""
    ctx1 = par.context_at_level(1)
    expanded = O.expands(par, gks, query, dim1 + dim2)
    dots = []
    for i in range(dim2):
        column = [O.Poly(ctx1, O.NTT, db_ntt[k * dim2 + i]) for k in range(dim1)]
        c = O.dot_product_scalar(expanded[:dim1], column)
        dots.append(c.switch_to_level(par.max_level()))
    in_bits, out_bits = par.moduli[0].bit_length(), par.plaintext.bit_length() - 1
    fold = []
    for c in dots:
        vals = []
        for p in c.c:
            vals += transcode_bidirectional(p.c.reshape(-1), in_bits, out_bits)
        fold.append(ER.try_encode(par, np.array(vals, dtype=np.uint64), False, 1))
    out = []
    for i in range(len(fold[0])):
        r = O.dot_product_scalar(expanded[dim1:], [O.Poly(ctx1, O.NTT, f[i]) for f in fold])
        out.append(r.switch_to_level(par.max_level()))
    return out


def fold_values(words: np.ndarray, in_bits: int, out_bits: int) -> np.ndarray:
    """the values the fold encodes for one ciphertext's words [parts][limbs][N]"""
    vals = []
    for p in words:
        vals += transcode_bidirectional(p.reshape(-1), in_bits, out_bits)
    return np.array(vals, dtype=np.uint64)


def client_answer(par: "O.BfvParameters", decrypt, responses: Sequence, index: int, elements_size: int) -> bytes:
    """sealpir.rs:222-273.  decrypt(ciphertext words [parts][limbs][N], level) -> N decoded u64 values"""
    n, t = par.degree, par.plaintext
    in_bits, nbits = par.moduli[0].bit_length(), t.bit_length() - 1
    vec = np.concatenate([decrypt(r, par.max_level()) for r in responses])
    e = -(-n * in_bits // nbits)
    assert len(vec) >= 2 * e
    polys = [transcode_bidirectional(vec[k * e:(k + 1) * e], nbits, in_bits)[:n] for k in range(2)]
    pt = decrypt(np.array(polys, dtype=np.uint64)[:, None, :], par.max_level())
    plaintext = O.transcode_to_bytes(pt, nbits)
    offset = index % number_elements_per_plaintext(n, nbits, elements_size)
    return plaintext[offset * elements_size:(offset + 1) * elements_size]
