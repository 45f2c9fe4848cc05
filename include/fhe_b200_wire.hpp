// fhe_b200_wire.hpp -- the protobuf messages either side of the accelerated path, for C++ hosts (header-only).
//
// The reference serialises with prost (paths under the reference's crates/):
//   fhers.rq.Rq                   fhe-math/src/proto/rq.proto:12-17, written by fhe-math/src/rq/convert.rs:17-44
//   fhers.bfv.Ciphertext          fhe/src/proto/bfv.proto:5-9,       fhe/src/bfv/ciphertext.rs:230-317
//   fhers.bfv.KeySwitchingKey     bfv.proto:16-23,                   fhe/src/bfv/keys/key_switching_key.rs:365-482
//   fhers.bfv.RelinearizationKey  bfv.proto:25-27 (keys/relinearization_key.rs:113-135), GaloisKey :29-32
//                                 (keys/galois_key.rs:146-173), EvaluationKey :34-38 (keys/evaluation_key.rs:293-310,
//                                 :494-550)
//   fhers.bfv.SecretKey           bfv.proto:54-56,                   fhe/src/bfv/keys/secret_key.rs:142-175
//   fhers.bfv.PublicKey           bfv.proto:50-52,                   fhe/src/bfv/keys/public_key.rs:95-149
//   fhers.bfv.Parameters          bfv.proto:40-48,                   fhe/src/bfv/parameters.rs:741-789
// `Rq.coefficients` -- the bit-packed power-basis words, all but a few bytes of every message -- is produced and consumed
// on the device (fhe_b200_batch_pack / fhe_b200_batch_unpack); this header is the proto3 framing around it, emitting
// what prost emits (fields in field-number order, a oneof at its lowest field number, zero scalars and empty singular
// `bytes` omitted) and accepting what prost accepts (any order, unknown fields skipped, last scalar wins), plus the
// checks of the reference's decoders under the reference's variant names (WireError::variant).  The Python mirror's fhe_rs_b200/wire.py is the same
// codec; both are tested byte for byte against the google.protobuf runtime.
//
// Seeded messages carry a 32-byte ChaCha8 seed instead of their last polynomial (row c1 for keys).  Expanding it is
// the Rust host's job (see fhe_b200.h): the *_from_bytes functions take the expanded words as an argument.
#pragma once
#include <cstring>
#include <string>
#include <vector>

#include "fhe_b200.hpp"

namespace fhe_b200 {

// PolynomialSerializationError (fhe-math/src/errors.rs) / SerializationError (fhe/src/errors.rs) by variant name
struct WireError : Error {
  std::string variant;
  WireError(const std::string& v, int c = FHE_B200_INVALID_ARGUMENT, const std::string& detail = "")
      : Error(c, detail.empty() ? v : v + ": " + detail), variant(v) {}
};

namespace wire {

enum : int32_t { REP_UNKNOWN = 0, REP_POWERBASIS = 1, REP_NTT = 2, REP_NTTSHOUP = 3 };  // rq.proto:5-10

struct Span {
  const uint8_t* p = nullptr;
  size_t n = 0;
};

inline void put_varint(std::string& out, uint64_t v) {
  while (v >= 0x80) {
    out.push_back((char)(v | 0x80));
    v >>= 7;
  }
  out.push_back((char)v);
}
inline void put_uint(std::string& out, uint32_t field, uint64_t v) {
  if (!v) return;  // proto3: default values are not written
  put_varint(out, (uint64_t)field << 3);
  put_varint(out, v);
}
inline void put_len(std::string& out, uint32_t field, const void* data, size_t n) {
  put_varint(out, ((uint64_t)field << 3) | 2);
  put_varint(out, n);
  out.append((const char*)data, n);
}
inline void put_len(std::string& out, uint32_t field, const std::string& s) { put_len(out, field, s.data(), s.size()); }

// one message, field by field.  Follows prost's decoder: keys are 32-bit with a field number >= 1, varints are at most
// ten bytes, unknown groups are skipped whole (they never occur in these messages), an unmatched end-group or wire
// types 6 / 7 are errors, a known field with another wire type is an error (expect()).
class Reader {
 public:
  Reader(const void* p, size_t n) : p_((const uint8_t*)p), end_((const uint8_t*)p + n) {}
  // false at the end of the message; otherwise field / wire_type and (varint, fixed) value or (bytes) span
  bool next() {
    if (p_ >= end_) return false;
    key(field, wire_type);
    skip_or_read(field, wire_type, 0, true);
    return true;
  }
  void expect(int wt) const {
    if (wire_type != wt) fail("unexpected wire type for a known field");
  }
  uint32_t field = 0;
  int wire_type = 0;
  uint64_t value = 0;
  Span span;

 private:
  [[noreturn]] static void fail(const char* why) { throw WireError("Decode", FHE_B200_INVALID_ARGUMENT, why); }
  uint64_t varint() {
    uint64_t v = 0;
    for (int shift = 0;; shift += 7) {
      if (p_ >= end_) fail("truncated varint");
      uint8_t b = *p_++;
      if (shift == 63 && b > 1) fail("varint overflows 64 bits");
      v |= (uint64_t)(b & 0x7f) << shift;
      if (!(b & 0x80)) return v;
    }
  }
  void key(uint32_t& f, int& wt) {
    uint64_t k = varint();
    if (k > 0xFFFFFFFFull) fail("key does not fit 32 bits");
    if ((k >> 3) == 0) fail("field number 0");
    f = (uint32_t)(k >> 3);
    wt = (int)(k & 7);
  }
  void skip_or_read(uint32_t f, int wt, int depth, bool keep) {
    switch (wt) {
      case 0: {
        uint64_t v = varint();
        if (keep) value = v;
        break;
      }
      case 2: {
        uint64_t n = varint();
        if (n > (uint64_t)(end_ - p_)) fail("length overruns the buffer");
        if (keep) { span.p = p_; span.n = (size_t)n; }
        p_ += n;
        break;
      }
      case 1:
      case 5: {
        size_t n = wt == 1 ? 8 : 4;
        if (n > (size_t)(end_ - p_)) fail("truncated fixed-width field");
        if (keep) {
          value = 0;
          for (size_t i = 0; i < n; i++) value |= (uint64_t)p_[i] << (8 * i);
        }
        p_ += n;
        break;
      }
      case 3: {
        if (depth >= 100) fail("recursion limit");
        for (;;) {
          if (p_ >= end_) fail("unterminated group");
          uint32_t gf;
          int gw;
          key(gf, gw);
          if (gw == 4) {
            if (gf != f) fail("mismatched end of group");
            break;
          }
          skip_or_read(gf, gw, depth + 1, false);
        }
        if (keep) value = 0;
        break;
      }
      default: fail("unsupported wire type");
    }
  }
  const uint8_t *p_, *end_;
};

// ---- Rq ---------------------------------------------------------------------------------------------------------
// Rq::from(&poly).encode_to_vec(); allow_variable_time is never true on the wire (rq/convert.rs:39-41)
inline std::string encode_rq(int32_t representation, uint32_t degree, const uint8_t* coeffs, size_t n) {
  std::string out;
  out.reserve(n + 16);
  put_uint(out, 1, (uint32_t)representation);
  put_uint(out, 2, degree);
  if (n) put_len(out, 3, coeffs, n);
  return out;
}
struct Rq {
  int32_t representation = 0;
  uint32_t degree = 0;
  Span coefficients;
};
// the context-free checks of parse_proto (rq/convert.rs:46-75)
inline Rq decode_rq(const void* data, size_t n) {
  Rq m;
  Reader r(data, n);
  while (r.next()) {
    if (r.field == 1) { r.expect(0); m.representation = (int32_t)(uint32_t)r.value; }
    else if (r.field == 2) { r.expect(0); m.degree = (uint32_t)r.value; }
    else if (r.field == 3) { r.expect(2); m.coefficients = r.span; }
    else if (r.field == 4) { r.expect(0); }   // the timing flag on the wire grants nothing
  }
  if (m.representation < 0 || m.representation > 3)
    throw WireError("InvalidRepresentation", FHE_B200_INVALID_REPRESENTATION, std::to_string(m.representation));
  if (m.representation == REP_UNKNOWN) throw WireError("UnknownRepresentation", FHE_B200_INVALID_REPRESENTATION);
  if (m.degree % 8 != 0 || m.degree < 8) throw WireError("InvalidDegree", FHE_B200_INVALID_DEGREE, std::to_string(m.degree));
  return m;
}

// ---- Ciphertext -------------------------------------------------------------------------------------------------
struct CiphertextMsg {
  std::vector<Span> c;
  Span seed;
  uint32_t level = 0;
};
inline std::string encode_ciphertext(const std::vector<std::string>& polys, const std::string& seed, uint32_t level) {
  std::string out;
  size_t total = 16 + seed.size();
  for (auto& p : polys) total += p.size() + 8;
  out.reserve(total);
  for (auto& p : polys) put_len(out, 1, p);
  if (!seed.empty()) put_len(out, 2, seed);
  put_uint(out, 3, level);
  return out;
}
inline CiphertextMsg decode_ciphertext(const void* data, size_t n) {
  CiphertextMsg m;
  Reader r(data, n);
  while (r.next()) {
    if (r.field == 1) { r.expect(2); m.c.push_back(r.span); }
    else if (r.field == 2) { r.expect(2); m.seed = r.span; }
    else if (r.field == 3) { r.expect(0); m.level = (uint32_t)r.value; }
  }
  if (m.c.empty() || (m.c.size() == 1 && m.seed.n == 0))   // ciphertext.rs:261-269
    throw WireError("InvalidCiphertextPolynomialCount", FHE_B200_BAD_POLY_COUNT);
  return m;
}

// ---- KeySwitchingKey and the messages that wrap it -----------------------------------------------------------------
struct KskMsg {
  std::vector<Span> c0, c1;
  Span seed;
  uint32_t ciphertext_level = 0, ksk_level = 0, log_base = 0;
};
inline std::string encode_ksk(const std::vector<std::string>& c0, const std::vector<std::string>& c1, const std::string& seed,
                              uint32_t ciphertext_level, uint32_t ksk_level, uint32_t log_base) {
  std::string out;
  for (auto& p : c0) put_len(out, 1, p);
  for (auto& p : c1) put_len(out, 2, p);
  if (!seed.empty()) put_len(out, 3, seed);
  put_uint(out, 4, ciphertext_level);
  put_uint(out, 5, ksk_level);
  put_uint(out, 6, log_base);
  return out;
}
inline KskMsg decode_ksk(const void* data, size_t n) {
  KskMsg m;
  Reader r(data, n);
  while (r.next()) {
    if (r.field == 1) { r.expect(2); m.c0.push_back(r.span); }
    else if (r.field == 2) { r.expect(2); m.c1.push_back(r.span); }
    else if (r.field == 3) { r.expect(2); m.seed = r.span; }
    else if (r.field == 4) { r.expect(0); m.ciphertext_level = (uint32_t)r.value; }
    else if (r.field == 5) { r.expect(0); m.ksk_level = (uint32_t)r.value; }
    else if (r.field == 6) { r.expect(0); m.log_base = (uint32_t)r.value; }
  }
  return m;
}
inline std::string encode_relinearization_key(const std::string& ksk) {   // relinearization_key.rs:113-119
  std::string out;
  put_len(out, 1, ksk);
  return out;
}
inline std::string encode_galois_key(const std::string& ksk, uint32_t exponent) {   // galois_key.rs:146-153
  std::string out;
  put_len(out, 1, ksk);
  put_uint(out, 2, exponent);
  return out;
}
// EvaluationKeyProto::from(&ek).encode_to_vec() (evaluation_key.rs:494-505): the GaloisKey messages in the order given
// (the reference writes HashMap order, so a reader may depend on none), then the two levels
inline std::string encode_evaluation_key(const std::vector<std::string>& gks, uint32_t ciphertext_level,
                                         uint32_t evaluation_key_level) {
  std::string out;
  for (auto& g : gks) put_len(out, 2, g);
  put_uint(out, 3, ciphertext_level);
  put_uint(out, 4, evaluation_key_level);
  return out;
}
struct EvaluationKeyMsg {
  std::vector<Span> gk;   // wire order
  uint32_t ciphertext_level = 0, evaluation_key_level = 0;
};
inline EvaluationKeyMsg decode_evaluation_key(const void* data, size_t n) {
  EvaluationKeyMsg m;
  Reader r(data, n);
  while (r.next()) {
    if (r.field == 2) { r.expect(2); m.gk.push_back(r.span); }
    else if (r.field == 3) { r.expect(0); m.ciphertext_level = (uint32_t)r.value; }
    else if (r.field == 4) { r.expect(0); m.evaluation_key_level = (uint32_t)r.value; }
  }
  return m;
}
inline std::string encode_rgsw(const std::string& ksk0, const std::string& ksk1) {   // rgsw_ciphertext.rs:30-37
  std::string out;
  put_len(out, 1, ksk0);
  put_len(out, 2, ksk1);
  return out;
}
// ---- SecretKey (bfv.proto:54-56: repeated sint64 coeffs = 1, packed, zig-zag) -------------------------------------
// SecretKey::to_bytes (secret_key.rs:142-148)
inline std::string encode_secret_key(const int64_t* coeffs, size_t n) {
  std::string payload, out;
  for (size_t i = 0; i < n; i++) put_varint(payload, ((uint64_t)coeffs[i] << 1) ^ (uint64_t)(coeffs[i] >> 63));
  if (n) put_len(out, 1, payload);
  return out;
}
// SecretKey::from_bytes (secret_key.rs:151-175): packed and unpacked coefficients are both accepted (as prost does);
// a count other than `degree` is InvalidSecretKeyCoefficientCount
inline std::vector<int64_t> decode_secret_key(const void* data, size_t n, size_t degree) {
  std::vector<int64_t> c;
  auto unzig = [](uint64_t v) { return (int64_t)((v >> 1) ^ (0 - (v & 1))); };
  Reader r(data, n);
  while (r.next()) {
    if (r.field != 1) continue;
    if (r.wire_type == 0) {
      c.push_back(unzig(r.value));
    } else {
      r.expect(2);
      // packed: the payload is a run of varints
      const uint8_t *p = r.span.p, *end = r.span.p + r.span.n;
      while (p < end) {
        uint64_t v = 0;
        for (int shift = 0;; shift += 7) {
          if (p >= end) throw WireError("Decode", FHE_B200_INVALID_ARGUMENT, "truncated varint");
          const uint8_t b = *p++;
          if (shift == 63 && b > 1) throw WireError("Decode", FHE_B200_INVALID_ARGUMENT, "varint overflows 64 bits");
          v |= (uint64_t)(b & 0x7f) << shift;
          if (!(b & 0x80)) break;
        }
        c.push_back(unzig(v));
      }
    }
  }
  if (c.size() != degree)
    throw WireError("InvalidSecretKeyCoefficientCount", FHE_B200_INVALID_ARGUMENT,
                    std::to_string(c.size()) + " coefficients, expected " + std::to_string(degree));
  return c;
}

// ---- Parameters (bfv.proto:40-48) ---------------------------------------------------------------------------------
// degree = 1 (uint32), moduli = 2 (repeated uint64, packed), the oneof plaintext_modulus { plaintext = 3 (uint64),
// plaintext_big = 5 (bytes, little-endian) }, variance = 4 (uint32)
struct ParametersMsg {
  uint32_t degree = 0, variance = 0;
  std::vector<uint64_t> moduli;
  bool has_plaintext = false;           // a member of the oneof was present
  std::vector<uint8_t> plaintext_le;    // the plaintext modulus, little-endian (either member)
};
// true when t (little-endian) is a zq::Modulus, 2 <= t < 2^62: where PlaintextModulus::as_u64 is Some
inline bool plaintext_is_small(const std::vector<uint8_t>& t_le, uint64_t* t = nullptr) {
  size_t n = t_le.size();
  while (n && !t_le[n - 1]) n--;
  if (n > 8) return false;
  uint64_t v = 0;
  for (size_t i = 0; i < n; i++) v |= (uint64_t)t_le[i] << (8 * i);
  if (t) *t = v;
  return v >= 2 && v < (1ull << 62);
}
// BfvParameters::to_bytes (parameters.rs:741-759).  prost writes a oneof at the position of its lowest field number,
// so plaintext_big (5) goes before variance (4), as plaintext (3) does.
inline std::string encode_parameters(uint32_t degree, const std::vector<uint64_t>& moduli,
                                     const std::vector<uint8_t>& plaintext_le, uint32_t variance) {
  std::string out, packed;
  put_uint(out, 1, degree);
  for (uint64_t q : moduli) put_varint(packed, q);
  if (!moduli.empty()) put_len(out, 2, packed);
  uint64_t t = 0;
  if (plaintext_is_small(plaintext_le, &t)) {
    put_varint(out, 3 << 3);   // a set oneof member is written even when it is zero
    put_varint(out, t);
  } else {
    size_t n = plaintext_le.size();
    while (n > 1 && !plaintext_le[n - 1]) n--;   // BigUint::to_bytes_le: no trailing zeros, one byte for zero
    const uint8_t zero = 0;
    put_len(out, 5, n ? plaintext_le.data() : &zero, n ? n : 1);
  }
  put_uint(out, 4, variance);
  return out;
}
// the fields of a Parameters message (parameters.rs:762-781): packed and unpacked moduli are both accepted, the last
// oneof member wins, malformed bytes are Decode and a missing oneof is MissingField (ParametersPlaintextModulus)
inline ParametersMsg decode_parameters(const void* data, size_t n) {
  ParametersMsg m;
  Reader r(data, n);
  while (r.next()) {
    if (r.field == 1) { r.expect(0); m.degree = (uint32_t)r.value; }
    else if (r.field == 4) { r.expect(0); m.variance = (uint32_t)r.value; }
    else if (r.field == 3) {
      r.expect(0);
      m.has_plaintext = true;
      m.plaintext_le.clear();
      for (int i = 0; i < 8; i++) m.plaintext_le.push_back((uint8_t)(r.value >> (8 * i)));
    } else if (r.field == 5) {
      r.expect(2);
      m.has_plaintext = true;
      m.plaintext_le.assign(r.span.p, r.span.p + r.span.n);
    } else if (r.field == 2) {
      if (r.wire_type == 0) { m.moduli.push_back(r.value); continue; }
      r.expect(2);
      const uint8_t *p = r.span.p, *end = r.span.p + r.span.n;
      while (p < end) {
        uint64_t v = 0;
        for (int shift = 0;; shift += 7) {
          if (p >= end) throw WireError("Decode", FHE_B200_INVALID_ARGUMENT, "truncated varint");
          const uint8_t b = *p++;
          if (shift == 63 && b > 1) throw WireError("Decode", FHE_B200_INVALID_ARGUMENT, "varint overflows 64 bits");
          v |= (uint64_t)(b & 0x7f) << shift;
          if (!(b & 0x80)) break;
        }
        m.moduli.push_back(v);
      }
    }
  }
  if (!m.has_plaintext) throw WireError("MissingField", FHE_B200_INVALID_ARGUMENT, "ParametersPlaintextModulus");
  return m;
}

inline std::string encode_public_key(const std::string& ciphertext) {   // public_key.rs:95-107, bfv.proto:50-52
  std::string out;
  put_len(out, 1, ciphertext);
  return out;
}

// sub-message `field` of a wrapper message; *scalar2 = varint field 2 when present
inline Span sub_message(const void* data, size_t n, uint32_t field, const char* missing, uint32_t* scalar2 = nullptr) {
  Span s;
  bool found = false;
  Reader r(data, n);
  while (r.next()) {
    if (r.field == field) { r.expect(2); s = r.span; found = true; }
    else if (scalar2 && r.field == 2 && r.wire_type == 0) *scalar2 = (uint32_t)r.value;
  }
  if (!found) throw WireError("MissingField", FHE_B200_INVALID_ARGUMENT, missing);
  return s;
}

}  // namespace wire

namespace bfv {

// `Poly::<R>::from_bytes` for every polynomial of `batch` (rq/serialize.rs:23-31, rq/convert.rs:46-161): msgs[i * parts + j]
// is the encoded Rq of part j of ciphertext i.  Framing and checks on the host, unpacking (+ forward NTT) on the device.
inline void unpack_rq(Ciphertext& batch, const std::vector<wire::Span>& msgs, int32_t want_rep) {
  const size_t nbytes = batch.packed_bytes(), deg = batch.par()->degree();
  const uint32_t count = batch.count(), parts = batch.len(), limbs = batch.limbs();
  if (msgs.size() != (size_t)count * parts) throw Error(FHE_B200_INVALID_ARGUMENT, "message count does not match the batch");
  std::vector<uint8_t> blobs(msgs.size() * nbytes, 0);
  for (size_t k = 0; k < msgs.size(); k++) {
    wire::Rq m = wire::decode_rq(msgs[k].p, msgs[k].n);
    if ((uint64_t)m.degree * nbytes != (uint64_t)m.coefficients.n * deg)    // convert.rs:76-88
      throw WireError("InvalidCoefficientCount");
    if (m.representation != want_rep) throw WireError("RepresentationMismatch", FHE_B200_INVALID_REPRESENTATION);
    // convert.rs:148-192: q.len() * degree words, or -- one modulus only -- a shorter low-order polynomial, zero-extended
    if (m.degree != deg && (limbs != 1 || m.degree > deg)) throw WireError("InvalidCoefficientCount");
    std::memcpy(blobs.data() + k * nbytes, m.coefficients.p, m.coefficients.n);
  }
  check(fhe_b200_batch_unpack(batch.handle(), 0, count, blobs.data(), batch.stream()));
  batch.sync();
}

// ct.to_bytes() for every ciphertext of the batch (ciphertext.rs:230-257, unseeded branch)
inline std::vector<std::string> to_bytes(const Ciphertext& ct) {
  const uint32_t count = ct.count(), parts = ct.len(), level = ct.level();
  const size_t nbytes = ct.packed_bytes();
  const uint32_t deg = (uint32_t)ct.par()->degree();
  std::vector<uint8_t> blobs = ct.to_packed();
  ct.sync();
  std::vector<std::string> out(count);
  for (uint32_t i = 0; i < count; i++) {
    std::vector<std::string> polys(parts);
    for (uint32_t j = 0; j < parts; j++)
      polys[j] = wire::encode_rq(wire::REP_NTT, deg, blobs.data() + ((size_t)i * parts + j) * nbytes, nbytes);
    out[i] = wire::encode_ciphertext(polys, std::string(), level);
  }
  return out;
}

// Ciphertext::from_bytes (ciphertext.rs:259-317) for a batch of messages of one level, part count and kind.
// seeded_halves: [count][limbs][N] NTT words of Poly::random_from_seed for messages that carry a seed (host-expanded).
inline Ciphertext ciphertext_from_bytes(std::shared_ptr<BfvParameters> par, const std::vector<std::string>& messages,
                                        const uint64_t* seeded_halves = nullptr) {
  if (messages.empty()) throw Error(FHE_B200_INVALID_ARGUMENT, "no messages");
  std::vector<wire::CiphertextMsg> dec;
  for (auto& m : messages) dec.push_back(wire::decode_ciphertext(m.data(), m.size()));
  const uint32_t level = dec[0].level;
  if (level > par->max_level()) throw WireError("InvalidLevel", FHE_B200_INVALID_LEVEL);
  const size_t n_rq = dec[0].c.size();
  const bool seeded = dec[0].seed.n != 0;
  std::vector<wire::Span> rq;
  for (auto& d : dec) {
    if (d.level != level || d.c.size() != n_rq || (d.seed.n != 0) != seeded)
      throw Error(FHE_B200_INVALID_ARGUMENT, "a batch holds ciphertexts of one level, part count and kind");
    if (d.seed.n && d.seed.n != 32) throw WireError("InvalidSeedSize");
    rq.insert(rq.end(), d.c.begin(), d.c.end());
  }
  const uint32_t count = (uint32_t)dec.size();
  Ciphertext body(par, count, (uint32_t)n_rq, level);
  unpack_rq(body, rq, wire::REP_NTT);
  if (!seeded) return body;
  if (!seeded_halves)
    throw WireError("SeedExpansion", FHE_B200_UNSUPPORTED, "pass the host-expanded last polynomial (ciphertext.rs:287-300)");
  const size_t poly = (size_t)body.limbs() * par->degree();
  std::vector<uint64_t> w = body.to_host(), all((size_t)count * (n_rq + 1) * poly);
  for (uint32_t i = 0; i < count; i++) {
    std::memcpy(&all[(size_t)i * (n_rq + 1) * poly], &w[(size_t)i * n_rq * poly], n_rq * poly * 8);
    std::memcpy(&all[((size_t)i * (n_rq + 1) + n_rq) * poly], seeded_halves + (size_t)i * poly, poly * 8);
  }
  return Ciphertext::from_host(par, all, count, (uint32_t)n_rq + 1, level);
}

// KeySwitchingKey::try_convert_from(&KeySwitchingKeyProto, par) (key_switching_key.rs:388-482).
// seeded_c1: [digits][limbs][N] NTT words of generate_c1 (:130-146) for a key that carries a seed.
inline std::shared_ptr<KeySwitchingKey> key_switching_key_from_bytes(std::shared_ptr<BfvParameters> par, const void* data,
                                                                     size_t n, const uint64_t* seeded_c1 = nullptr) {
  wire::KskMsg k = wire::decode_ksk(data, n);
  if (k.ksk_level > par->max_level() || k.ciphertext_level > par->max_level())
    throw WireError("InvalidLevel", FHE_B200_INVALID_LEVEL);
  auto bits = [](uint64_t v) { uint32_t b = 0; while (v) { b++; v >>= 1; } return b; };
  const std::vector<uint64_t> q = par->moduli();
  size_t c0_size;
  if (k.log_base) {
    if (k.ksk_level != par->max_level() || k.ciphertext_level != par->max_level())
      throw WireError("InvalidKeySwitchingDecompositionLevels", FHE_B200_INVALID_LEVEL);
    const uint32_t log_modulus = bits(q[0] - 1);   // as coded (:406-408): the first modulus of the parameter set
    c0_size = (log_modulus + k.log_base - 1) / k.log_base;
  } else {
    c0_size = q.size() - k.ciphertext_level;
  }
  if (k.c0.size() != c0_size) throw WireError("WrongPolynomialCount", FHE_B200_BAD_POLY_COUNT, "KeySwitchingKeyC0");
  const uint32_t ksk_limbs = (uint32_t)(q.size() - k.ksk_level);
  const uint32_t expect_base = ksk_limbs == 1 ? bits(q[0] - 1) / 2 : 0;   // key_switching_key.rs:92-97
  if (k.log_base != expect_base)   // the device derives the base from the key level; a message that disagrees is refused
    throw WireError("InvalidKeySwitchingDecompositionLevels", FHE_B200_UNSUPPORTED, "log_base does not match the key level");
  const size_t poly = (size_t)ksk_limbs * par->degree();
  std::vector<uint64_t> c0(c0_size * poly), c1(c0_size * poly);
  if (k.seed.n == 0) {
    if (k.c1.size() != c0_size) throw WireError("WrongPolynomialCount", FHE_B200_BAD_POLY_COUNT, "KeySwitchingKeyC1");
    Ciphertext tmp(par, (uint32_t)c0_size, 2, k.ksk_level);
    std::vector<wire::Span> rq;
    for (size_t i = 0; i < c0_size; i++) { rq.push_back(k.c0[i]); rq.push_back(k.c1[i]); }
    unpack_rq(tmp, rq, wire::REP_NTTSHOUP);
    std::vector<uint64_t> w = tmp.to_host();
    for (size_t i = 0; i < c0_size; i++) {
      std::memcpy(&c0[i * poly], &w[(2 * i) * poly], poly * 8);
      std::memcpy(&c1[i * poly], &w[(2 * i + 1) * poly], poly * 8);
    }
  } else {
    if (k.seed.n != 32) throw WireError("InvalidKeySwitchingSeedLength");
    if (!seeded_c1)
      throw WireError("SeedExpansion", FHE_B200_UNSUPPORTED, "pass the host-expanded c1 row (key_switching_key.rs:130-146)");
    Ciphertext tmp(par, (uint32_t)c0_size, 1, k.ksk_level);
    unpack_rq(tmp, k.c0, wire::REP_NTTSHOUP);
    c0 = tmp.to_host();
    std::memcpy(c1.data(), seeded_c1, c1.size() * 8);
  }
  return std::make_shared<KeySwitchingKey>(par, c0, c1, (uint32_t)c0_size, k.ciphertext_level, k.ksk_level);
}

// RelinearizationKey::from_bytes (relinearization_key.rs:121-135)
inline RelinearizationKey relinearization_key_from_bytes(std::shared_ptr<BfvParameters> par, const std::string& data) {
  wire::Span s = wire::sub_message(data.data(), data.size(), 1, "RelinearizationKeySwitchingKey");
  return RelinearizationKey(key_switching_key_from_bytes(std::move(par), s.p, s.n));
}
// GaloisKey::from_bytes (galois_key.rs:155-173)
// (seeded_c1 as for key_switching_key_from_bytes)
inline GaloisKey galois_key_from_bytes(std::shared_ptr<BfvParameters> par, const std::string& data,
                                       const uint64_t* seeded_c1 = nullptr) {
  uint32_t exponent = 0;
  wire::Span s = wire::sub_message(data.data(), data.size(), 1, "GaloisKeySwitchingKey", &exponent);
  const uint32_t two_n = 2 * (uint32_t)par->degree();
  auto ksk = key_switching_key_from_bytes(std::move(par), s.p, s.n, seeded_c1);
  exponent %= two_n;                        // SubstitutionExponent::new (rq/mod.rs:99-106)
  if (!(exponent & 1)) throw WireError("InvalidSubstitutionExponent", FHE_B200_INVALID_EXPONENT);
  return GaloisKey(exponent, std::move(ksk));
}
// KeySwitchingKeyProto::from(&ksk).encode_to_vec() (key_switching_key.rs:365-386), unseeded branch: the words read
// back from the device, every c0_i and c1_i as an Rq with representation NTTSHOUP (packed on the device)
inline std::string to_bytes(const KeySwitchingKey& k) {
  const auto w = k.arrays();
  const uint32_t nd = k.n_digits(), deg = (uint32_t)k.par()->degree();
  const size_t poly = w.first.size() / nd;
  std::vector<uint64_t> both(2 * w.first.size());   // [digit][c0, c1][limb][N]
  for (uint32_t i = 0; i < nd; i++) {
    std::memcpy(&both[(2 * (size_t)i) * poly], &w.first[(size_t)i * poly], poly * 8);
    std::memcpy(&both[(2 * (size_t)i + 1) * poly], &w.second[(size_t)i * poly], poly * 8);
  }
  const Ciphertext tmp = Ciphertext::from_host(k.par(), both, nd, 2, k.ksk_level());
  const size_t nbytes = tmp.packed_bytes();
  const std::vector<uint8_t> blobs = tmp.to_packed();
  tmp.sync();
  std::vector<std::string> c0(nd), c1(nd);
  for (uint32_t i = 0; i < nd; i++) {
    c0[i] = wire::encode_rq(wire::REP_NTTSHOUP, deg, blobs.data() + (2 * (size_t)i) * nbytes, nbytes);
    c1[i] = wire::encode_rq(wire::REP_NTTSHOUP, deg, blobs.data() + (2 * (size_t)i + 1) * nbytes, nbytes);
  }
  return wire::encode_ksk(c0, c1, std::string(), k.ciphertext_level(), k.ksk_level(), k.log_base());
}
// RelinearizationKey::to_bytes (relinearization_key.rs:113-119, :137-141), GaloisKey::to_bytes (galois_key.rs:146-153),
// RGSWCiphertext::to_bytes (rgsw_ciphertext.rs:30-37)
inline std::string to_bytes(const RelinearizationKey& rk) { return wire::encode_relinearization_key(to_bytes(*rk.ksk)); }
inline std::string to_bytes(const GaloisKey& gk) { return wire::encode_galois_key(to_bytes(*gk.ksk), gk.exponent); }
inline std::string to_bytes(const RGSWCiphertext& r) { return wire::encode_rgsw(to_bytes(*r.ksk0), to_bytes(*r.ksk1)); }
// EvaluationKey::to_bytes (evaluation_key.rs:293-297, :494-505), the Galois keys in ascending exponent order
inline std::string to_bytes(const EvaluationKey& ek) {
  std::vector<std::string> gks;
  for (auto& kv : ek.galois_keys()) gks.push_back(to_bytes(*kv.second));
  return wire::encode_evaluation_key(gks, ek.ciphertext_level(), ek.evaluation_key_level());
}
// EvaluationKey::from_bytes (evaluation_key.rs:299-310, :507-550): every key through galois_key_from_bytes; a key at
// other levels than the message's, or a message ciphertext level beyond the parameters', -> InvalidLevel; a repeated
// exponent keeps the later key (HashMap::insert).  seeded_c1: exponent (mod 2N) -> the host-expanded c1 of a compact key.
inline EvaluationKey evaluation_key_from_bytes(std::shared_ptr<BfvParameters> par, const std::string& data,
                                               const std::map<uint32_t, const uint64_t*>& seeded_c1 = {}) {
  const wire::EvaluationKeyMsg m = wire::decode_evaluation_key(data.data(), data.size());
  EvaluationKey ek(par, m.ciphertext_level, m.evaluation_key_level);
  const uint32_t two_n = 2 * (uint32_t)par->degree();
  for (const wire::Span& g : m.gk) {
    uint32_t exponent = 0;
    wire::sub_message(g.p, g.n, 1, "GaloisKeySwitchingKey", &exponent);
    auto it = seeded_c1.find(exponent % two_n);
    auto gk = std::make_shared<GaloisKey>(
        galois_key_from_bytes(par, std::string((const char*)g.p, g.n), it == seeded_c1.end() ? nullptr : it->second));
    if (gk->ksk->ciphertext_level() != m.ciphertext_level || gk->ksk->ksk_level() != m.evaluation_key_level)
      throw WireError("InvalidLevel", FHE_B200_INVALID_LEVEL);
    ek.add_galois_key(std::move(gk));
  }
  if (m.ciphertext_level > par->max_level()) throw WireError("InvalidLevel", FHE_B200_INVALID_LEVEL);
  return ek;
}

// SecretKey::to_bytes / from_bytes (secret_key.rs:142-175)
// A device-born key's coefficients come from fhe_b200_secret_key_coeffs and are erased once encoded.
inline std::string to_bytes(const SecretKey& sk) {
  std::vector<int64_t> c = sk.download_coeffs();
  std::string msg = wire::encode_secret_key(c.data(), c.size());
  volatile int64_t* w = c.data();
  for (size_t i = 0; i < c.size(); i++) w[i] = 0;
  return msg;
}
inline std::unique_ptr<SecretKey> secret_key_from_bytes(std::shared_ptr<BfvParameters> par, const std::string& data) {
  std::vector<int64_t> c = wire::decode_secret_key(data.data(), data.size(), par->degree());
  std::unique_ptr<SecretKey> sk(new SecretKey(std::move(par), c));
  volatile int64_t* w = c.data();
  for (size_t i = 0; i < c.size(); i++) w[i] = 0;
  return sk;
}

// PublicKey::to_bytes (public_key.rs:95-107): both parts (a device-encrypted key carries no seed)
inline std::string to_bytes(const PublicKey& pk) { return wire::encode_public_key(to_bytes(pk.c())[0]); }
// PublicKey::from_bytes (public_key.rs:109-149).  The reference writes a compact message (c0 and the seed of c1):
// decoding one needs seeded_c1, the [limbs][N] NTT words of c1 expanded by the Rust host.  A key at a level other than
// 0 is InvalidPublicKeyLevel.
inline PublicKey public_key_from_bytes(std::shared_ptr<BfvParameters> par, const std::string& data,
                                       const uint64_t* seeded_c1 = nullptr) {
  wire::Span s = wire::sub_message(data.data(), data.size(), 1, "PublicKeyCiphertext");
  const wire::CiphertextMsg m = wire::decode_ciphertext(s.p, s.n);
  if (m.level != 0) throw WireError("InvalidPublicKeyLevel", FHE_B200_INVALID_LEVEL);
  if (m.seed.n && !seeded_c1)
    throw WireError("SeedExpansion", FHE_B200_UNSUPPORTED, "pass the host-expanded c1 (ciphertext.rs:287-300)");
  Ciphertext c = ciphertext_from_bytes(par, {std::string((const char*)s.p, s.n)}, seeded_c1);
  return PublicKey(std::move(par), std::move(c));
}

// BfvParameters::to_bytes / try_deserialize (parameters.rs:741-789).  The decoder builds through BfvParametersBuilder
// with explicit moduli and the decoded variance, so every builder error keeps its code (variance 0 is InvalidVariance).
inline std::string parameters_to_bytes(const BfvParameters& par) {
  return wire::encode_parameters((uint32_t)par.degree(), par.moduli(), par.plaintext_le(), par.variance());
}
inline std::shared_ptr<BfvParameters> parameters_from_bytes(const std::string& data, int device = 0) {
  const wire::ParametersMsg m = wire::decode_parameters(data.data(), data.size());
  return BfvParametersBuilder()
      .set_degree(m.degree)
      .set_moduli(m.moduli)
      .set_plaintext_modulus_le(m.plaintext_le)
      .set_variance(m.variance)
      .set_device(device)
      .build_arc();
}

}  // namespace bfv
}  // namespace fhe_b200
