// fhe_b200.hpp -- C++17 host-side mirror of the reference's `fhe::bfv` interface for the
// accelerated path, header-only, implemented purely on the C ABI of fhe_b200.h.
//
// Names and argument meaning follow tlepoint/fhe.rs (paths under the reference's crates/fhe/src):
//   bfv::BfvParameters / BfvParametersBuilder   bfv/parameters.rs:88, :319
//   bfv::Ciphertext                             bfv/ciphertext.rs:18  (here: a device-resident batch)
//   bfv::KeySwitchingKey / RelinearizationKey   bfv/keys/key_switching_key.rs:22, relinearization_key.rs:23
//   bfv::RGSWCiphertext                         bfv/rgsw_ciphertext.rs:20 (external product = two key switches)
//   bfv::GaloisKey / EvaluationKey              bfv/keys/galois_key.rs:18, evaluation_key.rs:110-170
//   bfv::Multiplicator                          bfv/ops/mul.rs:22
//   bfv::Encoding / Plaintext / PlaintextVec    bfv/encoding.rs, bfv/plaintext.rs:20, plaintext_vec.rs:20
//   bfv::SecretKey / PublicKey                  bfv/keys/secret_key.rs:25, public_key.rs:17 (SecretKey::random,
//                                               encryption, decryption, measure_noise)
// Fallible reference calls return Result<_, fhe::Error>; here they throw fhe_b200::Error carrying
// the fhe_b200_status code (same variants, see fhe_b200.h).
#pragma once
#include <cstdint>
#include <cstring>
#include <map>
#include <algorithm>
#include <memory>
#include <mutex>
#include <set>
#include <stdexcept>
#include <string>
#include <type_traits>
#include <utility>
#include <vector>

#include <sys/random.h>

#include "fhe_b200.h"

namespace fhe_b200 {

struct Error : std::runtime_error {
  int code;
  Error(int c, const std::string& m) : std::runtime_error(m), code(c) {}
};
inline void check(int code) {
  if (code != FHE_B200_OK) throw Error(code, fhe_b200_last_error());
}

namespace mbfv {
class PlaintextAccess;
}

namespace bfv {

enum class Representation : int { PowerBasis = FHE_B200_POWER_BASIS, Ntt = FHE_B200_NTT };

class BfvParameters {
 public:
  BfvParameters(const BfvParameters&) = delete;
  BfvParameters& operator=(const BfvParameters&) = delete;
  size_t degree() const { return fhe_b200_params_degree(h_); }
  std::vector<uint64_t> moduli() const {
    std::vector<uint64_t> m(fhe_b200_params_n_moduli(h_));
    check(fhe_b200_params_moduli(h_, m.data()));
    return m;
  }
  size_t max_level() const { return fhe_b200_params_n_moduli(h_) - 1; }
  // BfvParameters::variance (parameters.rs:98-99): the centred binomial parameter of encryption's errors
  uint32_t variance() const { return variance_; }
  // the plaintext modulus as little-endian bytes without trailing zeros (BigUint::to_bytes_le, at least one byte)
  const std::vector<uint8_t>& plaintext_le() const { return plaintext_le_; }
  std::vector<uint64_t> mul_basis(uint32_t level) const {
    uint32_t n = 0;
    check(fhe_b200_params_mul_basis(h_, level, nullptr, &n));
    std::vector<uint64_t> m(n);
    check(fhe_b200_params_mul_basis(h_, level, m.data(), &n));
    return m;
  }
  const fhe_b200_params* handle() const { return h_; }
  // ntt_operator + matrix_reps_index_map of the plaintext modulus (parameters.rs:71-75, :713-726), built on first use
  const fhe_b200_encoder* encoder() const {
    std::call_once(enc_once_, [this] {
      check(fhe_b200_encoder_create(h_, has_plaintext_psi_ ? &plaintext_psi_ : nullptr, &enc_));
    });
    return enc_;
  }

 private:
  friend class BfvParametersBuilder;
  BfvParameters(fhe_b200_params* h, bool has_psi_t, uint64_t psi_t, uint32_t variance, std::vector<uint8_t> t_le)
      : h_(h), has_plaintext_psi_(has_psi_t), plaintext_psi_(psi_t), variance_(variance), plaintext_le_(std::move(t_le)) {}
  fhe_b200_params* h_;
  bool has_plaintext_psi_;
  uint64_t plaintext_psi_;
  uint32_t variance_;
  std::vector<uint8_t> plaintext_le_;
  mutable std::once_flag enc_once_;
  mutable fhe_b200_encoder* enc_ = nullptr;

 public:
  ~BfvParameters() { fhe_b200_encoder_free(enc_); fhe_b200_params_destroy(h_); }
};

class BfvParametersBuilder {
 public:
  BfvParametersBuilder& set_degree(size_t d) { degree_ = (uint32_t)d; return *this; }
  BfvParametersBuilder& set_plaintext_modulus(uint64_t t) {
    plaintext_.assign(8, 0);
    for (int i = 0; i < 8; i++) plaintext_[i] = (uint8_t)(t >> (8 * i));
    return *this;
  }
  // set_plaintext_modulus_biguint (parameters.rs:349-356): t as little-endian bytes of any length
  BfvParametersBuilder& set_plaintext_modulus_le(const std::vector<uint8_t>& t_le) { plaintext_ = t_le; return *this; }
  BfvParametersBuilder& set_moduli(const std::vector<uint64_t>& m) { moduli_ = m; return *this; }
  BfvParametersBuilder& set_moduli_sizes(const std::vector<uint32_t>& s) { sizes_ = s; return *this; }
  BfvParametersBuilder& set_ntt_roots(const std::vector<uint64_t>& psi) { psi_ = psi; return *this; }
  BfvParametersBuilder& set_device(int device) { device_ = device; return *this; }
  // the error variance, 1..32 (parameters.rs:384-388; build throws InvalidVariance outside)
  BfvParametersBuilder& set_variance(uint32_t v) { variance_ = v; return *this; }
  // 2N-th root for the plaintext modulus (the reference's NttOperator::new(t).omegas[N/2]); default rule otherwise
  BfvParametersBuilder& set_plaintext_ntt_root(uint64_t psi_t) { psi_t_ = psi_t; has_psi_t_ = true; return *this; }
  // BfvParametersBuilder::build_arc (bfv/parameters.rs:555)
  std::shared_ptr<BfvParameters> build_arc() const {
    std::vector<uint8_t> t_le = plaintext_;
    while (t_le.size() > 1 && !t_le.back()) t_le.pop_back();
    const uint8_t* pt = t_le.data();
    fhe_b200_params* h = nullptr;
    if (variance_ < 1 || variance_ > 32) throw Error(FHE_B200_INVALID_ARGUMENT, "InvalidVariance");
    if (!moduli_.empty() && !sizes_.empty())
      throw Error(FHE_B200_INVALID_ARGUMENT, "ConflictingCiphertextModulusSpecifications");
    if (!moduli_.empty())
      check(fhe_b200_params_create(device_, degree_, moduli_.data(), (uint32_t)moduli_.size(), pt, (uint32_t)t_le.size(),
                                   psi_.empty() ? nullptr : psi_.data(), &h));
    else
      check(fhe_b200_params_create_from_sizes(device_, degree_, sizes_.data(), (uint32_t)sizes_.size(), pt,
                                              (uint32_t)t_le.size(), &h));
    return std::shared_ptr<BfvParameters>(new BfvParameters(h, has_psi_t_, psi_t_, variance_, std::move(t_le)));
  }

 private:
  uint32_t degree_ = 0;
  std::vector<uint8_t> plaintext_ = std::vector<uint8_t>(8, 0);
  uint64_t psi_t_ = 0;
  bool has_psi_t_ = false;
  uint32_t variance_ = 10;
  std::vector<uint64_t> moduli_, psi_;
  std::vector<uint32_t> sizes_;
  int device_ = 0;
};

// A batch of `count` ciphertexts with `parts` polynomials each, at one level, resident in HBM.
// Page-locked host staging memory (fhe_b200_host_alloc) for the asynchronous transfers below; write_combined for
// upload-only buffers the host fills front to back.
class PinnedWords {
 public:
  explicit PinnedWords(size_t n_words, bool write_combined = false) : n_(n_words) {
    void* p = nullptr;
    check(fhe_b200_host_alloc(n_words * sizeof(uint64_t), write_combined ? 1 : 0, &p));
    p_ = static_cast<uint64_t*>(p);
  }
  PinnedWords(const PinnedWords&) = delete;
  PinnedWords& operator=(const PinnedWords&) = delete;
  ~PinnedWords() { fhe_b200_host_free(p_); }
  uint64_t* data() { return p_; }
  const uint64_t* data() const { return p_; }
  size_t size() const { return n_; }

 private:
  uint64_t* p_ = nullptr;
  size_t n_ = 0;
};

class PlaintextVec;
class RGSWCiphertext;

class Ciphertext {
 public:
  Ciphertext(std::shared_ptr<BfvParameters> par, uint32_t count, uint32_t parts = 2, uint32_t level = 0,
             Representation r = Representation::Ntt, void* stream = nullptr)
      : par_(std::move(par)), stream_(stream) {
    check(fhe_b200_batch_alloc(par_->handle(), count, parts, level, (int)r, &h_));
  }
  Ciphertext(Ciphertext&& o) noexcept : par_(std::move(o.par_)), h_(o.h_), stream_(o.stream_) { o.h_ = nullptr; }
  Ciphertext(const Ciphertext&) = delete;
  ~Ciphertext() { fhe_b200_batch_free(h_); }

  // host words [count][parts][limbs][N] == Vec<u64>::from(&Poly) per part (rq/convert.rs:474)
  static Ciphertext from_host(std::shared_ptr<BfvParameters> par, const std::vector<uint64_t>& words, uint32_t count,
                              uint32_t parts = 2, uint32_t level = 0, Representation r = Representation::Ntt) {
    Ciphertext ct(std::move(par), count, parts, level, r);
    if (words.size() != ct.words()) throw Error(FHE_B200_INVALID_ARGUMENT, "word count does not match the batch shape");
    check(fhe_b200_batch_upload(ct.h_, 0, count, words.data(), ct.stream_));
    check(fhe_b200_sync(ct.stream_));
    return ct;
  }
  std::vector<uint64_t> to_host() const {
    std::vector<uint64_t> w(words());
    check(fhe_b200_batch_download(h_, 0, count(), w.data(), stream_));
    return w;
  }
  // enqueue-only transfers of ciphertexts [first, first + n) on the batch's stream; `host` must be page-locked
  // (PinnedWords) for them to be asynchronous and must stay valid until sync()
  void upload_async(const uint64_t* host, uint32_t first, uint32_t n) { check(fhe_b200_batch_upload(h_, first, n, host, stream_)); }
  void download_async(uint64_t* host, uint32_t first, uint32_t n) const { check(fhe_b200_batch_download_async(h_, first, n, host, stream_)); }
  void sync() const { check(fhe_b200_sync(stream_)); }
  uint32_t count() const { uint32_t c; check(fhe_b200_batch_info(h_, &c, nullptr, nullptr, nullptr, nullptr)); return c; }
  uint32_t len() const { uint32_t p; check(fhe_b200_batch_info(h_, nullptr, &p, nullptr, nullptr, nullptr)); return p; }
  uint32_t level() const { uint32_t l; check(fhe_b200_batch_info(h_, nullptr, nullptr, &l, nullptr, nullptr)); return l; }
  uint32_t limbs() const { uint32_t l; check(fhe_b200_batch_info(h_, nullptr, nullptr, nullptr, &l, nullptr)); return l; }
  size_t words() const { return (size_t)count() * len() * limbs() * par_->degree(); }

  Ciphertext clone() const {
    Ciphertext c(par_, count(), len(), level(), representation(), stream_);
    check(fhe_b200_batch_copy(c.h_, h_, stream_));
    return c;
  }
  // the SealPIR reply fold (examples/sealpir.rs:176-200, fhe_b200_fold): plaintext i of ciphertext j is entry
  // i * count() + j of the result, encoded with Encoding::poly_at_level(level)
  PlaintextVec fold(uint32_t in_bits, uint32_t out_bits, uint32_t level) const;
  // a new batch of the n ciphertexts first, first + stride, ..., first + (n-1)*stride
  Ciphertext take(uint32_t first, uint32_t n, uint32_t stride = 1) const {
    Ciphertext c(par_, n, len(), level(), representation(), stream_);
    check(fhe_b200_batch_copy_range(c.h_, 0, h_, first, stride, n, stream_));
    return c;
  }
  // bfv/ops/mod.rs:54, :148, :205
  Ciphertext& operator+=(const Ciphertext& rhs) { check(fhe_b200_add(h_, rhs.h_, stream_)); return *this; }
  Ciphertext& operator-=(const Ciphertext& rhs) { check(fhe_b200_sub(h_, rhs.h_, stream_)); return *this; }
  Ciphertext operator-() const { Ciphertext c = clone(); check(fhe_b200_neg(c.h_, stream_)); return c; }
  // &Ciphertext * &Ciphertext -> 3 parts (bfv/ops/mod.rs:259)
  Ciphertext operator*(const Ciphertext& rhs) const {
    Ciphertext out(par_, count(), len() + rhs.len() - 1, level(), Representation::Ntt, stream_);
    check(fhe_b200_mul(h_, rhs.h_, out.h_, stream_));
    return out;
  }
  // Ciphertext += / -= &Plaintext (bfv/ops/mod.rs:88, :188): poly = Plaintext::to_poly() words, [limbs][N]
  Ciphertext& add_plain(const std::vector<uint64_t>& poly, bool subtract = false) {
    check(fhe_b200_add_plain(h_, poly.data(), 1, subtract ? 1 : 0, stream_));
    return *this;
  }
  // Ciphertext *= &Plaintext (bfv/ops/mod.rs:229): poly_ntt = [limbs][N] words shared by the batch
  Ciphertext& mul_plain(const std::vector<uint64_t>& poly_ntt) {
    check(fhe_b200_mul_plain(h_, poly_ntt.data(), 1, stream_));
    return *this;
  }
  // the same with device plaintexts (1 shared, or one per ciphertext); to_poly() is derived on the device
  inline Ciphertext& mul_plain(const PlaintextVec& pts);
  inline Ciphertext& add_plain(const PlaintextVec& pts, bool subtract = false);
  // Poly::into_ntt / into_power_basis on every polynomial (rq/mod.rs:535, :590)
  Ciphertext& into_ntt() { check(fhe_b200_ntt_forward(h_, stream_)); return *this; }
  Ciphertext& into_power_basis() { check(fhe_b200_ntt_backward(h_, stream_)); return *this; }
  Representation representation() const {
    int r;
    check(fhe_b200_batch_info(h_, nullptr, nullptr, nullptr, nullptr, &r));
    return (Representation)r;
  }
  // Poly::substitute on every polynomial, in either representation (rq/mod.rs:360-408)
  Ciphertext substitute(uint32_t exponent) const {
    Ciphertext out(par_, count(), len(), level(), representation(), stream_);
    check(fhe_b200_substitute(h_, exponent, out.h_, stream_));
    return out;
  }
  // Ciphertext::switch_down (bfv/ciphertext.rs:148)
  void switch_down() { check(fhe_b200_switch_down(h_, stream_)); }
  // Ciphertext::switch_to_level (ciphertext.rs:164-184): only moves down
  void switch_to_level(uint32_t target_level) {
    if (target_level < level() || target_level > par_->max_level())
      throw Error(FHE_B200_INVALID_LEVEL, "InvalidLevel");
    while (level() < target_level) switch_down();
  }
  // Rq.coefficients of every polynomial (rq/convert.rs:17-44): count*parts blobs of packed_bytes() each
  size_t packed_bytes() const {
    size_t n = 0;
    check(fhe_b200_batch_packed_bytes(h_, &n));   // per batch: a multiplication-basis batch has L + E limbs
    return n;
  }
  std::vector<uint8_t> to_packed() const {
    std::vector<uint8_t> out((size_t)count() * len() * packed_bytes());
    check(fhe_b200_batch_pack(h_, 0, count(), out.data(), stream_));
    return out;
  }
  // TryConvertFrom<&Rq> for Poly<Ntt> (rq/convert.rs:116-131) for every polynomial of the batch
  static Ciphertext from_packed(std::shared_ptr<BfvParameters> par, const std::vector<uint8_t>& blobs, uint32_t count,
                                uint32_t parts = 2, uint32_t level = 0, Representation r = Representation::Ntt) {
    Ciphertext ct(std::move(par), count, parts, level, r);
    if (blobs.size() != (size_t)count * parts * ct.packed_bytes())
      throw Error(FHE_B200_INVALID_ARGUMENT, "InvalidCoefficientCount");
    check(fhe_b200_batch_unpack(ct.h_, 0, count, blobs.data(), ct.stream_));
    check(fhe_b200_sync(ct.stream_));
    return ct;
  }

  fhe_b200_batch* handle() const { return h_; }
  const std::shared_ptr<BfvParameters>& par() const { return par_; }
  void* stream() const { return stream_; }

 private:
  std::shared_ptr<BfvParameters> par_;
  fhe_b200_batch* h_ = nullptr;
  void* stream_ = nullptr;
};

// fhe::bfv::Encoding (bfv/encoding.rs)
struct Encoding {
  int kind;
  uint32_t level;
  static Encoding poly() { return {FHE_B200_ENCODING_POLY, 0}; }
  static Encoding simd() { return {FHE_B200_ENCODING_SIMD, 0}; }
  static Encoding poly_at_level(uint32_t level) { return {FHE_B200_ENCODING_POLY, level}; }
  static Encoding simd_at_level(uint32_t level) { return {FHE_B200_ENCODING_SIMD, level}; }
  bool operator==(const Encoding& o) const { return kind == o.kind && level == o.level; }
  bool operator!=(const Encoding& o) const { return !(*this == o); }
};

// fhe::bfv::PlaintextVec (bfv/plaintext_vec.rs:20-103): the poly_ntt of every plaintext in a 1-part device batch.
// `values` of try_encode may be host (pageable or PinnedWords) or device memory; SIMD values must be below t.
class PlaintextVec {
 public:
  static PlaintextVec try_encode(const uint64_t* values, size_t n, const Encoding& e,
                                 const std::shared_ptr<BfvParameters>& par) {
    return encode(values, n, false, e, par);
  }
  static PlaintextVec try_encode(const int64_t* values, size_t n, const Encoding& e,
                                 const std::shared_ptr<BfvParameters>& par) {
    return encode(values, n, true, e, par);
  }
  template <typename T>
  static PlaintextVec try_encode(const std::vector<T>& values, const Encoding& e, const std::shared_ptr<BfvParameters>& par) {
    return try_encode(values.data(), values.size(), e, par);
  }
  size_t len() const { return batch_.count(); }
  // the stored encoding; false for plaintexts without one (SecretKey::try_decrypt's)
  bool has_encoding() const { return has_encoding_; }
  const Encoding& encoding() const { return encoding_; }
  const Ciphertext& batch() const { return batch_; }
  std::vector<uint64_t> poly_ntt() const { return batch_.to_host(); }   // [count][limbs][N]

  // Plaintext::resolve_encoding (plaintext.rs:137-153); `e` may be null
  Encoding resolve_encoding(const Encoding* e) const {
    if (!has_encoding_ && !e) throw Error(FHE_B200_INVALID_ARGUMENT, "PlaintextError::MissingEncoding");
    if (has_encoding_ && e && *e != encoding_) throw Error(FHE_B200_INVALID_ARGUMENT, "EncodingError::Mismatch");
    return has_encoding_ ? encoding_ : *e;
  }
  // Vec<u64>::try_decode (T = uint64_t) / Vec<i64>::try_decode (T = int64_t) (plaintext.rs:374-459) of every plaintext
  // on the device: count * N values, plaintext k at [k*N, (k+1)*N)
  template <typename T>
  std::vector<T> try_decode(const Encoding* e = nullptr) const {
    static_assert(std::is_same<T, uint64_t>::value || std::is_same<T, int64_t>::value, "u64 or i64 values");
    const Encoding enc = resolve_encoding(e);
    std::vector<T> out(len() * batch_.par()->degree());
    check(fhe_b200_decode(batch_.par()->encoder(), enc.kind, std::is_signed<T>::value ? 1 : 0, batch_.handle(),
                          out.data(), out.size(), batch_.stream()));
    batch_.sync();
    return out;
  }

 protected:
  friend class SecretKey;
  friend class Ciphertext;              // Ciphertext::fold
  friend class mbfv::PlaintextAccess;   // Plaintext::from_shares builds plaintexts without an encoding
  PlaintextVec(Ciphertext b, const Encoding& e) : batch_(std::move(b)), encoding_(e) {}
  explicit PlaintextVec(Ciphertext b) : batch_(std::move(b)), encoding_(Encoding::poly()), has_encoding_(false) {}
  static PlaintextVec encode(const void* values, size_t n, bool is_signed, const Encoding& e,
                             const std::shared_ptr<BfvParameters>& par) {
    const size_t N = par->degree();
    Ciphertext b(par, (uint32_t)std::max<size_t>(1, (n + N - 1) / N), 1, e.level, Representation::Ntt);
    check(fhe_b200_encode(par->encoder(), e.kind, is_signed ? 1 : 0, values, n, b.handle(), b.stream()));
    b.sync();   // `values` may be released by the caller once this returns
    return PlaintextVec(std::move(b), e);
  }
  Ciphertext batch_;
  Encoding encoding_;
  bool has_encoding_ = true;
};

// fhe::bfv::Plaintext (bfv/plaintext.rs:20-27): one plaintext of at most N values (TooManyValues, :311-345)
class Plaintext : public PlaintextVec {
 public:
  template <typename T>
  static Plaintext try_encode(const std::vector<T>& values, const Encoding& e, const std::shared_ptr<BfvParameters>& par) {
    if (values.size() > par->degree()) throw Error(FHE_B200_INVALID_ARGUMENT, "TooManyValues");
    return Plaintext(PlaintextVec::try_encode(values, e, par));
  }

 private:
  explicit Plaintext(PlaintextVec&& v) : PlaintextVec(std::move(v)) {}
};

inline PlaintextVec Ciphertext::fold(uint32_t in_bits, uint32_t out_bits, uint32_t level) const {
  const uint64_t n = par_->degree();
  uint64_t per_ct = 1;
  if (in_bits >= 1 && in_bits <= 64 && out_bits >= 1 && out_bits <= 64) {   // (otherwise fhe_b200_fold refuses them)
    const uint64_t e = (limbs() * n * in_bits + out_bits - 1) / out_bits;
    per_ct = (len() * e + n - 1) / n;
  }
  Ciphertext out(par_, (uint32_t)(per_ct * count()), 1, level, Representation::Ntt, stream_);
  check(fhe_b200_fold(h_, in_bits, out_bits, out.h_, stream_));
  return PlaintextVec(std::move(out), Encoding::poly_at_level(level));
}

// fhe_util::transcode_bidirectional / transcode_to_bytes / transcode_from_bytes (fhe-util/src/lib.rs:68-187) on the
// device of `par` (fhe_b200_transcode), one row
inline std::vector<uint64_t> transcode_bidirectional(const std::shared_ptr<BfvParameters>& par, const std::vector<uint64_t>& a,
                                                     uint32_t input_nbits, uint32_t output_nbits) {
  const size_t n = output_nbits ? (a.size() * input_nbits + output_nbits - 1) / output_nbits : 0;
  std::vector<uint64_t> out(n);
  check(fhe_b200_transcode(par->handle(), a.empty() ? nullptr : a.data(), 8, a.size(), a.size(), input_nbits,
                           out.empty() ? nullptr : out.data(), 8, n, n, output_nbits, 1, nullptr));
  check(fhe_b200_sync(nullptr));
  return out;
}
inline std::vector<uint8_t> transcode_to_bytes(const std::shared_ptr<BfvParameters>& par, const std::vector<uint64_t>& a,
                                               uint32_t nbits) {
  const size_t n = (a.size() * nbits + 7) / 8;
  std::vector<uint8_t> out(n);
  check(fhe_b200_transcode(par->handle(), a.empty() ? nullptr : a.data(), 8, a.size(), a.size(), nbits,
                           out.empty() ? nullptr : out.data(), 1, n, n, 8, 1, nullptr));
  check(fhe_b200_sync(nullptr));
  return out;
}
inline std::vector<uint64_t> transcode_from_bytes(const std::shared_ptr<BfvParameters>& par, const std::vector<uint8_t>& b,
                                                  uint32_t nbits) {
  const size_t n = nbits ? (b.size() * 8 + nbits - 1) / nbits : 0;
  std::vector<uint64_t> out(n);
  check(fhe_b200_transcode(par->handle(), b.empty() ? nullptr : b.data(), 1, b.size(), b.size(), 8,
                           out.empty() ? nullptr : out.data(), 8, n, n, nbits, 1, nullptr));
  check(fhe_b200_sync(nullptr));
  return out;
}

inline Ciphertext& Ciphertext::mul_plain(const PlaintextVec& pts) {
  check(fhe_b200_mul_plain_batch(h_, pts.batch().handle(), stream_));
  return *this;
}
inline Ciphertext& Ciphertext::add_plain(const PlaintextVec& pts, bool subtract) {
  check(fhe_b200_add_plain_batch(h_, pts.batch().handle(), subtract ? 1 : 0, stream_));
  return *this;
}

// fhe::bfv::SecretKey (keys/secret_key.rs:25-53) on the device, from its N signed coefficients (SecretKey.coeffs; a
// Rust host reads them from sk.to_bytes(), see fhe_b200_wire.hpp).  The device copy of s is erased when the key is
// released; the host copy kept for to_bytes is erased with the object.
class SecretKey {
 public:
  SecretKey(std::shared_ptr<BfvParameters> par, const std::vector<int64_t>& coeffs) : par_(std::move(par)), coeffs_(coeffs) {
    if (coeffs_.size() != par_->degree()) throw Error(FHE_B200_INVALID_ARGUMENT, "a secret key has N coefficients");
    check(fhe_b200_secret_key_create(par_->handle(), coeffs_.data(), &h_));
  }
  SecretKey(const SecretKey&) = delete;
  SecretKey& operator=(const SecretKey&) = delete;
  // SecretKey::random (secret_key.rs:42-45): s = sample_vec_cbd(N, par.variance()) drawn on the device from the
  // stream of fhe_b200.h (role 18, key 0).  seed: 32 bytes (nullptr: fresh getrandom bytes).
  static std::unique_ptr<SecretKey> random(const std::shared_ptr<BfvParameters>& par, const uint8_t* seed = nullptr) {
    return std::move(random_vec(par, 1, seed)[0]);
  }
  // n independent SecretKey::random keys in one device call (key k is stream word 13 = k), e.g. one per party of
  // multiparty BFV.  Their coefficients stay on the device: coeffs() is empty and to_bytes downloads them.
  static inline std::vector<std::unique_ptr<SecretKey>> random_vec(const std::shared_ptr<BfvParameters>& par, uint32_t n,
                                                                   const uint8_t* seed = nullptr);
  // the N signed coefficients (fhe_b200_secret_key_coeffs for a device-born key); the caller erases them
  std::vector<int64_t> download_coeffs() const {
    if (!coeffs_.empty()) return coeffs_;
    std::vector<int64_t> c(par_->degree());
    check(fhe_b200_secret_key_coeffs(h_, c.data(), nullptr));
    return c;
  }
  ~SecretKey() {
    fhe_b200_secret_key_free(h_);
    volatile int64_t* c = coeffs_.data();
    for (size_t i = 0; i < coeffs_.size(); i++) c[i] = 0;
  }
  // SecretKey::try_encrypt (secret_key.rs:100-136, :181-193) of every plaintext of pts: one fresh ciphertext per
  // plaintext at their level.  seed: the 32 bytes keying the stream of fhe_b200.h (nullptr: fresh getrandom bytes).
  Ciphertext try_encrypt(const PlaintextVec& pts, const uint8_t* seed = nullptr) const {
    return encrypt_into(&pts.batch(), pts.len(), pts.batch().level(), seed, pts.batch().stream());
  }
  // `count` encryptions of zero at `level` (PublicKey::new takes one at level 0)
  Ciphertext try_encrypt_zero(uint32_t count, uint32_t level, const uint8_t* seed = nullptr) const {
    return encrypt_into(nullptr, count, level, seed, nullptr);
  }
  // SecretKey::try_decrypt (secret_key.rs:198-260) of every ciphertext of the batch: plaintexts without an encoding
  PlaintextVec try_decrypt(const Ciphertext& ct) const {
    Ciphertext out(par_, ct.count(), 1, ct.level(), Representation::Ntt, ct.stream());
    check(fhe_b200_decrypt(h_, ct.handle(), out.handle(), ct.stream()));
    return PlaintextVec(std::move(out));
  }
  // SecretKey::measure_noise (secret_key.rs:55-98) of every ciphertext of the batch
  std::vector<uint32_t> measure_noise(const Ciphertext& ct) const {
    std::vector<uint32_t> out(ct.count());
    check(fhe_b200_measure_noise(h_, ct.handle(), out.data(), ct.stream()));
    ct.sync();
    return out;
  }
  // SecretKey::try_encrypt into RGSWCiphertext (rgsw_ciphertext.rs:94-120) of every plaintext of pts, at their level,
  // in one device call; seed as for try_encrypt
  inline std::vector<RGSWCiphertext> try_encrypt_rgsw(const PlaintextVec& pts, const uint8_t* seed = nullptr) const;
  const std::vector<int64_t>& coeffs() const { return coeffs_; }   // empty for a device-born key
  const std::shared_ptr<BfvParameters>& par() const { return par_; }
  const fhe_b200_secret_key* handle() const { return h_; }

 private:
  SecretKey(std::shared_ptr<BfvParameters> par, fhe_b200_secret_key* h) : par_(std::move(par)), h_(h) {}
  Ciphertext encrypt_into(const Ciphertext* pts, uint32_t count, uint32_t level, const uint8_t* seed, void* stream) const;
  std::shared_ptr<BfvParameters> par_;
  std::vector<int64_t> coeffs_;
  fhe_b200_secret_key* h_ = nullptr;
};

// 32 bytes of fresh entropy for one encryption call (getrandom(2), the system CSPRNG)
struct EncryptionSeed {
  uint8_t bytes[32];
  explicit EncryptionSeed(const uint8_t* given) {
    if (given) { std::memcpy(bytes, given, 32); return; }
    for (size_t got = 0; got < 32;) {
      const ssize_t r = getrandom(bytes + got, 32 - got, 0);
      if (r < 0) throw Error(FHE_B200_INVALID_ARGUMENT, "getrandom failed");
      got += (size_t)r;
    }
  }
};

inline std::vector<std::unique_ptr<SecretKey>> SecretKey::random_vec(const std::shared_ptr<BfvParameters>& par,
                                                                    uint32_t n, const uint8_t* seed) {
  const EncryptionSeed s(seed);
  std::vector<fhe_b200_secret_key*> hs(std::max<uint32_t>(1, n), nullptr);
  check(fhe_b200_secret_keys_random(par->handle(), n, par->variance(), s.bytes, hs.data(), nullptr));
  std::vector<std::unique_ptr<SecretKey>> out;
  for (uint32_t k = 0; k < n; k++) out.emplace_back(new SecretKey(par, hs[k]));
  return out;
}

inline Ciphertext SecretKey::encrypt_into(const Ciphertext* pts, uint32_t count, uint32_t level, const uint8_t* seed,
                                          void* stream) const {
  const EncryptionSeed s(seed);
  Ciphertext out(par_, count, 2, level, Representation::Ntt, stream);
  check(fhe_b200_encrypt_sk(h_, pts ? pts->handle() : nullptr, par_->variance(), s.bytes, out.handle(), stream));
  return out;
}

// fhe::bfv::PublicKey (keys/public_key.rs:17-22): its c, one 2-part ciphertext at level 0, on the device
class PublicKey {
 public:
  PublicKey(std::shared_ptr<BfvParameters> par, Ciphertext c) : par_(std::move(par)), c_(std::move(c)) {
    if (c_.count() != 1 || c_.len() != 2) throw Error(FHE_B200_INVALID_ARGUMENT, "a public key is one 2-part ciphertext");
    if (c_.level() != 0) throw Error(FHE_B200_INVALID_LEVEL, "InvalidPublicKeyLevel");
  }
  // PublicKey::new (public_key.rs:26-38): a secret-key encryption of zero at level 0
  static PublicKey new_key(const SecretKey& sk, const uint8_t* seed = nullptr) {
    return PublicKey(sk.par(), sk.try_encrypt_zero(1, 0, seed));
  }
  // PublicKey::try_encrypt (public_key.rs:45-92) of every plaintext of pts, as SecretKey::try_encrypt
  Ciphertext try_encrypt(const PlaintextVec& pts, const uint8_t* seed = nullptr) const {
    const EncryptionSeed s(seed);
    void* stream = pts.batch().stream();
    Ciphertext out(par_, pts.len(), 2, pts.batch().level(), Representation::Ntt, stream);
    check(fhe_b200_encrypt_pk(c_.handle(), pts.batch().handle(), par_->variance(), s.bytes, out.handle(), stream));
    return out;
  }
  const Ciphertext& c() const { return c_; }
  const std::shared_ptr<BfvParameters>& par() const { return par_; }

 private:
  std::shared_ptr<BfvParameters> par_;
  Ciphertext c_;
};

class KeySwitchingKey {
 public:
  // c0, c1: NTT-domain words [n_digits][ksk_limbs][N] of the key polynomials (key_switching_key.rs:22-45)
  KeySwitchingKey(std::shared_ptr<BfvParameters> par, const std::vector<uint64_t>& c0, const std::vector<uint64_t>& c1,
                  uint32_t n_digits, uint32_t ciphertext_level = 0, uint32_t ksk_level = 0)
      : par_(std::move(par)), ciphertext_level_(ciphertext_level), ksk_level_(ksk_level), n_digits_(n_digits) {
    check(fhe_b200_ksk_upload(par_->handle(), ciphertext_level, ksk_level, c0.data(), c1.data(), n_digits, &h_));
  }
  // takes ownership of a key the library generated on `stream` (fhe_b200_relin_key_generate and the other generators)
  KeySwitchingKey(std::shared_ptr<BfvParameters> par, fhe_b200_ksk* generated, uint32_t ciphertext_level,
                  uint32_t ksk_level, void* stream)
      : par_(std::move(par)), h_(generated), ciphertext_level_(ciphertext_level), ksk_level_(ksk_level),
        stream_(stream) {
    const std::vector<uint64_t> q = par_->moduli();   // key_switching_key.rs:92-126
    n_digits_ = log_base() ? (bits(q[0] - 1) + log_base() - 1) / log_base() : (uint32_t)(q.size() - ciphertext_level);
  }
  KeySwitchingKey(const KeySwitchingKey&) = delete;
  ~KeySwitchingKey() { fhe_b200_ksk_free(h_); }
  const fhe_b200_ksk* handle() const { return h_; }
  uint32_t ciphertext_level() const { return ciphertext_level_; }
  uint32_t ksk_level() const { return ksk_level_; }
  uint32_t n_digits() const { return n_digits_; }
  // a key level with one modulus decomposes in base 2^(log_modulus / 2) (key_switching_key.rs:92-97), else 0
  uint32_t log_base() const {
    const std::vector<uint64_t> q = par_->moduli();
    return q.size() - ksk_level_ == 1 ? bits(q[0] - 1) / 2 : 0;
  }
  // the key's words read back from the device: c0, c1 [n_digits][ksk_limbs][N] (NTT)
  std::pair<std::vector<uint64_t>, std::vector<uint64_t>> arrays() const {
    const size_t n = (size_t)n_digits_ * (par_->moduli().size() - ksk_level_) * par_->degree();
    std::pair<std::vector<uint64_t>, std::vector<uint64_t>> w{std::vector<uint64_t>(n), std::vector<uint64_t>(n)};
    check(fhe_b200_ksk_download(h_, w.first.data(), w.second.data(), stream_));
    return w;
  }
  // KeySwitchingKey::key_switch (key_switching_key.rs:241-270, :323-362) on polynomial `part` of a power-basis batch:
  // the (c0, c1) pair as a 2-part NTT batch at the key level
  Ciphertext key_switch(const Ciphertext& p, uint32_t part = 0) const {
    Ciphertext out(par_, p.count(), 2, ksk_level_, Representation::Ntt, p.stream());
    check(fhe_b200_key_switch(p.handle(), part, h_, out.handle(), p.stream()));
    return out;
  }
  const std::shared_ptr<BfvParameters>& par() const { return par_; }

 private:
  static uint32_t bits(uint64_t v) { uint32_t b = 0; while (v) { b++; v >>= 1; } return b; }
  std::shared_ptr<BfvParameters> par_;
  fhe_b200_ksk* h_ = nullptr;
  uint32_t ciphertext_level_, ksk_level_, n_digits_ = 0;
  void* stream_ = nullptr;
};

class RelinearizationKey {
 public:
  explicit RelinearizationKey(std::shared_ptr<KeySwitchingKey> ksk) : ksk(std::move(ksk)) {}
  // RelinearizationKey::new / new_leveled (relinearization_key.rs:28-65), generated on the device from the seeded
  // stream (seed as for SecretKey::try_encrypt)
  static RelinearizationKey new_key(const SecretKey& sk, const uint8_t* seed = nullptr) { return new_leveled(sk, 0, 0, seed); }
  static RelinearizationKey new_leveled(const SecretKey& sk, uint32_t ciphertext_level, uint32_t key_level,
                                        const uint8_t* seed = nullptr) {
    const EncryptionSeed s(seed);
    fhe_b200_ksk* h = nullptr;
    check(fhe_b200_relin_key_generate(sk.handle(), ciphertext_level, key_level, sk.par()->variance(), s.bytes, &h,
                                      nullptr));
    return RelinearizationKey(std::make_shared<KeySwitchingKey>(sk.par(), h, ciphertext_level, key_level, nullptr));
  }
  // RelinearizationKey::relinearizes (relinearization_key.rs:70): (c0,c1,c2) -> (c0,c1)
  Ciphertext relinearizes(const Ciphertext& ct) const {
    Ciphertext out(ct.par(), ct.count(), 2, ct.level(), Representation::Ntt, ct.stream());
    check(fhe_b200_relinearize(ct.handle(), ksk->handle(), out.handle(), ct.stream()));
    return out;
  }
  std::shared_ptr<KeySwitchingKey> ksk;
};

class GaloisKey {
 public:
  GaloisKey(uint32_t exponent, std::shared_ptr<KeySwitchingKey> ksk) : exponent(exponent), ksk(std::move(ksk)) {}
  // GaloisKey::new (galois_key.rs:26-60), generated on the device (seed as for SecretKey::try_encrypt)
  static GaloisKey new_key(const SecretKey& sk, uint64_t exponent, uint32_t ciphertext_level = 0, uint32_t key_level = 0,
                           const uint8_t* seed = nullptr) {
    return std::move(generate(sk, {exponent}, ciphertext_level, key_level, seed)[0]);
  }
  // one device call for every exponent (reduced mod 2N): key k of the call (stream word 13) is exponents[k]
  static std::vector<GaloisKey> generate(const SecretKey& sk, const std::vector<uint64_t>& exponents,
                                         uint32_t ciphertext_level, uint32_t key_level, const uint8_t* seed = nullptr) {
    const EncryptionSeed s(seed);
    const uint64_t two_n = 2 * (uint64_t)sk.par()->degree();
    std::vector<uint32_t> e;
    for (uint64_t x : exponents) e.push_back((uint32_t)(x % two_n));   // SubstitutionExponent::new (rq/mod.rs:99-106)
    std::vector<fhe_b200_ksk*> h(std::max<size_t>(1, e.size()), nullptr);
    check(fhe_b200_galois_keys_generate(sk.handle(), e.data(), (uint32_t)e.size(), ciphertext_level, key_level,
                                        sk.par()->variance(), s.bytes, h.data(), nullptr));
    std::vector<GaloisKey> out;
    for (size_t k = 0; k < e.size(); k++)
      out.emplace_back(e[k], std::make_shared<KeySwitchingKey>(sk.par(), h[k], ciphertext_level, key_level, nullptr));
    return out;
  }
  // GaloisKey::relinearize (galois_key.rs:63)
  Ciphertext relinearize(const Ciphertext& ct) const {
    Ciphertext out(ct.par(), ct.count(), 2, ct.level(), Representation::Ntt, ct.stream());
    check(fhe_b200_galois(ct.handle(), exponent, ksk->handle(), out.handle(), ct.stream()));
    return out;
  }
  uint32_t exponent;
  std::shared_ptr<KeySwitchingKey> ksk;
};

// rotation subset of EvaluationKey (evaluation_key.rs:110-170)
// fhe::bfv::RGSWCiphertext (bfv/rgsw_ciphertext.rs:20-24): two key-switching keys (for m and m*s) of one level
class RGSWCiphertext {
 public:
  RGSWCiphertext(std::shared_ptr<KeySwitchingKey> k0, std::shared_ptr<KeySwitchingKey> k1) : ksk0(std::move(k0)), ksk1(std::move(k1)) {
    if (ksk0->ksk_level() != ksk0->ciphertext_level() || ksk1->ksk_level() != ksk1->ciphertext_level() ||
        ksk0->ciphertext_level() != ksk1->ciphertext_level())
      throw Error(FHE_B200_INVALID_LEVEL, "InconsistentKeySwitchingLevels");   // rgsw_ciphertext.rs:58-70
  }
  // &Ciphertext * &RGSWCiphertext (rgsw_ciphertext.rs:122-155): key-switch both parts, add
  Ciphertext external_product(const Ciphertext& ct) const {
    if (ct.level() != ksk0->ciphertext_level()) throw Error(FHE_B200_INVALID_LEVEL, "Ciphertext and RGSWCiphertext must have the same level");
    if (ct.len() != 2) throw Error(FHE_B200_BAD_POLY_COUNT, "Ciphertext must have two parts");
    Ciphertext pb = ct.clone();
    pb.into_power_basis();
    Ciphertext out = ksk0->key_switch(pb, 0);
    out += ksk1->key_switch(pb, 1);
    return out;
  }
  std::shared_ptr<KeySwitchingKey> ksk0, ksk1;
};

// fhe::bfv::EvaluationKey (keys/evaluation_key.rs:21-310): Galois keys by exponent, and the levels of the ciphertexts
// it takes and of its keys (both 0 unless an EvaluationKeyBuilder or a message sets them)
// the column rotation steps a linear transform of n_diags diagonals with baby step `baby` needs keys for (to enable in
// EvaluationKeyBuilder): the baby steps 1 .. baby - 1, then the giant steps baby, 2 baby, ..
inline std::vector<uint32_t> linear_transform_steps(uint32_t n_diags, uint32_t baby) {
  if (baby < 1 || baby > n_diags) throw Error(FHE_B200_INVALID_ARGUMENT, "the baby step must be 1 .. n_diags");
  std::vector<uint32_t> s;
  for (uint32_t i = 1; i < baby; i++) s.push_back(i);
  for (uint32_t g = baby; g < n_diags; g += baby) s.push_back(g);
  return s;
}

class EvaluationKey {
 public:
  explicit EvaluationKey(std::shared_ptr<BfvParameters> par, uint32_t ciphertext_level = 0,
                         uint32_t evaluation_key_level = 0)
      : par_(std::move(par)), ciphertext_level_(ciphertext_level), evaluation_key_level_(evaluation_key_level) {}
  uint32_t ciphertext_level() const { return ciphertext_level_; }
  uint32_t evaluation_key_level() const { return evaluation_key_level_; }
  const std::map<uint32_t, std::shared_ptr<GaloisKey>>& galois_keys() const { return gk_; }   // ascending exponents
  void add_galois_key(std::shared_ptr<GaloisKey> gk) { gk_[gk->exponent % (2 * (uint32_t)par_->degree())] = std::move(gk); }
  Ciphertext rotates_rows(const Ciphertext& ct) const { return at(2 * (uint32_t)par_->degree() - 1).relinearize(ct); }
  Ciphertext rotates_columns_by(const Ciphertext& ct, uint32_t i) const { return at(column_exponent(i)).relinearize(ct); }
  // sum_k diag_k (.) rotates_columns_by(ct, k) of every ciphertext by baby-step/giant-step diagonals in one device call
  // (fhe_b200_linear_transform); diags from encode_diagonals, n_diags shared by every ciphertext or n_diags per one
  Ciphertext linear_transform(const Ciphertext& ct, const Ciphertext& diags, uint32_t baby, uint32_t n_diags) const {
    std::vector<const fhe_b200_ksk*> keys;
    std::vector<uint32_t> exps;
    for (uint32_t i : linear_transform_steps(n_diags, baby)) {
      exps.push_back(column_exponent(i));
      keys.push_back(at(exps.back()).ksk->handle());
    }
    Ciphertext out(ct.par(), ct.count(), 2, ct.level(), Representation::Ntt, ct.stream());
    check(fhe_b200_linear_transform(ct.handle(), diags.handle(), n_diags, baby, keys.data(), exps.data(),
                                    (uint32_t)keys.size(), out.handle(), nullptr, ct.stream()));
    return out;
  }
  Ciphertext linear_transform(const Ciphertext& ct, const PlaintextVec& diags, uint32_t baby, uint32_t n_diags) const {
    return linear_transform(ct, diags.batch(), baby, n_diags);
  }
  // evaluation_key.rs:40-53
  bool supports_inner_sum() const {
    const uint32_t n = (uint32_t)par_->degree();
    bool ok = gk_.count(2 * n - 1) != 0;
    for (uint32_t i = 1; i < n / 2; i *= 2) ok = ok && gk_.count(column_exponent(i)) != 0;
    return ok;
  }
  // the keys of the inner sum's log2 N steps: column rotations by 1, 2, 4, ..., N/4, then the row rotation
  std::vector<const fhe_b200_ksk*> inner_sum_keys() const {
    if (!supports_inner_sum()) throw Error(FHE_B200_INVALID_ARGUMENT, "EvaluationKeyError: inner sum not supported by this key");
    const uint32_t n = (uint32_t)par_->degree();
    std::vector<const fhe_b200_ksk*> keys;
    for (uint32_t i = 1; i < n / 2; i *= 2) keys.push_back(at(column_exponent(i)).ksk->handle());
    keys.push_back(at(2 * n - 1).ksk->handle());
    return keys;
  }
  // EvaluationKey::computes_inner_sum (evaluation_key.rs:56-100) of every ciphertext of ct, one device call
  Ciphertext computes_inner_sum(const Ciphertext& ct) const {
    const std::vector<const fhe_b200_ksk*> keys = inner_sum_keys();
    Ciphertext out(ct.par(), ct.count(), 2, ct.level(), Representation::Ntt, ct.stream());
    check(fhe_b200_inner_sum(ct.handle(), keys.data(), (uint32_t)keys.size(), out.handle(), ct.stream()));
    return out;
  }
  // rotates_columns_by(ct_q, steps[i]) for every step and every ciphertext of ct (Q = ct.count()) in one device call
  // (fhe_b200_galois_many): entry i*Q + q of the result is ciphertext q rotated by steps[i]
  Ciphertext rotates_columns_by_many(const Ciphertext& ct, const std::vector<uint32_t>& steps) const {
    return rotates_many(ct, steps, false);
  }
  // rotates_columns_by_many, word for word, with each ciphertext's rotations computed from one digit decomposition of
  // it when it has two or more (fhe_b200_galois_many_hoisted; synchronises ct's stream once when it hoists)
  Ciphertext rotates_columns_by_many_hoisted(const Ciphertext& ct, const std::vector<uint32_t>& steps) const {
    return rotates_many(ct, steps, true);
  }

 private:
  Ciphertext rotates_many(const Ciphertext& ct, const std::vector<uint32_t>& steps, bool hoisted) const {
    std::vector<const fhe_b200_ksk*> keys;
    std::vector<uint32_t> exps, index, source;
    const uint32_t q = ct.count();
    for (uint32_t i : steps) {
      const uint32_t e = column_exponent(i);
      const GaloisKey& gk = at(e);
      uint32_t k = 0;
      while (k < exps.size() && exps[k] != e) k++;
      if (k == exps.size()) {
        exps.push_back(e);
        keys.push_back(gk.ksk->handle());
      }
      for (uint32_t j = 0; j < q; j++) {
        index.push_back(k);
        source.push_back(j);
      }
    }
    if (keys.empty()) keys.push_back(nullptr);   // no steps: refused by the call
    Ciphertext out(ct.par(), std::max<uint32_t>((uint32_t)index.size(), 1), 2, ct.level(), Representation::Ntt,
                   ct.stream());
    if (hoisted)
      check(fhe_b200_galois_many_hoisted(ct.handle(), source.data(), keys.data(), exps.data(), (uint32_t)exps.size(),
                                         index.data(), out.handle(), nullptr, ct.stream()));
    else
      check(fhe_b200_galois_many(ct.handle(), source.data(), keys.data(), exps.data(), (uint32_t)exps.size(),
                                 index.data(), out.handle(), ct.stream()));
    return out;
  }

 public:
  // evaluation_key.rs:175-189
  bool supports_expansion(uint32_t level) const {
    const uint32_t n = (uint32_t)par_->degree();
    if (level == 0) return true;
    if ((1ull << level) > n) return false;
    for (uint32_t l = 0; l < level; l++)
      if (!gk_.count((n >> l) + 1)) return false;
    return true;
  }
  // EvaluationKey::expands (evaluation_key.rs:192-256) of every ciphertext of `ct` (Q queries) as one batch of
  // size * Q: entry i*Q + q is output i of query q (fhe_b200_expand)
  Ciphertext expands_batch(const Ciphertext& ct, uint32_t size) const {
    const uint32_t n = (uint32_t)par_->degree();
    if (size == 0 || size > n) throw Error(FHE_B200_INVALID_ARGUMENT, "EvaluationKeyError: InvalidExpansionSize");
    uint32_t level = 0;
    while ((1u << level) < size) level++;
    std::vector<const fhe_b200_ksk*> keys(level, nullptr);
    for (uint32_t l = 0; l < level; l++) {
      auto it = gk_.find((n >> l) + 1);
      if (it != gk_.end()) keys[l] = it->second->ksk->handle();
    }
    Ciphertext out(ct.par(), size * ct.count(), 2, ct.level(), Representation::Ntt, ct.stream());
    check(fhe_b200_expand(ct.handle(), size, keys.data(), level, out.handle(), ct.stream()));
    return out;
  }
  // the reference's return shape: `size` batches of ct.count() ciphertexts, output i of every query
  std::vector<Ciphertext> expands(const Ciphertext& ct, uint32_t size) const {
    const Ciphertext whole = expands_batch(ct, size);
    const uint32_t q = ct.count();
    std::vector<Ciphertext> out;
    out.reserve(size);
    for (uint32_t i = 0; i < size; i++) out.push_back(whole.take(i * q, q));
    return out;
  }

 private:
  uint32_t column_exponent(uint32_t i) const {   // evaluation_key.rs:278-286
    uint64_t e = 1, m = 2 * par_->degree();
    for (uint32_t k = 0; k < i; k++) e = e * 3 % m;
    return (uint32_t)e;
  }
  const GaloisKey& at(uint32_t e) const {
    auto it = gk_.find(e);
    if (it == gk_.end()) throw Error(FHE_B200_INVALID_ARGUMENT, "EvaluationKeyError: rotation not supported by this key");
    return *it->second;
  }
  std::shared_ptr<BfvParameters> par_;
  uint32_t ciphertext_level_, evaluation_key_level_;
  std::map<uint32_t, std::shared_ptr<GaloisKey>> gk_;
};

inline std::vector<RGSWCiphertext> SecretKey::try_encrypt_rgsw(const PlaintextVec& pts, const uint8_t* seed) const {
  const EncryptionSeed s(seed);
  const Ciphertext& b = pts.batch();
  std::vector<fhe_b200_ksk*> h(2 * (size_t)b.count(), nullptr);
  check(fhe_b200_rgsw_encrypt(h_, b.handle(), par_->variance(), s.bytes, h.data(), b.stream()));
  std::vector<std::shared_ptr<KeySwitchingKey>> k;   // adopt every handle before anything can throw
  for (fhe_b200_ksk* x : h) k.push_back(std::make_shared<KeySwitchingKey>(par_, x, b.level(), b.level(), b.stream()));
  std::vector<RGSWCiphertext> out;
  for (size_t p = 0; p < b.count(); p++) out.emplace_back(k[2 * p], k[2 * p + 1]);
  return out;
}

// fhe::bfv::EvaluationKeyBuilder (keys/evaluation_key.rs:318-491): the Galois keys of an EvaluationKey, generated on
// the device in one call
class EvaluationKeyBuilder {
 public:
  explicit EvaluationKeyBuilder(const SecretKey& sk) : sk_(sk) {}
  // evaluation_key.rs:353-383
  static EvaluationKeyBuilder new_leveled(const SecretKey& sk, uint32_t ciphertext_level, uint32_t evaluation_key_level) {
    if (ciphertext_level > sk.par()->max_level()) throw Error(FHE_B200_INVALID_LEVEL, "InvalidLevel");
    if (evaluation_key_level > ciphertext_level) throw Error(FHE_B200_INVALID_LEVEL, "InvalidLevel");
    EvaluationKeyBuilder b(sk);
    b.ciphertext_level_ = ciphertext_level;
    b.key_level_ = evaluation_key_level;
    return b;
  }
  EvaluationKeyBuilder& enable_expansion(uint32_t level) {   // evaluation_key.rs:386-398
    uint32_t max_level = 0;
    while ((2ull << max_level) <= sk_.par()->degree()) max_level++;
    if (level > max_level) throw Error(FHE_B200_INVALID_LEVEL, "InvalidLevel");
    expansion_level_ = level;
    return *this;
  }
  EvaluationKeyBuilder& enable_inner_sum() { inner_sum_ = true; return *this; }
  EvaluationKeyBuilder& enable_row_rotation() { row_rotation_ = true; return *this; }
  EvaluationKeyBuilder& enable_column_rotation(uint32_t i) {   // evaluation_key.rs:414-426: steps 1 .. N/2 - 1
    if (i < 1 || i >= sk_.par()->degree() / 2) throw Error(FHE_B200_INVALID_ARGUMENT, "EvaluationKeyError::InvalidRotationStep");
    columns_.insert(column_exponent(i));
    return *this;
  }
  // the Galois exponents build() generates keys for (evaluation_key.rs:439-463), ascending
  std::vector<uint64_t> exponents() const {
    const uint64_t n = sk_.par()->degree();
    std::set<uint64_t> idx(columns_.begin(), columns_.end());
    if (row_rotation_ || inner_sum_) idx.insert(2 * n - 1);
    if (inner_sum_)
      for (uint64_t i = 1; i < n / 2; i *= 2) idx.insert(column_exponent((uint32_t)i));
    for (uint32_t l = 0; l < expansion_level_; l++) idx.insert((n >> l) + 1);
    return std::vector<uint64_t>(idx.begin(), idx.end());
  }
  // EvaluationKeyBuilder::build (evaluation_key.rs:429-491): every Galois key in one device call, the exponents
  // ascending, so a seed fixes the key of each exponent
  EvaluationKey build(const uint8_t* seed = nullptr) const {
    EvaluationKey ek(sk_.par(), ciphertext_level_, key_level_);
    const std::vector<uint64_t> e = exponents();
    if (e.empty()) return ek;
    for (GaloisKey& gk : GaloisKey::generate(sk_, e, ciphertext_level_, key_level_, seed))
      ek.add_galois_key(std::make_shared<GaloisKey>(std::move(gk)));
    return ek;
  }

 private:
  uint64_t column_exponent(uint32_t i) const {   // evaluation_key.rs:278-286
    uint64_t e = 1, m = 2 * sk_.par()->degree();
    for (uint32_t k = 0; k < i; k++) e = e * 3 % m;
    return e;
  }
  const SecretKey& sk_;
  uint32_t ciphertext_level_ = 0, key_level_ = 0, expansion_level_ = 0;
  bool inner_sum_ = false, row_rotation_ = false;
  std::set<uint64_t> columns_;
};

// fhe::bfv::dot_product_scalar (bfv/ops/dot_product.rs:55): out[g] = sum_{i<n_terms} cts[g*n_terms+i] * pts[g*n_terms+i];
// pts is a batch of one-part NTT polynomials (Plaintext::poly_ntt).  An operand with exactly n_terms entries is shared
// by every group.
inline Ciphertext dot_product_scalar(const Ciphertext& cts, const Ciphertext& pts, uint32_t n_terms) {
  if (n_terms == 0) throw Error(FHE_B200_INVALID_ARGUMENT, "DotProductError::EmptyInput");
  const uint32_t groups = std::max(cts.count(), pts.count()) / n_terms;
  Ciphertext out(cts.par(), groups ? groups : 1, cts.len(), cts.level(), Representation::Ntt, cts.stream());
  check(fhe_b200_dot_product_scalar(cts.handle(), pts.handle(), n_terms, out.handle(), cts.stream()));
  return out;
}
inline Ciphertext dot_product_scalar(const Ciphertext& cts, const PlaintextVec& pts, uint32_t n_terms) {
  return dot_product_scalar(cts, pts.batch(), n_terms);
}

// fhe_math::rns::ScalingFactor (rns/scaler.rs:20-58): numerator / denominator as little-endian byte strings
// (BigUint::to_bytes_le)
struct ScalingFactor {
  std::vector<uint8_t> numerator, denominator;
  static ScalingFactor one() { return ScalingFactor{{1}, {1}}; }
  static ScalingFactor from_u64(uint64_t num, uint64_t den) {
    auto le = [](uint64_t v) {
      std::vector<uint8_t> b;
      do { b.push_back((uint8_t)v); v >>= 8; } while (v);
      return b;
    };
    return ScalingFactor{le(num), le(den)};
  }
};

class Multiplicator {
 public:
  // Multiplicator::default (ops/mul.rs:101)
  static Multiplicator default_(const RelinearizationKey& rk) {
    Multiplicator m(rk.ksk->par(), rk.ksk->ciphertext_level());
    m.rk_ = std::make_shared<RelinearizationKey>(rk);
    return m;
  }
  // Multiplicator::new (ops/mul.rs:37-53)
  static Multiplicator new_(const ScalingFactor& lhs, const ScalingFactor& rhs, const std::vector<uint64_t>& extended_basis,
                            const ScalingFactor& post, std::shared_ptr<BfvParameters> par) {
    return new_leveled(lhs, rhs, extended_basis, post, 0, std::move(par));
  }
  // Multiplicator::new_leveled (ops/mul.rs:56-75)
  static Multiplicator new_leveled(const ScalingFactor& lhs, const ScalingFactor& rhs,
                                   const std::vector<uint64_t>& extended_basis, const ScalingFactor& post,
                                   uint32_t level, std::shared_ptr<BfvParameters> par) {
    Multiplicator m(par, level);
    fhe_b200_multiplicator* h = nullptr;
    check(fhe_b200_multiplicator_create(par->handle(), level, lhs.numerator.data(), (uint32_t)lhs.numerator.size(),
                                        lhs.denominator.data(), (uint32_t)lhs.denominator.size(), rhs.numerator.data(),
                                        (uint32_t)rhs.numerator.size(), rhs.denominator.data(),
                                        (uint32_t)rhs.denominator.size(), extended_basis.data(),
                                        (uint32_t)extended_basis.size(), nullptr, post.numerator.data(),
                                        (uint32_t)post.numerator.size(), post.denominator.data(),
                                        (uint32_t)post.denominator.size(), &h));
    m.h_ = std::shared_ptr<fhe_b200_multiplicator>(h, [](fhe_b200_multiplicator* x) { fhe_b200_multiplicator_free(x); });
    return m;
  }
  // Multiplicator::enable_relinearization (ops/mul.rs:141-151)
  void enable_relinearization(const RelinearizationKey& rk) {
    if (rk.ksk->par() != par_ || rk.ksk->ciphertext_level() != level_)
      throw Error(FHE_B200_CONTEXT_MISMATCH, "ParameterMismatch");
    rk_ = std::make_shared<RelinearizationKey>(rk);
  }
  // Multiplicator::enable_mod_switching (ops/mul.rs:155)
  void enable_mod_switching() {
    if (level_ >= par_->max_level()) throw Error(FHE_B200_NO_MORE_CONTEXT, "NoMoreContext");
    mod_switch_ = true;
  }
  // Multiplicator::multiply (ops/mul.rs:165)
  Ciphertext multiply(const Ciphertext& lhs, const Ciphertext& rhs) const {
    if (lhs.level() != level_ || rhs.level() != level_) throw Error(FHE_B200_INVALID_LEVEL, "InvalidLevel");
    const uint32_t parts = rk_ ? 2 : 3;
    Ciphertext out(lhs.par(), lhs.count(), parts, level_ + (mod_switch_ ? 1 : 0), Representation::Ntt, lhs.stream());
    if (!h_) {
      check(fhe_b200_mul_relin(lhs.handle(), rhs.handle(), rk_->ksk->handle(), mod_switch_ ? 1 : 0, out.handle(),
                               lhs.stream()));
    } else {
      check(fhe_b200_multiplicator_multiply(h_.get(), lhs.handle(), rhs.handle(), rk_ ? rk_->ksk->handle() : nullptr,
                                            mod_switch_ ? 1 : 0, out.handle(), lhs.stream()));
    }
    return out;
  }

 private:
  Multiplicator(std::shared_ptr<BfvParameters> par, uint32_t level) : par_(std::move(par)), level_(level) {}
  std::shared_ptr<BfvParameters> par_;
  std::shared_ptr<RelinearizationKey> rk_;
  std::shared_ptr<fhe_b200_multiplicator> h_;   // custom strategy; empty = fused default path
  uint32_t level_;
  bool mod_switch_ = false;
};

// ---- per-ciphertext keys (the fhe_b200_*_keyed entry points): index[j] names the key of ciphertext j (for
// expands_keyed: of query j), and output j is what the single-key method gives on ciphertext j with that key
namespace keyed_detail {
inline void check_index(const std::vector<uint32_t>& index, uint32_t count) {
  if (index.size() != count) throw Error(FHE_B200_INVALID_ARGUMENT, "expected one key index per ciphertext");
}
template <class K, class F>
std::vector<const fhe_b200_ksk*> handles(const std::vector<const K*>& keys, F ksk_of) {
  std::vector<const fhe_b200_ksk*> h;
  for (const K* k : keys) h.push_back(k ? ksk_of(*k) : nullptr);
  if (h.empty()) h.push_back(nullptr);   // n_keys = 0: refused by the call
  return h;
}
inline std::vector<const GaloisKey*> galois_of(const std::vector<const EvaluationKey*>& eks, uint32_t exponent) {
  std::vector<const GaloisKey*> g;
  for (const EvaluationKey* ek : eks) {
    auto it = ek->galois_keys().find(exponent);
    if (it == ek->galois_keys().end())
      throw Error(FHE_B200_INVALID_ARGUMENT, "EvaluationKeyError: rotation not supported by this key");
    g.push_back(it->second.get());
  }
  return g;
}
}  // namespace keyed_detail

inline Ciphertext key_switch_keyed(const Ciphertext& p, uint32_t part, const std::vector<const KeySwitchingKey*>& ksks,
                                   const std::vector<uint32_t>& index) {
  keyed_detail::check_index(index, p.count());
  const auto h = keyed_detail::handles(ksks, [](const KeySwitchingKey& k) { return k.handle(); });
  Ciphertext out(p.par(), p.count(), 2, ksks.empty() || !ksks[0] ? p.level() : ksks[0]->ksk_level(),
                 Representation::Ntt, p.stream());
  check(fhe_b200_key_switch_keyed(p.handle(), part, h.data(), (uint32_t)ksks.size(), index.data(), out.handle(),
                                  p.stream()));
  return out;
}
inline Ciphertext relinearizes_keyed(const Ciphertext& ct, const std::vector<const RelinearizationKey*>& rks,
                                     const std::vector<uint32_t>& index) {
  keyed_detail::check_index(index, ct.count());
  const auto h = keyed_detail::handles(rks, [](const RelinearizationKey& k) { return k.ksk->handle(); });
  Ciphertext out(ct.par(), ct.count(), 2, ct.level(), Representation::Ntt, ct.stream());
  check(fhe_b200_relinearize_keyed(ct.handle(), h.data(), (uint32_t)rks.size(), index.data(), out.handle(), ct.stream()));
  return out;
}
// Multiplicator::default(rks[index[j]]).multiply of pair j, with enable_mod_switching when mod_switch
inline Ciphertext multiply_keyed(const Ciphertext& a, const Ciphertext& b, const std::vector<const RelinearizationKey*>& rks,
                                 const std::vector<uint32_t>& index, bool mod_switch = false) {
  keyed_detail::check_index(index, a.count());
  const auto h = keyed_detail::handles(rks, [](const RelinearizationKey& k) { return k.ksk->handle(); });
  Ciphertext out(a.par(), a.count(), 2, a.level() + (mod_switch ? 1 : 0), Representation::Ntt, a.stream());
  check(fhe_b200_mul_relin_keyed(a.handle(), b.handle(), h.data(), (uint32_t)rks.size(), index.data(),
                                 mod_switch ? 1 : 0, out.handle(), a.stream()));
  return out;
}
// every key must be for the same exponent
inline Ciphertext galois_keyed(const Ciphertext& ct, const std::vector<const GaloisKey*>& gks,
                               const std::vector<uint32_t>& index) {
  keyed_detail::check_index(index, ct.count());
  for (const GaloisKey* g : gks)
    if (g && gks[0] && g->exponent != gks[0]->exponent)
      throw Error(FHE_B200_INVALID_ARGUMENT, "the Galois keys of one call must share their exponent");
  const auto h = keyed_detail::handles(gks, [](const GaloisKey& k) { return k.ksk->handle(); });
  Ciphertext out(ct.par(), ct.count(), 2, ct.level(), Representation::Ntt, ct.stream());
  check(fhe_b200_galois_keyed(ct.handle(), gks.empty() || !gks[0] ? 1 : gks[0]->exponent, h.data(),
                              (uint32_t)gks.size(), index.data(), out.handle(), ct.stream()));
  return out;
}
inline Ciphertext rotates_columns_by_keyed(const Ciphertext& ct, const std::vector<const EvaluationKey*>& eks,
                                           const std::vector<uint32_t>& index, uint32_t i) {
  uint64_t e = 1, m = 2 * ct.par()->degree();   // evaluation_key.rs:278-286
  for (uint32_t k = 0; k < i; k++) e = e * 3 % m;
  return galois_keyed(ct, keyed_detail::galois_of(eks, (uint32_t)e), index);
}
inline Ciphertext rotates_rows_keyed(const Ciphertext& ct, const std::vector<const EvaluationKey*>& eks,
                                     const std::vector<uint32_t>& index) {
  return galois_keyed(ct, keyed_detail::galois_of(eks, 2 * (uint32_t)ct.par()->degree() - 1), index);
}
// GaloisKey::relinearize of ciphertext source[j] (j when source is empty) with gks[index[j]], each key with its own
// exponent (fhe_b200_galois_many)
inline Ciphertext galois_many(const Ciphertext& ct, const std::vector<const GaloisKey*>& gks,
                              const std::vector<uint32_t>& index, const std::vector<uint32_t>& source = {}) {
  const uint32_t count = source.empty() ? ct.count() : (uint32_t)source.size();
  keyed_detail::check_index(index, count);
  const auto h = keyed_detail::handles(gks, [](const GaloisKey& k) { return k.ksk->handle(); });
  std::vector<uint32_t> exps;
  for (const GaloisKey* g : gks) exps.push_back(g ? g->exponent : 1);
  if (exps.empty()) exps.push_back(1);
  Ciphertext out(ct.par(), std::max<uint32_t>(count, 1), 2, ct.level(), Representation::Ntt, ct.stream());
  check(fhe_b200_galois_many(ct.handle(), source.empty() ? nullptr : source.data(), h.data(), exps.data(),
                             (uint32_t)gks.size(), index.data(), out.handle(), ct.stream()));
  return out;
}
// galois_many, word for word, with the rotations of each source that has two or more outputs computed from one digit
// decomposition of its c1 (fhe_b200_galois_many_hoisted); *n_hoisted (when given) receives how many were
inline Ciphertext galois_many_hoisted(const Ciphertext& ct, const std::vector<const GaloisKey*>& gks,
                                      const std::vector<uint32_t>& index, const std::vector<uint32_t>& source = {},
                                      uint32_t* n_hoisted = nullptr) {
  const uint32_t count = source.empty() ? ct.count() : (uint32_t)source.size();
  keyed_detail::check_index(index, count);
  const auto h = keyed_detail::handles(gks, [](const GaloisKey& k) { return k.ksk->handle(); });
  std::vector<uint32_t> exps;
  for (const GaloisKey* g : gks) exps.push_back(g ? g->exponent : 1);
  if (exps.empty()) exps.push_back(1);
  Ciphertext out(ct.par(), std::max<uint32_t>(count, 1), 2, ct.level(), Representation::Ntt, ct.stream());
  check(fhe_b200_galois_many_hoisted(ct.handle(), source.empty() ? nullptr : source.data(), h.data(), exps.data(),
                                     (uint32_t)gks.size(), index.data(), out.handle(), n_hoisted, ct.stream()));
  return out;
}
// out[c] = sum_g rot_{g baby}(sum_i diags[g baby + i] (.) rot_i(ct[c])), rot_0 the identity, word for word the
// composition of rotates_columns_by, mul_plain and + (fhe_b200_linear_transform); gks: Galois keys holding at least the
// steps of linear_transform_steps; *n_fallback (when given) receives how many baby-step rotations were unhoisted
inline Ciphertext linear_transform(const Ciphertext& ct, const Ciphertext& diags, uint32_t n_diags, uint32_t baby,
                                   const std::vector<const GaloisKey*>& gks, uint32_t* n_fallback = nullptr) {
  const auto h = keyed_detail::handles(gks, [](const GaloisKey& k) { return k.ksk->handle(); });
  std::vector<uint32_t> exps;
  for (const GaloisKey* g : gks) exps.push_back(g ? g->exponent : 1);
  Ciphertext out(ct.par(), ct.count(), 2, ct.level(), Representation::Ntt, ct.stream());
  check(fhe_b200_linear_transform(ct.handle(), diags.handle(), n_diags, baby, gks.empty() ? nullptr : h.data(),
                                  exps.empty() ? nullptr : exps.data(), (uint32_t)gks.size(), out.handle(), n_fallback,
                                  ct.stream()));
  return out;
}
// The diagonals of `count` slot-wise linear maps for linear_transform, SIMD-encoded at `level`: matrices holds count
// pairs of (N/2) x (N/2) matrices, [count][2][N/2][N/2] (one per slot row), entries taken mod t.  Diagonal k of a map is
// M[r][(r + k) mod N/2] in slot r of each row, rotated right by its giant step (k / baby) * baby; the result holds
// diagonals 0 .. n_diags - 1 (0: N/2) of each map.  A non-zero diagonal from n_diags on is refused.
inline PlaintextVec encode_diagonals(const std::shared_ptr<BfvParameters>& par, const std::vector<uint64_t>& matrices,
                                     uint32_t count, uint32_t baby, uint32_t level = 0, uint32_t n_diags = 0) {
  const size_t half = par->degree() / 2;
  uint64_t t = 0;
  const std::vector<uint8_t>& t_le = par->plaintext_le();
  if (t_le.size() > 8) throw Error(FHE_B200_INVALID_ARGUMENT, "EncodingError::SimdUnavailable");
  for (size_t i = t_le.size(); i-- > 0;) t = (t << 8) | t_le[i];
  if (!n_diags) n_diags = (uint32_t)half;
  if (matrices.size() != count * 2 * half * half || n_diags > half || baby < 1 || baby > n_diags)
    throw Error(FHE_B200_INVALID_ARGUMENT, "expected [count][2][N/2][N/2] matrices, n_diags <= N/2, 1 <= baby <= n_diags");
  std::vector<uint64_t> v((size_t)count * n_diags * 2 * half);
  for (size_t c = 0; c < count; c++)
    for (size_t q = 0; q < 2; q++)
      for (size_t k = 0; k < half; k++)
        for (size_t r = 0; r < half; r++) {
          const uint64_t x = matrices[((c * 2 + q) * half + r) * half + (r + k) % half] % t;
          if (k >= n_diags) {
            if (x) throw Error(FHE_B200_INVALID_ARGUMENT, "a diagonal beyond the first n_diags is not zero");
            continue;
          }
          const size_t shift = (k / baby) * baby;
          v[((c * n_diags + k) * 2 + q) * half + (r + shift) % half] = x;
        }
  return PlaintextVec::try_encode(v, Encoding::simd_at_level(level), par);
}
// EvaluationKey::computes_inner_sum of ciphertext j with eks[index[j]] (fhe_b200_inner_sum_keyed)
inline Ciphertext computes_inner_sum_keyed(const Ciphertext& ct, const std::vector<const EvaluationKey*>& eks,
                                           const std::vector<uint32_t>& index) {
  keyed_detail::check_index(index, ct.count());
  std::vector<const fhe_b200_ksk*> keys;
  uint32_t n_gks = 0;
  for (const EvaluationKey* ek : eks) {
    const std::vector<const fhe_b200_ksk*> k = ek->inner_sum_keys();
    n_gks = (uint32_t)k.size();
    keys.insert(keys.end(), k.begin(), k.end());
  }
  if (keys.empty()) keys.push_back(nullptr);
  Ciphertext out(ct.par(), ct.count(), 2, ct.level(), Representation::Ntt, ct.stream());
  check(fhe_b200_inner_sum_keyed(ct.handle(), keys.data(), n_gks, (uint32_t)eks.size(), index.data(), out.handle(),
                                 ct.stream()));
  return out;
}
// Ciphertext += folded over runs of n_terms entries (bfv/ops/mod.rs:54-69; n_terms 0: the whole batch), one
// ciphertext per run (fhe_b200_batch_sum)
inline Ciphertext batch_sum(const Ciphertext& in, uint32_t n_terms = 0) {
  const uint32_t n = n_terms ? n_terms : in.count();
  if (n == 0 || in.count() % n)
    throw Error(FHE_B200_INVALID_ARGUMENT, "a batch of " + std::to_string(in.count()) + " entries does not split into runs of " +
                                              std::to_string(n_terms));
  Ciphertext out(in.par(), in.count() / n, in.len(), in.level(), in.representation(), in.stream());
  check(fhe_b200_batch_sum(in.handle(), n, 0, out.handle(), in.stream()));
  return out;
}
namespace keyed_detail {
inline uint32_t dot_groups(const Ciphertext& a, const Ciphertext& b, uint32_t n_terms) {
  const uint32_t count = std::max(a.count(), b.count());
  if (n_terms == 0 || count % n_terms)
    throw Error(FHE_B200_INVALID_ARGUMENT, "DotProductError::OperandCountMismatch");
  return count / n_terms;
}
}  // namespace keyed_detail
// sum_{i<n_terms} a[g*n_terms+i] * b[g*n_terms+i] for every group g, relinearized with rk (3 parts when rk is null) and
// switched to `level` (-1: the operands' level); an operand of n_terms entries is shared (fhe_b200_dot_product)
inline Ciphertext dot_product(const Ciphertext& a, const Ciphertext& b, uint32_t n_terms,
                              const RelinearizationKey* rk = nullptr, int level = -1) {
  const uint32_t groups = keyed_detail::dot_groups(a, b, n_terms);
  Ciphertext out(a.par(), groups, rk ? 2 : 3, level < 0 ? a.level() : (uint32_t)level, Representation::Ntt, a.stream());
  check(fhe_b200_dot_product(a.handle(), b.handle(), n_terms, rk ? rk->ksk->handle() : nullptr, out.handle(),
                             a.stream()));
  return out;
}
// dot_product with group g relinearized by rks[index[g]] (fhe_b200_dot_product_keyed)
inline Ciphertext dot_product_keyed(const Ciphertext& a, const Ciphertext& b, uint32_t n_terms,
                                    const std::vector<const RelinearizationKey*>& rks, const std::vector<uint32_t>& index,
                                    int level = -1) {
  const uint32_t groups = keyed_detail::dot_groups(a, b, n_terms);
  keyed_detail::check_index(index, groups);
  const auto h = keyed_detail::handles(rks, [](const RelinearizationKey& k) { return k.ksk->handle(); });
  Ciphertext out(a.par(), groups, 2, level < 0 ? a.level() : (uint32_t)level, Representation::Ntt, a.stream());
  check(fhe_b200_dot_product_keyed(a.handle(), b.handle(), n_terms, h.data(), (uint32_t)rks.size(), index.data(),
                                   out.handle(), a.stream()));
  return out;
}
// EvaluationKey::expands of query q with eks[index[q]]: `size` batches, batch i holding output i of every query
inline std::vector<Ciphertext> expands_keyed(const Ciphertext& ct, const std::vector<const EvaluationKey*>& eks,
                                             const std::vector<uint32_t>& index, uint32_t size) {
  const uint32_t n = (uint32_t)ct.par()->degree();
  if (size == 0 || size > n) throw Error(FHE_B200_INVALID_ARGUMENT, "EvaluationKeyError: InvalidExpansionSize");
  keyed_detail::check_index(index, ct.count());
  uint32_t level = 0;
  while ((1u << level) < size) level++;
  std::vector<const fhe_b200_ksk*> keys((size_t)level * eks.size() + 1, nullptr);
  for (size_t s = 0; s < eks.size(); s++)
    for (uint32_t l = 0; l < level; l++) {
      auto it = eks[s]->galois_keys().find((n >> l) + 1);
      if (it != eks[s]->galois_keys().end()) keys[s * level + l] = it->second->ksk->handle();
    }
  Ciphertext whole(ct.par(), size * ct.count(), 2, ct.level(), Representation::Ntt, ct.stream());
  check(fhe_b200_expand_keyed(ct.handle(), size, keys.data(), level, (uint32_t)eks.size(), index.data(), whole.handle(),
                              ct.stream()));
  const uint32_t q = ct.count();
  std::vector<Ciphertext> out;
  out.reserve(size);
  for (uint32_t i = 0; i < size; i++) out.push_back(whole.take(i * q, q));
  return out;
}
// &cts[j] * &rgsws[index[j]] (rgsw_ciphertext.rs:122-155): two keyed key switches and an add
inline Ciphertext external_products_keyed(const Ciphertext& cts, const std::vector<const RGSWCiphertext*>& rgsws,
                                          const std::vector<uint32_t>& index) {
  for (const RGSWCiphertext* r : rgsws)
    if (r && r->ksk0->ciphertext_level() != cts.level())
      throw Error(FHE_B200_INVALID_LEVEL, "Ciphertext and RGSWCiphertext must have the same level");
  if (cts.len() != 2) throw Error(FHE_B200_BAD_POLY_COUNT, "Ciphertext must have two parts");
  std::vector<const KeySwitchingKey*> k0, k1;
  for (const RGSWCiphertext* r : rgsws) {
    k0.push_back(r ? r->ksk0.get() : nullptr);
    k1.push_back(r ? r->ksk1.get() : nullptr);
  }
  Ciphertext pb = cts.clone();
  pb.into_power_basis();
  Ciphertext out = key_switch_keyed(pb, 0, k0, index);
  out += key_switch_keyed(pb, 1, k1, index);
  return out;
}

}  // namespace bfv

// fhe::mbfv (multiparty BFV, crates/fhe/src/mbfv).  WARNING: experimental, incomplete and not audited, as the
// reference's module: the share errors are the ordinary variance errors, not smudging noise, and none is added.  Every
// share holds device batches and covers a whole batch of ciphertexts; seeds as for SecretKey::try_encrypt.
namespace mbfv {
using bfv::BfvParameters;
using bfv::Ciphertext;
using bfv::EncryptionSeed;
using bfv::KeySwitchingKey;
using bfv::PlaintextVec;
using bfv::PublicKey;
using bfv::RelinearizationKey;
using bfv::Representation;
using bfv::SecretKey;

inline std::vector<fhe_b200_batch*> handles(const std::vector<const Ciphertext*>& b) {
  std::vector<fhe_b200_batch*> h;
  for (const Ciphertext* c : b) h.push_back(c->handle());
  return h;
}
inline const fhe_b200_batch* const* table(const std::vector<fhe_b200_batch*>& h) {
  return reinterpret_cast<const fhe_b200_batch* const*>(h.data());
}

// CommonRandomPoly (crp.rs:8-44): a 1-part batch, one CRP per entry
struct CommonRandomPoly {
  std::shared_ptr<Ciphertext> batch;
  static CommonRandomPoly new_leveled(const std::shared_ptr<BfvParameters>& par, uint32_t level,
                                      const uint8_t* seed = nullptr) {
    return {generate(par, 1, level, seed)};
  }
  static CommonRandomPoly new_key(const std::shared_ptr<BfvParameters>& par, const uint8_t* seed = nullptr) {
    return new_leveled(par, 0, seed);
  }
  // one CRP per modulus, drawn in one call (entry k of the call is CRP k)
  static std::vector<CommonRandomPoly> new_vec(const std::shared_ptr<BfvParameters>& par, const uint8_t* seed = nullptr) {
    const auto b = generate(par, (uint32_t)par->moduli().size(), 0, seed);
    std::vector<CommonRandomPoly> v;
    for (uint32_t k = 0; k < b->count(); k++) v.push_back({std::make_shared<Ciphertext>(b->take(k, 1))});
    return v;
  }
  static std::shared_ptr<Ciphertext> generate(const std::shared_ptr<BfvParameters>& par, uint32_t count, uint32_t level,
                                              const uint8_t* seed) {
    const EncryptionSeed s(seed);
    auto b = std::make_shared<Ciphertext>(par, count, 1, level);
    check(fhe_b200_crp_generate(par->handle(), s.bytes, b->handle(), b->stream()));
    return b;
  }
};

// PublicKeyShare (public_key_gen.rs:11-58): p0 = -crp s + e
struct PublicKeyShare {
  CommonRandomPoly crp;
  Ciphertext p0_share;
  PublicKeyShare(const SecretKey& sk, CommonRandomPoly c, const uint8_t* seed = nullptr)
      : crp(std::move(c)), p0_share(sk.par(), crp.batch->count(), 1, 0) {
    const EncryptionSeed s(seed);
    check(fhe_b200_pk_share(sk.handle(), crp.batch->handle(), sk.par()->variance(), s.bytes, p0_share.handle(),
                            p0_share.stream()));
  }
};

// SecretKeySwitchShare (secret_key_switch.rs:14-96): h = (s_in - s_out) c1 + e for every ciphertext of ct; a null
// output key is DecryptionShare's zero key (:117-143)
struct SecretKeySwitchShare {
  const Ciphertext* ct;
  Ciphertext h_share;
  SecretKeySwitchShare(const SecretKey& sk_in, const SecretKey* sk_out, const Ciphertext& c, const uint8_t* seed = nullptr)
      : ct(&c), h_share(sk_in.par(), c.count(), 1, c.level(), Representation::Ntt, c.stream()) {
    const EncryptionSeed s(seed);
    check(fhe_b200_sks_share(sk_in.handle(), sk_out ? sk_out->handle() : nullptr, c.handle(), sk_in.par()->variance(),
                             s.bytes, h_share.handle(), c.stream()));
  }
};
struct DecryptionShare : SecretKeySwitchShare {
  DecryptionShare(const SecretKey& sk, const Ciphertext& c, const uint8_t* seed = nullptr)
      : SecretKeySwitchShare(sk, nullptr, c, seed) {}
};

// PublicKeySwitchShare (public_key_switch.rs:13-93): (u pk0 + s c1 + e0, u pk1 + e1), a 2-part batch
struct PublicKeySwitchShare {
  const Ciphertext* ct;
  Ciphertext h_share;
  PublicKeySwitchShare(const SecretKey& sk, const PublicKey& pk, const Ciphertext& c, const uint8_t* seed = nullptr)
      : ct(&c), h_share(sk.par(), c.count(), 2, c.level(), Representation::Ntt, c.stream()) {
    const EncryptionSeed s(seed);
    check(fhe_b200_pks_share(sk.handle(), pk.c().handle(), c.handle(), sk.par()->variance(), s.bytes, h_share.handle(),
                             c.stream()));
  }
};

// RelinKeyShare<R> (relin_key_gen.rs:14-34): h0, h1, one polynomial per level-0 modulus each; a round-2 share keeps
// the round-1 aggregate it was made from
enum class Round { R1, R1Aggregated, R2 };
struct RelinKeyShare {
  Round round;
  std::shared_ptr<Ciphertext> h0, h1;
  std::shared_ptr<const RelinKeyShare> last_round;
};

// RelinKeyGenerator (relin_key_gen.rs:36-110): u lives on the device and is erased when the generator is destroyed
class RelinKeyGenerator {
 public:
  RelinKeyGenerator(const SecretKey& sk, const std::vector<CommonRandomPoly>& crp, const uint8_t* seed = nullptr)
      : par_(sk.par()), crp_(par_, (uint32_t)par_->moduli().size(), 1, 0) {
    if (crp.size() != par_->moduli().size())
      throw Error(FHE_B200_INVALID_ARGUMENT, "MultipartyError::InvalidCommonRandomPolynomialCount");
    for (uint32_t i = 0; i < crp.size(); i++)
      check(fhe_b200_batch_copy_range(crp_.handle(), i, crp[i].batch->handle(), 0, 1, 1, crp_.stream()));
    const EncryptionSeed s(seed);
    check(fhe_b200_rkg_create(sk.handle(), crp_.handle(), par_->variance(), s.bytes, &h_, crp_.stream()));
  }
  RelinKeyGenerator(const RelinKeyGenerator&) = delete;
  RelinKeyGenerator& operator=(const RelinKeyGenerator&) = delete;
  ~RelinKeyGenerator() { fhe_b200_rkg_free(h_); }
  RelinKeyShare round_1(const uint8_t* seed = nullptr) const {
    const EncryptionSeed s(seed);
    RelinKeyShare r = pair(Round::R1);
    check(fhe_b200_rkg_round1(h_, s.bytes, r.h0->handle(), r.h1->handle(), r.h0->stream()));
    return r;
  }
  RelinKeyShare round_2(const std::shared_ptr<const RelinKeyShare>& r1, const uint8_t* seed = nullptr) const {
    if (r1->round != Round::R1Aggregated) throw Error(FHE_B200_INVALID_ARGUMENT, "round 2 takes the round-1 aggregate");
    const EncryptionSeed s(seed);
    RelinKeyShare r = pair(Round::R2);
    r.last_round = r1;
    check(fhe_b200_rkg_round2(h_, r1->h0->handle(), r1->h1->handle(), s.bytes, r.h0->handle(), r.h1->handle(),
                              r.h0->stream()));
    return r;
  }

 private:
  RelinKeyShare pair(Round round) const {
    const uint32_t L = (uint32_t)par_->moduli().size();
    return {round, std::make_shared<Ciphertext>(par_, L, 1, 0), std::make_shared<Ciphertext>(par_, L, 1, 0), nullptr};
  }
  std::shared_ptr<BfvParameters> par_;
  Ciphertext crp_;   // the CRPs side by side, as long as the generator
  fhe_b200_rkg* h_ = nullptr;
};

// Aggregate::from_shares (aggregate.rs and the impls beside each share); the first share supplies the CRP / ciphertext
inline PublicKey public_key_from_shares(const std::vector<PublicKeyShare>& shares) {
  if (shares.empty()) throw Error(FHE_B200_INVALID_ARGUMENT, "MultipartyError::NoShares");
  std::vector<const Ciphertext*> b;
  for (const auto& s : shares) b.push_back(&s.p0_share);
  const auto h = handles(b);
  const Ciphertext& crp = *shares[0].crp.batch;
  Ciphertext pk(crp.par(), crp.count(), 2, 0, Representation::Ntt, crp.stream());
  check(fhe_b200_pk_aggregate(table(h), (uint32_t)h.size(), crp.handle(), pk.handle(), pk.stream()));
  return PublicKey(crp.par(), std::move(pk));
}
template <class Share>
inline Ciphertext ciphertext_from_shares(const std::vector<Share>& shares) {
  if (shares.empty()) throw Error(FHE_B200_INVALID_ARGUMENT, "MultipartyError::NoShares");
  std::vector<const Ciphertext*> b;
  for (const auto& s : shares) b.push_back(&s.h_share);
  const auto h = handles(b);
  const Ciphertext& ct = *shares[0].ct;
  Ciphertext out(ct.par(), ct.count(), 2, ct.level(), Representation::Ntt, ct.stream());
  const bool sks = std::is_base_of<SecretKeySwitchShare, Share>::value;
  check((sks ? fhe_b200_sks_aggregate : fhe_b200_pks_aggregate)(ct.handle(), table(h), (uint32_t)h.size(), out.handle(),
                                                                out.stream()));
  return out;
}
class PlaintextAccess {
 public:
  static PlaintextVec without_encoding(Ciphertext b) { return PlaintextVec(std::move(b)); }
};
// Plaintext::from_shares: one plaintext per ciphertext, no encoding
inline PlaintextVec plaintext_from_shares(const std::vector<DecryptionShare>& shares) {
  if (shares.empty()) throw Error(FHE_B200_INVALID_ARGUMENT, "MultipartyError::NoShares");
  std::vector<const Ciphertext*> b;
  for (const auto& s : shares) b.push_back(&s.h_share);
  const auto h = handles(b);
  const Ciphertext& ct = *shares[0].ct;
  Ciphertext out(ct.par(), ct.count(), 1, ct.level(), Representation::Ntt, ct.stream());
  check(fhe_b200_decryption_aggregate(ct.par()->encoder(), ct.handle(), table(h), (uint32_t)h.size(), out.handle(),
                                      out.stream()));
  return PlaintextAccess::without_encoding(std::move(out));
}
// RelinKeyShare<R1Aggregated>::from_shares (round-1 shares) or RelinearizationKey::from_shares (round-2 shares)
inline RelinKeyShare r1_from_shares(const std::vector<RelinKeyShare>& shares) {
  if (shares.empty()) throw Error(FHE_B200_INVALID_ARGUMENT, "MultipartyError::NoShares");
  std::vector<const Ciphertext*> b0, b1;
  for (const auto& s : shares) {
    if (s.round != Round::R1) throw Error(FHE_B200_INVALID_ARGUMENT, "round-1 shares expected");
    b0.push_back(s.h0.get());
    b1.push_back(s.h1.get());
  }
  const Ciphertext& f = *shares[0].h0;
  RelinKeyShare r{Round::R1Aggregated, std::make_shared<Ciphertext>(f.par(), f.count(), 1, 0),
                  std::make_shared<Ciphertext>(f.par(), f.count(), 1, 0), nullptr};
  const auto h0 = handles(b0), h1 = handles(b1);
  check(fhe_b200_shares_sum(table(h0), (uint32_t)h0.size(), r.h0->handle(), r.h0->stream()));
  check(fhe_b200_shares_sum(table(h1), (uint32_t)h1.size(), r.h1->handle(), r.h1->stream()));
  return r;
}
inline RelinearizationKey relin_key_from_shares(const std::vector<RelinKeyShare>& shares) {
  if (shares.empty()) throw Error(FHE_B200_INVALID_ARGUMENT, "MultipartyError::NoShares");
  std::vector<const Ciphertext*> b0, b1;
  for (const auto& s : shares) {
    if (s.round != Round::R2) throw Error(FHE_B200_INVALID_ARGUMENT, "round-2 shares expected");
    b0.push_back(s.h0.get());
    b1.push_back(s.h1.get());
  }
  const auto h0 = handles(b0), h1 = handles(b1);
  const Ciphertext& f = *shares[0].h0;
  fhe_b200_ksk* k = nullptr;
  check(fhe_b200_rkg_aggregate(table(h0), table(h1), (uint32_t)h0.size(), shares[0].last_round->h1->handle(), &k,
                               f.stream()));
  return RelinearizationKey(std::make_shared<KeySwitchingKey>(f.par(), k, 0, 0, f.stream()));
}
}  // namespace mbfv
}  // namespace fhe_b200
