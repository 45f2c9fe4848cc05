/*
 * fhe_b200.h -- C ABI of the H100-native BFV ciphertext-arithmetic engine.
 *
 * Drop-in boundary for the fhe-math / fhe::bfv hot path of tlepoint/fhe.rs @ e248cd28
 * (pure Rust; it has no FFI of its own -- SURVEY.md section 8b).  Each entry point
 * names the reference item it replaces (file:line under the reference's crates/).
 * A Rust host binds these with `extern "C"` (see INTEGRATION.md); in this repository the
 * same symbols are driven from C++ (include/fhe_b200.hpp) and Python ctypes
 * (fhe_rs_b200/_capi.py).
 *
 * Conventions
 *  - plain pointers and sizes only; all polynomial words are u64 residues.
 *  - every call returns 0 on success or a negative fhe_b200_status mirroring the
 *    reference's error enums (fhe-math/src/errors.rs:14-113, fhe/src/errors.rs:17-66);
 *    nothing throws or aborts across the boundary.  fhe_b200_last_error() returns the
 *    message of the calling thread's last failure.  (The reference's operators `+ - *`
 *    panic on mismatched operands, ops/mod.rs:19-29; here the same conditions return
 *    FHE_B200_CONTEXT_MISMATCH / FHE_B200_INVALID_LEVEL.)
 *  - caller owns host memory; the library owns device memory behind opaque handles,
 *    released by the matching *_destroy / *_free.  params and ksk handles are immutable
 *    after creation and may be shared by host threads (like Arc<BfvParameters>,
 *    bfv/parameters.rs:125); a batch handle must not be mutated concurrently.
 *  - `stream` is a cudaStream_t passed as void* (NULL = default stream).  Work is
 *    enqueued asynchronously; fhe_b200_sync() or a download waits for it.  `stream` is the only
 *    stream the caller has to reason about: a batched operation over more ciphertexts than one chunk
 *    (FHE_B200_CHUNK, default 256) runs its chunks on side streams owned by the parameter set, but
 *    these start behind everything already enqueued on `stream` and `stream` waits for them before
 *    the call returns, so the operation is ordered on `stream` like a single kernel would be.
 *  - host layout of a batch == Vec<u64>::from(&Poly) of the reference
 *    (rq/convert.rs:474-503) concatenated over parts and ciphertexts:
 *    [ciphertext][part][limb][coefficient], row-major, limb i modulo moduli[i].
 *  - there is NO CPU fallback: compute entry points fail with FHE_B200_NO_DEVICE when the
 *    parameter set was created without a CUDA device.
 */
#ifndef FHE_B200_H
#define FHE_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef enum {
  FHE_B200_OK = 0,
  FHE_B200_INVALID_ARGUMENT = -1,       /* null pointer, zero count, bad size                        */
  FHE_B200_INVALID_MODULUS = -2,        /* fhe_math::Error::InvalidModulus / NonCoprimeModuli        */
  FHE_B200_INVALID_DEGREE = -3,         /* fhe_math::Error::InvalidPolynomialDegree                   */
  FHE_B200_NTT_UNAVAILABLE = -4,        /* fhe_math::Error::NttOperatorUnavailable                    */
  FHE_B200_CONTEXT_MISMATCH = -5,       /* PolynomialContextMismatch / fhe::Error::ParameterMismatch  */
  FHE_B200_INVALID_LEVEL = -6,          /* fhe::Error::InvalidLevel / InvalidContextLevel             */
  FHE_B200_BAD_POLY_COUNT = -7,         /* CiphertextError::{MultiplicationPolynomialCount,InvalidPolynomialCount} */
  FHE_B200_INVALID_REPRESENTATION = -8, /* fhe_math::Error::IncorrectRepresentation                   */
  FHE_B200_NO_MORE_CONTEXT = -9,        /* fhe_math::Error::NoMoreContext                             */
  FHE_B200_INVALID_EXPONENT = -10,      /* fhe_math::Error::InvalidSubstitutionExponent               */
  FHE_B200_UNSUPPORTED = -11,           /* feature outside the accelerated path                       */
  FHE_B200_CUDA_ERROR = -20,
  FHE_B200_OUT_OF_MEMORY = -21,
  FHE_B200_NO_DEVICE = -22
} fhe_b200_status;

/* Poly representation tag (rq/mod.rs Representation). */
typedef enum { FHE_B200_POWER_BASIS = 0, FHE_B200_NTT = 1 } fhe_b200_repr;

typedef struct fhe_b200_params fhe_b200_params; /* == Arc<BfvParameters> (bfv/parameters.rs:88-114)            */
typedef struct fhe_b200_batch fhe_b200_batch;   /* == Vec<Ciphertext> of one level (bfv/ciphertext.rs:18-32),
                                                   device resident, [count][parts][limbs][N] u64               */
typedef struct fhe_b200_ksk fhe_b200_ksk;       /* == KeySwitchingKey (bfv/keys/key_switching_key.rs:22-45)     */
typedef struct fhe_b200_multiplicator fhe_b200_multiplicator; /* == Multiplicator with a custom strategy
                                                   (bfv/ops/mul.rs:22-98)                                        */
typedef struct fhe_b200_encoder fhe_b200_encoder; /* == the plaintext side of BfvParameters: the NTT operator of t
                                                     and the SIMD slot map (parameters.rs:71-75, :713-726)      */
typedef struct fhe_b200_secret_key fhe_b200_secret_key; /* == SecretKey (bfv/keys/secret_key.rs:25-53)               */
typedef struct fhe_b200_rkg fhe_b200_rkg;             /* == mbfv::RelinKeyGenerator (mbfv/relin_key_gen.rs:36-96)  */

/* Encoding (bfv/encoding.rs): the level comes from the output batch (Encoding::{poly,simd}_at_level). */
typedef enum { FHE_B200_ENCODING_POLY = 0, FHE_B200_ENCODING_SIMD = 1 } fhe_b200_encoding;

const char* fhe_b200_version(void);
const char* fhe_b200_last_error(void);

/* ---- parameters ---------------------------------------------------------------------
 * BfvParametersBuilder::build (bfv/parameters.rs:560-738) for explicit moduli
 * (`set_moduli`) or generated ones (`set_moduli_sizes`, parameters.rs:391-431).
 * plaintext_le: plaintext modulus as little-endian bytes (as bfv.proto PlaintextBig).
 * psi: optional 2N-th primitive roots, one per prime in the order
 *      [moduli..., extended_basis...] (n_moduli + n_moduli + 1 entries); NULL selects the
 *      documented default root.  A Rust host passes the reference's roots
 *      (NttOperator.omegas[N/2], ntt/native.rs:50-56) so that NTT-domain data is
 *      interchangeable bit for bit.
 * device: CUDA device ordinal, or -1 for a host-only handle (table inspection only). */
int fhe_b200_params_create(int device, uint32_t degree, const uint64_t* moduli, uint32_t n_moduli,
                           const uint8_t* plaintext_le, uint32_t plaintext_len, const uint64_t* psi,
                           fhe_b200_params** out);
int fhe_b200_params_create_from_sizes(int device, uint32_t degree, const uint32_t* moduli_sizes,
                                      uint32_t n_moduli, const uint8_t* plaintext_le,
                                      uint32_t plaintext_len, fhe_b200_params** out);
int fhe_b200_params_destroy(fhe_b200_params* p);
uint32_t fhe_b200_params_degree(const fhe_b200_params* p);                 /* BfvParameters::degree          */
uint32_t fhe_b200_params_n_moduli(const fhe_b200_params* p);               /* BfvParameters::moduli().len()  */
int fhe_b200_params_moduli(const fhe_b200_params* p, uint64_t* out);       /* BfvParameters::moduli          */
/* multiplication basis of `level`: the level's moduli followed by the extension primes
 * (parameters.rs:660-700); *n receives the count, out may be NULL to query it. */
int fhe_b200_params_mul_basis(const fhe_b200_params* p, uint32_t level, uint64_t* out, uint32_t* n);
/* psi actually used for prime `q` of this parameter set. */
int fhe_b200_params_psi(const fhe_b200_params* p, uint64_t q, uint64_t* psi);

/* ---- batches --------------------------------------------------------------------------
 * parts = polynomials per ciphertext (2 fresh, 3 after `&ct * &ct`); level = modulus-
 * switching level (ciphertext.rs:31); limbs = n_moduli - level. */
int fhe_b200_batch_alloc(const fhe_b200_params* p, uint32_t count, uint32_t parts, uint32_t level,
                         int repr, fhe_b200_batch** out);
int fhe_b200_batch_free(fhe_b200_batch* b);
int fhe_b200_batch_info(const fhe_b200_batch* b, uint32_t* count, uint32_t* parts, uint32_t* level,
                        uint32_t* limbs, int* repr);
/* host <-> device copy of ciphertexts [first, first+n); host may be pageable or pinned.  Uploads (and the host_polys
 * of fhe_b200_mul_plain / fhe_b200_add_plain) are only enqueued: a pinned source must stay valid until `stream` has
 * passed the call (a pageable one has been staged by the CUDA runtime when the call returns). */
int fhe_b200_batch_upload(fhe_b200_batch* b, uint32_t first, uint32_t n, const uint64_t* host, void* stream);
int fhe_b200_batch_download(const fhe_b200_batch* b, uint32_t first, uint32_t n, uint64_t* host, void* stream);
/* same as download, but only enqueues the copy on `stream` (host must be pinned for it to be asynchronous);
 * the caller waits with fhe_b200_sync(stream) before reading `host` */
int fhe_b200_batch_download_async(const fhe_b200_batch* b, uint32_t first, uint32_t n, uint64_t* host, void* stream);
/* Ciphertext::clone: dst <- src (same parameters, shape, level; representation is copied) */
int fhe_b200_batch_copy(fhe_b200_batch* dst, const fhe_b200_batch* src, void* stream);
/* dst[dst_first + k] = src[src_first + k*src_stride] for k < n: same parameters, parts, level and representation,
 * dst != src, n > 0, src_stride > 0 (one cudaMemcpy2DAsync).  Splits or gathers the entries of a batch, e.g. the
 * per-index batches of an fhe_b200_expand output. */
int fhe_b200_batch_copy_range(fhe_b200_batch* dst, uint32_t dst_first, const fhe_b200_batch* src,
                              uint32_t src_first, uint32_t src_stride, uint32_t n, void* stream);
/* Page-locked host staging memory for asynchronous uploads / downloads (cudaHostAlloc, portable across devices).
 * write_combined != 0 asks for write-combining pages: faster for the device to read over PCIe and invisible to the
 * CPU caches, slow for the CPU to read -- meant for upload-only buffers the host fills once, front to back. */
int fhe_b200_host_alloc(size_t bytes, int write_combined, void** out);
int fhe_b200_host_free(void* p);
/* raw device pointer of the batch storage (for zero-copy producers such as bench.py). */
int fhe_b200_batch_device_ptr(const fhe_b200_batch* b, uint64_t** dptr, size_t* n_words);

/* ---- keys -----------------------------------------------------------------------------
 * KeySwitchingKey (key_switching_key.rs:22-45): c0, c1 are the NTT-domain values of the
 * n_digits key polynomials at the key level, host layout [digit][limb][coeff];
 * n_digits must equal the limb count of ciphertext_level (:113) -- or, when the key level has a
 * single modulus q, ceil(log_modulus / log_base) with log_modulus = ilog2(next_power_of_two(q)),
 * log_base = log_modulus / 2: the base-2^log_base decomposition variant (:92-110), whose key switch
 * (key_switch_decomposition, :323-362) the library then runs.  Shoup companions (Poly<NttShoup>) are
 * not needed by the device inner product. */
int fhe_b200_ksk_upload(const fhe_b200_params* p, uint32_t ciphertext_level, uint32_t ksk_level,
                        const uint64_t* c0, const uint64_t* c1, uint32_t n_digits, fhe_b200_ksk** out);
int fhe_b200_ksk_free(fhe_b200_ksk* k);
/* the key's words back in the host layout of fhe_b200_ksk_upload: c0, c1 [n_digits][key limbs][N] (NTT); waits for
 * `stream` (a generated key is complete once the stream reaches this call) */
int fhe_b200_ksk_download(const fhe_b200_ksk* k, uint64_t* c0, uint64_t* c1, void* stream);

/* ---- primitives (each parity-tested one by one) --------------------------------------- */
/* Poly::into_ntt / NttOperator::forward[_vt] on every row (rq/mod.rs:535, ntt/native.rs:77,183) */
int fhe_b200_ntt_forward(fhe_b200_batch* b, void* stream);
/* Poly::into_power_basis / NttOperator::backward[_vt] (rq/mod.rs:590, ntt/native.rs:106,197) */
int fhe_b200_ntt_backward(fhe_b200_batch* b, void* stream);
/* Ciphertext += / -= / unary - (bfv/ops/mod.rs:54, :148, :205; rq/ops.rs:92-172, :354-418) */
int fhe_b200_add(fhe_b200_batch* a, const fhe_b200_batch* b, void* stream);
int fhe_b200_sub(fhe_b200_batch* a, const fhe_b200_batch* b, void* stream);
int fhe_b200_neg(fhe_b200_batch* a, void* stream);
/* Ciphertext *= &Plaintext (bfv/ops/mod.rs:229-238; Poly<Ntt> *= &Poly<Ntt>, rq/ops.rs:174): every part of every
 * ciphertext is multiplied coefficient-wise by an NTT-domain polynomial.  host_polys holds n_polys polynomials of
 * [limbs][N] words (Plaintext::poly_ntt, or a monomial of EvaluationKey::expands); n_polys is 1 (shared) or count. */
int fhe_b200_mul_plain(fhe_b200_batch* a, const uint64_t* host_polys, uint32_t n_polys, void* stream);
/* Ciphertext += &Plaintext / -= &Plaintext (bfv/ops/mod.rs:88-97, :188-197): part 0 of every ciphertext gets
 * +/- Plaintext::to_poly() (the delta-scaled NTT polynomial the host computes, plaintext.rs:172-197); host_polys as for
 * fhe_b200_mul_plain. */
int fhe_b200_add_plain(fhe_b200_batch* a, const uint64_t* host_polys, uint32_t n_polys, int subtract, void* stream);
/* dot_product_scalar (bfv/ops/dot_product.rs:55-184): out[g] = sum_{i < n_terms} cts[g*n_terms + i] (.) pts[g*n_terms + i]
 * for g < out.count.  pts is a batch with one NTT polynomial per entry (Plaintext::poly_ntt); either operand may hold
 * n_terms entries only, shared by every group (the PIR loops of examples/mulpir.rs:153-181 share the expanded query
 * across database columns), or out.count * n_terms.  Errors: EmptyInput / OperandCountMismatch -> INVALID_ARGUMENT,
 * CiphertextPolynomialCountMismatch -> BAD_POLY_COUNT, mixed levels -> INVALID_LEVEL. */
int fhe_b200_dot_product_scalar(const fhe_b200_batch* cts, const fhe_b200_batch* pts, uint32_t n_terms,
                                fhe_b200_batch* out, void* stream);

/* ---- plaintexts on the device ---------------------------------------------------------------
 * A device plaintext batch is an fhe_b200_batch with 1 part, in the NTT representation: entry k holds
 * Plaintext::poly_ntt of one plaintext (plaintext.rs:20-27), at the level of its encoding.
 * Encoder handle: psi_t (nullable) is the 2N-th root of unity for t, as `psi` of fhe_b200_params_create
 * (a Rust host passes NttOperator::new(t).omegas[N/2], NULL selects the default rule).  Creation succeeds on every
 * valid parameter set, host-only ones included; when t has no NTT operator (t not prime, or t != 1 mod 2N) SIMD
 * encoding fails with FHE_B200_NTT_UNAVAILABLE (EncodingError::SimdUnavailable) and Poly encoding still works.
 * The handle holds a reference on the parameter set. */
int fhe_b200_encoder_create(const fhe_b200_params* p, const uint64_t* psi_t, fhe_b200_encoder** out);
int fhe_b200_encoder_free(fhe_b200_encoder* e);
/* PlaintextVec::try_encode (plaintext_vec.rs:37-103) of n_values u64 (is_signed == 0) or i64 (is_signed != 0) words
 * into `out`, a 1-part batch of max(1, ceil(n_values / N)) entries at the encoding level; entry k encodes
 * values[k*N, min(n_values, (k+1)*N)) and zero in its other slots; `out` becomes NTT.
 *  - POLY, u64: the words are coefficients, not reduced mod t; each is reduced modulo every q_i (rq/convert.rs:160-183).
 *  - SIMD, u64: slot i holds values[i]; the values must be below t (the reference's NTT assumes reduced input).
 *  - i64 (either encoding): each word is first reduced into [0, t) (Modulus::reduce_vec_i64, plaintext.rs:347-372).
 *  - At a level with a single modulus q_0 the reference keeps the N coefficient words unreduced (rq/convert.rs:150-159)
 *    while the device reduces every word: the results agree for words below q_0 (SIMD words and reduced i64 words are
 *    below t, so they differ only for t > q_0).
 * values: pageable host, pinned host or device memory, copied with cudaMemcpyDefault and only enqueued, as for
 * fhe_b200_batch_upload.  Errors: t beyond a u64 Modulus -> UNSUPPORTED; SIMD without an NTT for t -> NTT_UNAVAILABLE;
 * parts != 1 -> BAD_POLY_COUNT; wrong count, NULL values with n_values > 0 -> INVALID_ARGUMENT; host-only
 * parameters -> NO_DEVICE. */
int fhe_b200_encode(const fhe_b200_encoder* e, int encoding, int is_signed, const void* values, size_t n_values,
                    fhe_b200_batch* out, void* stream);
/* fhe_b200_mul_plain with a device plaintext batch (ops/mod.rs:229-238): pts holds 1 (shared) or a.count entries at
 * a's level.  Same checks and error codes, plus BAD_POLY_COUNT when pts has more than one part. */
int fhe_b200_mul_plain_batch(fhe_b200_batch* a, const fhe_b200_batch* pts, void* stream);
/* fhe_b200_add_plain with a device plaintext batch (ops/mod.rs:88-97, :188-197): Plaintext::to_poly is derived from
 * poly_ntt on the device as the reference does (plaintext.rs:103-135, :172-197).  t >= q_0 -> UNSUPPORTED. */
int fhe_b200_add_plain_batch(fhe_b200_batch* a, const fhe_b200_batch* pts, int subtract, void* stream);

/* ---- decryption, decoding and noise measurement ---------------------------------------------
 * SecretKey (keys/secret_key.rs:25-53) from its N signed coefficients (SecretKey.coeffs, the `coeffs` of the bfv.proto
 * SecretKey message, bfv.proto:54-56; a Rust host reads them from sk.to_bytes(), see INTEGRATION.md).  The key is
 * uploaded once as NTT words modulo every modulus of the parameter set; it also holds, per level, the tables of the
 * cipher -> plaintext scaler (cipher_plain_context.scaler, parameters.rs:638-643) and of the noise measurement.  It
 * holds a reference on the parameter set.  fhe_b200_secret_key_free waits for the device (like every *_free, work
 * still queued with the key may be in flight), then erases the device words of s before releasing them (SecretKey's
 * Zeroize, secret_key.rs:28-40), and scratch holding s-dependent values is zeroed before it goes back
 * to the pool.  The decryption kernels have no branch that depends on the data.  Errors: t beyond a u64 Modulus ->
 * UNSUPPORTED (the large-t branch of try_decrypt is not implemented); host-only parameters -> NO_DEVICE. */
int fhe_b200_secret_key_create(const fhe_b200_params* p, const int64_t* coeffs, fhe_b200_secret_key** out);
int fhe_b200_secret_key_free(fhe_b200_secret_key* sk);
/* SecretKey::try_decrypt (secret_key.rs:198-260) of every ciphertext of `ct` (NTT, any number of parts >= 1): out is
 * a 1-part batch of ct.count entries at ct's level; entry k becomes Plaintext::poly_ntt of the decryption of ct[k]
 * (encoding None), word for word, also when t >= q_0.  The phase c0 + c1 s + c2 s^2 + ... is taken to the power basis,
 * scaled by t / Q into limb 0 of the plaintext context, and w = ((v + t) mod q_0) mod t is lifted and transformed.
 * Errors: ct or out of another parameter set, or over the multiplication basis -> CONTEXT_MISMATCH; power-basis ct ->
 * INVALID_REPRESENTATION; out not 1-part, ct.count entries at ct's level -> INVALID_ARGUMENT. */
int fhe_b200_decrypt(const fhe_b200_secret_key* sk, const fhe_b200_batch* ct, fhe_b200_batch* out, void* stream);
/* Vec<u64>::try_decode (is_signed == 0) / Vec<i64>::try_decode (is_signed != 0) (plaintext.rs:103-135, :155-170,
 * :374-459) of every plaintext of pts, a 1-part NTT batch at any level: values receives pts.count * N words, plaintext
 * k at values[k*N, (k+1)*N).  Signed words are centred as Modulus::center does (a - t when a >= t >> 1, zq/mod.rs:448-457).
 * values: pageable host, pinned host or device memory; the copy is only enqueued (cudaMemcpyDefault), read it after
 * fhe_b200_sync(stream).  The encoding is the caller's (a batch does not record it; resolve_encoding is host work).
 * Errors: t beyond a u64 Modulus, or t >= q_0 (the reference then lifts every limb) -> UNSUPPORTED; SIMD without an
 * NTT for t -> NTT_UNAVAILABLE; parts != 1 -> BAD_POLY_COUNT; power basis -> INVALID_REPRESENTATION; another parameter
 * set -> CONTEXT_MISMATCH; n_values != pts.count * N or NULL values -> INVALID_ARGUMENT; host-only parameters -> NO_DEVICE. */
int fhe_b200_decode(const fhe_b200_encoder* e, int encoding, int is_signed, const fhe_b200_batch* pts, void* values,
                    size_t n_values, void* stream);
/* SecretKey::measure_noise (secret_key.rs:55-98) of every ciphertext of ct: noise_bits[k] = max over the coefficients
 * of min(bits(x), bits(Q - x)), x in [0, Q) the CRT lift of phase - to_poly(decrypt(ct[k])) at ct's level.  Exact
 * for every x.  noise_bits: ct.count words in host or device memory, only enqueued as for fhe_b200_decode.  Variable
 * time, as the reference's (unsafe) function.  Errors: as fhe_b200_decrypt; t >= q_0 -> UNSUPPORTED. */
int fhe_b200_measure_noise(const fhe_b200_secret_key* sk, const fhe_b200_batch* ct, uint32_t* noise_bits, void* stream);

/* ---- encryption ----------------------------------------------------------------------------------
 * The random words come from a seeded ChaCha20 stream that this library defines (the reference draws from rand::rng()
 * and a caller-supplied rng, secret_key.rs:100-136, public_key.rs:45-92, so no host depends on which words are drawn;
 * what it depends on is their distribution and the algebra built on them).  Block b of a row is the RFC 8439 block
 * function (20 rounds) of the state
 *     words 0..3   "expand 32-byte k"
 *     words 4..11  the 32-byte seed as eight little-endian u32
 *     word 12      b, the block index within the row
 *     word 13      the index of the ciphertext within the call (0 .. out.count - 1)
 *     word 14      role << 8 | limb: role 0 = a, 1 = e (secret-key encryption), 2 = u, 3 = e1, 4 = e2 (public-key
 *                  encryption), 5 = c1, 6 = e (key generation, below), 7 - 17 (multiparty BFV, below), 18 = s
 *                  (fhe_b200_secret_keys_random, below, word 13 = the key's index); the small polynomials use limb 0
 *     word 15      0 (encryption, multiparty BFV, secret keys), the digit of the key (key generation)
 * Each block is addressed only by its position, so the words do not depend on chunking or streams.  One 64-byte block
 * gives four 128-bit values: value m is u64 words 2m (low) and 2m + 1 (high) of the block, and coefficient 4b + m of
 * the row takes value m of block b.
 *  - a (uniform, drawn directly as NTT words like Poly::random_from_seed into Ntt): (hi 2^64 + lo) mod q_j.  Its
 *    statistical distance from uniform is below q_j / 2^128 <= 2^-66 per word (the reference samples exactly).
 *  - e, u, e1, e2 (centred binomial, sample_vec_cbd, fhe-util/src/lib.rs:22-67): popc(v & mask_add) - popc(v & mask_sub)
 *    of the 128-bit value v, mask_add the low 2 variance bits and mask_sub the next 2 variance bits.  Same distribution
 *    as the reference for every variance in 1..32 (which reads its bits differently).
 * seed: 32 bytes of fresh entropy per call (a Rust host passes OsRng bytes); reusing a seed repeats a and the errors
 * and breaks security.  variance: BfvParameters::variance, 1..32 (reference default 10).  Both calls write out whole
 * (2-part NTT batch) and are only enqueued.  Scratch holding e, u, e1, e2 or the plaintext is zeroed before it goes
 * back to the pool; the kernels have no branch that depends on the data.
 * Errors: variance outside 1..32 (InvalidVariance), a NULL key, seed or out, out not 2-part, pts not 1-part or with a
 * count other than out.count -> INVALID_ARGUMENT; a batch of another parameter set or over the multiplication basis ->
 * CONTEXT_MISMATCH; pts at another level than out -> INVALID_LEVEL; power-basis pts -> INVALID_REPRESENTATION;
 * t >= q_0 (as fhe_b200_add_plain_batch's to_poly) -> UNSUPPORTED. */
/* SecretKey::try_encrypt (secret_key.rs:100-136, :181-193) into out: b = e - a s + to_poly(m), a.  pts: a 1-part NTT
 * batch from fhe_b200_encode (one plaintext per output ciphertext, at out's level), or NULL to encrypt zeros at out's
 * level (PublicKey::new, public_key.rs:26-38: a 1 x 2 batch at level 0 is then the public key's c). */
int fhe_b200_encrypt_sk(const fhe_b200_secret_key* sk, const fhe_b200_batch* pts, uint32_t variance,
                        const uint8_t* seed, fhe_b200_batch* out, void* stream);
/* PublicKey::try_encrypt (public_key.rs:45-92) into out: (u pk0 + e1 + to_poly(m), u pk1 + e2).  pk: the public key's
 * c as a 1-ciphertext, 2-part, level-0 NTT batch, switched down to out's level on every call as the reference does;
 * pts as for fhe_b200_encrypt_sk.  Extra errors: pk not at level 0 -> INVALID_LEVEL (InvalidPublicKeyLevel); pk not
 * one 2-part ciphertext -> INVALID_ARGUMENT; power-basis pk -> INVALID_REPRESENTATION. */
int fhe_b200_encrypt_pk(const fhe_b200_batch* pk, const fhe_b200_batch* pts, uint32_t variance, const uint8_t* seed,
                        fhe_b200_batch* out, void* stream);
/* SecretKey::random (secret_key.rs:42-45) for n_keys independent keys in one call (one per party of multiparty BFV):
 * key k is s = sample_vec_cbd(N, variance) (fhe-util/src/lib.rs:22-67) drawn from the stream above as role 18, limb 0,
 * word 13 = k, word 15 = 0, by the same 128-bit value -> centred binomial rule as e (the reference's distribution for
 * every variance in 1..32).  The coefficients never pass through host memory: one kernel writes the canonical residue
 * of every coefficient on every modulus (Poly::try_convert_from(&[i64])) and the NTT transforms them, so key k holds
 * exactly the device words fhe_b200_secret_key_create makes from the same coefficients.  Scratch goes back to the pool
 * zeroed, each key is erased when freed, and no kernel branches on the data.  out receives n_keys handles; the call
 * returns once they are ready on every stream.  seed: 32 bytes of fresh entropy (a Rust host passes OsRng bytes);
 * variance: BfvParameters::variance.  Errors: as fhe_b200_secret_key_create (t beyond a u64 Modulus -> UNSUPPORTED;
 * host-only parameters -> NO_DEVICE); variance outside 1..32 (InvalidVariance), a NULL parameter set, seed or out,
 * n_keys == 0 -> INVALID_ARGUMENT.  A failed call returns no handle and frees every key it made. */
int fhe_b200_secret_keys_random(const fhe_b200_params* p, uint32_t n_keys, uint32_t variance, const uint8_t* seed,
                                fhe_b200_secret_key** out, void* stream);
/* SecretKey.coeffs (secret_key.rs:25-30), what SecretKey::to_bytes (:142-148) writes: out (N words of host memory)
 * receives the inverse NTT of the key's limb 0, each word centred modulo q_0 (v - q_0 when v > q_0 / 2).  These are
 * the key's coefficients whenever they lie within (-q_0 / 2, q_0 / 2], as every fhe_b200_secret_keys_random key's
 * do.  The only way a device-born key's coefficients reach the host; the call returns once out is written.  Errors: a
 * NULL key or out -> INVALID_ARGUMENT. */
int fhe_b200_secret_key_coeffs(const fhe_b200_secret_key* sk, int64_t* out, void* stream);

/* ---- key generation ------------------------------------------------------------------------------
 * KeySwitchingKey::new (key_switching_key.rs:71-238) on the device, for every digit i of every key of the call:
 * c1_i uniform at the key level and c0_i = e_i - c1_i s + g_i from, computed in the NTT domain (every value is a
 * canonical residue and the NTT is linear, so the words are those of the reference's power-basis computation).  The
 * words come from the stream above with word 13 = the index k of the key within the call, word 15 = the digit i:
 *  - c1 (role 5, limb j of the key level): (hi 2^64 + lo) mod q_j, drawn directly as NTT words;
 *  - e_i (role 6, limb 0): the centred binomial sample, lifted to every key limb.
 * Key indices: 0 for the relinearization key, the position in `exponents` for Galois keys, 2p (ksk0) and 2p + 1
 * (ksk1) for plaintext p of an RGSW encryption.  The digits: one per ciphertext limb, g_i the Garner coefficient of the
 * ciphertext basis and `from` x switched up to the key level; or, when the key level has a single modulus (then the
 * last level, as fhe_b200_ksk_upload requires), the base-2^log_base decomposition with g_i = 2^(i log_base).  The
 * handles are ordinary keys: fhe_b200_relinearize, fhe_b200_galois, fhe_b200_expand, fhe_b200_key_switch and the
 * multiplicator take them.  Compact (seeded) key messages need the reference's ChaCha8 stream, which this library does
 * not reproduce: fhe_b200_ksk_download gives both rows for an uncompact message.  Scratch holding errors or x is zeroed
 * before it goes back to the pool.  Errors: variance outside 1..32 (InvalidVariance), a NULL argument ->
 * INVALID_ARGUMENT; key_level > ciphertext_level or ciphertext_level above the max level -> INVALID_LEVEL; a
 * decomposition base below 1 -> UNSUPPORTED.  A failed call returns no handle and frees every key it made. */
/* RelinearizationKey::new_leveled (relinearization_key.rs:43-65): x = s s.  A single-modulus key level ->
 * UNSUPPORTED (EvaluationKeyError::KeySwitchingNotSupported). */
int fhe_b200_relin_key_generate(const fhe_b200_secret_key* sk, uint32_t ciphertext_level, uint32_t key_level,
                                uint32_t variance, const uint8_t* seed, fhe_b200_ksk** out, void* stream);
/* GaloisKey::new (galois_key.rs:26-60) for each of n_keys exponents (reduced mod 2N): x = s substituted by the
 * exponent; out receives n_keys handles.  An even exponent -> INVALID_EXPONENT. */
int fhe_b200_galois_keys_generate(const fhe_b200_secret_key* sk, const uint32_t* exponents, uint32_t n_keys,
                                  uint32_t ciphertext_level, uint32_t key_level, uint32_t variance,
                                  const uint8_t* seed, fhe_b200_ksk** out, void* stream);
/* SecretKey::try_encrypt into RGSWCiphertext (rgsw_ciphertext.rs:94-120) of every plaintext of pts (a 1-part NTT
 * batch from fhe_b200_encode) at its level: out receives 2 pts.count handles, ksk0 (x = m) and ksk1 (x = m s) of each
 * plaintext.  pts of another parameter set or over the multiplication basis -> CONTEXT_MISMATCH, not 1-part ->
 * INVALID_ARGUMENT, power basis -> INVALID_REPRESENTATION. */
int fhe_b200_rgsw_encrypt(const fhe_b200_secret_key* sk, const fhe_b200_batch* pts, uint32_t variance,
                          const uint8_t* seed, fhe_b200_ksk** out, void* stream);

/* ---- multiparty BFV (fhe::mbfv, crates/fhe/src/mbfv) ----------------------------------------------
 * WARNING: experimental, incomplete and not audited, as the reference's module.  As there, the errors of every share
 * are the ordinary BfvParameters::variance errors, not smudging noise (the reference's own TODO): a decryption share
 * may leak information about the secret key share.  No noise flooding is added here.
 * A share is an ordinary batch; every call takes whole batches (one share per ciphertext or per CRP) and is only
 * enqueued.  The random words come from the stream above with word 15 = 0 and word 13 = the index within the call
 * (the CRP, or the ciphertext of `ct`):
 *  - role 7: the CRP, (hi 2^64 + lo) mod q_j of limb j's row, drawn directly as NTT words (Poly::<Ntt>::random);
 *  - role 8: e of PublicKeyShare;  role 14: e of SecretKeySwitchShare / DecryptionShare;  roles 15, 16, 17: u, e0, e1
 *    of PublicKeySwitchShare;  role 9: u of RelinKeyGenerator::new;  roles 10, 11: the errors of round 1's h0_i, h1_i and
 *    roles 12, 13 those of round 2's h0'_i, h1'_i, with word 13 = 0 and word 15 = i; all centred binomial samples of
 *    limb 0's row lifted to every limb.
 * Scratch holding errors, u, s-dependent values or the aggregated phase is zeroed before it goes back to the pool; the
 * kernels have no branch that depends on the data.  Aggregation reads every share word once and reduces each output word
 * once.  Errors: variance outside 1..32 (InvalidVariance), a NULL argument, n == 0 (MultipartyError::NoShares), shares
 * whose shape (count, parts, level) differs from the one the call needs, an output of the wrong shape ->
 * INVALID_ARGUMENT; operands of different parameter sets or over the multiplication basis (ParameterMismatch) ->
 * CONTEXT_MISMATCH; ct not 2-part (InvalidPolynomialCount) -> BAD_POLY_COUNT; a crp or public key not at level 0 ->
 * INVALID_LEVEL; power-basis operands -> INVALID_REPRESENTATION.  A refused call allocates nothing. */
/* CommonRandomPoly::new / new_vec / new_leveled (crp.rs:15-43): every entry of `out` (a 1-part batch) becomes one CRP
 * at out's level; new_vec is a batch of n_moduli entries at level 0. */
int fhe_b200_crp_generate(const fhe_b200_params* p, const uint8_t* seed, fhe_b200_batch* out, void* stream);
/* PublicKeyShare::new (public_key_gen.rs:32-58): out entry k = p0 = -crp_k s + e_k at level 0.  crp: a 1-part level-0
 * batch; out: a 1-part level-0 batch of crp.count entries. */
int fhe_b200_pk_share(const fhe_b200_secret_key* sk, const fhe_b200_batch* crp, uint32_t variance, const uint8_t* seed,
                      fhe_b200_batch* out, void* stream);
/* PublicKey::from_shares (public_key_gen.rs:60-77): pk entry k = (sum_i shares[i]_k, crp_k), a 2-part level-0 batch of
 * crp.count entries; an entry is a public key fhe_b200_encrypt_pk takes as it is. */
int fhe_b200_pk_aggregate(const fhe_b200_batch* const* shares, uint32_t n, const fhe_b200_batch* crp,
                          fhe_b200_batch* pk, void* stream);
/* out = sum of the n shares, word by word, for shares of out's shape (the sum inside every aggregation, and
 * RelinKeyShare<R1Aggregated>::from_shares, relin_key_gen.rs:200-222, for h0 and h1 each).  out may be any of the
 * shares.  Shares are summed in launches of 64: each output word is reduced once per launch. */
int fhe_b200_shares_sum(const fhe_b200_batch* const* shares, uint32_t n, fhe_b200_batch* out, void* stream);
/* SecretKeySwitchShare::new (secret_key_switch.rs:38-96) of every ciphertext of ct (2-part): out entry k =
 * h = (s_in - s_out) c1_k + e_k at ct's level, a 1-part batch of ct.count entries.  sk_out NULL is the zero key of
 * DecryptionShare::new (:133-143). */
int fhe_b200_sks_share(const fhe_b200_secret_key* sk_in, const fhe_b200_secret_key* sk_out, const fhe_b200_batch* ct,
                       uint32_t variance, const uint8_t* seed, fhe_b200_batch* out, void* stream);
/* Ciphertext::from_shares of SecretKeySwitchShares (secret_key_switch.rs:98-115): out = (c0 + sum h_i, c1), a 2-part
 * batch of ct's shape (out may be ct). */
int fhe_b200_sks_aggregate(const fhe_b200_batch* ct, const fhe_b200_batch* const* shares, uint32_t n,
                           fhe_b200_batch* out, void* stream);
/* PublicKeySwitchShare::new (public_key_switch.rs:33-93) of every ciphertext of ct: out entry k = (u pk0 + s c1_k + e0,
 * u pk1 + e1), pk (a level-0 public key, as for fhe_b200_encrypt_pk) switched down to ct's level; out has ct's shape. */
int fhe_b200_pks_share(const fhe_b200_secret_key* sk, const fhe_b200_batch* pk, const fhe_b200_batch* ct,
                       uint32_t variance, const uint8_t* seed, fhe_b200_batch* out, void* stream);
/* Ciphertext::from_shares of PublicKeySwitchShares (public_key_switch.rs:95-112): out = (c0 + sum h0_i, sum h1_i). */
int fhe_b200_pks_aggregate(const fhe_b200_batch* ct, const fhe_b200_batch* const* shares, uint32_t n,
                           fhe_b200_batch* out, void* stream);
/* RelinKeyGenerator::new (relin_key_gen.rs:76-96): u (role 9) is drawn and kept on the device in *out; the generator
 * also refers to sk and to crp, a 1-part level-0 batch of the n_moduli CRPs of CommonRandomPoly::new_vec, which must
 * outlive it (the reference borrows both).  fhe_b200_rkg_free waits for the device, erases u and releases it.
 * Errors: a single modulus -> UNSUPPORTED (KeySwitchingNotSupported); crp.count != n_moduli ->
 * INVALID_ARGUMENT (InvalidCommonRandomPolynomialCount); crp not at level 0 -> INVALID_LEVEL. */
int fhe_b200_rkg_create(const fhe_b200_secret_key* sk, const fhe_b200_batch* crp, uint32_t variance,
                        const uint8_t* seed, fhe_b200_rkg** out, void* stream);
int fhe_b200_rkg_free(fhe_b200_rkg* r);
/* RelinKeyGenerator::round_1 (relin_key_gen.rs:112-198): entry i of h0 / h1 (1-part level-0 batches of n_moduli
 * entries) = -a_i u + w_i s + e, a_i s + e; w_i is the Garner coefficient of the level-0 basis (s on limb i, 0 on the
 * others).  Aggregate the parties' h0 and h1 with fhe_b200_shares_sum (RelinKeyShare<R1Aggregated>). */
int fhe_b200_rkg_round1(const fhe_b200_rkg* r, const uint8_t* seed, fhe_b200_batch* h0, fhe_b200_batch* h1,
                        void* stream);
/* RelinKeyGenerator::round_2 (relin_key_gen.rs:224-297) from the round-1 aggregate (r1_h0, r1_h1): entry i of h0 / h1
 * = r1_h0_i s + e, r1_h1_i (u - s) + e. */
int fhe_b200_rkg_round2(const fhe_b200_rkg* r, const fhe_b200_batch* r1_h0, const fhe_b200_batch* r1_h1,
                        const uint8_t* seed, fhe_b200_batch* h0, fhe_b200_batch* h1, void* stream);
/* RelinearizationKey::from_shares (relin_key_gen.rs:299-350) of the n parties' round-2 shares (h0s[k], h1s[k]) and the
 * round-1 aggregate's r1_h1: *out = a new level-0 RNS-digit key with c0_i = sum h0'_i + sum h1'_i, c1_i = r1_h1_i,
 * written straight into the key's device layout.  It is an ordinary key for fhe_b200_relinearize, fhe_b200_mul_relin
 * and the multiplicator, released with fhe_b200_ksk_free. */
int fhe_b200_rkg_aggregate(const fhe_b200_batch* const* h0s, const fhe_b200_batch* const* h1s, uint32_t n,
                           const fhe_b200_batch* r1_h1, fhe_b200_ksk** out, void* stream);
/* Plaintext::from_shares of DecryptionShares (secret_key_switch.rs:145-186): c = c0 + sum h_i to the power basis, scaled
 * by t / Q (cipher_plain_context.scaler), w = ((v + t) mod Q_p) mod t with Q_p the product of the plaintext-context
 * moduli (the first moduli whose sizes add up to bits(t) + 60, parameters.rs:579-595), lifted and transformed into
 * pts_out (a 1-part batch of ct.count entries at ct's level, encoding None).  The scaled value v is the rounding of
 * t x / Q for the centred lift x of the phase, |v| <= t / 2, and from_shares gives v mod t.  fhe_b200_decrypt lifts
 * ((v + t) mod q_0) mod t instead; the two differ when the plaintext context has two or more moduli, q_0 / 2 < t < q_0
 * and v >= q_0 - t.  The aggregator holds no secret key: the scaler tables of each level live on the encoder `e`, built
 * on first use.  t >= q_0 or t beyond a u64 Modulus -> UNSUPPORTED. */
int fhe_b200_decryption_aggregate(const fhe_b200_encoder* e, const fhe_b200_batch* ct,
                                  const fhe_b200_batch* const* shares, uint32_t n, fhe_b200_batch* pts_out,
                                  void* stream);

/* &Ciphertext * &Ciphertext (bfv/ops/mod.rs:259-358): n parts x m parts -> n + m - 1 parts (out3 must have that many;
 * 2 x 2 -> 3 is the fused path) */
int fhe_b200_mul(const fhe_b200_batch* a, const fhe_b200_batch* b, fhe_b200_batch* out3, void* stream);
/* RelinearizationKey::relinearizes: (c0,c1,c2) -> (c0,c1) (keys/relinearization_key.rs:70-103) */
int fhe_b200_relinearize(const fhe_b200_batch* ct3, const fhe_b200_ksk* rk, fhe_b200_batch* out2, void* stream);
/* Multiplicator::default(rk).multiply (bfv/ops/mul.rs:101-138, :165-243); mod_switch != 0
 * additionally applies Ciphertext::switch_down (mul.rs:238) and out2 must be at level+1. */
int fhe_b200_mul_relin(const fhe_b200_batch* a, const fhe_b200_batch* b, const fhe_b200_ksk* rk,
                       int mod_switch, fhe_b200_batch* out2, void* stream);
/* Multiplicator::new / new_leveled (bfv/ops/mul.rs:37-98): custom strategy.  Each ScalingFactor (rns/scaler.rs:20-58)
 * is a numerator / denominator pair of little-endian byte strings (BigUint::to_bytes_le).  extended_basis are the
 * n_basis moduli of the multiplication context (Context::new(extended_basis), mul.rs:82); psi (nullable) gives the
 * 2N-th root per basis prime (default rule of fhe_b200_params_create otherwise; primes shared with the parameter set
 * reuse its tables).  As in rq/scaler.rs:35-43 an extender keeps the common prefix of the two bases only when its
 * factor is one.  Errors: InvalidLevel, DuplicateModuli / InvalidModulus, NTT_UNAVAILABLE. */
int fhe_b200_multiplicator_create(const fhe_b200_params* p, uint32_t level, const uint8_t* lhs_num, uint32_t lhs_num_len,
                                  const uint8_t* lhs_den, uint32_t lhs_den_len, const uint8_t* rhs_num,
                                  uint32_t rhs_num_len, const uint8_t* rhs_den, uint32_t rhs_den_len,
                                  const uint64_t* extended_basis, uint32_t n_basis, const uint64_t* psi,
                                  const uint8_t* post_num, uint32_t post_num_len, const uint8_t* post_den,
                                  uint32_t post_den_len, fhe_b200_multiplicator** out);
int fhe_b200_multiplicator_free(fhe_b200_multiplicator* m);
/* Multiplicator::multiply (mul.rs:165-243) with that strategy.  rk == NULL: no relinearization, out has 3 parts;
 * otherwise enable_relinearization(rk) semantics (mul.rs:141-151: the key must be for the multiplicator's level,
 * ParameterMismatch if not) and out has 2 parts.  mod_switch != 0: enable_mod_switching (mul.rs:155-162,
 * NoMoreContext at the last level), out must be at level+1. */
int fhe_b200_multiplicator_multiply(const fhe_b200_multiplicator* m, const fhe_b200_batch* a, const fhe_b200_batch* b,
                                    const fhe_b200_ksk* rk, int mod_switch, fhe_b200_batch* out, void* stream);
/* GaloisKey::relinearize (keys/galois_key.rs:63-86) for substitution exponent `exponent`
 * (column rotation by i <-> 3^i mod 2N, row swap <-> 2N-1; evaluation_key.rs:118, :278-286) */
int fhe_b200_galois(const fhe_b200_batch* ct, uint32_t exponent, const fhe_b200_ksk* gk,
                    fhe_b200_batch* out, void* stream);
/* EvaluationKey::expands (keys/evaluation_key.rs:192-256) of each of the Q = ct.count ciphertexts of `ct`
 * (oblivious expansion, eprint 2019/1483).  out: size*Q ciphertexts, 2 parts, ct's level; entry i*Q + q is expansion
 * output i of query q (for Q = 1 the reference's Vec order); out becomes NTT.  gks[l], l < ceil(log2 size), is the
 * key-switching key of the GaloisKey for element (N >> l) + 1, for ct's level (its key level may be lower, as with
 * EvaluationKeyBuilder::new_leveled); the caller vouches for the element, as for fhe_b200_galois.  The monomials
 * -x^(N - 2^l) (:465-474) are fixed by the parameters and built by the library.  Each level is one batched Galois call
 * over all step*Q inputs and one butterfly kernel; size == 1 is a copy.  Errors: size == 0 or size > N, n_gks too small,
 * a NULL key -> INVALID_ARGUMENT; a key for another level or parameter set -> as fhe_b200_galois; ct.parts != 2 ->
 * BAD_POLY_COUNT; power basis -> INVALID_REPRESENTATION; wrong out shape or out aliasing ct -> INVALID_ARGUMENT. */
int fhe_b200_expand(const fhe_b200_batch* ct, uint32_t size, const fhe_b200_ksk* const* gks, uint32_t n_gks,
                    fhe_b200_batch* out, void* stream);
/* Poly::substitute on every row of a batch: the slot permutation of an NTT batch (rq/mod.rs:360-389) or the signed
 * coefficient permutation x^j -> x^(j*exponent) of a power-basis batch (rq/mod.rs:390-408); `out` takes `in`'s
 * representation.  Even exponents: FHE_B200_INVALID_EXPONENT. */
int fhe_b200_substitute(const fhe_b200_batch* in, uint32_t exponent, fhe_b200_batch* out, void* stream);
/* Ciphertext::switch_down: drop the last modulus with rounding (ciphertext.rs:148-161, rq/mod.rs:433-492).
 * Stream-ordered and in place: the batch keeps its allocation (fhe_b200_batch_device_ptr stays valid, the words of the
 * lower level are compacted at its start), nothing is allocated or synchronised. */
int fhe_b200_switch_down(fhe_b200_batch* b, void* stream);
/* KeySwitchingKey::key_switch on part `part` of a POWER_BASIS batch (key_switching_key.rs:241-270):
 * out (2 parts, NTT, ksk level) = (sum_i NTT(d_i) * c0_i, sum_i NTT(d_i) * c1_i) */
int fhe_b200_key_switch(const fhe_b200_batch* pb, uint32_t part, const fhe_b200_ksk* k,
                        fhe_b200_batch* out2, void* stream);
/* ---- per-ciphertext keys ----------------------------------------------------------------------------
 * A server that answers many clients holds one relinearization, Galois or expansion key per client.  The _keyed
 * calls below take a list of key handles and, in key_index (host memory, read during the call only), one u32 per
 * ciphertext of the batch naming its key: entry j of the output is, word for word, what the single-key call gives on
 * entry j alone with keys[key_index[j]].  An index may repeat, a key may go unused and a handle may be listed more
 * than once.
 * What stays shared by the whole batch: the levels, the Galois exponent, the expansion size and mod_switch.  Each
 * key is checked as the single-key call checks it, and all keys of one call (for expand: of one expansion level) must
 * have the same key level, digit count and base.  INVALID_ARGUMENT: a NULL key list, key or index, n_keys == 0, an
 * index >= n_keys, keys that differ in key level, digit count or base; every other error is the single-key call's.
 * Every check runs before anything is enqueued: a refused call writes nothing and keeps no device memory.  Streams
 * and chunks behave as in the single-key calls.  The digit transforms of a key switch do not depend on the key; its
 * inner product stages each run of ciphertexts with the same key once, and a chunk with more than 64 distinct keys
 * takes one inner-product launch per range of at most 64.  With one key the calls launch exactly the single-key
 * calls' kernels. */
/* fhe_b200_key_switch of entry j with keys[key_index[j]] */
int fhe_b200_key_switch_keyed(const fhe_b200_batch* pb, uint32_t part, const fhe_b200_ksk* const* keys,
                              uint32_t n_keys, const uint32_t* key_index, fhe_b200_batch* out2, void* stream);
/* fhe_b200_relinearize of entry j with rks[key_index[j]] */
int fhe_b200_relinearize_keyed(const fhe_b200_batch* ct3, const fhe_b200_ksk* const* rks, uint32_t n_keys,
                               const uint32_t* key_index, fhe_b200_batch* out2, void* stream);
/* fhe_b200_mul_relin of entry j with rks[key_index[j]] (Multiplicator::default of each key) */
int fhe_b200_mul_relin_keyed(const fhe_b200_batch* a, const fhe_b200_batch* b, const fhe_b200_ksk* const* rks,
                             uint32_t n_keys, const uint32_t* key_index, int mod_switch, fhe_b200_batch* out2,
                             void* stream);
/* fhe_b200_galois of entry j with gks[key_index[j]]; the exponent is shared, so every key must be for it (the caller
 * vouches for that, as for fhe_b200_galois) */
int fhe_b200_galois_keyed(const fhe_b200_batch* ct, uint32_t exponent, const fhe_b200_ksk* const* gks,
                          uint32_t n_keys, const uint32_t* key_index, fhe_b200_batch* out, void* stream);
/* fhe_b200_expand of every query with its own key set: gks[s * n_gks + l] is the key of expansion level l of key set
 * s, set_index[q] (one per query, Q = ct.count) the key set of query q.  Entry i*Q + q of out is output i of query q
 * expanded with key set set_index[q].  n_gks below the expansion level, n_sets == 0 or a NULL set_index ->
 * INVALID_ARGUMENT. */
int fhe_b200_expand_keyed(const fhe_b200_batch* ct, uint32_t size, const fhe_b200_ksk* const* gks, uint32_t n_gks,
                          uint32_t n_sets, const uint32_t* set_index, fhe_b200_batch* out, void* stream);
/* ---- per-ciphertext Galois exponents --------------------------------------------------------------------
 * Many rotations in one call: of one ciphertext by many steps, or of many ciphertexts by their own steps.  gks[k] is
 * the Galois key for exponents[k] (the caller vouches that they match, as for fhe_b200_galois); entry j of out is, word
 * for word, fhe_b200_galois(ct[src_j], exponents[key_index[j]], gks[key_index[j]]) with src_j = source[j], or j when
 * source is NULL (then ct.count must equal out.count).  source and key_index are host memory with out.count entries,
 * read during the call only.  Each exponent is reduced mod 2N; an even one -> INVALID_EXPONENT.  INVALID_ARGUMENT: a
 * NULL key list, key, exponent list or index, n_keys == 0, key_index[j] >= n_keys, source[j] >= ct.count, out aliasing
 * ct, keys that differ in key level, digit count or base.  Every other error is fhe_b200_galois's, and every check runs
 * before anything is enqueued.  The substitution reads each output's exponent and source from its kernel parameters: no
 * table is built, nothing is allocated beyond the stream-ordered scratch and nothing is synchronised. */
int fhe_b200_galois_many(const fhe_b200_batch* ct, const uint32_t* source, const fhe_b200_ksk* const* gks,
                         const uint32_t* exponents, uint32_t n_keys, const uint32_t* key_index, fhe_b200_batch* out,
                         void* stream);
/* fhe_b200_galois_many with hoisting: the same arguments, checks and error codes, and entry j of out is word for word
 * entry j of fhe_b200_galois_many.  The outputs of a source ciphertext that has two or more outputs share one digit
 * decomposition of its c1: its L x Lk digit transforms (rq/mod.rs:563-586) run once, and each output's key switch
 * (key_switching_key.rs:241-270, galois_key.rs:63-86) reads them through the NTT-domain permutation of its exponent
 * (rq/mod.rs:360-389).  The reference's digits of sigma(c1) differ from sigma applied to the digits of c1 by q_k at the
 * coefficients the substitution negates (rq/mod.rs:390-408); the kernel adds that difference back, which is exact
 * except where such a coefficient's residue is zero.  The outputs whose exponent negates a position s >= 1 at which
 * some residue of their source's c1 is zero, the outputs of sources with one output, and every output of a call whose
 * keys have a base-2^b decomposition (log_base != 0) take fhe_b200_galois_many's path.
 * n_hoisted (host memory, nullable) receives how many outputs were computed from shared digits.
 * Synchronisation: when any output is a candidate for hoisting, the call synchronises `stream` once, after the zero
 * check and before the first output is computed, to read the check on the host.  A call that hoists nothing (every
 * source used once, or base-2^b keys) does not synchronise.
 * Scratch: stream-ordered, per hoisted source of a chunk L x Lk x N words of digits plus L x N of its power-basis c1
 * (51 MB at N = 2^15 with 14 moduli), and per distinct exponent of a chunk Lk x N words; a chunk holds at most
 * FHE_B200_CHUNK outputs.  Nothing outlives the call. */
int fhe_b200_galois_many_hoisted(const fhe_b200_batch* ct, const uint32_t* source, const fhe_b200_ksk* const* gks,
                                 const uint32_t* exponents, uint32_t n_keys, const uint32_t* key_index,
                                 fhe_b200_batch* out, uint32_t* n_hoisted, void* stream);
/* Plaintext-matrix x ciphertext-vector products by baby-step/giant-step diagonals, for every ciphertext c of ct:
 *   out[c] = sum_{g < G} rot_{g b}( sum_{i < b, g b + i < n_diags} diags[g b + i] (.) B_i(ct[c]) ),  G = ceil(n_diags / b),
 * with B_0 the identity (no key switch) and B_i = rot_i, rot_k = EvaluationKey::rotates_columns_by(k) (exponent
 * 3^k mod 2N, keys/evaluation_key.rs:145-170).  The words are those of that composition of galois, mul_plain_batch and
 * add calls.  ct: 2-part NTT batch; diags: 1-part NTT batch at ct's level (fhe_b200_encode) holding n_diags entries
 * shared by every ciphertext, or ct.count * n_diags (entry c * n_diags + k is diagonal k of ciphertext c), already
 * rotated for the giant steps; out: ct's shape, must not alias ct or diags, becomes NTT.  gks / exponents / n_keys: a
 * key list as fhe_b200_galois_many takes it (one level, digit count and base); the call uses the keys of the steps
 * 1 .. b - 1 and b, 2b, .., (G - 1) b and ignores the others.
 * Keys at the ciphertext level with RNS digits run one hoisted digit decomposition per ciphertext and one kernel that
 * multiplies each baby step's key switch by its diagonals and sums them, without writing the rotations; a baby-step
 * term whose ciphertext fails the zero check of fhe_b200_galois_many_hoisted is rotated unhoisted instead.  Leveled
 * keys and base-2^b keys run the composition itself.  n_fallback (host memory, nullable) receives how many
 * (ciphertext, baby step >= 1) rotations were computed unhoisted: the zero-check failures, or count * (b - 1) for
 * leveled and base-2^b keys.
 * Errors: a step without a key, baby = 0, baby > n_diags, n_diags = 0 or > N/2, a diags count other than n_diags or
 * ct.count * n_diags, an output of another shape, aliasing, a null key -> INVALID_ARGUMENT (a transform with
 * n_diags = 1 needs no key and takes n_keys = 0); ct, diags,
 * out or a key at different levels -> INVALID_LEVEL; power-basis operands -> INVALID_REPRESENTATION; even exponents
 * -> INVALID_EXPONENT.  A refused call enqueues nothing.
 * Synchronisation: with b >= 2 and keys at the ciphertext level without base-2^b digits, the call synchronises
 * `stream` once, after the zero check, to read it on the host.
 * Scratch: stream-ordered and released by the call; per chunk of ciphertexts their digits (L x L x N words each) and
 * two buffers of partial sums, and b x L x N words of correction rows per call. */
int fhe_b200_linear_transform(const fhe_b200_batch* ct, const fhe_b200_batch* diags, uint32_t n_diags, uint32_t baby,
                              const fhe_b200_ksk* const* gks, const uint32_t* exponents, uint32_t n_keys,
                              fhe_b200_batch* out, uint32_t* n_fallback, void* stream);
/* EvaluationKey::computes_inner_sum (keys/evaluation_key.rs:56-100) of every ciphertext of ct into out (same shape,
 * must not alias ct; ct is left unchanged; out becomes NTT).  gks holds n_gks = log2 N keys: the Galois keys of the
 * column rotations by 1, 2, 4, ..., N/4 (exponents 3^i mod 2N), then of the row rotation (2N - 1); any other n_gks or a
 * NULL key -> INVALID_ARGUMENT.  Levels and leveled keys as in fhe_b200_galois.  Each step is one substitution kernel
 * that also forms sigma(c0) + c0 and one key switch that adds in place: no separate add launch, no host
 * synchronisation between steps. */
int fhe_b200_inner_sum(const fhe_b200_batch* ct, const fhe_b200_ksk* const* gks, uint32_t n_gks, fhe_b200_batch* out,
                       void* stream);
/* fhe_b200_inner_sum of every ciphertext with its own key set: gks[s * n_gks + l] is the key of step l of key set s
 * and set_index[c] the key set of ciphertext c (host memory, ct.count entries).  The keys of one step must share their
 * key level, digit count and base.  n_sets == 0, a NULL set_index or set_index[c] >= n_sets -> INVALID_ARGUMENT. */
int fhe_b200_inner_sum_keyed(const fhe_b200_batch* ct, const fhe_b200_ksk* const* gks, uint32_t n_gks, uint32_t n_sets,
                             const uint32_t* set_index, fhe_b200_batch* out, void* stream);
/* ---- sums over many ciphertexts --------------------------------------------------------------------------
 * A run is n_terms consecutive entries: run g of a batch is entries g*n_terms .. g*n_terms + n_terms - 1, and an output
 * batch of out.count entries takes one run each.  Every check runs before anything is enqueued. */
/* Ciphertext += &Ciphertext (bfv/ops/mod.rs:54-69) folded over each run, from Ciphertext::zero (accumulate == 0) or
 * from out's own entries: out[g] = (accumulate ? out[g] : 0) + sum_{i < n_terms} in[g*n_terms + i], for g < out.count.
 * Any part count, either representation, and batches over the multiplication basis; out takes in's representation.
 * Errors: in.count != out.count * n_terms, n_terms == 0, a NULL argument or out == in -> INVALID_ARGUMENT; parts that
 * differ -> BAD_POLY_COUNT; levels that differ -> INVALID_LEVEL; another parameter set, or one batch over the
 * multiplication basis and the other not -> CONTEXT_MISMATCH; accumulate into an out of the other representation ->
 * INVALID_REPRESENTATION.  One kernel: each output word is accumulated in 128 bits and reduced once, so n_terms may
 * reach 2^32 - 1.  The voting tally of examples/voting.rs:142-147 is one call with n_terms = the number of ballots. */
int fhe_b200_batch_sum(const fhe_b200_batch* in, uint32_t n_terms, int accumulate, fhe_b200_batch* out, void* stream);
/* The dot product of two ciphertext vectors, one relinearization per run (examples/mulpir.rs:176-183):
 *   out[g] = switch_to_level(out.level, relinearizes(sum_{i < n_terms} a[g*n_terms + i] * b[g*n_terms + i]))
 * Each term is &Ciphertext * &Ciphertext (bfv/ops/mod.rs:259-358) of two 2-part NTT ciphertexts, the sum is AddAssign
 * (ops/mod.rs:54-69) from Ciphertext::zero.  rk == NULL: no relinearization, out is 3-part; otherwise out is 2-part,
 * RelinearizationKey::relinearizes (relinearization_key.rs:70-103), with keys at another key level as in
 * fhe_b200_relinearize.  out.level > a.level applies Ciphertext::switch_to_level (ciphertext.rs:164-186) to the result.
 * Either operand may hold n_terms entries only, shared by every group, or out.count * n_terms (the rule of
 * fhe_b200_dot_product_scalar).  The words equal the reference's loop of mul, +=, relinearizes and switch_to_level.
 * Errors: operand parts other than 2 x 2, or out parts other than 3 (no key) / 2 -> BAD_POLY_COUNT; counts that fit
 * neither rule, n_terms == 0, a NULL argument, out aliasing an operand -> INVALID_ARGUMENT; operands at different
 * levels, out.level below a.level -> INVALID_LEVEL; POWER_BASIS operands -> INVALID_REPRESENTATION; another parameter
 * set or a multiplication-basis batch -> CONTEXT_MISMATCH; the key as fhe_b200_relinearize checks it.
 * The products are summed before their forward NTT (linear on canonical residues), so each group transforms 2 parts
 * (with a key) or 3 instead of 3 per term, and c2 goes from the power basis straight into the key switch. */
int fhe_b200_dot_product(const fhe_b200_batch* a, const fhe_b200_batch* b, uint32_t n_terms, const fhe_b200_ksk* rk,
                         fhe_b200_batch* out, void* stream);
/* fhe_b200_dot_product with group g relinearized by rks[key_index[g]]: many clients' MulPIR responses in one call.
 * key_index holds one u32 per group (out.count entries, host memory), not per term; the key rules and errors are those
 * of the other _keyed calls above. */
int fhe_b200_dot_product_keyed(const fhe_b200_batch* a, const fhe_b200_batch* b, uint32_t n_terms,
                               const fhe_b200_ksk* const* rks, uint32_t n_keys, const uint32_t* key_index,
                               fhe_b200_batch* out, void* stream);
/* rq::scaler::Scaler::scale with the level's multiplication scalers (rq/scaler.rs:55-127):
 * which = 0: extender (level basis -> multiplication basis, factor 1),
 * which = 1: down scaler (multiplication basis -> level basis, factor t/Q).
 * `in` is an NTT batch whose limb count equals the source basis; out gets the target basis. */
int fhe_b200_scale(const fhe_b200_batch* in, int which, fhe_b200_batch* out, void* stream);
/* batch over the multiplication basis of `level` (limbs = L + E), for fhe_b200_scale */
int fhe_b200_batch_alloc_mul_basis(const fhe_b200_params* p, uint32_t count, uint32_t parts, uint32_t level,
                                   int repr, fhe_b200_batch** out);

/* ---- wire format of polynomials (SURVEY section 8f row 1) -------------------------------------------
 * `Rq.coefficients` of the reference's protobuf message (fhe-math/src/proto/rq.proto:12-17) is, for every limb
 * in order, the power-basis coefficients bit-packed LSB first with ceil(log2 q_i) bits each
 * (Modulus::serialize_vec zq/mod.rs:783-786, fhe_util::transcode_to_bytes fhe-util/src/lib.rs:71-108).
 * The protobuf framing itself (tags, varints, `representation`, `degree`) is host work: a Rust host keeps its prost
 * code; C++ and Python hosts have the same messages in include/fhe_b200_wire.hpp / fhe_rs_b200/wire.py. */
/* Seeded ("compact") ciphertexts and keys are NOT expanded here.  The reference serialises a fresh ciphertext as c0 plus
 * the 32-byte seed of c1 (bfv/ciphertext.rs:231-317; keys: key_switching_key.rs:365-482) and regenerates c1 with
 * Poly::random_from_seed (rq/mod.rs:276-292): ChaCha8Rng::from_seed(seed) driving rand's uniform u64 sampling per
 * limb.  That stream is defined by rand 0.10.2 / rand_chacha 0.10.0, which are not vendored in the reference tree
 * and cannot be run or pinned in this build environment, so a device-side expansion could not be proven identical.
 * The Rust host therefore expands c1 with the reference's own code (ciphertext.rs:287-300) and uploads both halves
 * as words (fhe_b200_batch_upload) or as Rq blobs (fhe_b200_batch_unpack); the device never guesses the RNG. */
/* Modulus::serialization_length summed over the limbs of `level` (rq/convert.rs:78-82): bytes per polynomial */
int fhe_b200_poly_packed_bytes(const fhe_b200_params* p, uint32_t level, size_t* nbytes);
/* the same for the polynomials of one batch -- use this one to size the host buffers of pack / unpack: a batch over
 * the multiplication basis (fhe_b200_batch_alloc_mul_basis) has L + E limbs, not the level's L */
int fhe_b200_batch_packed_bytes(const fhe_b200_batch* b, size_t* nbytes);
/* From<&Poly<R>> for Rq (rq/convert.rs:17-44): polynomials of ciphertexts [first, first+n) -> power basis
 * (if the batch is NTT) -> packed bytes; host_out receives n*parts blobs of packed_bytes each. */
int fhe_b200_batch_pack(const fhe_b200_batch* b, uint32_t first, uint32_t n, uint8_t* host_out, void* stream);
/* TryConvertFrom<&Rq> for Poly<PowerBasis|Ntt> (rq/convert.rs:100-131): unpack n*parts blobs into ciphertexts
 * [first, first+n) of `b`; when `b` is an NTT batch the rows are forward-transformed afterwards (as
 * `p.into_ntt()` does).  The whole batch must be filled with one call per disjoint range before it is used. */
int fhe_b200_batch_unpack(fhe_b200_batch* b, uint32_t first, uint32_t n, const uint8_t* host_in, void* stream);

/* ---- bit transcoding and the SealPIR reply fold ---------------------------------------------
 * fhe_util::transcode_bidirectional, transcode_to_bytes and transcode_from_bytes (fhe-util/src/lib.rs:68-187) over
 * n_rows independent rows in one call, on the device of `p`.  Row r of `in` is in_len elements starting r * in_stride
 * elements from `in`; an element is a u64 word (in_elem = 8), masked to in_bits as the reference's release build does,
 * or a byte (in_elem = 1, in_bits = 8).  Value k of output row r is bits [k*out_bits, (k+1)*out_bits) of the row's
 * LSB-first bit stream for k < ceil(in_len * in_bits / out_bits), the last one holding the leftover bits, exactly as
 * the reference's loop; row r receives its first out_len values, zeros after them (the truncation of
 * examples/sealpir.rs:249-252, the zero padding of examples/util.rs:97-145), at out + r * out_stride elements, as u64
 * words (out_elem = 8) or bytes (out_elem = 1, out_bits = 8: transcode_to_bytes).  in_len = 0 is valid (an empty
 * stream, lib.rs:364-371).  `in` and `out` may be pageable host, pinned host or device memory; the call is only
 * enqueued, read `out` after fhe_b200_sync(stream).  Errors: bits outside 1..64, an element size other than 1 or 8, a
 * byte element with bits != 8, n_rows == 0, a stride shorter than its length, NULL with a non-zero length, or
 * overlapping `in` and `out` ranges -> INVALID_ARGUMENT; host-only parameters -> NO_DEVICE. */
int fhe_b200_transcode(const fhe_b200_params* p, const void* in, uint32_t in_elem, size_t in_len, size_t in_stride,
                       uint32_t in_bits, void* out, uint32_t out_elem, size_t out_len, size_t out_stride,
                       uint32_t out_bits, uint32_t n_rows, void* stream);
/* The reply fold of the SealPIR server (examples/sealpir.rs:176-200) for every ciphertext j of `ct` in one call: the
 * stored words of each part ([limb][N], whatever the representation, as Poly::coefficients returns them) are
 * transcoded from in_bits to out_bits, E = ceil(L * N * in_bits / out_bits) values per part; the values of the parts,
 * concatenated, are encoded as PlaintextVec::try_encode(values, Encoding::poly_at_level(out.level)) with the words of
 * fhe_b200_encode (POLY, u64): P = ceil(parts * E / N) plaintexts per ciphertext.  Plaintext i of ciphertext j is entry
 * i * ct.count + j of `out`, a 1-part batch of P * ct.count entries that becomes NTT: fhe_b200_dot_product_scalar of
 * the dim2 selectors (shared) with `out` and n_terms = ct.count gives all P response ciphertexts in one call.
 * Errors: operands of different parameter sets or over the multiplication basis -> CONTEXT_MISMATCH; `out` not 1-part
 * -> BAD_POLY_COUNT; a wrong `out` count, bits outside 1..64 or `out` == `ct` -> INVALID_ARGUMENT. */
int fhe_b200_fold(const fhe_b200_batch* ct, uint32_t in_bits, uint32_t out_bits, fhe_b200_batch* out, void* stream);

int fhe_b200_sync(void* stream);
/* kernels launched by this library in the calling process so far (bench.py "gpu_launches") */
uint64_t fhe_b200_launch_count(void);
/* polynomial rows (one limb of one polynomial) transformed by the batched NTT so far in the calling process:
 * inverse == 0 forward, otherwise inverse.  Transforms fused into other kernels (the tensor product, the key switch
 * digits) are not counted. */
uint64_t fhe_b200_ntt_row_count(int inverse);

/* ---- inspection of the host precompute (CPU-only tests of the parameter builder) -------
 * RnsScaler tables (rns/scaler.rs:52-73) of the level's extender (which=0), down scaler
 * (which=1) or decryption scaler t / Q_l into the plaintext context (which=2, parameters.rs:638-643;
 * its n_to is the plaintext context's modulus count).  Any output pointer may be NULL.
 * omega is [n_to][n_from]. */
int fhe_b200_debug_scaler_tables(const fhe_b200_params* p, uint32_t level, int which, uint32_t* n_from,
                                 uint32_t* n_to, uint32_t* shift, uint64_t* gamma, uint64_t* omega,
                                 uint64_t* theta_gamma /* lo,hi,sign */, uint64_t* theta_omega_lo,
                                 uint64_t* theta_omega_hi, uint8_t* theta_omega_sign,
                                 uint64_t* theta_garner_lo, uint64_t* theta_garner_hi);
/* NTT tables of prime q: any of omegas/zetas_inv (N words each) may be NULL. */
int fhe_b200_debug_ntt_tables(const fhe_b200_params* p, uint64_t q, uint64_t* omegas, uint64_t* omegas_shoup,
                              uint64_t* zetas_inv, uint64_t* zetas_inv_shoup, uint64_t* size_inv);
/* NTT words [limbs][N] at `level` of the expansion monomial -x^(N - 2^l), l < log2 N (evaluation_key.rs:465-474), as
 * fhe_b200_expand uses them; works on host-only handles. */
int fhe_b200_debug_expansion_monomial(const fhe_b200_params* p, uint32_t level, uint32_t l, uint64_t* out);
/* Encoder tables: matrix_reps_index_map (N words), the NTT tables of t (N words each; NTT_UNAVAILABLE when t has none),
 * and for `level` q_mod_t (one word) and delta = (-t)^-1 mod q_i (one word per limb).  Any output may be NULL. */
int fhe_b200_debug_encoder_tables(const fhe_b200_encoder* e, uint32_t level, uint32_t* index_map, uint64_t* omegas,
                                  uint64_t* zetas_inv, uint64_t* q_mod_t, uint64_t* delta);

#ifdef __cplusplus
}
#endif
#endif /* FHE_B200_H */
