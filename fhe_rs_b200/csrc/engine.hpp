// Internal launch interfaces shared by ntt.cu / kernels.cu / capi.cu.
#pragma once
#include <atomic>
#include <cuda.h>
#include <cuda_runtime.h>
#include <vector>

#include "ntt.cuh"

namespace fhe_b200 {

extern std::atomic<unsigned long long> g_launches;
// rows transformed by launch_ntt so far: [0] forward, [1] inverse (fhe_b200_ntt_row_count)
extern std::atomic<unsigned long long> g_ntt_rows[2];

// The FHE_B200_* environment switches (DESIGN.md, appendix), read once per process by switches() (ntt.cu).  Every
// value the appendix lists is set by a bit-for-bit rerun test.
struct Switches {
  enum Ntt { NTT_FAST, NTT_AUTO, NTT_TMA };
  enum Ksmac { KSMAC_FUSED, KSMAC_TMA, KSMAC_CLASSIC };
  u32 chunk;              // FHE_B200_CHUNK: ciphertexts per chunk of a batched call (>= 1, default 256)
  u32 streams;            // FHE_B200_STREAMS: side streams the chunks are dealt over (1..4, default 2)
  Ntt ntt;                // FHE_B200_NTT = fast | tma (default auto)
  bool generic_ntt;       // FHE_B200_GENERIC_NTT
  bool solinas_ntt;       // FHE_B200_SOLINAS_NTT: Solinas twiddle pairs (generic tile kernels only)
  bool no_solinas;        // FHE_B200_NO_SOLINAS: Barrett instead of the 2^62 = c folds everywhere
  bool no_tensor_fusion;  // FHE_B200_NO_TENSOR_FUSION
  bool classic_scaler;    // FHE_B200_SCALER=classic
  Ksmac ksmac;            // FHE_B200_KSMAC = tma | classic (default fused)
  int tma_cols;           // FHE_B200_TMA_COLS: 2 = ring depth 2 of the TMA cols pass (default 3)
  int scale_unroll;       // FHE_B200_SCALE_UNROLL: 4 = unroll 4 of the TMA scaler's multiply loop (default 2)
  u32 ks_stages;          // FHE_B200_KS_STAGES: digit ring depth of the key-switch kernels (2..4, default 2)
  // every NTT of N > 4096 runs on the generic tile kernels
  bool generic_tiles() const { return generic_ntt || solinas_ntt; }
  // the TMA-fed NTT kernels may serve a launch
  bool tma_allowed() const { return ntt != NTT_FAST && !generic_tiles(); }
};
const Switches& switches();

// cuTensorMapEncodeTiled, fetched through the runtime so the library does not link against libcuda; null when the
// driver lacks it
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn tensor_map_encoder();
// the buffer [rows][N] u64 as {box_cols, box_rows} boxes, no swizzle; false when the encoder is missing or refuses
bool box_map(CUtensorMap* m, const u64* base, u64 rows, u32 logn, u32 box_cols, u32 box_rows);
// multiprocessors of the current device (cached per device)
int sm_count();

struct CudaFail {
  cudaError_t err;
  const char* what;
};
#define FHE_CUDA(x)                                         \
  do {                                                      \
    cudaError_t e__ = (x);                                  \
    if (e__ != cudaSuccess) throw CudaFail{e__, #x};        \
  } while (0)

// cudaFuncAttributeMaxDynamicSharedMemorySize is a per-device attribute of a kernel: remember, per (device, kernel),
// the largest size already granted and raise it when a launch needs more (thread-safe; a parameter set may live on
// any device of the process).  Throws CudaFail when the device refuses.
void ensure_dynamic_smem(const void* kernel, size_t bytes);

// position -> limb id map of the rows of a buffer
struct RowIds {
  u32 limbs_per_poly;
  unsigned short ids[kMaxPos];
};

// ---- NTT (ntt.cu)
// Transforms n_rows rows of N words.  in may differ from out (first pass reads in).
// in_div / reduce_on_load / lazy_out: see NttArgs.
// digit_adjacent (forward, in_div == limbs_per_poly only): polynomial p = (ct, digit d) writes its limb-j row at
// ((ct*limbs_per_poly + j)*n_dig + d)*N instead of (p*limbs_per_poly + j)*N -- the layout the key-switch inner
// product reads fastest (all digits of one (ct, limb) adjacent).
void launch_ntt(const u64* in, u64* out, u32 n_rows, const RowIds& ids, const LimbDev* limbs, u32 logn,
                bool inverse, u32 in_div, bool reduce_on_load, cudaStream_t st, bool lazy_out = false,
                bool digit_adjacent = false, u32 n_dig = 1);

// Tensor product of two 2-part ciphertexts (as launch_tensor with nca == ncb == L) fused with the inverse transform of
// its 3K output rows: T [ct][3][K][N] receives the POWER-BASIS products.  Returns false when the TMA kernels do not
// serve the shape (the caller then runs launch_tensor + launch_ntt).
bool launch_tensor_inverse_ntt(const u64* a, const u64* b, const u64* xa, const u64* xb, u64* T, u32 cts, u32 L, u32 K,
                               const RowIds& mul_ids, const LimbDev* limbs, u32 logn, cudaStream_t st);

// ---- element-wise (kernels.cu)
enum EwOp { EW_ADD = 0, EW_SUB = 1, EW_NEG = 2 };
void launch_ew(EwOp op, u64* a, const u64* b, size_t n_rows, const RowIds& ids, const LimbDev* limbs, u32 logn,
               cudaStream_t st);

// op 0: a[ct][part][limb][:] *= pt[ct % n_pt][limb][:]   (Modulus::mul_vec, zq/mod.rs:332)
// op 1 / 2: a[ct][0][limb][:] +=/-= pt[ct % n_pt][limb][:]   (Ciphertext +=/-= &Plaintext, ops/mod.rs:88-97, :188-197)
void launch_mul_plain(u64* a, const u64* pt, u32 cts, u32 parts, u32 n_pt, const RowIds& ids, const LimbDev* limbs,
                      u32 logn, cudaStream_t st, u32 op = 0);

// one level of EvaluationKey::expands (evaluation_key.rs:229-241) over `pairs` 2-part ciphertexts, all NTT:
// lo [pairs][2][L][N] += s;  hi [n_hi][2][L][N] = (lo - s) * mono (mono: [L][N] (value, Shoup) pairs).
// s of pair k is hi[k] for k < n_hi (read, then overwritten) and spill[k - n_hi] otherwise.
void launch_expand_butterfly(u64* lo, u64* hi, const u64* spill, u32 pairs, u32 n_hi, const ulonglong2* mono,
                             const RowIds& ids, const LimbDev* limbs, u32 logn, cudaStream_t st);

// dot_product_scalar (bfv/ops/dot_product.rs:55-184): out[g] = sum_{i<n_terms} ct[(g*n+i) % ct_count] (.) pt[(g*n+i) % pt_count]
// ct: [ct_count][parts][limbs][N], pt: [pt_count][limbs][N], out: [groups][parts][limbs][N], all NTT
void launch_dot(const u64* ct, const u64* pt, u64* out, u32 groups, u32 n_terms, u32 parts, u32 ct_count,
                u32 pt_count, const RowIds& ids, const LimbDev* limbs, u32 logn, cudaStream_t st);

// tensor product of two 2-part ciphertexts over the multiplication basis (mul.rs:198-201).
// a,b: [ct][2][L][N] NTT (supply the first nca / ncb mul-basis limbs of their side: the common prefix a factor-one
// extender keeps); xa: [ct][2][K-nca][N], xb: [ct][2][K-ncb][N] (the scaled limbs, NTT); out: [ct][3][K][N].
void launch_tensor(const u64* a, const u64* b, const u64* xa, const u64* xb, u64* out, u32 cts, u32 L, u32 nca,
                   u32 ncb, u32 K, const RowIds& mul_ids, const LimbDev* limbs, u32 logn, cudaStream_t st);

// general part counts (ops/mod.rs:259-358): a [ct][na][L][N], b [ct][nb][L][N], xa [ct][na][E][N], xb [ct][nb][E][N]
// -> out [ct][na+nb-1][K][N], c[k] = sum_{i+j=k} a_i * b_j
void launch_tensor_nm(const u64* a, const u64* b, const u64* xa, const u64* xb, u64* out, u32 cts, u32 L, u32 E, u32 na,
                      u32 nb, const RowIds& mul_ids, const LimbDev* limbs, u32 logn, cudaStream_t st);

// exact RNS scaler (rns/scaler.rs:249-352), tables resident on the device
struct ScalerDev {
  u32 n_from, n_to, is_one, shift;
  u64 tg_lo, tg_hi;
  u32 tg_sign;
  u32 all_solinas;   // every `to` limb is 2^62 - c, c < 2^28 (the persistent TMA kernel's epilogue needs it)
  const u64* gamma;       // [n_to]
  const u64* omega;       // [n_to][n_from]
  const u64* to_lo;       // theta_omega [n_from]
  const u64* to_hi;
  const unsigned char* to_sign;
  const unsigned char* to_order;   // source indices, the theta_omega terms with positive sign first
  u32 n_pos, n_terms;              // positive-sign terms, all non-zero terms (<= n_from)
  const u64* tgar_lo;     // theta_garner [n_from]
  const u64* tgar_hi;
  unsigned short to_ids[kMaxPos];
};
// in: [polys][n_from][N] power basis.  Output rows `start .. start+n_out` of the `to` basis:
//  split3 == 0: out0 + (poly * out_rows_per_poly + row) * N
//  split3 == 1: polys come in triples (c0,c1,c2); c0,c1 -> out0 as [ct][2][n_out][N], c2 -> out1 as [ct][n_out][N]
void launch_scale(const ScalerDev& S, const LimbDev* limbs, const u64* in, u64* out0, u64* out1, u32 polys,
                  u32 out_rows_per_poly, u32 start, u32 n_out, int split3, u32 logn, cudaStream_t st);

// The keys of one inner-product launch, carried in its kernel parameters: pair s is (k0[s], k1[s]), each
// [Lk][n_dig][N], and ciphertext c of the launch uses pair slot[c].  With n == 1 every ciphertext uses pair 0 and
// `slot` is not read, so a one-key launch may hold any number of ciphertexts; otherwise at most kKeySlots.
constexpr u32 kKeyPairs = 64;
constexpr u32 kKeySlots = 512;
struct KeyTable {
  const u64* k0[kKeyPairs];
  const u64* k1[kKeyPairs];
  u32 n;
  unsigned char slot[kKeySlots];
};
// ciphertexts [ct0, ct0 + cts) of a key switch and their keys: one inner-product launch each
struct KeyRange {
  u32 ct0, cts;
  KeyTable keys;
};
#ifdef __CUDACC__
__device__ __forceinline__ u32 key_slot(const KeyTable& K, u32 ct) { return K.n > 1 ? K.slot[ct] : 0; }
#endif

// key-switch inner product (key_switching_key.rs:256-268) on already transformed digits, one launch per range:
// inter: [ct][n_dig][Lk][N] NTT values (lazy, any 64-bit word), or [ct][Lk][n_dig][N] when `adjacent`;
// keys: [Lk][n_dig][N] (limb-major: the device copy of a key is transposed once at upload);
// out0/out1 row (ct, j) at out + (ct*out_ct_rows + j)*N ; base0/base1 (nullable) same indexing.
void launch_ksmac(const u64* inter, const std::vector<KeyRange>& ranges, const u64* base0, const u64* base1, u64* out0,
                  u64* out1, u32 n_dig, u32 Lk, u32 out_ct_rows, const RowIds& ids, const LimbDev* limbs, u32 logn,
                  cudaStream_t st, bool adjacent = false);

// whether launch_ntt will take the TMA kernels for this shape (they can write the digit-adjacent layout)
bool ntt_uses_tma(u32 n_rows, const RowIds& ids, u32 logn, u32 in_div, const u64* in, const u64* out);

// the RNS-digit key switch on the TMA kernels: digit broadcast + forward cols pass of c2 [cts][n_dig][N] into
// `inter` (scratch, cts*n_dig*Lk rows, digit-adjacent), then the forward rows pass fused with the inner product of
// launch_ksmac (same outputs, same indexing), one rows+MAC launch per range over the same `inter`.  Returns false,
// having launched nothing, outside the kernels' domain.
bool launch_key_switch_tma(const u64* c2, u64* inter, const std::vector<KeyRange>& ranges, const u64* base0,
                           const u64* base1, u64* out0, u64* out1, u32 cts, u32 n_dig, u32 Lk, u32 out_ct_rows,
                           const RowIds& ids, const LimbDev* limbs, u32 logn, bool reduce, cudaStream_t st);

// base-2^log_base digit decomposition of single-limb polynomials (key_switching_key.rs:339-345):
// in [polys][N] -> out [polys][n_dig][N]
void launch_decompose(const u64* in, u64* out, size_t polys, u32 n_dig, u32 log_base, u32 logn, cudaStream_t st);

// out[row][t] = in[row][perm[t]] (the SIMD decoder's slot map)
void launch_gather(const u64* in, u64* out, size_t n_rows, const int* perm, u32 logn, cudaStream_t st);
// The substitutions of one launch, carried in its kernel parameters: ciphertexts ct0[r] .. ct0[r+1]-1 of the launch
// (run r) use exponent[r] and read sources src0[r], src0[r] + 1, ...  A call with more runs takes more launches.
constexpr u32 kSubstRuns = 64;
struct SubstTable {
  u32 n;
  u32 ct0[kSubstRuns], exponent[kSubstRuns], src0[kSubstRuns];
};
// Poly::substitute of NTT rows (rq/mod.rs:360-389) for `cts` ciphertexts: ciphertext c reads ciphertext source[c]
// (c when source is null) of `in`, L rows per part, and uses exponent[c] (odd, < 2N); host arrays.
//  sum == false: out0 + c*out0_stride = sigma(part 0); out1 (nullable) + c*out1_stride = sigma(part 1).
//  sum == true (2-part): out0 + c*out0_stride = (sigma(c0) + c0, c1), out1 = sigma(c1).  ids/limbs: the rows' moduli.
// Every word stays in [0, q) when the input's are.  No table, allocation or host synchronisation.
void launch_substitute_ntt(const u64* in, size_t in_stride, u64* out0, size_t out0_stride, u64* out1,
                           size_t out1_stride, const u32* exponent, const u32* source, u32 cts, u32 L, bool sum,
                           const RowIds& ids, const LimbDev* limbs, u32 logn, cudaStream_t st);
// Poly<PowerBasis>::substitute (rq/mod.rs:390-408): signed coefficient scatter x^j -> x^(j*exponent)
void launch_substitute_power(const u64* in, u64* out, size_t n_rows, u32 exponent, const RowIds& ids,
                             const LimbDev* limbs, u32 logn, cudaStream_t st);

// ---- hoisted rotations (DESIGN §8): many Galois key switches of one ciphertext from one digit decomposition of c1.
// One hoisted output: its key pair ([Lk][n_dig][N] each), exponent (odd, < 2N), the slot of its source's digits and
// power-basis c1 in the call's buffers, its source ciphertext in the batch, its correction row and where it is written.
struct HoistOut {
  const u64 *k0, *k1;
  u32 exponent, src, src_ct, mrow, dst;
};
// flags[i] = 1 when output i's substitution negates a position s >= 1 at which some residue row of its source's c1 is
// zero: x [slot][L][N] power basis, canonical; output i negates s when (s * exponent mod 2N) >= N.  Writes only 1s (the
// caller clears the flags).
void launch_hoist_zero(const HoistOut* outs, u32 n, const u64* x, u32* flags, u32 L, u32 logn, cudaStream_t st);
// out [m][Lk][N] power basis: row (m, j) is N_e of exponent exps[m] in every limb j, 1 at each destination x^d whose
// source x^s has (s * e mod 2N) >= N (the negated coefficients of rq/mod.rs:390-408), 0 elsewhere
void launch_negation_rows(u64* out, const u32* exps, u32 n_exp, u32 Lk, u32 logn, cudaStream_t st);
// The key switch of sigma_e(c1) from the digit transforms of c1 (key_switching_key.rs:256-268 with the identity of
// DESIGN §8): for output i with source slot s, exponent e and correction row m, limb j < Lk,
//   out_p[j] = sum_{k < L} key_p,k[j] (.) pi_e(D_k[j]) + M_m[j] (.) sum_{k < L} [q_k]_{q_j} key_p,k[j]   (+ sigma_e(c0)[j])
// D: digits [slot][L][Lk][N] (lazy NTT words), or [slot][Lk][L][N] when `adjacent`; mrows: [m][Lk][N] NTT of N_e,
// canonical.  Output i's rows (p, j) go to out + dst * out_stride + (p * Lk + j) * N.  c0 (nullable, Lk == L): the
// batch, whose part 0 of ciphertext src_ct (at c0 + src_ct * c0_stride) is added through pi_e.  ids: the key level's.
void launch_hoist_mac(const HoistOut* outs, u32 n, const u64* D, bool adjacent, const u64* mrows, const u64* c0,
                      size_t c0_stride, u64* out, size_t out_stride, u32 L, u32 Lk, const RowIds& ids,
                      const LimbDev* limbs, u32 logn, cudaStream_t st);

// ---- linear transforms (DESIGN §3.4): baby-step/giant-step diagonal products from one hoisted decomposition.
// Baby step i >= 1 of a transform: its Galois key pair ([L][L][N] each) and exponent (3^i mod 2N).
struct LtStep {
  const u64 *k0, *k1;
  u32 exponent, pad;
};
// The partial sums of giant groups [g0, g0 + n_groups) of `cts` ciphertexts, NTT, keys at the ciphertext level (L):
//   out[c][g - g0][p] = sum_{i < baby, g*baby + i < n_diags} diag[g*baby + i] (.) T_i,p(ct[c])
// T_0 = ct[c]; T_i (i >= 1) = GaloisKey::relinearize of ct[c] for steps[i] from the digits D of its c1 (layout of
// launch_hoist_mac, slot c) and the correction rows mrows [baby][L][N] (row i: NTT of N_e of steps[i]), as
// hoist_mac_kernel computes it -- or, when fallback (nullable, [cts][baby]) gives f >= 0 for (c, i), item f of fb.
// ct, fb, out: items of ct_stride words; diag: [.][L][N], entry k of ciphertext c at (per_ct ? (diag_ct0 + c) *
// n_diags : 0) + k.  Every word canonical.
void launch_hoist_dot(const LtStep* steps, const int* fallback, const u64* fb, const u64* D, bool adjacent,
                      const u64* mrows, const u64* ct, size_t ct_stride, u32 cts, const u64* diag, u32 diag_ct0,
                      bool per_ct, u32 n_diags, u32 baby, u32 g0, u32 n_groups, u64* out, u32 L, const RowIds& ids,
                      const LimbDev* limbs, u32 logn, cudaStream_t st);

// Poly<PowerBasis>::switch_down (rq/mod.rs:433-492): in [polys][L][N] -> out [polys][L-1][N]
struct SwitchDownDev {
  u64 q_last, q_last_half;
  const u64* half_mod;  // [L-1]: q_i - (q_last/2 mod q_i)
  const u64* inv;       // [L-1]: q_last^-1 mod q_i
  const u64* inv_s;     // shoup
};
void launch_switch_down(const SwitchDownDev& S, const u64* in, u64* out, u32 polys, u32 L, const RowIds& ids,
                        const LimbDev* limbs, u32 logn, cudaStream_t st);

// ---- plaintext encoding (plaintext_vec.rs:37-103, plaintext.rs:103-197)
// constants of the plaintext modulus t (a zq::Modulus, t < 2^62)
struct PlainMod {
  u64 t, bhi, blo;
};
// coeffs [n_pt][N]: word c of plaintext k is value k*N + (inv_map ? inv_map[c] : c) of `staged` (the SIMD scatter
// coeffs[map[i]] = v[i] written as a gather), or 0 past n_values; is_signed: the values are i64, reduced into [0, t)
// (Modulus::reduce_vec_i64)
void launch_encode_load(const u64* staged, u64* coeffs, u32 n_pt, size_t n_values, const u32* inv_map, bool is_signed,
                        const PlainMod& T, u32 logn, cudaStream_t st);
// Plaintext::to_poly from power-basis residues modulo q_0 (t < q_0, plaintext.rs:103-135, :172-181), in place:
// x <- ((x mod t) * q_mod_t) mod t
void launch_to_poly_load(u64* x, size_t n_words, const PlainMod& T, u64 q_mod_t, cudaStream_t st);
// a[ct][0][j][:] +/-= m[ct % n_pt][j][:] * delta[j] mod q_j   (delta_s: Shoup companions; plaintext.rs:195 and
// ops/mod.rs:88-97, :188-197)
void launch_add_scaled(u64* a, const u64* m, u32 cts, u32 parts, u32 n_pt, const u64* delta, const u64* delta_s,
                       bool subtract, const RowIds& ids, const LimbDev* limbs, u32 logn, cudaStream_t st);

// ---- decryption (keys/secret_key.rs:55-98, :198-260)
// out [cts][L][N] = c0 + c1*s + c2*s^2 + ... of ct [cts][parts][L][N] (NTT, canonical); s row j at s + j*N
void launch_phase(const u64* ct, const u64* s, u64* out, u32 cts, u32 parts, const RowIds& ids, const LimbDev* limbs,
                  u32 logn, cudaStream_t st);
// in place: v <- ((v + t) mod q_0) mod t   (Q0 = {q_0, Barrett constants})
void launch_decrypt_epilogue(u64* v, size_t n_words, const PlainMod& Q0, const PlainMod& T, cudaStream_t st);
// in place: the lift of Plaintext::from_shares over two or more plaintext moduli from limb 0 of the scaled value (t < q_0)
void launch_from_shares_epilogue(u64* v, size_t n_words, u64 q0, const PlainMod& T, cudaStream_t st);
// in place: Modulus::center, a - t when a >= t >> 1 (the words are read back as i64)
void launch_center(u64* x, size_t n_words, u64 t, cudaStream_t st);
// out[ct] = max(out[ct], max over the N coefficients of min(bits(x), bits(Q - x))), x the CRT lift of the L residues of
// x [cts][L][N] (power basis, canonical; limb j modulo limbs[j]).  garner [L][L]: (i, j < i) = q_j^-1 mod q_i;
// q_words: Q as W little-endian words.  L <= 32.
void launch_noise(const u64* x, u32* out, u32 cts, u32 L, const u64* garner, const u64* q_words, u32 W,
                  const LimbDev* limbs, u32 logn, cudaStream_t st);

// ---- encryption (keys/secret_key.rs:100-136, keys/public_key.rs:45-92) from the seeded ChaCha20 stream of
// include/fhe_b200.h; ct_base is the call-wide index of the first ciphertext (state word 13)
struct EncSeed {
  u32 w[8];   // the 32-byte seed as eight little-endian words (state words 4..11)
};
// out [cts][2][L][N]: part 1 = a (role 0, uniform NTT words), part 0 = e - a*s; e [cts][L][N] NTT; s row j at s + j*N
void launch_encrypt_sk(const u64* s, const u64* e, u64* out, u32 cts, u32 ct_base, const EncSeed& K, const RowIds& ids,
                       const LimbDev* limbs, u32 logn, cudaStream_t st);
// out [cts][n_roles][L][N]: the centred binomial polynomial of roles role0 .. role0 + n_roles - 1 (drawn from limb 0's
// row) as canonical residues in every limb; variance 1..32
// digits > 1 addresses the rows as key generation does: row c of the call is digit c % digits (state word 15) of key
// c / digits (state word 13)
void launch_cbd(u64* out, u32 cts, u32 ct_base, u32 role0, u32 n_roles, u32 variance, const EncSeed& K,
                const RowIds& ids, const LimbDev* limbs, u32 logn, cudaStream_t st, u32 digits = 1);
// out [cts][2][L][N] = (u*pk0 + e1, u*pk1 + e2); uee [cts][3][L][N] = (u, e1, e2), pk [2][L][N], all NTT
void launch_encrypt_pk(const u64* uee, const u64* pk, u64* out, u32 cts, const RowIds& ids, const LimbDev* limbs,
                       u32 logn, cudaStream_t st);

// key generation (key_switching_key.rs:71-238): G, the gadget factor of digit i on key limb j, as Shoup pairs.  RNS
// digits (decomp = 0): G[i][j] = (i == j) g[j], g[j] = (Q_key / Q_ct) mod q_j; decomposition (decomp = 1, one key
// limb): G[i][0] = g[i] = 2^(i log_base) mod q_0
struct KskG {
  u32 decomp;
  u64 g[kMaxPos], g_s[kMaxPos];
};
// digits digit0 .. digit0 + digits - 1 of key `key` of the call: k0/k1 [Lk][n_dig][N] receive c0 = NTT(e_i) - c1 s +
// G[i][j] x and c1 (role 5, drawn directly as NTT words); e [digits][Lk][N] NTT, x [L_ct][N] NTT, s row j at s + j*N
void launch_ksk_gen(const u64* s, const u64* e, const u64* x, u64* k0, u64* k1, u32 key, u32 digit0, u32 digits,
                    u32 n_dig, const KskG& G, const EncSeed& K, const RowIds& ids, const LimbDev* limbs, u32 logn,
                    cudaStream_t st);

// ---- multiparty BFV (fhe::mbfv).  Experimental, incomplete, not audited, as the reference's module.
// out [cts][L][N]: CommonRandomPoly k = ct_base + c (role 7, uniform NTT words)
void launch_crp(u64* out, u32 cts, u32 ct_base, const EncSeed& K, const RowIds& ids, const LimbDev* limbs, u32 logn,
                cudaStream_t st);
// the share of one protocol per ciphertext (kernels.cu mbfv_share_kernel gives the operands of each)
enum MbfvShare { SHARE_PK = 0, SHARE_SKS = 1, SHARE_PKS = 2, SHARE_RKG1 = 3, SHARE_RKG2 = 4 };
void launch_mbfv_share(MbfvShare kind, const u64* s, const u64* s_out, const u64* x, const u64* pk, const u64* e,
                       u64* out, u32 cts, const RowIds& ids, const LimbDev* limbs, u32 logn, cudaStream_t st,
                       const u64* u = nullptr, u64* out1 = nullptr, u32 ct_base = 0);
// Aggregate: for items k < items, out item k = base item k (nullable) + sum_i src[i] item k, item_words words each
// (rows of limb (row % limbs_per_poly)); sources are read once, in launches of kSumGroup sources, each output word
// reduced once per launch.  Row r of an out item is at + r * out_row (0: N, contiguous rows; the key layout
// [limb][digit][N] of fhe_b200_rkg_aggregate takes n_dig * N).  A source may be out.
constexpr u32 kSumGroup = 64;
void launch_shares_sum(const u64* const* src, u32 n_src, size_t src_stride, const u64* base, size_t base_stride,
                       u64* out, size_t out_stride, u32 items, size_t item_words, const RowIds& ids,
                       const LimbDev* limbs, u32 logn, cudaStream_t st, size_t out_row = 0);
// Segment sums (AddAssign folded over runs, bfv/ops/mod.rs:54-69): for g < groups, out item g = (accumulate ? out item
// g : 0) + sum_{i < n_terms} in item g * n_terms + i.  An item is item_words words of rows of limb (row %
// limbs_per_poly); input item j starts at in + j * in_stride.  Rows r < split_rows of out item g are at out0 +
// g * out0_stride + r * N, the others at out1 + g * out1_stride + (r - split_rows) * N (split_rows = item_words / N:
// one output).  Every input word is read once and every output word reduced and written once.
void launch_segment_sum(const u64* in, size_t in_stride, u32 n_terms, u64* out0, size_t out0_stride, u64* out1,
                        size_t out1_stride, u32 split_rows, u32 groups, size_t item_words, bool accumulate,
                        const RowIds& ids, const LimbDev* limbs, u32 logn, cudaStream_t st);

// bit (un)packing of power-basis rows (fhe-util/src/lib.rs:71-146): row r of `rows` uses nbits[r % limbs] bits per
// coefficient; packed row r starts at byte  (r / limbs) * poly_bytes + offs[r % limbs]
struct PackDev {
  u32 limbs;
  unsigned char nbits[kMaxPos];
  u32 offs[kMaxPos];
  u32 poly_bytes;
};
void launch_pack(const PackDev& P, const u64* words, unsigned char* bytes, size_t n_rows, u32 logn, cudaStream_t st);
void launch_unpack(const PackDev& P, const unsigned char* bytes, u64* words, size_t n_rows, u32 logn, cudaStream_t st);

// fhe_util::transcode_bidirectional / _to_bytes / _from_bytes (fhe-util/src/lib.rs:68-187) over independent rows, one
// output value per thread.  Row r reads in_len elements (u64 words when in_elem == 8, bytes when 1) at
// in + r * in_stride elements and writes out_len values (u64 or bytes) at out + r * out_stride: value k is bits
// [k*out_bits, (k+1)*out_bits) of the row's LSB-first stream of in_bits-bit fields, zero past the stream's end.
struct TranscodeRows {
  const void* in;
  void* out;
  size_t in_len, in_stride, out_len, out_stride;
  u32 in_elem, in_bits, out_elem, out_bits;
};
void launch_transcode(const TranscodeRows& T, size_t n_rows, cudaStream_t st);
// The reply fold of the SealPIR server (examples/sealpir.rs:176-200) up to its plaintext coefficients: every part of
// the n_ct ciphertexts at `ct` ([n_ct][parts][row_words]) is transcoded from in_bits to out_bits, giving E values per
// part; the parts' values are concatenated and cut into P rows of N.  Row i of ciphertext j goes to
// coeffs + (i * n_ct + j) * N, zero past the parts * E values.
void launch_fold_stage(const u64* ct, u32 n_ct, u32 parts, size_t row_words, u32 in_bits, u32 out_bits, u32 P,
                       u64* coeffs, u32 logn, cudaStream_t st);

}  // namespace fhe_b200
