// Element-wise ring ops, tensor product, exact RNS scaler, key-switch inner product,
// Galois gather and modulus switch-down kernels (sm_90a).  64-bit integer modular
// arithmetic, HBM / integer-pipe bound: no tensor cores.
#include <algorithm>
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "engine.hpp"
#include "ntt_tma.cuh"

namespace fhe_b200 {

typedef unsigned __int128 u128;

namespace {

// ------------------------------------------------------------------ element-wise
struct EwArgs {
  u64* a;
  const u64* b;
  size_t n_words;
  u32 logn, limbs_per_poly;
  const LimbDev* limbs;
  unsigned short ids[kMaxPos];
};

// Modulus::{add,sub,neg}_vec (zq/mod.rs:240-326, :534-550) over every row of a batch
template <int OP>
__global__ void ew_kernel(EwArgs A) {
  size_t i = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) * 2;
  if (i >= A.n_words) return;
  const u64 p = A.limbs[A.ids[(i >> A.logn) % A.limbs_per_poly]].p;
  ulonglong2 x = *reinterpret_cast<ulonglong2*>(A.a + i);
  if (OP == EW_NEG) {
    x.x = csub(p - x.x, p);
    x.y = csub(p - x.y, p);
  } else {
    ulonglong2 y = *reinterpret_cast<const ulonglong2*>(A.b + i);
    if (OP == EW_ADD) {
      x.x = csub(x.x + y.x, p);
      x.y = csub(x.y + y.y, p);
    } else {
      x.x = csub(x.x + p - y.x, p);
      x.y = csub(x.y + p - y.y, p);
    }
  }
  *reinterpret_cast<ulonglong2*>(A.a + i) = x;
}

// ------------------------------------------------------------------ ciphertext x plaintext polynomial
struct MulPlainArgs {
  u64* a;
  const u64* pt;
  u32 cts, parts, n_pt, logn, limbs_per_poly;
  u32 op;   // 0: every part *= pt (ops/mod.rs:229); 1: part 0 += pt (:88-97); 2: part 0 -= pt (:188-197)
  const LimbDev* limbs;
  unsigned short ids[kMaxPos];
};
__global__ void mul_plain_kernel(MulPlainArgs A) {
  size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t total = ((size_t)A.cts * A.parts * A.limbs_per_poly) << A.logn;
  if (idx >= total) return;
  const u32 c = idx & ((1u << A.logn) - 1);
  const size_t row = idx >> A.logn;
  const u32 limb = row % A.limbs_per_poly;
  const u32 ct = (u32)(row / ((size_t)A.limbs_per_poly * A.parts));
  const LimbDev& M = A.limbs[A.ids[limb]];
  const u64 w = A.pt[((((size_t)(ct % A.n_pt)) * A.limbs_per_poly + limb) << A.logn) + c];
  if (A.op == 0) {
    A.a[idx] = mulmod_limb(A.a[idx], w, M);
  } else if ((row / A.limbs_per_poly) % A.parts == 0) {
    const u64 x = A.a[idx];
    A.a[idx] = A.op == 1 ? csub(x + w, M.p) : csub(x + M.p - w, M.p);   // Modulus::add / sub, zq/mod.rs:103-128
  }
}

// ------------------------------------------------------------------ oblivious expansion butterfly
struct ExpandArgs {
  u64* lo;              // [pairs][2][L][N], in place
  u64* hi;              // [n_hi][2][L][N]: s of the first n_hi pairs, replaced by the monomial product
  const u64* spill;     // [pairs - n_hi][2][L][N]: s of the pairs without a slot in `hi`
  const ulonglong2* mono;   // [L][N] (value, Shoup companion)
  size_t n_words, hi_words;
  u32 logn, limbs_per_poly;
  const LimbDev* limbs;
  unsigned short ids[kMaxPos];
};
// One level of EvaluationKey::expands (evaluation_key.rs:229-241) for every (i, query) pair:
// hi = (lo - s) * m_l, lo = lo + s.  Two 64-bit words per thread (128-bit accesses); s is read from hi (or the spill
// buffer) before the same thread overwrites it.  All values canonical, so the result equals the reference's
// sub / mul_shoup / add sequence bit for bit.
__global__ void expand_butterfly_kernel(ExpandArgs A) {
  const size_t i = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) * 2;
  if (i >= A.n_words) return;
  const u32 j = (u32)((i >> A.logn) % A.limbs_per_poly);
  const u32 slot = (u32)i & ((1u << A.logn) - 1);
  const u64 p = A.limbs[A.ids[j]].p;
  const bool has_hi = i < A.hi_words;
  const u64* sp = has_hi ? A.hi + i : A.spill + (i - A.hi_words);
  const ulonglong2 s = *reinterpret_cast<const ulonglong2*>(sp);
  ulonglong2 x = *reinterpret_cast<ulonglong2*>(A.lo + i);
  if (has_hi) {
    const ulonglong2 m0 = A.mono[((size_t)j << A.logn) + slot];
    const ulonglong2 m1 = A.mono[((size_t)j << A.logn) + slot + 1];
    ulonglong2 d;
    d.x = mul_shoup(csub(x.x + p - s.x, p), m0.x, m0.y, p);
    d.y = mul_shoup(csub(x.y + p - s.y, p), m1.x, m1.y, p);
    *reinterpret_cast<ulonglong2*>(A.hi + i) = d;
  }
  x.x = csub(x.x + s.x, p);
  x.y = csub(x.y + s.y, p);
  *reinterpret_cast<ulonglong2*>(A.lo + i) = x;
}

// ------------------------------------------------------------------ dot_product_scalar
struct DotArgs {
  const u64 *ct, *pt;
  u64* out;
  u32 groups, n_terms, parts, ct_count, pt_count, limbs_per_poly, logn;
  const LimbDev* limbs;
  unsigned short ids[kMaxPos];
};
// out[g][part][limb][:] = sum_i ct[g*n + i][part][limb][:] * pt[g*n + i][limb][:]   (an operand with only n entries
// is shared by all groups)
// (bfv/ops/dot_product.rs:55-184: u128 fused multiply-adds per coefficient, one reduction at the end; the lazy
// register here is 160 bits wide, so no term-count threshold / fallback path is needed).  HBM-bound: two words
// read per multiply; four terms in flight per trip.
__global__ void dot_kernel(DotArgs A) {
  const u32 N = 1u << A.logn;
  size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;  // over groups*parts*limbs*N
  size_t total = ((size_t)A.groups * A.parts * A.limbs_per_poly) << A.logn;
  if (idx >= total) return;
  const u32 c = idx & (N - 1);
  size_t row = idx >> A.logn;
  const u32 limb = row % A.limbs_per_poly;
  row /= A.limbs_per_poly;
  const u32 part = row % A.parts, g = (u32)(row / A.parts);
  const LimbDev& M = A.limbs[A.ids[limb]];
  const size_t ct_stride = ((size_t)A.parts * A.limbs_per_poly) << A.logn, pt_stride = (size_t)A.limbs_per_poly << A.logn;
  const u64* cp = A.ct + (((size_t)part * A.limbs_per_poly + limb) << A.logn) + c;
  const u64* pp = A.pt + ((size_t)limb << A.logn) + c;
  Acc192 acc;
  acc.clear();
  // an operand holds either n_terms entries (shared by every group) or groups * n_terms (checked by the caller)
  cp += (A.ct_count == A.n_terms ? 0 : (size_t)g * A.n_terms) * ct_stride;
  pp += (A.pt_count == A.n_terms ? 0 : (size_t)g * A.n_terms) * pt_stride;
  u32 i = 0;
  for (; i + 4 <= A.n_terms; i += 4) {   // eight independent loads in flight
    u64 x[4], y[4];
#pragma unroll
    for (int k = 0; k < 4; k++) {
      x[k] = cp[(size_t)(i + k) * ct_stride];
      y[k] = pp[(size_t)(i + k) * pt_stride];
    }
#pragma unroll
    for (int k = 0; k < 4; k++) acc.mac(x[k], y[k]);
  }
  for (; i < A.n_terms; i++) acc.mac(cp[(size_t)i * ct_stride], pp[(size_t)i * pt_stride]);
  A.out[idx] = acc.reduce(M);
}

// ------------------------------------------------------------------ tensor
struct TensorArgs {
  const u64 *a, *b, *xa, *xb;
  u64* out;
  u32 cts, L, nca, ncb, K, logn;
  const LimbDev* limbs;
  unsigned short ids[kMaxPos];
};
// c0 = a0*b0, c1 = a0*b1 + a1*b0, c2 = a1*b1 (bfv/ops/mul.rs:198-201; Modulus::mul_vec zq/mod.rs:332).
// Operand x (x = a, b) supplies its first nc_x mul-basis limbs from the ciphertext itself ([ct][2][L][N], the
// common prefix a factor-one extender keeps, rq/scaler.rs:61-65) and the other K - nc_x from the scaled rows
// ([ct][2][K - nc_x][N]).
__global__ void tensor_kernel(TensorArgs A) {
  const u32 N = 1u << A.logn, K = A.K;
  size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;  // over cts*K*N
  size_t total = (size_t)A.cts * K << A.logn;
  if (idx >= total) return;
  u32 c = idx & (N - 1);
  size_t row = idx >> A.logn;
  u32 pos = row % K, ct = row / K;
  const LimbDev& M = A.limbs[A.ids[pos]];
  u64 a0, a1, b0, b1;
  if (pos < A.nca) {
    size_t o = (((size_t)ct * 2) * A.L + pos) << A.logn;
    a0 = A.a[o + c]; a1 = A.a[o + ((size_t)A.L << A.logn) + c];
  } else {
    const u32 E = K - A.nca;
    size_t o = (((size_t)ct * 2) * E + (pos - A.nca)) << A.logn;
    a0 = A.xa[o + c]; a1 = A.xa[o + ((size_t)E << A.logn) + c];
  }
  if (pos < A.ncb) {
    size_t o = (((size_t)ct * 2) * A.L + pos) << A.logn;
    b0 = A.b[o + c]; b1 = A.b[o + ((size_t)A.L << A.logn) + c];
  } else {
    const u32 E = K - A.ncb;
    size_t o = (((size_t)ct * 2) * E + (pos - A.ncb)) << A.logn;
    b0 = A.xb[o + c]; b1 = A.xb[o + ((size_t)E << A.logn) + c];
  }
  u64 c0 = mulmod_limb(a0, b0, M);
  u64 c2 = mulmod_limb(a1, b1, M);
  Acc192 s;                                 // a0*b1 + a1*b0 < 2^125, one reduction
  s.clear();
  s.mac(a0, b1);
  s.mac(a1, b0);
  u64 c1 = s.reduce(M);
  size_t o = (((size_t)ct * 3) * K + pos) << A.logn;
  A.out[o + c] = c0;
  A.out[o + ((size_t)K << A.logn) + c] = c1;
  A.out[o + ((size_t)2 * K << A.logn) + c] = c2;
}

// General part counts of &ct * &ct (bfv/ops/mod.rs:259-358): c[k] = sum_{i+j=k} a_i * b_j over the multiplication
// basis, one thread per (ciphertext, output part k, limb, coefficient).  a: [ct][na][L][N], xa: [ct][na][E][N] etc.
struct TensorNmArgs {
  const u64 *a, *b, *xa, *xb;
  u64* out;
  u32 cts, L, E, na, nb, logn;
  const LimbDev* limbs;
  unsigned short ids[kMaxPos];
};
__global__ void tensor_nm_kernel(TensorNmArgs A) {
  const u32 N = 1u << A.logn, K = A.L + A.E, nc = A.na + A.nb - 1;
  size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;  // over cts*nc*K*N
  size_t total = ((size_t)A.cts * nc * K) << A.logn;
  if (idx >= total) return;
  const u32 c = idx & (N - 1);
  size_t row = idx >> A.logn;
  const u32 pos = row % K;
  row /= K;
  const u32 k = row % nc, ct = (u32)(row / nc);
  const LimbDev& M = A.limbs[A.ids[pos]];
  const bool ext = pos >= A.L;
  const u32 rows = ext ? A.E : A.L, r = ext ? pos - A.L : pos;
  const u64* pa = (ext ? A.xa : A.a) + ((((size_t)ct * A.na) * rows + r) << A.logn) + c;
  const u64* pb = (ext ? A.xb : A.b) + ((((size_t)ct * A.nb) * rows + r) << A.logn) + c;
  const size_t ps = (size_t)rows << A.logn;
  Acc192 acc;
  acc.clear();
  const u32 lo = k + 1 > A.nb ? k + 1 - A.nb : 0, hi = k < A.na - 1 ? k : A.na - 1;
  for (u32 i = lo; i <= hi; i++) acc.mac(pa[i * ps], pb[(k - i) * ps]);
  A.out[idx] = acc.reduce(M);
}

// ------------------------------------------------------------------ exact RNS scaler
struct ScaleArgs {
  ScalerDev S;
  const LimbDev* limbs;
  const u64* in;
  u64 *out0, *out1;
  u32 polys, out_rows_per_poly, start, n_out, split3, logn;
};

// 256-bit two's-complement helpers on 4 x u64 (stand-in for ethnum::U256 wrapping arithmetic)
struct U256 {
  u64 w0, w1, w2, w3;
};
__device__ __forceinline__ U256 u256_from_acc(const u32 (&a)[7]) {
  U256 r;
  r.w0 = ((u64)a[1] << 32) | a[0];
  r.w1 = ((u64)a[3] << 32) | a[2];
  r.w2 = ((u64)a[5] << 32) | a[4];
  r.w3 = a[6];
  return r;
}
__device__ __forceinline__ U256 u256_add(U256 a, U256 b) {
  U256 r;
  asm("add.cc.u64 %0, %4, %8;\n\t"
      "addc.cc.u64 %1, %5, %9;\n\t"
      "addc.cc.u64 %2, %6, %10;\n\t"
      "addc.u64 %3, %7, %11;"
      : "=l"(r.w0), "=l"(r.w1), "=l"(r.w2), "=l"(r.w3)
      : "l"(a.w0), "l"(a.w1), "l"(a.w2), "l"(a.w3), "l"(b.w0), "l"(b.w1), "l"(b.w2), "l"(b.w3));
  return r;
}
__device__ __forceinline__ U256 u256_sub(U256 a, U256 b) {
  U256 r;
  asm("sub.cc.u64 %0, %4, %8;\n\t"
      "subc.cc.u64 %1, %5, %9;\n\t"
      "subc.cc.u64 %2, %6, %10;\n\t"
      "subc.u64 %3, %7, %11;"
      : "=l"(r.w0), "=l"(r.w1), "=l"(r.w2), "=l"(r.w3)
      : "l"(a.w0), "l"(a.w1), "l"(a.w2), "l"(a.w3), "l"(b.w0), "l"(b.w1), "l"(b.w2), "l"(b.w3));
  return r;
}
// (128-bit v) * (128-bit theta) mod 2^256
__device__ __forceinline__ U256 u256_mul_128(u128 v, u64 tlo, u64 thi) {
  u32 a[7] = {0, 0, 0, 0, 0, 0, 0}, b[7] = {0, 0, 0, 0, 0, 0, 0};
  mac_theta(a, (u64)v, tlo, thi);
  mac_theta(b, (u64)(v >> 64), tlo, thi);
  U256 lo = u256_from_acc(a), hi = u256_from_acc(b);
  U256 hs = {0, hi.w0, hi.w1, hi.w2};
  return u256_add(lo, hs);
}

// RnsScaler::scale (rns/scaler.rs:249-352): one thread per coefficient column, 128 columns per CTA.
// The n_from source residues of the tile are staged in shared memory (coalesced load, conflict-free
// reads) so the thread keeps only accumulators in registers; the fixed-point sums (v, w) are computed
// exactly as coded in the reference; the output limbs are produced four at a time (four independent
// lazy accumulators per thread give the instruction-level parallelism the single dependent carry
// chain lacks; the register-resident one-limb-at-a-time form was latency-bound on that chain).
constexpr int kScaleTC = 128;

// The omega table in shared memory: omega_ji (< q_j < 2^62) split at bit 31 into three u32 planes per source row i,
// [i][w0, w1, w0 + w1][n_out4], so the four output limbs of a group take three 128-bit loads per term.
__device__ __forceinline__ void stage_omega_split(u32* s_om, const ScalerDev& S, u32 start, u32 n_out, u32 n_out4) {
  const u32 nf = S.n_from;
  for (u32 idx = threadIdx.x; idx < nf * n_out4; idx += blockDim.x) {
    const u32 ii = idx / n_out4, jj = idx - ii * n_out4;
    const Split31 w = split31(jj < n_out ? S.omega[(size_t)(start + jj) * nf + ii] : 0);
    u32* row = s_om + (size_t)ii * 3 * n_out4 + jj;
    row[0] = w.lo;
    row[n_out4] = w.hi;
    row[2 * n_out4] = w.sum;
  }
}

// sum_i r_i * omega_{j0+k, i} for the G (<= 4) output limbs of one group, three products per term (AccKara: every
// r_i is a canonical residue and every omega_ji is reduced, both < 2^62).  The unroll stays bounded: fully unrolled,
// ptxas keeps carry predicates alive across terms and parks them in registers.
template <int G, int UNR = 2>
__device__ __forceinline__ void scale_mac_group(AccKara (&acc)[4], const u64* r_col, const u32* om, u32 nf,
                                                u32 n_out4) {
#pragma unroll UNR
  for (u32 i = 0; i < nf; i++) {
    const Split31 r = split31(r_col[i * kScaleTC]);
    const u32* row = om + (size_t)i * 3 * n_out4;
    const uint4 w0 = *reinterpret_cast<const uint4*>(row);
    const uint4 w1 = *reinterpret_cast<const uint4*>(row + n_out4);
    const uint4 ws = *reinterpret_cast<const uint4*>(row + 2 * n_out4);
    acc[0].mac(r.lo, r.hi, r.sum, w0.x, w1.x, ws.x);
    if (G > 1) acc[1].mac(r.lo, r.hi, r.sum, w0.y, w1.y, ws.y);
    if (G > 2) acc[2].mac(r.lo, r.hi, r.sum, w0.z, w1.z, ws.z);
    if (G > 3) acc[3].mac(r.lo, r.hi, r.sum, w0.w, w1.w, ws.w);
  }
}

__global__ void __launch_bounds__(kScaleTC) scale_kernel(ScaleArgs A) {
  extern __shared__ __align__(16) u64 smem[];
  const ScalerDev& S = A.S;
  const u32 nf = S.n_from, n_out = A.n_out;
  const u32 n_out4 = (n_out + 3) & ~3u;
  constexpr u32 TC = kScaleTC;
  u64* s_r = smem;                                // [n_from][TC]
  u32* s_omega = reinterpret_cast<u32*>(s_r + (size_t)nf * TC);   // [n_from][3][n_out4]  (stage_omega_split)
  u64* s_gamma = reinterpret_cast<u64*>(s_omega + (size_t)nf * 3 * n_out4);   // [n_out4]
  u64* s_tgl = s_gamma + n_out4;                  // theta tables [n_from]
  u64* s_tgh = s_tgl + nf;
  u64* s_tol = s_tgh + nf;
  u64* s_toh = s_tol + nf;
  u32* s_ord = reinterpret_cast<u32*>(s_toh + nf);   // [n_from] term order of the w sum

  const u32 N = 1u << A.logn;
  const u32 per_poly = N / TC;
  const u32 poly = blockIdx.x / per_poly;
  const u32 c0 = (blockIdx.x % per_poly) * TC;
  const u64* src = A.in + (((size_t)poly * nf) << A.logn) + c0;
  const u32 cc = threadIdx.x;

  // Every thread fetches its own column of the source residues with asynchronous 8-byte copies (all n_from
  // requests in flight at once, no registers held, and no CTA barrier is needed for them: a thread only ever reads
  // back what it copied itself).  A load-then-store loop would leave warps waiting at the barrier behind eight
  // dependent HBM round trips.
  {
    const u32 dst0 = (u32)__cvta_generic_to_shared(s_r + cc);
    for (u32 i = 0; i < nf; i++)
      asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(dst0 + i * TC * 8u),
                   "l"(src + ((size_t)i << A.logn) + cc)
                   : "memory");
    asm volatile("cp.async.commit_group;" ::: "memory");
  }
  // the (L2-resident) tables, spread over the whole CTA
  stage_omega_split(s_omega, S, A.start, n_out, n_out4);
  for (u32 i = cc; i < n_out4; i += TC) s_gamma[i] = i < n_out ? S.gamma[A.start + i] : 0;
  for (u32 i = cc; i < nf; i += TC) {
    s_tgl[i] = S.tgar_lo[i];
    s_tgh[i] = S.tgar_hi[i];
    s_tol[i] = S.to_lo[i];
    s_toh[i] = S.to_hi[i];
    s_ord[i] = i < S.n_terms ? S.to_order[i] : 0;
  }
  asm volatile("cp.async.wait_all;" ::: "memory");
  __syncthreads();

  // v = round(sum_i r_i * theta_garner_i / 2^shift)   (:260-272)
  u128 v;
  {
    AccTheta at;
    at.clear();
#pragma unroll 2
    for (u32 i = 0; i < nf; i++) at.mac(s_r[i * TC + cc], s_tgl[i], s_tgh[i]);
    u32 acc[7];
    at.words(acc);
    U256 sg = u256_from_acc(acc);
    // theta_garner_shift is in [123,127] for moduli < 2^62 and <= 64 limbs (:130-142): shift-1 = 64 + bs, 58 <= bs <= 62
    const u32 bs = S.shift - 1 - 64;
    u64 lo = (sg.w1 >> bs) | (sg.w2 << (64 - bs));
    u64 hi = (sg.w2 >> bs) | (sg.w3 << (64 - bs));
    u128 x = ((u128)hi << 64) | lo;
    v = (x >> 1) + (x & 1);
  }
  // w = round((sum_i +/- r_i * theta_omega_i -/+ v * theta_gamma) / 2^127)   (:276-314)
  bool w_sign = false;
  u128 w = 0;
  if (!S.is_one) {
    // one pass per sign keeps a single accumulator set live; the table lists the positive terms first
    U256 s_pos = {0, 0, 0, 0}, s_neg = {0, 0, 0, 0};
#pragma unroll 1
    for (u32 sg = 0; sg < 2; sg++) {
      AccTheta at;
      at.clear();
      const u32 k0 = sg ? S.n_pos : 0, k1 = sg ? S.n_terms : S.n_pos;
#pragma unroll 2
      for (u32 k = k0; k < k1; k++) {
        const u32 i = s_ord[k];
        at.mac(s_r[i * TC + cc], s_tol[i], s_toh[i]);
      }
      u32 wds[7];
      at.words(wds);
      if (sg == 0) s_pos = u256_from_acc(wds);
      else s_neg = u256_from_acc(wds);
    }
    U256 so = u256_sub(s_pos, s_neg);
    U256 vt = u256_mul_128(v, S.tg_lo, S.tg_hi);
    so = S.tg_sign ? u256_add(so, vt) : u256_sub(so, vt);
    w_sign = (so.w3 != 0) || (so.w2 >> 63);
    if (w_sign) {
      u64 n1 = ~so.w1, n2 = ~so.w2, n3 = ~so.w3;
      u128 y = ((u128)((n2 >> 62) | (n3 << 2)) << 64) | ((n1 >> 62) | (n2 << 2));
      w = (y + 1) >> 1;
    } else {
      u128 y = ((u128)((so.w2 >> 62) | (so.w3 << 2)) << 64) | ((so.w1 >> 62) | (so.w2 << 2));
      w = (y >> 1) + (y & 1);
    }
  }

  // outputs (:316-351): y_j = (-(v mod q_j) * gamma_j +/- w + sum_i r_i * omega_ji) mod q_j, four limbs at a time
  for (u32 j0 = 0; j0 < n_out; j0 += 4) {
    AccKara acc[4];
#pragma unroll
    for (int k = 0; k < 4; k++) acc[k].clear();
    const u32* om = s_omega + j0;
    // the multiplier pipe bounds this loop (bench_micro/mac_bench.cu), so the last group only multiplies for the
    // limbs it really has (14 outputs = 4+4+4+2, not 16)
    switch (min(4u, n_out - j0)) {
      case 4: scale_mac_group<4>(acc, s_r + cc, om, nf, n_out4); break;
      case 3: scale_mac_group<3>(acc, s_r + cc, om, nf, n_out4); break;
      case 2: scale_mac_group<2>(acc, s_r + cc, om, nf, n_out4); break;
      default: scale_mac_group<1>(acc, s_r + cc, om, nf, n_out4); break;
    }
#pragma unroll
    for (int k = 0; k < 4; k++) {
      const u32 jj = j0 + k;
      if (jj >= n_out) break;
      const LimbDev& M = A.limbs[S.to_ids[A.start + jj]];
      u64 vr = reduce94_limb((u64)v, (u64)(v >> 64), M);   // v < n_from * 2^63
      acc[k].mac(split31(vr ? M.p - vr : 0), split31(s_gamma[jj]));
      if (!S.is_one) {
        u64 wr = reduce94_limb((u64)w, (u64)(w >> 64), M); // w < 2^70
        acc[k].add64(w_sign ? (wr ? M.p - wr : 0) : wr);
      }
      u64 y = acc[k].reduce(M);
      u64* dst;
      if (A.split3) {
        u32 ct = poly / 3, part = poly % 3;
        dst = part < 2 ? A.out0 + ((((size_t)ct * 2 + part) * n_out + jj) << A.logn)
                       : A.out1 + (((size_t)ct * n_out + jj) << A.logn);
      } else {
        dst = A.out0 + (((size_t)poly * A.out_rows_per_poly + jj) << A.logn);
      }
      dst[c0 + cc] = y;
    }
  }
}


// ------------------------------------------------------------------ exact RNS scaler, persistent TMA-fed form
// Same arithmetic as scale_kernel (RnsScaler::scale, rns/scaler.rs:249-352: v and w "as coded", one lazy accumulator
// and one reduction per output limb); what changes is everything around the multiply loop, which kept the per-tile
// kernel far below the multiplier-pipe bound that the loop alone reaches:
//   * persistent CTAs: the scaler tables (omega, gamma, theta_*, per-limb constants) are staged in shared memory once
//     per CTA instead of once per 128-column tile;
//   * the n_from x 128 source residues of a tile arrive with ONE TMA box copy (tensor map over [rows][N], box
//     {128 columns, n_from rows}) tracked by an mbarrier; the next tile's copy is issued as soon as the last multiply
//     group has read the current one;
//   * the per-limb epilogue works on Solinas limbs only (q_j = 2^62 - c_j; the caller checks): v and w are folded with
//     2^62 == c_j (one IMAD.WIDE each, no conditional subtraction, no canonical intermediate), -(v mod q_j)*gamma_j
//     enters the accumulator as (2q_j - v')*gamma_j, +/-w as one 64-bit addend, and the per-limb constants come from
//     shared memory (the old epilogue fetched the LimbDev record from global memory through two dependent loads).
struct ScaleTmaArgs {
  ScalerDev S;
  const LimbDev* limbs;
  u64 *out0, *out1;
  u32 polys, out_rows_per_poly, start, n_out, split3, logn;
  u32 tiles_total;   // polys * N / 128
};

template <bool IS_ONE, int UNR>
__global__ void __launch_bounds__(kScaleTC) scale_tma_kernel(const __grid_constant__ CUtensorMap tm_in, const ScaleTmaArgs A) {
  using namespace tma;
  extern __shared__ __align__(128) u64 smem[];
  const ScalerDev& S = A.S;
  const u32 nf = S.n_from, n_out = A.n_out;
  const u32 n_out4 = (n_out + 3) & ~3u;
  constexpr u32 TC = kScaleTC;
  u64* s_r = smem;                                // [n_from][TC]   (TMA destination, 128-byte aligned)
  u32* s_omega = reinterpret_cast<u32*>(s_r + (size_t)nf * TC);   // [n_from][3][n_out4]  (stage_omega_split)
  u64* s_gamma = reinterpret_cast<u64*>(s_omega + (size_t)nf * 3 * n_out4);   // [n_out4]
  u64* s_p2 = s_gamma + n_out4;                   // [n_out4]  2 q_j
  u64* s_c = s_p2 + n_out4;                       // [n_out4]  c_j = 2^62 - q_j
  u64* s_tgl = s_c + n_out4;                      // theta_garner [n_from]
  u64* s_tgh = s_tgl + nf;
  u64* s_tol = s_tgh + nf;                        // theta_omega of the non-zero terms, positive sign first [n_terms]
  u64* s_toh = s_tol + nf;
  u32* s_ord = reinterpret_cast<u32*>(s_toh + nf);   // their source rows, as byte offsets into s_r
  u64* s_bar = reinterpret_cast<u64*>(s_ord + ((nf + 1) & ~1u));
  const u32 bar = smem_u32(s_bar);
  const u32 cc = threadIdx.x;

  stage_omega_split(s_omega, S, A.start, n_out, n_out4);
  for (u32 i = cc; i < n_out4; i += TC) {
    const bool live = i < n_out;
    const LimbDev& M = A.limbs[S.to_ids[A.start + (live ? i : 0)]];
    s_gamma[i] = live ? S.gamma[A.start + i] : 0;
    s_p2[i] = M.p2;
    s_c[i] = M.sol_c;
  }
  for (u32 i = cc; i < nf; i += TC) {
    s_tgl[i] = S.tgar_lo[i];
    s_tgh[i] = S.tgar_hi[i];
    const u32 src = (!IS_ONE && i < S.n_terms) ? S.to_order[i] : 0;
    s_tol[i] = IS_ONE ? 0 : S.to_lo[src];
    s_toh[i] = IS_ONE ? 0 : S.to_hi[src];
    s_ord[i] = src * TC * 8;
  }
  if (cc == 0) {
    mbar_init(bar, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  const u32 N = 1u << A.logn;
  const u32 per_poly = N / TC;
  const u32 dst_r = smem_u32(s_r);
  const u32 tile_bytes = nf * TC * 8;
  u32 tile = blockIdx.x;
  if (cc == 0 && tile < A.tiles_total) {
    mbar_expect_tx(bar, tile_bytes);
    load_2d(dst_r, &tm_in, (tile % per_poly) * TC, (tile / per_poly) * nf, bar);
  }
  const u32 my_r = dst_r + cc * 8;   // this thread's column of the tile
  for (u32 it = 0; tile < A.tiles_total; tile += gridDim.x, it++) {
    const u32 poly = tile / per_poly;
    const u32 c0 = (tile - poly * per_poly) * TC;
    mbar_wait(bar, it & 1);

    // v = round(sum_i r_i * theta_garner_i / 2^shift)   (:260-272)
    u128 v;
    {
      AccTheta at;
      at.clear();
#pragma unroll 2
      for (u32 i = 0; i < nf; i++) at.mac(lds64(my_r + i * TC * 8), s_tgl[i], s_tgh[i]);
      u32 acc[7];
      at.words(acc);
      U256 sg = u256_from_acc(acc);
      const u32 bs = S.shift - 1 - 64;
      u64 lo = (sg.w1 >> bs) | (sg.w2 << (64 - bs));
      u64 hi = (sg.w2 >> bs) | (sg.w3 << (64 - bs));
      u128 x = ((u128)hi << 64) | lo;
      v = (x >> 1) + (x & 1);
    }
    // w = round((sum_i +/- r_i * theta_omega_i -/+ v * theta_gamma) / 2^127)   (:276-314)
    bool w_sign = false;
    u128 w = 0;
    if (!IS_ONE) {
      U256 s_pos = {0, 0, 0, 0}, s_neg = {0, 0, 0, 0};
#pragma unroll 1
      for (u32 sg = 0; sg < 2; sg++) {
        AccTheta at;
        at.clear();
        const u32 k0 = sg ? S.n_pos : 0, k1 = sg ? S.n_terms : S.n_pos;
#pragma unroll 2
        for (u32 k = k0; k < k1; k++) at.mac(lds64(my_r + s_ord[k]), s_tol[k], s_toh[k]);
        u32 wds[7];
        at.words(wds);
        if (sg == 0) s_pos = u256_from_acc(wds);
        else s_neg = u256_from_acc(wds);
      }
      U256 so = u256_sub(s_pos, s_neg);
      U256 vt = u256_mul_128(v, S.tg_lo, S.tg_hi);
      so = S.tg_sign ? u256_add(so, vt) : u256_sub(so, vt);
      w_sign = (so.w3 != 0) || (so.w2 >> 63);
      if (w_sign) {
        u64 n1 = ~so.w1, n2 = ~so.w2, n3 = ~so.w3;
        u128 y = ((u128)((n2 >> 62) | (n3 << 2)) << 64) | ((n1 >> 62) | (n2 << 2));
        w = (y + 1) >> 1;
      } else {
        u128 y = ((u128)((so.w2 >> 62) | (so.w3 << 2)) << 64) | ((so.w1 >> 62) | (so.w2 << 2));
        w = (y >> 1) + (y & 1);
      }
    }
    // v = vh * 2^62 + vl, w likewise: modulo q_j = 2^62 - c_j they are vh * c_j + vl < 2 q_j
    const u64 mask62 = (1ull << 62) - 1;
    const u64 vl = (u64)v & mask62, wl = (u64)w & mask62;
    const u32 vh = (u32)(v >> 62), wh = (u32)(w >> 62);

    // destination of output limb 0 of this column
    u64* dst;
    size_t dstride = (size_t)1 << A.logn;
    if (A.split3) {
      const u32 ct = poly / 3, part = poly - ct * 3;
      dst = part < 2 ? A.out0 + ((((size_t)ct * 2 + part) * n_out) << A.logn) : A.out1 + (((size_t)ct * n_out) << A.logn);
    } else {
      dst = A.out0 + (((size_t)poly * A.out_rows_per_poly) << A.logn);
    }
    dst += c0 + cc;

    // outputs (:316-351): y_j = (-(v mod q_j) * gamma_j +/- w + sum_i r_i * omega_ji) mod q_j, four limbs at a time
    for (u32 j0 = 0; j0 < n_out; j0 += 4) {
      AccKara acc[4];
#pragma unroll
      for (int k = 0; k < 4; k++) acc[k].clear();
      const u32* om = s_omega + j0;
      const u32 g = min(4u, n_out - j0);
      switch (g) {
        case 4: scale_mac_group<4, UNR>(acc, s_r + cc, om, nf, n_out4); break;
        case 3: scale_mac_group<3, UNR>(acc, s_r + cc, om, nf, n_out4); break;
        case 2: scale_mac_group<2, UNR>(acc, s_r + cc, om, nf, n_out4); break;
        default: scale_mac_group<1, UNR>(acc, s_r + cc, om, nf, n_out4); break;
      }
      if (j0 + 4 >= n_out) {
        // the tile has been read for the last time: fetch the next one while the last epilogue runs
        __syncthreads();
        const u32 nxt = tile + gridDim.x;
        if (cc == 0 && nxt < A.tiles_total) {
          mbar_expect_tx(bar, tile_bytes);
          load_2d(dst_r, &tm_in, (nxt % per_poly) * TC, (nxt / per_poly) * nf, bar);
        }
      }
#pragma unroll
      for (int k = 0; k < 4; k++) {
        const u32 jj = j0 + k;
        if (jj >= n_out) break;
        const u64 p2 = s_p2[jj];
        const u32 c = (u32)s_c[jj];
        // -(v mod q) * gamma as a positive multiple: 2q - v' is in (0, 2q], brought to [0, q] for the split
        acc[k].mac(split31(csub(p2 - ((u64)vh * c + vl), p2 >> 1)), split31(s_gamma[jj]));
        if (!IS_ONE) {
          const u64 wr = (u64)wh * c + wl;                     // w mod q in [0, 2q)
          acc[k].add64(w_sign ? p2 - wr : wr);
        }
        u64 lo, mid;
        u32 hi32;
        acc[k].merged(lo, mid, hi32);
        dst[(size_t)jj * dstride] = csub(fold192_solinas(lo, mid, hi32, c), p2 >> 1);
      }
    }
  }
}

// fallback for rings smaller than one tile (N < 64): one thread per coefficient, same arithmetic
__global__ void scale_small_kernel(ScaleArgs A) {
  const ScalerDev& S = A.S;
  const u32 nf = S.n_from, n_out = A.n_out;
  const u32 N = 1u << A.logn;
  const u32 idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= A.polys * N) return;
  const u32 poly = idx >> A.logn, c = idx & (N - 1);
  const u64* src = A.in + (((size_t)poly * nf) << A.logn) + c;
  u32 av[7] = {0, 0, 0, 0, 0, 0, 0}, ap[7] = {0, 0, 0, 0, 0, 0, 0}, an[7] = {0, 0, 0, 0, 0, 0, 0};
  for (u32 i = 0; i < nf; i++) {
    const u64 r = src[(size_t)i << A.logn];
    mac_theta(av, r, S.tgar_lo[i], S.tgar_hi[i]);
    if (!S.is_one) {
      if (S.to_sign[i]) mac_theta(an, r, S.to_lo[i], S.to_hi[i]);
      else mac_theta(ap, r, S.to_lo[i], S.to_hi[i]);
    }
  }
  U256 sg = u256_from_acc(av);
  const u32 bs = S.shift - 1 - 64;
  u64 lo = (sg.w1 >> bs) | (sg.w2 << (64 - bs));
  u64 hi = (sg.w2 >> bs) | (sg.w3 << (64 - bs));
  u128 x = ((u128)hi << 64) | lo;
  u128 v = (x >> 1) + (x & 1);
  bool w_sign = false;
  u128 w = 0;
  if (!S.is_one) {
    U256 so = u256_sub(u256_from_acc(ap), u256_from_acc(an));
    U256 vt = u256_mul_128(v, S.tg_lo, S.tg_hi);
    so = S.tg_sign ? u256_add(so, vt) : u256_sub(so, vt);
    w_sign = (so.w3 != 0) || (so.w2 >> 63);
    if (w_sign) {
      u64 n1 = ~so.w1, n2 = ~so.w2, n3 = ~so.w3;
      u128 y = ((u128)((n2 >> 62) | (n3 << 2)) << 64) | ((n1 >> 62) | (n2 << 2));
      w = (y + 1) >> 1;
    } else {
      u128 y = ((u128)((so.w2 >> 62) | (so.w3 << 2)) << 64) | ((so.w1 >> 62) | (so.w2 << 2));
      w = (y >> 1) + (y & 1);
    }
  }
  for (u32 j = 0; j < n_out; j++) {
    const LimbDev& M = A.limbs[S.to_ids[A.start + j]];
    Acc192 acc;
    acc.clear();
    for (u32 i = 0; i < nf; i++) acc.mac(src[(size_t)i << A.logn], S.omega[(size_t)(A.start + j) * nf + i]);
    u64 vr = reduce128_limb((u64)v, (u64)(v >> 64), M);
    acc.mac(vr ? M.p - vr : 0, S.gamma[A.start + j]);
    if (!S.is_one) {
      u64 wr = reduce128_limb((u64)w, (u64)(w >> 64), M);
      acc.add64(w_sign ? (wr ? M.p - wr : 0) : wr);
    }
    u64 y = acc.reduce(M);
    u64* dst;
    if (A.split3) {
      u32 ct = poly / 3, part = poly % 3;
      dst = part < 2 ? A.out0 + ((((size_t)ct * 2 + part) * n_out + j) << A.logn)
                     : A.out1 + (((size_t)ct * n_out + j) << A.logn);
    } else {
      dst = A.out0 + (((size_t)poly * A.out_rows_per_poly + j) << A.logn);
    }
    dst[c] = y;
  }
}

// ------------------------------------------------------------------ key-switch MAC
struct KsMacArgs {
  KeyTable keys;
  const u64 *inter, *base0, *base1;
  u64 *out0, *out1;
  u32 cts, n_dig, Lk, out_ct_rows, logn;
  u32 adjacent;   // digit rows of one (ciphertext, limb) adjacent: inter is [ct][limb][digit][N], else [ct][digit][limb][N]
  const LimbDev* limbs;
  unsigned short ids[kMaxPos];
};
// out0 = base0 + sum_i t_i * k0_i ; out1 = base1 + sum_i t_i * k1_i   (key_switching_key.rs:256-268)
// One thread per (limb j, ciphertext, coefficient), limb-major: consecutive CTAs work on the same key limb for
// every ciphertext of the chunk, so the 2 x n_dig key rows of that limb (7 MB at set C, stored limb-major
// [limb][digit][N]) stay in L2 while the digit rows stream through -- each key word leaves HBM once per chunk instead
// of once per ciphertext.  Each ciphertext reads the key pair its slot names.
__global__ void ksmac_kernel(const __grid_constant__ KsMacArgs A) {
  const u32 N = 1u << A.logn;
  size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;  // over Lk*cts*N
  size_t total = ((size_t)A.cts * A.Lk) << A.logn;
  if (idx >= total) return;
  u32 c = idx & (N - 1);
  size_t row = idx >> A.logn;
  u32 ct = row % A.cts, j = row / A.cts;
  const LimbDev& M = A.limbs[A.ids[j]];
  Acc192 a0, a1;
  a0.clear();
  a1.clear();
  const u64* t_ptr = A.adjacent ? A.inter + ((((size_t)ct * A.Lk + j) * A.n_dig) << A.logn) + c
                                : A.inter + ((((size_t)ct * A.n_dig) * A.Lk + j) << A.logn) + c;
  const size_t dstride = A.adjacent ? (size_t)1 << A.logn : (size_t)A.Lk << A.logn;
  const size_t kstride = (size_t)1 << A.logn;
  const u32 slot = key_slot(A.keys, ct);
  const u64* k0_ptr = A.keys.k0[slot] + (((size_t)j * A.n_dig) << A.logn) + c;
  const u64* k1_ptr = A.keys.k1[slot] + (((size_t)j * A.n_dig) << A.logn) + c;
  // two digits per trip, the six words of the next trip requested before the multiplies of this one (the kernel
  // is bound by HBM latency, not by the multiplier: 2 x n_dig x 8 IMAD.WIDE per 48 bytes read).  Two
  // coefficients per thread with 16-byte accesses, and four ciphertexts per thread sharing each key word (a third
  // of the L2 -> SM bytes), both measured the same or slower
  u32 i = 0;
  u64 t0 = 0, t1 = 0, x0 = 0, x1 = 0, y0 = 0, y1 = 0;
  if (A.n_dig >= 2) {
    t0 = t_ptr[0], t1 = t_ptr[dstride];
    x0 = __ldg(k0_ptr), x1 = __ldg(k0_ptr + kstride);
    y0 = __ldg(k1_ptr), y1 = __ldg(k1_ptr + kstride);
  }
  for (; i + 2 <= A.n_dig; i += 2) {
    const u64 ct0 = t0, ct1 = t1, cx0 = x0, cx1 = x1, cy0 = y0, cy1 = y1;
    if (i + 4 <= A.n_dig) {
      t0 = t_ptr[(size_t)(i + 2) * dstride], t1 = t_ptr[(size_t)(i + 3) * dstride];
      x0 = __ldg(k0_ptr + (size_t)(i + 2) * kstride), x1 = __ldg(k0_ptr + (size_t)(i + 3) * kstride);
      y0 = __ldg(k1_ptr + (size_t)(i + 2) * kstride), y1 = __ldg(k1_ptr + (size_t)(i + 3) * kstride);
    }
    a0.mac(ct0, cx0);
    a1.mac(ct0, cy0);
    a0.mac(ct1, cx1);
    a1.mac(ct1, cy1);
  }
  if (i < A.n_dig) {
    const u64 tl = t_ptr[(size_t)i * dstride];
    a0.mac(tl, __ldg(k0_ptr + (size_t)i * kstride));
    a1.mac(tl, __ldg(k1_ptr + (size_t)i * kstride));
  }
  const size_t o = (((size_t)ct * A.out_ct_rows + j) << A.logn) + c;
  if (A.base0) a0.add64(A.base0[o]);
  if (A.base1) a1.add64(A.base1[o]);
  A.out0[o] = a0.reduce(M);
  A.out1[o] = a1.reduce(M);
}


// ------------------------------------------------------------------ key-switch MAC, persistent TMA-fed form
// The same sums as ksmac_kernel for the digit-adjacent layout (inter [ct][limb][digit][N], keys [limb][digit][N]).
// The inner product is HBM-bound (14 digit words streamed per pair of outputs) but the per-thread form was bound by
// load latency (about half of the device's copy rate): here one elected thread streams every operand with TMA box
// copies and the compute threads only read shared memory.
//   work item = (limb j, 128-coefficient tile tau, ciphertext ct), ct innermost: the two key tiles of (j, tau)
//   (2 n_dig row segments of 1 KiB) are fetched once and stay in shared memory for every ciphertext of the CTA's
//   range that uses the same key pair; the digit tile of each ciphertext ({128, n_dig} box: its n_dig rows are adjacent) arrives through a ring of
//   KS_STAGES buffers, refilled as soon as the CTA has consumed it.
constexpr int kKsTC = 128;
struct KsTmaArgs {
  KeyTable keys;
  const u64 *base0, *base1;
  u64 *out0, *out1;
  u32 cts, n_dig, Lk, out_ct_rows, logn;
  u32 items_total;   // Lk * (N / 128) * cts, item = (j * tiles + tau) * cts + ct
  const LimbDev* limbs;
  unsigned short ids[kMaxPos];
};

template <int KS_STAGES>
__global__ void __launch_bounds__(kKsTC) ksmac_tma_kernel(const __grid_constant__ CUtensorMap tm_t,
                                                          const __grid_constant__ KsTmaArgs A) {
  using namespace tma;
  extern __shared__ __align__(128) u64 smem[];
  constexpr u32 TC = kKsTC, S = KS_STAGES;
  const u32 nd = A.n_dig;
  const u32 box_bytes = nd * TC * 8;
  u64* s_k0 = smem;                       // [n_dig][TC]
  u64* s_k1 = s_k0 + (size_t)nd * TC;
  u64* s_t = s_k1 + (size_t)nd * TC;      // [S][n_dig][TC]
  u64* s_bar = s_t + (size_t)S * nd * TC; // S full barriers + 1 key barrier
  const u32 bar_full = smem_u32(s_bar), bar_key = bar_full + 8 * S;
  const u32 cc = threadIdx.x;
  if (cc == 0) {
    for (u32 s = 0; s < S; s++) mbar_init(bar_full + 8 * s, 1);
    mbar_init(bar_key, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  const u32 tiles = (1u << A.logn) / TC;
  const u32 lo = (u32)(((u64)A.items_total * blockIdx.x) / gridDim.x);
  const u32 hi = (u32)(((u64)A.items_total * (blockIdx.x + 1)) / gridDim.x);
  const u32 n = hi - lo;
  // item -> (jt, ct) walkers: `wl` for the loads thread 0 issues ahead, `w` for the item being computed
  TileWalk wl, w;
  wl.init(lo, A.cts);
  w.init(lo, A.cts);
  u32 loaded = 0;
  auto load_next = [&]() {   // thread 0 only
    const u32 s = loaded % S;
    const u32 j = wl.jt / tiles, tau = wl.jt - j * tiles;
    mbar_expect_tx(bar_full + 8 * s, box_bytes);
    load_2d(smem_u32(s_t + (size_t)s * nd * TC), &tm_t, tau * TC, (wl.p * A.Lk + j) * nd, bar_full + 8 * s);
    wl.next();
    loaded++;
  };
  if (cc == 0)
    while (loaded < n && loaded < S) load_next();

  u32 cur_jt = 0xffffffffu, cur_slot = 0, key_phase = 0;
  const LimbDev* Mp = A.limbs;
  for (u32 i = 0; i < n; i++) {
    const u32 slot = key_slot(A.keys, w.p);
    if (w.jt != cur_jt || slot != cur_slot) {
      // new (limb, tile) or new key: its two key tiles replace the previous ones (every thread has finished with
      // those: the item loop ends with a CTA barrier)
      cur_jt = w.jt;
      cur_slot = slot;
      const u32 j = cur_jt / tiles, tau = cur_jt - j * tiles;
      Mp = A.limbs + A.ids[j];
      if (cc == 0)
        load_key_tiles<TC>(smem_u32(s_k0), smem_u32(s_k1), A.keys.k0[slot], A.keys.k1[slot], j, tau, nd, A.logn,
                           bar_key);
      mbar_wait(bar_key, key_phase);
      key_phase ^= 1;
    }
    const u32 j = cur_jt / tiles, tau = cur_jt - j * tiles;
    const u32 s = i % S;
    const size_t o = (((size_t)w.p * A.out_ct_rows + j) << A.logn) + tau * TC + cc;
    u64 b0 = 0, b1 = 0;
    if (A.base0) b0 = A.base0[o];
    if (A.base1) b1 = A.base1[o];
    mbar_wait(bar_full + 8 * s, (i / S) & 1);
    const u64* t = s_t + (size_t)s * nd * TC + cc;
    Acc192 a0, a1;
    a0.clear();
    a1.clear();
#pragma unroll 2
    for (u32 d = 0; d < nd; d++) {
      const u64 td = t[d * TC];
      a0.mac(td, s_k0[d * TC + cc]);
      a1.mac(td, s_k1[d * TC + cc]);
    }
    a0.add64(b0);
    a1.add64(b1);
    A.out0[o] = a0.reduce(*Mp);
    A.out1[o] = a1.reduce(*Mp);
    __syncthreads();                       // stage s (and, before a key change, the key tiles) are free again
    if (cc == 0 && loaded < n) load_next();
    w.next();
  }
}

// base-2^log_base digits of a single-limb power-basis polynomial (key_switching_key.rs:339-345):
// out[poly][d][:] = (in[poly][:] >> (d * log_base)) & (2^log_base - 1)
__global__ void decompose_kernel(const u64* in, u64* out, size_t n_words, u32 n_dig, u32 log_base, u32 logn) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_words) return;
  const size_t poly = i >> logn;
  const u32 c = i & ((1u << logn) - 1);
  u64 v = in[i];
  const u64 mask = (1ull << log_base) - 1;
  for (u32 d = 0; d < n_dig; d++) {
    out[((poly * n_dig + d) << logn) + c] = v & mask;
    v >>= log_base;
  }
}

// ------------------------------------------------------------------ gather / switch_down
__global__ void gather_kernel(const u64* in, u64* out, size_t n_words, const int* perm, u32 logn) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_words) return;
  size_t row = i >> logn;
  u32 t = i & ((1u << logn) - 1);
  out[i] = in[(row << logn) + perm[t]];
}

// Poly::substitute, Ntt branch (rq/mod.rs:360-389), with SubstitutionExponent::new (:99-121) and the bit reversal of
// the evaluation points folded into the index: out[brev(j)] = in[brev((j*e + (e-1)/2) mod N)].  One CTA row (blockIdx.y)
// per ciphertext; its exponent and source come from the run table (SubstTable).  The 2-part form writes
// sigma(c0) to out0 and sigma(c1) to out1 in one pass; the inner-sum form writes out0 = (sigma(c0) + c0, c1) instead.
struct SubstArgs {
  SubstTable T;
  const u64* in;
  u64 *out0, *out1;
  size_t in_stride, out0_stride, out1_stride;   // words per ciphertext
  u32 L, logn;
  int sum;
  const LimbDev* limbs;
  unsigned short ids[kMaxPos];
};
__global__ void subst_kernel(SubstArgs A) {
  const u32 N = 1u << A.logn;
  const size_t w = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (w >= ((size_t)A.L << A.logn)) return;
  const u32 c = blockIdx.y;
  const SubstTable& T = A.T;
  u32 lo = 0, hi = T.n;   // the run holding c: the last r with T.ct0[r] <= c
  while (hi - lo > 1) {
    const u32 mid = (lo + hi) >> 1;
    if (T.ct0[mid] <= c) lo = mid;
    else hi = mid;
  }
  const u32 e = T.exponent[lo];
  const u64* src = A.in + (size_t)(T.src0[lo] + (c - T.ct0[lo])) * A.in_stride;
  const u32 o = (u32)w & (N - 1);
  const size_t row = w - o;
  const u32 j = __brev(o) >> (32 - A.logn);
  const u32 s = __brev((j * e + ((e - 1) >> 1)) & (N - 1)) >> (32 - A.logn);   // mod 2^32 keeps the low logn bits
  const size_t part1 = (size_t)A.L << A.logn;
  u64 v0 = src[row + s];
  u64* d0 = A.out0 + (size_t)blockIdx.y * A.out0_stride;
  if (A.sum) {
    const u64 p = A.limbs[A.ids[row >> A.logn]].p;
    v0 = csub(v0 + src[w], p);
    d0[part1 + w] = src[part1 + w];
  }
  d0[w] = v0;
  if (A.out1) A.out1[(size_t)blockIdx.y * A.out1_stride + w] = src[part1 + row + s];
}

// Poly::substitute, PowerBasis branch (rq/mod.rs:390-408): coefficient j of x^j moves to x^(j*e mod 2N), i.e. to slot
// (j*e) & (N-1), negated when bit N of j*e is set (x^N = -1).  e is odd, so the map is a bijection: a scatter in which
// every output word is written exactly once (reads coalesced, writes strided by e).
struct SubstPowerArgs {
  const u64* in;
  u64* out;
  size_t n_words;
  u32 logn, limbs_per_poly, exponent;
  const LimbDev* limbs;
  unsigned short ids[kMaxPos];
};
__global__ void substitute_power_kernel(SubstPowerArgs A) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= A.n_words) return;
  const u32 N = 1u << A.logn;
  const size_t row = i >> A.logn;
  const u32 j = (u32)i & (N - 1);
  const u64 p = A.limbs[A.ids[row % A.limbs_per_poly]].p;
  const u32 power = j * A.exponent;          // mod 2^32 keeps the low logn+1 bits exact
  const u64 v = A.in[i];
  A.out[(row << A.logn) + (power & (N - 1))] = (power & N) ? csub(p - v, p) : v;   // Modulus::sub(0, v) / add(0, v)
}

// ------------------------------------------------------------------ hoisted rotations (DESIGN §8)
// The outputs of one launch, carried in its kernel parameters (HoistOut without the key pointers, which go to the
// KeyTable).  96 outputs keep the MAC kernel's parameters under 4 KiB.
constexpr u32 kHoistOuts = 96;
struct HoistTable {
  u32 n;
  u32 exponent[kHoistOuts], src_ct[kHoistOuts], dst[kHoistOuts];
  unsigned short src[kHoistOuts], mrow[kHoistOuts];
};

// the source word of NTT position o under exponent e: pi_e of subst_kernel
__device__ __forceinline__ u32 subst_source(u32 o, u32 e, u32 logn) {
  const u32 j = __brev(o) >> (32 - logn);
  return __brev((j * e + ((e - 1) >> 1)) & ((1u << logn) - 1)) >> (32 - logn);
}

// One CTA row (blockIdx.y) per output, one thread per coefficient s of its source's c1; only the positions the
// exponent negates read the L residues.
__global__ void hoist_zero_kernel(const __grid_constant__ HoistTable T, const u64* x, u32* flags, u32 L, u32 logn) {
  const u32 N = 1u << logn, s = blockIdx.x * blockDim.x + threadIdx.x, i = blockIdx.y;
  if (s == 0 || s >= N || !((s * T.exponent[i]) & N)) return;   // mod 2^32 keeps bit logn of s*e exact
  const u64* r = x + (((size_t)T.src[i] * L) << logn) + s;
  bool zero = false;
  for (u32 k = 0; k < L; k++) zero |= r[(size_t)k << logn] == 0;
  if (zero) flags[i] = 1;
}

// Row (m, j) of N_e: thread s writes destination (s * e) mod N, so every word is written once.
__global__ void negation_rows_kernel(const __grid_constant__ HoistTable T, u64* out, u32 Lk, u32 logn) {
  const u32 N = 1u << logn, s = blockIdx.x * blockDim.x + threadIdx.x, m = blockIdx.y;
  if (s >= N) return;
  const u32 power = s * T.exponent[m];
  u64* row = out + (((size_t)m * Lk) << logn) + (power & (N - 1));
  for (u32 j = 0; j < Lk; j++) row[(size_t)j << logn] = (power & N) ? 1 : 0;
}

struct HoistMacArgs {
  HoistTable T;
  KeyTable keys;
  const u64 *D, *mrows, *c0;
  u64* out;
  size_t c0_stride, out_stride;
  u32 L, Lk, logn, adjacent;
  const LimbDev* limbs;
  unsigned short ids[kMaxPos];
};
// One thread per (coefficient o, output i = blockIdx.y, limb j = blockIdx.z), limb outermost: at any time the resident
// CTAs work on one limb of consecutive outputs, which the caller orders by (source, key), so the L digit rows of a
// source's limb j (3.7 MB at set C) and the key rows of a repeated key are read from L2 by every output that uses
// them.  pi_e permutes the words of each aligned group of 32 among themselves, so a warp's digit reads stay one 256-byte
// segment.  The correction sum_k [q_k]_{q_j} key_p,k[j] is accumulated beside the inner product from the key words
// already in registers, reduced, and multiplied by the correction row once.
__global__ void hoist_mac_kernel(const __grid_constant__ HoistMacArgs A) {
  __shared__ u64 qk[kMaxPos];
  const u32 N = 1u << A.logn, i = blockIdx.y, j = blockIdx.z;
  const LimbDev& M = A.limbs[A.ids[j]];
  if (threadIdx.x < A.L) qk[threadIdx.x] = A.limbs[A.ids[threadIdx.x]].p % M.p;   // [q_k]_{q_j}
  __syncthreads();
  const u32 o = blockIdx.x * blockDim.x + threadIdx.x;
  if (o >= N) return;
  const u32 s = subst_source(o, A.T.exponent[i], A.logn);
  const u64* d = A.adjacent ? A.D + ((((size_t)A.T.src[i] * A.Lk + j) * A.L) << A.logn) + s
                            : A.D + ((((size_t)A.T.src[i] * A.L) * A.Lk + j) << A.logn) + s;
  const size_t dstride = A.adjacent ? (size_t)1 << A.logn : (size_t)A.Lk << A.logn;
  const u32 slot = key_slot(A.keys, i);
  const u64* k0 = A.keys.k0[slot] + (((size_t)j * A.L) << A.logn) + o;
  const u64* k1 = A.keys.k1[slot] + (((size_t)j * A.L) << A.logn) + o;
  Acc192 a0, a1, h0, h1;
  a0.clear();
  a1.clear();
  h0.clear();
  h1.clear();
#pragma unroll 2
  for (u32 k = 0; k < A.L; k++) {
    const u64 t = d[k * dstride], x = __ldg(k0 + ((size_t)k << A.logn)), y = __ldg(k1 + ((size_t)k << A.logn));
    a0.mac(t, x);
    a1.mac(t, y);
    h0.mac(qk[k], x);
    h1.mac(qk[k], y);
  }
  const u64 m = A.mrows[(((size_t)A.T.mrow[i] * A.Lk + j) << A.logn) + o];
  a0.mac(h0.reduce(M), m);
  a1.mac(h1.reduce(M), m);
  if (A.c0) a0.add64(A.c0[A.T.src_ct[i] * A.c0_stride + ((size_t)j << A.logn) + s]);
  u64* out = A.out + A.T.dst[i] * A.out_stride + ((size_t)j << A.logn) + o;
  out[0] = a0.reduce(M);
  out[(size_t)A.Lk << A.logn] = a1.reduce(M);
}

// ------------------------------------------------------------------ linear transforms (DESIGN §3.4)
constexpr u32 kDotCts = 2;      // ciphertexts per thread: each key word loaded serves this many digit rows
constexpr u32 kDotGroups = 8;   // giant groups per thread: each baby-step term computed serves this many groups
struct HoistDotArgs {
  const LtStep* steps;
  const int* fallback;
  const u64 *D, *mrows, *ct, *diag, *fb;
  u64* out;
  size_t ct_stride;
  u32 cts, ct_tiles, diag_ct0, per_ct, n_diags, baby, g0, n_groups, L, logn, adjacent;
  const LimbDev* limbs;
  unsigned short ids[kMaxPos];
};
// One thread per (coefficient o, limb j = blockIdx.z), kDotCts ciphertexts and kDotGroups giant groups
// (blockIdx.x = group tile * ct_tiles + ciphertext tile, fastest): the CTAs resident at any time work on the same
// coefficients and limb of every tile, so each key and digit word they share comes from HBM once and from L2 after.
// Baby step i >= 1 is hoist_mac_kernel's key switch of sigma_i(c1) plus sigma_i(c0), computed once for the thread's
// ciphertexts from one load of the key words; step 0 is the ciphertext itself.  Each term is reduced, multiplied by
// the diagonal of every group of the tile that uses it and added into that group's partial sum; nothing per baby
// step leaves the registers.
__global__ void __launch_bounds__(256) hoist_dot_kernel(const __grid_constant__ HoistDotArgs A) {
  __shared__ u64 qk[kMaxPos];
  const u32 N = 1u << A.logn, j = blockIdx.z;
  const u32 gt = (blockIdx.x / A.ct_tiles) * kDotGroups, t0 = (blockIdx.x % A.ct_tiles) * kDotCts;
  const LimbDev& M = A.limbs[A.ids[j]];
  for (u32 k = threadIdx.x; k < A.L; k += blockDim.x) qk[k] = A.limbs[A.ids[k]].p % M.p;   // [q_k]_{q_j}
  __syncthreads();
  const u32 o = blockIdx.y * blockDim.x + threadIdx.x;
  if (o >= N) return;
  const u32 nt = min(kDotCts, A.cts - t0), ng = min(kDotGroups, A.n_groups - gt), g1 = A.g0 + gt;
  // the tile's first group is full unless it is the last: baby steps beyond its terms serve no group of the tile
  const u32 steps = min(A.baby, A.n_diags - g1 * A.baby);
  const size_t row = (size_t)1 << A.logn, jo = ((size_t)j << A.logn) + o, part1 = (size_t)A.L << A.logn;
  const size_t dstride = A.adjacent ? row : (size_t)A.L << A.logn, plane = ((size_t)A.L * A.L) << A.logn;
  const size_t dbase = A.adjacent ? ((size_t)j * A.L) << A.logn : (size_t)j << A.logn;
  const u64* ct = A.ct + t0 * A.ct_stride;
  u64 r0[kDotGroups][kDotCts], r1[kDotGroups][kDotCts];
#pragma unroll
  for (u32 g = 0; g < kDotGroups; g++)
#pragma unroll
    for (u32 c = 0; c < kDotCts; c++) r0[g][c] = r1[g][c] = 0;
  for (u32 i = 0; i < steps; i++) {
    u64 v0[kDotCts], v1[kDotCts];
    if (i == 0) {
#pragma unroll
      for (u32 c = 0; c < kDotCts; c++)
        if (c < nt) {
          v0[c] = ct[c * A.ct_stride + jo];
          v1[c] = ct[c * A.ct_stride + part1 + jo];
        }
    } else {
      const LtStep S = A.steps[i];
      const u32 s = subst_source(o, S.exponent, A.logn);
      const u64* k0 = S.k0 + (((size_t)j * A.L) << A.logn) + o;
      const u64* k1 = S.k1 + (((size_t)j * A.L) << A.logn) + o;
      const u64* d = A.D + t0 * plane + dbase + s;
      Acc192 a0[kDotCts], a1[kDotCts], h0, h1;
#pragma unroll
      for (u32 c = 0; c < kDotCts; c++) {
        a0[c].clear();
        a1[c].clear();
      }
      h0.clear();
      h1.clear();
      for (u32 k = 0; k < A.L; k++) {
        const u64 x = __ldg(k0 + ((size_t)k << A.logn)), y = __ldg(k1 + ((size_t)k << A.logn));
        h0.mac(qk[k], x);
        h1.mac(qk[k], y);
#pragma unroll
        for (u32 c = 0; c < kDotCts; c++)
          if (c < nt) {
            const u64 t = d[c * plane + k * dstride];
            a0[c].mac(t, x);
            a1[c].mac(t, y);
          }
      }
      const u64 m = A.mrows[(((size_t)i * A.L + j) << A.logn) + o], e0 = h0.reduce(M), e1 = h1.reduce(M);
#pragma unroll
      for (u32 c = 0; c < kDotCts; c++)
        if (c < nt) {
          const int f = A.fallback ? A.fallback[(t0 + c) * A.baby + i] : -1;
          if (f >= 0) {   // rot_i of this ciphertext, computed unhoisted
            v0[c] = A.fb[f * A.ct_stride + jo];
            v1[c] = A.fb[f * A.ct_stride + part1 + jo];
            continue;
          }
          a0[c].mac(e0, m);
          a1[c].mac(e1, m);
          a0[c].add64(ct[c * A.ct_stride + ((size_t)j << A.logn) + s]);
          v0[c] = a0[c].reduce(M);
          v1[c] = a1[c].reduce(M);
        }
    }
#pragma unroll
    for (u32 g = 0; g < kDotGroups; g++) {
      const u32 k = (g1 + g) * A.baby + i;
      if (g >= ng || k >= A.n_diags) continue;
#pragma unroll
      for (u32 c = 0; c < kDotCts; c++)
        if (c < nt) {
          const size_t dk = (A.per_ct ? (size_t)(A.diag_ct0 + t0 + c) * A.n_diags : 0) + k;
          const u64 w = A.diag[dk * part1 + jo];
          r0[g][c] = csub(r0[g][c] + mulmod_limb(v0[c], w, M), M.p);
          r1[g][c] = csub(r1[g][c] + mulmod_limb(v1[c], w, M), M.p);
        }
    }
  }
#pragma unroll
  for (u32 g = 0; g < kDotGroups; g++)
#pragma unroll
    for (u32 c = 0; c < kDotCts; c++)
      if (g < ng && c < nt) {
        u64* out = A.out + ((size_t)(t0 + c) * A.n_groups + gt + g) * A.ct_stride + jo;
        out[0] = r0[g][c];
        out[part1] = r1[g][c];
      }
}

struct SwitchDownArgs {
  SwitchDownDev S;
  const u64* in;
  u64* out;
  u32 polys, L, logn;
  const LimbDev* limbs;
  unsigned short ids[kMaxPos];
};
__global__ void switch_down_kernel(SwitchDownArgs A) {
  const u32 N = 1u << A.logn;
  size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;  // over polys*N
  if (idx >= ((size_t)A.polys << A.logn)) return;
  u32 c = idx & (N - 1);
  size_t poly = idx >> A.logn;
  const u64* src = A.in + ((poly * A.L) << A.logn) + c;
  u64* dst = A.out + ((poly * (A.L - 1)) << A.logn) + c;
  u64 xl = csub(src[(size_t)(A.L - 1) << A.logn] + A.S.q_last_half, A.S.q_last);  // rq/mod.rs:456-458
  for (u32 i = 0; i + 1 < A.L; i++) {
    const LimbDev& M = A.limbs[A.ids[i]];
    u64 tmp = barrett64(xl, M.p, M.bhi, M.blo) + A.S.half_mod[i];   // :469
    u64 v = src[(size_t)i << A.logn] + 3 * M.p - tmp;              // :473
    dst[(size_t)i << A.logn] = mul_shoup(v, A.S.inv[i], A.S.inv_s[i], M.p);  // :476 (always a Shoup pair)
  }
}

// ------------------------------------------------------------------ wire-format bit packing
// transcode_to_bytes / transcode_from_bytes (fhe-util/src/lib.rs:71-146): eight coefficients of nbits bits are
// exactly nbits bytes, so one thread converts one 8-coefficient group.
__global__ void pack_kernel(PackDev P, const u64* words, unsigned char* bytes, size_t n_groups, u32 logn) {
  size_t g = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= n_groups) return;
  const u32 gpr = (1u << logn) >> 3;            // groups per row
  const size_t row = g / gpr;
  const u32 k = (u32)(g % gpr), limb = (u32)(row % P.limbs);
  const u32 nb = P.nbits[limb];
  const u64* src = words + (row << logn) + ((size_t)k << 3);
  unsigned char* dst = bytes + (row / P.limbs) * P.poly_bytes + P.offs[limb] + (size_t)k * nb;
  const u64 mask = nb == 64 ? ~0ull : ((1ull << nb) - 1);
  unsigned __int128 cur = 0;
  u32 have = 0, o = 0;
#pragma unroll
  for (int e = 0; e < 8; e++) {
    cur |= (unsigned __int128)(src[e] & mask) << have;
    have += nb;
    while (have >= 8) {
      dst[o++] = (unsigned char)cur;
      cur >>= 8;
      have -= 8;
    }
  }
}
__global__ void unpack_kernel(PackDev P, const unsigned char* bytes, u64* words, size_t n_groups, u32 logn) {
  size_t g = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= n_groups) return;
  const u32 gpr = (1u << logn) >> 3;
  const size_t row = g / gpr;
  const u32 k = (u32)(g % gpr), limb = (u32)(row % P.limbs);
  const u32 nb = P.nbits[limb];
  const unsigned char* src = bytes + (row / P.limbs) * P.poly_bytes + P.offs[limb] + (size_t)k * nb;
  u64* dst = words + (row << logn) + ((size_t)k << 3);
  const u64 mask = nb == 64 ? ~0ull : ((1ull << nb) - 1);
  unsigned __int128 cur = 0;
  u32 have = 0, o = 0;
#pragma unroll
  for (int e = 0; e < 8; e++) {
    while (have < nb) {
      cur |= (unsigned __int128)src[o++] << have;
      have += 8;
    }
    dst[e] = (u64)cur & mask;
    cur >>= nb;
    have -= nb;
  }
}

// ------------------------------------------------------------------ row transcoding
// Value k of a row of `len` in_bits-bit fields read as one LSB-first bit stream: bits [k*out_bits, (k+1)*out_bits),
// cut at the stream's end (the leftover bits of the reference's last value), zero past it.  Fields are masked to
// in_bits, as the reference's release build does.  It reads elements floor(k*out_bits / in_bits) through
// floor((min((k+1)*out_bits, len*in_bits) - 1) / in_bits), at most ceil(out_bits / in_bits) + 1 of them, so no value
// depends on another.
template <class T>
__device__ __forceinline__ u64 bit_window(const T* row, size_t len, u32 in_bits, u32 out_bits, size_t k) {
  const u64 total = (u64)len * in_bits, b0 = (u64)k * out_bits;
  if (b0 >= total) return 0;
  const u64 b1 = b0 + out_bits < total ? b0 + out_bits : total;
  const u64 in_mask = in_bits == 64 ? ~0ull : ((1ull << in_bits) - 1);
  u64 v = 0;
  for (u64 e = b0 / in_bits, s = e * in_bits; s < b1; e++, s += in_bits) {
    const u64 w = (u64)row[e] & in_mask;
    v |= s >= b0 ? w << (s - b0) : w >> (b0 - s);   // both shifts are below 64
  }
  return out_bits == 64 ? v : v & ((1ull << out_bits) - 1);
}

template <class TI, class TO>
__global__ void transcode_kernel(TranscodeRows T, size_t n_values) {
  const TI* in = (const TI*)T.in;
  TO* out = (TO*)T.out;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_values; i += (size_t)gridDim.x * blockDim.x) {
    const size_t r = i / T.out_len, k = i - r * T.out_len;
    out[r * T.out_stride + k] = (TO)bit_window(in + r * T.in_stride, T.in_len, T.in_bits, T.out_bits, k);
  }
}

// one thread per coefficient of the staged plaintext rows [P][n_ct][N]
__global__ void fold_stage_kernel(const u64* ct, u32 n_ct, u32 parts, size_t row_words, u32 in_bits, u32 out_bits,
                                  u64 E, u64* coeffs, size_t n_words, u32 logn) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_words) return;
  const size_t c = i & ((1ull << logn) - 1), row = i >> logn;
  const size_t p = row / n_ct, j = row - p * n_ct;
  const u64 v = ((u64)p << logn) + c, part = v / E;
  coeffs[i] = part < parts ? bit_window(ct + (j * parts + part) * row_words, row_words, in_bits, out_bits, v - part * E)
                           : 0;
}

// ------------------------------------------------------------------ plaintext encoding
// one thread per (plaintext, coefficient): reads are coalesced for Poly, writes always are
__global__ void encode_load_kernel(const u64* staged, u64* coeffs, size_t n_words, size_t n_values, const u32* inv_map,
                                   u32 is_signed, PlainMod T, u32 logn) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_words) return;
  const u32 c = (u32)i & ((1u << logn) - 1);
  const size_t v = inv_map ? ((i >> logn) << logn) + inv_map[c] : i;
  u64 w = 0;
  if (v < n_values) {
    w = staged[v];
    if (is_signed) {   // zq/mod.rs reduce_i64: the canonical residue of a signed word
      const bool neg = (long long)w < 0;
      const u64 r = barrett64(neg ? 0 - w : w, T.t, T.bhi, T.blo);
      w = (neg && r) ? T.t - r : r;
    }
  }
  coeffs[i] = w;
}

__global__ void to_poly_load_kernel(u64* x, size_t n_words, PlainMod T, u64 q_mod_t) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_words) return;
  x[i] = mulmod(barrett64(x[i], T.t, T.bhi, T.blo), q_mod_t, T.t, T.bhi, T.blo);   // Modulus::scalar_mul_vec
}

struct AddScaledArgs {
  u64* a;
  const u64* m;
  const u64 *delta, *delta_s;
  u32 cts, parts, n_pt, logn, limbs_per_poly, subtract;
  const LimbDev* limbs;
  unsigned short ids[kMaxPos];
};
// delta is a constant in every NTT slot (parameters.rs:604-633), so m * delta is one Shoup product per word
__global__ void add_scaled_kernel(AddScaledArgs A) {
  const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t total = ((size_t)A.cts * A.limbs_per_poly) << A.logn;
  if (idx >= total) return;
  const u32 c = (u32)idx & ((1u << A.logn) - 1);
  const size_t row = idx >> A.logn;
  const u32 j = (u32)(row % A.limbs_per_poly), ct = (u32)(row / A.limbs_per_poly);
  const u64 p = A.limbs[A.ids[j]].p;
  const u64 w = mul_shoup(A.m[((((size_t)(ct % A.n_pt)) * A.limbs_per_poly + j) << A.logn) + c], A.delta[j],
                          A.delta_s[j], p);
  u64* dst = A.a + ((((size_t)ct * A.parts) * A.limbs_per_poly + j) << A.logn) + c;
  const u64 x = *dst;
  *dst = A.subtract ? csub(x + p - w, p) : csub(x + w, p);
}

// ------------------------------------------------------------------ decryption (keys/secret_key.rs:55-98, :198-260)
struct PhaseArgs {
  const u64* ct;   // [cts][parts][L][N]
  const u64* s;    // row j: s modulo the j-th limb
  u64* out;        // [cts][L][N]
  u32 cts, parts, logn, limbs_per_poly;
  const LimbDev* limbs;
  unsigned short ids[kMaxPos];
};
// c0 + c1 s + c2 s^2 + ... as a Horner sum, one coefficient per thread.  Every product and sum is reduced to the
// canonical residue (the reference's sum of canonical terms gives the same word).  No branch depends on the data.
__global__ void phase_kernel(PhaseArgs A) {
  const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t total = ((size_t)A.cts * A.limbs_per_poly) << A.logn;
  if (idx >= total) return;
  const u32 c = (u32)idx & ((1u << A.logn) - 1);
  const size_t row = idx >> A.logn;
  const u32 j = (u32)(row % A.limbs_per_poly), ct = (u32)(row / A.limbs_per_poly);
  const LimbDev& M = A.limbs[A.ids[j]];
  const u64 s = A.s[((size_t)j << A.logn) + c];
  const size_t stride = (size_t)A.limbs_per_poly << A.logn;
  const u64* src = A.ct + (size_t)ct * A.parts * stride + ((size_t)j << A.logn) + c;
  u64 acc = src[(size_t)(A.parts - 1) * stride];
  for (int p = (int)A.parts - 2; p >= 0; p--) acc = csub(mulmod_limb(acc, s, M) + src[(size_t)p * stride], M.p);
  A.out[idx] = acc;
}

// w = ((v + t) mod q_0) mod t on row 0 of the scaled phase (secret_key.rs:228-236): two Barrett reductions, no branch
__global__ void decrypt_epilogue_kernel(u64* v, size_t n_words, PlainMod Q0, PlainMod T) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_words) return;
  v[i] = barrett64(barrett64(v[i] + T.t, Q0.t, Q0.bhi, Q0.blo), T.t, T.bhi, T.blo);
}

// Plaintext::from_shares' lift (mbfv/secret_key_switch.rs:164-173) over a plaintext context of two or more moduli, from
// limb 0 of the scaled value v = round(t x / Q), x the centred lift of the phase: |v| <= t / 2 < q_0 / 2, so v < 0
// exactly when its residue r > q_0 / 2, and w = ((v + t) mod Q_p) mod t = (r + t - (v < 0 ? q_0 : 0)) mod t, as a
// select
__global__ void from_shares_epilogue_kernel(u64* v, size_t n_words, u64 q0, PlainMod T) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_words) return;
  const u64 r = v[i];
  v[i] = barrett64(r + T.t - (r > (q0 >> 1) ? q0 : 0), T.t, T.bhi, T.blo);
}

// Modulus::center (zq/mod.rs:448-457): a - t when a >= t >> 1, else a, as a select
__global__ void center_kernel(u64* x, size_t n_words, u64 t) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_words) return;
  const u64 a = x[i];
  x[i] = a >= (t >> 1) ? a - t : a;
}

struct NoiseArgs {
  const u64* x;         // [cts][L][N] power basis, canonical
  u32* out;             // [cts]
  const u64* garner;    // [L][L]: entry (i, j), j < i, is q_j^-1 mod q_i
  const u64* q_words;   // Q, W little-endian 64-bit words
  u32 L, W, logn;
  const LimbDev* limbs;   // limb j of the context is limbs[j]
};
// the bit length of a W-word integer
__device__ __forceinline__ u32 bits_of(const u64* a, u32 W) {
  for (int w = (int)W - 1; w >= 0; w--)
    if (a[w]) return 64u * (u32)w + 64u - (u32)__clzll((long long)a[w]);
  return 0;
}
// measure_noise's per-coefficient term min(bits(x), bits(Q - x)) (secret_key.rs:85-95) for the CRT lift x in [0, Q):
// Garner's mixed-radix digits y_i (x = y_0 + y_1 q_0 + y_2 q_0 q_1 + ...), then a Horner sum into W words.  Exact for
// every x.  The maximum over a block goes to out[ct] with one atomic.  Variable time, as the reference's unsafe fn.
__global__ void __launch_bounds__(256) noise_kernel(NoiseArgs A) {
  constexpr int kMax = 32;   // limbs of a context (parameter sets have fewer than 32 moduli)
  const u32 N = 1u << A.logn, ct = blockIdx.y;
  const u32 c = blockIdx.x * blockDim.x + threadIdx.x;
  u32 noise = 0;
  if (c < N) {
    const u64* src = A.x + (((size_t)ct * A.L) << A.logn) + c;
    u64 y[kMax], X[kMax];
    for (u32 i = 0; i < A.L; i++) {
      const LimbDev& M = A.limbs[i];
      u64 r = src[(size_t)i << A.logn];
      for (u32 j = 0; j < i; j++) {
        const u64 yj = barrett64(y[j], M.p, M.bhi, M.blo);
        r = mulmod_limb(csub(r + M.p - yj, M.p), A.garner[(size_t)i * A.L + j], M);
      }
      y[i] = r;
    }
    for (u32 w = 0; w < A.W; w++) X[w] = 0;
    for (int i = (int)A.L - 1; i >= 0; i--) {   // X = X * q_i + y_i
      u64 carry = y[i];
      const u64 q = A.limbs[i].p;
      for (u32 w = 0; w < A.W; w++) {
        const unsigned __int128 p = (unsigned __int128)X[w] * q + carry;
        X[w] = (u64)p;
        carry = (u64)(p >> 64);
      }
    }
    const u32 bx = bits_of(X, A.W);
    u64 borrow = 0;
    for (u32 w = 0; w < A.W; w++) {   // X <- Q - X
      const u64 a = A.q_words[w], b = X[w];
      const u64 d = a - b - borrow;
      borrow = (a < b) || (a - b < borrow);
      X[w] = d;
    }
    noise = min(bx, bits_of(X, A.W));
  }
  noise = __reduce_max_sync(0xffffffffu, noise);
  __shared__ u32 s_max[8];
  if ((threadIdx.x & 31) == 0) s_max[threadIdx.x >> 5] = noise;
  __syncthreads();
  if (threadIdx.x == 0) {
    u32 m = 0;
    for (u32 w = 0; w < (blockDim.x + 31) / 32; w++) m = max(m, s_max[w]);
    atomicMax(A.out + ct, m);
  }
}

// ------------------------------------------------------------------ encryption (keys/secret_key.rs:100-136,
// keys/public_key.rs:45-92) and key generation.  The random words come from the seeded ChaCha20 stream of
// include/fhe_b200.h: block b of the row (ciphertext or key ct, role, limb, digit) is the RFC 8439 block function of
// the state (constants, seed, b, ct, role << 8 | limb, digit); value m of the block (u64 words 2m, 2m + 1) drives
// coefficient 4b + m.  Encryption rows have digit 0.
__device__ __forceinline__ void chacha_qr(u32& a, u32& b, u32& c, u32& d) {
  a += b; d = __funnelshift_l(d ^ a, d ^ a, 16);
  c += d; b = __funnelshift_l(b ^ c, b ^ c, 12);
  a += b; d = __funnelshift_l(d ^ a, d ^ a, 8);
  c += d; b = __funnelshift_l(b ^ c, b ^ c, 7);
}
// the four 128-bit values (lo[m], hi[m]) of one block
__device__ __forceinline__ void chacha_block(const EncSeed& K, u32 b, u32 ct, u32 role_limb, u32 digit, u64 (&lo)[4],
                                             u64 (&hi)[4]) {
  const u32 in[16] = {0x61707865u, 0x3320646eu, 0x79622d32u, 0x6b206574u, K.w[0], K.w[1], K.w[2], K.w[3],
                      K.w[4],      K.w[5],      K.w[6],      K.w[7],      b,      ct,     role_limb, digit};
  u32 x[16];
#pragma unroll
  for (int i = 0; i < 16; i++) x[i] = in[i];
#pragma unroll 2
  for (int r = 0; r < 10; r++) {
    chacha_qr(x[0], x[4], x[8], x[12]);
    chacha_qr(x[1], x[5], x[9], x[13]);
    chacha_qr(x[2], x[6], x[10], x[14]);
    chacha_qr(x[3], x[7], x[11], x[15]);
    chacha_qr(x[0], x[5], x[10], x[15]);
    chacha_qr(x[1], x[6], x[11], x[12]);
    chacha_qr(x[2], x[7], x[8], x[13]);
    chacha_qr(x[3], x[4], x[9], x[14]);
  }
#pragma unroll
  for (int m = 0; m < 4; m++) {
    lo[m] = (u64)(x[4 * m] + in[4 * m]) | ((u64)(x[4 * m + 1] + in[4 * m + 1]) << 32);
    hi[m] = (u64)(x[4 * m + 2] + in[4 * m + 2]) | ((u64)(x[4 * m + 3] + in[4 * m + 3]) << 32);
  }
}

struct EncSkArgs {
  const u64* s;       // row j: s modulo the j-th limb (NTT)
  const u64* e;       // [cts][L][N] NTT of the error
  u64* out;           // [cts][2][L][N]
  EncSeed K;
  u32 cts, ct_base, logn, limbs_per_poly;
  const LimbDev* limbs;
  unsigned short ids[kMaxPos];
};
// SecretKey::encrypt_poly up to + m: a = (hi 2^64 + lo) mod q_j drawn as NTT words (Poly::random_from_seed into Ntt),
// part 1 = a, part 0 = e - a s.  One thread per (ciphertext, limb, 4 coefficients): a never leaves the registers.  No
// branch depends on the data.
__global__ void encrypt_sk_kernel(EncSkArgs A) {
  const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const u32 g_per_row = 1u << (A.logn - 2);
  const size_t total = (size_t)A.cts * A.limbs_per_poly * g_per_row;
  if (idx >= total) return;
  const u32 g = (u32)(idx % g_per_row);
  const size_t row = idx / g_per_row;
  const u32 j = (u32)(row % A.limbs_per_poly), ct = (u32)(row / A.limbs_per_poly);
  const LimbDev& M = A.limbs[A.ids[j]];
  u64 lo[4], hi[4];
  chacha_block(A.K, g, A.ct_base + ct, j, 0, lo, hi);   // role 0 (a), limb j
  const size_t c = (size_t)g * 4;
  const ulonglong2* sp = reinterpret_cast<const ulonglong2*>(A.s + ((size_t)j << A.logn) + c);
  const ulonglong2* ep = reinterpret_cast<const ulonglong2*>(A.e + (row << A.logn) + c);
  const ulonglong2 s01 = sp[0], s23 = sp[1], e01 = ep[0], e23 = ep[1];
  const u64 s[4] = {s01.x, s01.y, s23.x, s23.y}, e[4] = {e01.x, e01.y, e23.x, e23.y};
  u64 a[4], b[4];
#pragma unroll
  for (int m = 0; m < 4; m++) {
    a[m] = reduce128_limb(lo[m], hi[m], M);
    b[m] = csub(e[m] + M.p - mulmod_limb(a[m], s[m], M), M.p);
  }
  const size_t stride = (size_t)A.limbs_per_poly << A.logn;
  u64* b_row = A.out + (size_t)ct * 2 * stride + ((size_t)j << A.logn) + c;
  reinterpret_cast<ulonglong2*>(b_row)[0] = make_ulonglong2(b[0], b[1]);
  reinterpret_cast<ulonglong2*>(b_row)[1] = make_ulonglong2(b[2], b[3]);
  reinterpret_cast<ulonglong2*>(b_row + stride)[0] = make_ulonglong2(a[0], a[1]);
  reinterpret_cast<ulonglong2*>(b_row + stride)[1] = make_ulonglong2(a[2], a[3]);
}

struct CbdArgs {
  u64* out;           // [cts][n_roles][L][N]
  EncSeed K;
  u64 add_lo, add_hi, sub_lo, sub_hi;   // mask_add = low 2 variance bits, mask_sub = the next 2 variance bits
  u32 cts, ct_base, role0, n_roles, logn, limbs_per_poly;
  u32 digits;         // rows per key: row c of the call is digit c % digits of key c / digits (encryption: 1)
  const LimbDev* limbs;
  unsigned short ids[kMaxPos];
};
// Poly::small (rq/mod.rs, fhe-util sample_vec_cbd): x = popc(v & mask_add) - popc(v & mask_sub) on the 128-bit value
// of the (ct, role, limb 0, digit) row, written as its canonical residue into every limb of the level (q_j - |x| for
// x < 0, by a select).  One thread per (ciphertext or (key, digit), role, 4 coefficients).
__global__ void cbd_kernel(CbdArgs A) {
  const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const u32 g_per_row = 1u << (A.logn - 2);
  const size_t total = (size_t)A.cts * A.n_roles * g_per_row;
  if (idx >= total) return;
  const u32 g = (u32)(idx % g_per_row);
  const size_t poly = idx / g_per_row;
  const u32 r = (u32)(poly % A.n_roles), row = A.ct_base + (u32)(poly / A.n_roles);
  u64 lo[4], hi[4];
  chacha_block(A.K, g, row / A.digits, (A.role0 + r) << 8, row % A.digits, lo, hi);
  long long x[4];
#pragma unroll
  for (int m = 0; m < 4; m++)
    x[m] = (long long)(__popcll(lo[m] & A.add_lo) + __popcll(hi[m] & A.add_hi)) -
           (long long)(__popcll(lo[m] & A.sub_lo) + __popcll(hi[m] & A.sub_hi));
  const size_t c = (size_t)g * 4;
  u64* dst = A.out + ((poly * A.limbs_per_poly) << A.logn) + c;
  for (u32 j = 0; j < A.limbs_per_poly; j++) {
    const u64 p = A.limbs[A.ids[j]].p;
    u64 w[4];
#pragma unroll
    for (int m = 0; m < 4; m++) w[m] = (u64)x[m] + (p & (u64)(x[m] >> 63));
    reinterpret_cast<ulonglong2*>(dst)[0] = make_ulonglong2(w[0], w[1]);
    reinterpret_cast<ulonglong2*>(dst)[1] = make_ulonglong2(w[2], w[3]);
    dst += (size_t)1 << A.logn;
  }
}

struct EncPkArgs {
  const u64* uee;     // [cts][3][L][N]: u, e1, e2 (NTT)
  const u64* pk;      // [2][L][N] (NTT, at the level)
  u64* out;           // [cts][2][L][N]
  u32 cts, logn, limbs_per_poly;
  const LimbDev* limbs;
  unsigned short ids[kMaxPos];
};
// PublicKey::try_encrypt up to + m: c0 = u pk0 + e1, c1 = u pk1 + e2, one coefficient per thread
__global__ void encrypt_pk_kernel(EncPkArgs A) {
  const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t stride = (size_t)A.limbs_per_poly << A.logn;
  if (idx >= (size_t)A.cts * stride) return;
  const size_t ct = idx / stride, in_ct = idx % stride;
  const u32 j = (u32)(in_ct >> A.logn);
  const LimbDev& M = A.limbs[A.ids[j]];
  const u64* src = A.uee + ct * 3 * stride + in_ct;
  const u64 u = src[0], e1 = src[stride], e2 = src[2 * stride];
  u64* dst = A.out + ct * 2 * stride + in_ct;
  dst[0] = csub(mulmod_limb(u, A.pk[in_ct], M) + e1, M.p);
  dst[stride] = csub(mulmod_limb(u, A.pk[stride + in_ct], M) + e2, M.p);
}

struct KskGenArgs {
  const u64* s;       // row j: s modulo the j-th limb (NTT)
  const u64* e;       // [digits][Lk][N]: NTT(e_i) of the digits digit0 .. digit0 + digits - 1
  const u64* x;       // [L_ct][N]: the key's x at the ciphertext level (NTT)
  u64 *k0, *k1;       // the key, [Lk][n_dig][N]
  EncSeed K;
  u32 key, digit0, digits, n_dig, logn, limbs_per_poly, decomp;
  const LimbDev* limbs;
  // G as Shoup pairs: RNS digits G[i][j] = (i == j) g[j]; decomposition G[i][0] = g[i]
  u64 g[kMaxPos], g_s[kMaxPos];
  unsigned short ids[kMaxPos];
};
// KeySwitchingKey::new (key_switching_key.rs:71-238) in the NTT domain, for digits of one key: c1 = (hi 2^64 + lo) mod
// q_j of the role-5 row (key, limb j, digit i), c0 = NTT(e_i) - c1 s + G[i][j] x.  One thread per (digit, key limb, 4
// coefficients); both words go from the registers straight into the [limb][digit][N] layout the key switch reads.
// x is read only where G[i][j] is not zero, which depends on the indices alone; no branch depends on the data.
__global__ void ksk_gen_kernel(KskGenArgs A) {
  const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const u32 g_per_row = 1u << (A.logn - 2);
  const size_t total = (size_t)A.digits * A.limbs_per_poly * g_per_row;
  if (idx >= total) return;
  const u32 g = (u32)(idx % g_per_row);
  const size_t row = idx / g_per_row;
  const u32 j = (u32)(row % A.limbs_per_poly), d = (u32)(row / A.limbs_per_poly), i = A.digit0 + d;
  const LimbDev& M = A.limbs[A.ids[j]];
  u64 lo[4], hi[4];
  chacha_block(A.K, g, A.key, (5u << 8) | j, i, lo, hi);   // role 5 (c1), limb j, digit i
  const size_t c = (size_t)g * 4;
  const ulonglong2* sp = reinterpret_cast<const ulonglong2*>(A.s + ((size_t)j << A.logn) + c);
  const ulonglong2* ep = reinterpret_cast<const ulonglong2*>(A.e + (row << A.logn) + c);
  const ulonglong2 s01 = sp[0], s23 = sp[1], e01 = ep[0], e23 = ep[1];
  const u64 s[4] = {s01.x, s01.y, s23.x, s23.y}, e[4] = {e01.x, e01.y, e23.x, e23.y};
  const u32 gi = A.decomp ? i : j;
  u64 x[4] = {0, 0, 0, 0};
  if (A.decomp || i == j) {
    const ulonglong2* xp = reinterpret_cast<const ulonglong2*>(A.x + ((size_t)(A.decomp ? 0 : j) << A.logn) + c);
    const ulonglong2 x01 = xp[0], x23 = xp[1];
    x[0] = x01.x; x[1] = x01.y; x[2] = x23.x; x[3] = x23.y;
  }
  const u64 gw = A.g[gi], gw_s = A.g_s[gi];
  u64 a[4], b[4];
#pragma unroll
  for (int m = 0; m < 4; m++) {
    a[m] = reduce128_limb(lo[m], hi[m], M);
    b[m] = csub(e[m] + M.p - mulmod_limb(a[m], s[m], M), M.p);
    b[m] = csub(b[m] + mul_shoup(x[m], gw, gw_s, M.p), M.p);
  }
  const size_t off = ((size_t)j * A.n_dig + i) << A.logn;
  reinterpret_cast<ulonglong2*>(A.k0 + off + c)[0] = make_ulonglong2(b[0], b[1]);
  reinterpret_cast<ulonglong2*>(A.k0 + off + c)[1] = make_ulonglong2(b[2], b[3]);
  reinterpret_cast<ulonglong2*>(A.k1 + off + c)[0] = make_ulonglong2(a[0], a[1]);
  reinterpret_cast<ulonglong2*>(A.k1 + off + c)[1] = make_ulonglong2(a[2], a[3]);
}

// ------------------------------------------------------------------ multiparty BFV (fhe::mbfv)
struct CrpArgs {
  u64* out;           // [cts][L][N]
  EncSeed K;
  u32 cts, ct_base, logn, limbs_per_poly;
  const LimbDev* limbs;
  unsigned short ids[kMaxPos];
};
// CommonRandomPoly::new_leveled (crp.rs:35-43): (hi 2^64 + lo) mod q_j of the role-7 row (crp, limb j), drawn directly
// as NTT words.  One thread per (crp, limb, 4 coefficients).
__global__ void crp_kernel(CrpArgs A) {
  const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const u32 g_per_row = 1u << (A.logn - 2);
  const size_t total = (size_t)A.cts * A.limbs_per_poly * g_per_row;
  if (idx >= total) return;
  const u32 g = (u32)(idx % g_per_row);
  const size_t row = idx / g_per_row;
  const u32 j = (u32)(row % A.limbs_per_poly), ct = (u32)(row / A.limbs_per_poly);
  const LimbDev& M = A.limbs[A.ids[j]];
  u64 lo[4], hi[4];
  chacha_block(A.K, g, A.ct_base + ct, (7u << 8) | j, 0, lo, hi);
  u64 a[4];
#pragma unroll
  for (int m = 0; m < 4; m++) a[m] = reduce128_limb(lo[m], hi[m], M);
  u64* dst = A.out + (row << A.logn) + (size_t)g * 4;
  reinterpret_cast<ulonglong2*>(dst)[0] = make_ulonglong2(a[0], a[1]);
  reinterpret_cast<ulonglong2*>(dst)[1] = make_ulonglong2(a[2], a[3]);
}

struct MbfvShareArgs {
  const u64* s;       // row j: s modulo the j-th limb (NTT)
  const u64* s_out;   // SHARE_SKS: the output key's rows, or null for DecryptionShare's zero key
  const u64* x;       // SHARE_PK: crp [cts][L][N]; SHARE_SKS / SHARE_PKS: the ciphertexts [cts][2][L][N];
                      // SHARE_RKG1: crp a_i [cts][L][N]; SHARE_RKG2: round-1 aggregate h0_i [cts][L][N]
  const u64* pk;      // SHARE_PKS: the public key at the level, [2][L][N]; SHARE_RKG2: round-1 aggregate h1_i
  const u64* u;       // SHARE_RKG1 / SHARE_RKG2: the generator's u, rows as s
  const u64* e;       // SHARE_PK / SHARE_SKS: [cts][L][N]; SHARE_PKS: [cts][3][L][N] = (u, e0, e1);
                      // SHARE_RKG1 / SHARE_RKG2: [cts][2][L][N] = (e0, e1), all NTT
  u64* out;           // SHARE_PK / SHARE_SKS: [cts][L][N]; SHARE_PKS: [cts][2][L][N]; SHARE_RKG*: h0 [cts][L][N]
  u64* out1;          // SHARE_RKG1 / SHARE_RKG2: h1 [cts][L][N]
  u32 cts, ct_base, logn, limbs_per_poly;
  const LimbDev* limbs;
  unsigned short ids[kMaxPos];
};
// The share of one protocol in one pass, one coefficient per thread, every term a canonical residue:
//  SHARE_PK  (public_key_gen.rs:32-58):    p0 = -crp s + e
//  SHARE_SKS (secret_key_switch.rs:38-96): h = (s_in - s_out) c1 + e
//  SHARE_PKS (public_key_switch.rs:33-93): (h0, h1) = (u pk0 + s c1 + e0, u pk1 + e1)
//  SHARE_RKG1 (relin_key_gen.rs:112-198), item i = ct_base + ct: (h0_i, h1_i) = (-a_i u + w_i s + e0, a_i s + e1), w_i
//    the Garner coefficient of the level-0 basis: w_i s is s on limb i and 0 on the others (a select on the indices)
//  SHARE_RKG2 (relin_key_gen.rs:224-297): (h0'_i, h1'_i) = (h0_i s + e0, h1_i (u - s) + e1)
// No branch depends on the data (s_out == null is a property of the call).
template <int P>
__global__ void mbfv_share_kernel(MbfvShareArgs A) {
  const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t stride = (size_t)A.limbs_per_poly << A.logn;
  if (idx >= (size_t)A.cts * stride) return;
  const size_t ct = idx / stride, in_ct = idx % stride;
  const u32 j = (u32)(in_ct >> A.logn);
  const LimbDev& M = A.limbs[A.ids[j]];
  const u64 s = A.s[in_ct];
  if (P == SHARE_PK) {
    A.out[idx] = csub(A.e[idx] + M.p - mulmod_limb(A.x[idx], s, M), M.p);
  } else if (P == SHARE_SKS) {
    const u64 so = A.s_out ? A.s_out[in_ct] : 0;
    const u64 c1 = A.x[(2 * ct + 1) * stride + in_ct];
    A.out[idx] = csub(mulmod_limb(csub(s + M.p - so, M.p), c1, M) + A.e[idx], M.p);
  } else if (P == SHARE_RKG1) {
    const u64 a = A.x[idx], u = A.u[in_ct];
    const u64 ws = (j == A.ct_base + (u32)ct) ? s : 0;
    const u64* ee = A.e + ct * 2 * stride + in_ct;
    A.out[idx] = csub(csub(ee[0] + M.p - mulmod_limb(a, u, M), M.p) + ws, M.p);
    A.out1[idx] = csub(mulmod_limb(a, s, M) + ee[stride], M.p);
  } else if (P == SHARE_RKG2) {
    const u64 u = A.u[in_ct];
    const u64* ee = A.e + ct * 2 * stride + in_ct;
    A.out[idx] = csub(mulmod_limb(A.x[idx], s, M) + ee[0], M.p);
    A.out1[idx] = csub(mulmod_limb(A.pk[idx], csub(u + M.p - s, M.p), M) + ee[stride], M.p);
  } else {
    const u64* uee = A.e + ct * 3 * stride + in_ct;
    const u64 u = uee[0], e0 = uee[stride], e1 = uee[2 * stride];
    const u64 c1 = A.x[(2 * ct + 1) * stride + in_ct];
    u64* dst = A.out + ct * 2 * stride + in_ct;
    dst[0] = csub(csub(mulmod_limb(u, A.pk[in_ct], M) + mulmod_limb(s, c1, M), M.p) + e0, M.p);
    dst[stride] = csub(mulmod_limb(u, A.pk[stride + in_ct], M) + e1, M.p);
  }
}

struct SumArgs {
  const u64* src[kSumGroup];   // item k of source i at src[i] + k * src_stride
  const u64* base;             // nullable, item k at base + k * base_stride
  u64* out;                    // item k at out + k * out_stride
  size_t src_stride, base_stride, out_stride, item_words;
  size_t base_row, out_row;    // row r of a base / out item at + r * base_row / out_row (N: contiguous rows)
  u32 n_src, items, logn, limbs_per_poly;
  const LimbDev* limbs;
  unsigned short ids[kMaxPos];
};
// out = base + sum_i src_i, two words per thread.  The words are canonical (< 2^62): the sum is accumulated in 128 bits
// with a carry count and reduced once per word, so every source word is read once and the reduction count does not grow
// with the number of sources.
__global__ void shares_sum_kernel(SumArgs A) {
  const size_t i = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) * 2;
  if (i >= (size_t)A.items * A.item_words) return;
  const size_t item = i / A.item_words, w = i % A.item_words;
  const size_t r = w >> A.logn, c = w & ((1u << A.logn) - 1);
  const LimbDev& M = A.limbs[A.ids[(u32)r % A.limbs_per_poly]];
  u64 lo0 = 0, lo1 = 0, hi0 = 0, hi1 = 0;
  if (A.base) {
    const ulonglong2 b = *reinterpret_cast<const ulonglong2*>(A.base + item * A.base_stride + r * A.base_row + c);
    lo0 = b.x;
    lo1 = b.y;
  }
  const size_t off = item * A.src_stride + w;
  for (u32 k = 0; k < A.n_src; k++) {
    const ulonglong2 v = *reinterpret_cast<const ulonglong2*>(A.src[k] + off);
    lo0 += v.x;
    hi0 += lo0 < v.x;
    lo1 += v.y;
    hi1 += lo1 < v.y;
  }
  *reinterpret_cast<ulonglong2*>(A.out + item * A.out_stride + r * A.out_row + c) =
      make_ulonglong2(reduce128_limb(lo0, hi0, M), reduce128_limb(lo1, hi1, M));
}

struct SegSumArgs {
  const u64* in;               // input item j at in + j * in_stride
  u64 *out0, *out1;            // rows r < split_rows of out item g at out0 + g * out0_stride + r * N, the rest in out1
  size_t in_stride, out0_stride, out1_stride, item_words;
  u32 n_terms, groups, split_rows, logn, limbs_per_poly, accumulate;
  const LimbDev* limbs;
  unsigned short ids[kMaxPos];
};
// out[g] = (accumulate ? out[g] : 0) + sum_i in[g * n_terms + i], two words per thread.  The words are canonical
// (< 2^62), so the 128-bit sum with a carry count holds any n_terms < 2^32 (< 2^94) and is reduced once.  Memory
// bound: four terms (eight words) in flight per trip; the branch on the row only picks the output buffer.
__global__ void segment_sum_kernel(SegSumArgs A) {
  const size_t i = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) * 2;
  if (i >= (size_t)A.groups * A.item_words) return;
  const size_t g = i / A.item_words, w = i % A.item_words;
  const u32 r = (u32)(w >> A.logn), c = (u32)w & ((1u << A.logn) - 1);
  const LimbDev& M = A.limbs[A.ids[r % A.limbs_per_poly]];
  u64* o = r < A.split_rows ? A.out0 + g * A.out0_stride + ((size_t)r << A.logn) + c
                            : A.out1 + g * A.out1_stride + ((size_t)(r - A.split_rows) << A.logn) + c;
  u64 lo0 = 0, lo1 = 0, hi0 = 0, hi1 = 0;
  if (A.accumulate) {
    const ulonglong2 b = *reinterpret_cast<const ulonglong2*>(o);
    lo0 = b.x;
    lo1 = b.y;
  }
  const u64* p = A.in + g * A.n_terms * A.in_stride + w;
  u32 k = 0;
  for (; k + 4 <= A.n_terms; k += 4) {
    ulonglong2 v[4];
#pragma unroll
    for (int j = 0; j < 4; j++) v[j] = *reinterpret_cast<const ulonglong2*>(p + (size_t)(k + j) * A.in_stride);
#pragma unroll
    for (int j = 0; j < 4; j++) {
      lo0 += v[j].x;
      hi0 += lo0 < v[j].x;
      lo1 += v[j].y;
      hi1 += lo1 < v[j].y;
    }
  }
  for (; k < A.n_terms; k++) {
    const ulonglong2 v = *reinterpret_cast<const ulonglong2*>(p + (size_t)k * A.in_stride);
    lo0 += v.x;
    hi0 += lo0 < v.x;
    lo1 += v.y;
    hi1 += lo1 < v.y;
  }
  *reinterpret_cast<ulonglong2*>(o) = make_ulonglong2(reduce128_limb(lo0, hi0, M), reduce128_limb(lo1, hi1, M));
}

void copy_ids(unsigned short* dst, const RowIds& ids) {
  for (int i = 0; i < kMaxPos; i++) dst[i] = ids.ids[i];
}

}  // namespace

void launch_crp(u64* out, u32 cts, u32 ct_base, const EncSeed& K, const RowIds& ids, const LimbDev* limbs, u32 logn,
                cudaStream_t st) {
  CrpArgs A;
  A.out = out; A.K = K; A.cts = cts; A.ct_base = ct_base; A.logn = logn; A.limbs_per_poly = ids.limbs_per_poly;
  A.limbs = limbs;
  copy_ids(A.ids, ids);
  const size_t total = ((size_t)cts * ids.limbs_per_poly) << (logn - 2);
  if (!total) return;
  crp_kernel<<<(unsigned)((total + 127) / 128), 128, 0, st>>>(A);
  g_launches++;
}

void launch_mbfv_share(MbfvShare kind, const u64* s, const u64* s_out, const u64* x, const u64* pk, const u64* e,
                       u64* out, u32 cts, const RowIds& ids, const LimbDev* limbs, u32 logn, cudaStream_t st,
                       const u64* u, u64* out1, u32 ct_base) {
  MbfvShareArgs A;
  A.s = s; A.s_out = s_out; A.x = x; A.pk = pk; A.u = u; A.e = e; A.out = out; A.out1 = out1; A.cts = cts;
  A.ct_base = ct_base; A.logn = logn;
  A.limbs_per_poly = ids.limbs_per_poly; A.limbs = limbs;
  copy_ids(A.ids, ids);
  const size_t total = ((size_t)cts * ids.limbs_per_poly) << logn;
  if (!total) return;
  const unsigned blocks = (unsigned)((total + 255) / 256);
  if (kind == SHARE_PK) mbfv_share_kernel<SHARE_PK><<<blocks, 256, 0, st>>>(A);
  else if (kind == SHARE_SKS) mbfv_share_kernel<SHARE_SKS><<<blocks, 256, 0, st>>>(A);
  else if (kind == SHARE_PKS) mbfv_share_kernel<SHARE_PKS><<<blocks, 256, 0, st>>>(A);
  else if (kind == SHARE_RKG1) mbfv_share_kernel<SHARE_RKG1><<<blocks, 256, 0, st>>>(A);
  else mbfv_share_kernel<SHARE_RKG2><<<blocks, 256, 0, st>>>(A);
  g_launches++;
}

void launch_shares_sum(const u64* const* src, u32 n_src, size_t src_stride, const u64* base, size_t base_stride,
                       u64* out, size_t out_stride, u32 items, size_t item_words, const RowIds& ids,
                       const LimbDev* limbs, u32 logn, cudaStream_t st, size_t out_row) {
  const size_t total = (size_t)items * item_words;
  if (!total || !n_src) return;
  const size_t N = (size_t)1 << logn;
  SumArgs A;
  A.out = out; A.src_stride = src_stride; A.out_stride = out_stride; A.item_words = item_words; A.items = items;
  A.out_row = out_row ? out_row : N;
  A.logn = logn; A.limbs_per_poly = ids.limbs_per_poly; A.limbs = limbs;
  copy_ids(A.ids, ids);
  // one launch per group of kSumGroup sources; every group after the first adds to what the previous one wrote.  A
  // source that is also the output goes into the first group, which reads it before anything is written.
  std::vector<const u64*> order(src, src + n_src);
  for (u32 k = 0; k < n_src; k++)
    if (order[k] == out) std::swap(order[k], order[0]);
  for (u32 g0 = 0; g0 < n_src; g0 += kSumGroup) {
    A.n_src = std::min(kSumGroup, n_src - g0);
    for (u32 k = 0; k < A.n_src; k++) A.src[k] = order[g0 + k];
    A.base = g0 ? out : base;
    A.base_stride = g0 ? out_stride : base_stride;
    A.base_row = g0 ? A.out_row : N;
    shares_sum_kernel<<<(unsigned)((total / 2 + 255) / 256), 256, 0, st>>>(A);
    g_launches++;
  }
}

void launch_segment_sum(const u64* in, size_t in_stride, u32 n_terms, u64* out0, size_t out0_stride, u64* out1,
                        size_t out1_stride, u32 split_rows, u32 groups, size_t item_words, bool accumulate,
                        const RowIds& ids, const LimbDev* limbs, u32 logn, cudaStream_t st) {
  const size_t total = (size_t)groups * item_words;
  if (!total) return;
  SegSumArgs A;
  A.in = in; A.out0 = out0; A.out1 = out1;
  A.in_stride = in_stride; A.out0_stride = out0_stride; A.out1_stride = out1_stride; A.item_words = item_words;
  A.n_terms = n_terms; A.groups = groups; A.split_rows = split_rows; A.logn = logn;
  A.limbs_per_poly = ids.limbs_per_poly; A.accumulate = accumulate ? 1 : 0; A.limbs = limbs;
  copy_ids(A.ids, ids);
  segment_sum_kernel<<<(unsigned)((total / 2 + 255) / 256), 256, 0, st>>>(A);
  g_launches++;
}

void launch_encode_load(const u64* staged, u64* coeffs, u32 n_pt, size_t n_values, const u32* inv_map, bool is_signed,
                        const PlainMod& T, u32 logn, cudaStream_t st) {
  const size_t n_words = (size_t)n_pt << logn;
  if (!n_words) return;
  encode_load_kernel<<<(unsigned)((n_words + 255) / 256), 256, 0, st>>>(staged, coeffs, n_words, n_values, inv_map,
                                                                         is_signed ? 1 : 0, T, logn);
  g_launches++;
}

void launch_to_poly_load(u64* x, size_t n_words, const PlainMod& T, u64 q_mod_t, cudaStream_t st) {
  if (!n_words) return;
  to_poly_load_kernel<<<(unsigned)((n_words + 255) / 256), 256, 0, st>>>(x, n_words, T, q_mod_t);
  g_launches++;
}

void launch_add_scaled(u64* a, const u64* m, u32 cts, u32 parts, u32 n_pt, const u64* delta, const u64* delta_s,
                       bool subtract, const RowIds& ids, const LimbDev* limbs, u32 logn, cudaStream_t st) {
  AddScaledArgs A;
  A.a = a; A.m = m; A.delta = delta; A.delta_s = delta_s;
  A.cts = cts; A.parts = parts; A.n_pt = n_pt; A.logn = logn; A.limbs_per_poly = ids.limbs_per_poly;
  A.subtract = subtract ? 1 : 0;
  A.limbs = limbs;
  copy_ids(A.ids, ids);
  const size_t total = ((size_t)cts * ids.limbs_per_poly) << logn;
  if (!total) return;
  add_scaled_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(A);
  g_launches++;
}

void launch_phase(const u64* ct, const u64* s, u64* out, u32 cts, u32 parts, const RowIds& ids, const LimbDev* limbs,
                  u32 logn, cudaStream_t st) {
  PhaseArgs A;
  A.ct = ct; A.s = s; A.out = out; A.cts = cts; A.parts = parts; A.logn = logn;
  A.limbs_per_poly = ids.limbs_per_poly; A.limbs = limbs;
  copy_ids(A.ids, ids);
  const size_t total = ((size_t)cts * ids.limbs_per_poly) << logn;
  if (!total || !parts) return;
  phase_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(A);
  g_launches++;
}

void launch_decrypt_epilogue(u64* v, size_t n_words, const PlainMod& Q0, const PlainMod& T, cudaStream_t st) {
  if (!n_words) return;
  decrypt_epilogue_kernel<<<(unsigned)((n_words + 255) / 256), 256, 0, st>>>(v, n_words, Q0, T);
  g_launches++;
}

void launch_from_shares_epilogue(u64* v, size_t n_words, u64 q0, const PlainMod& T, cudaStream_t st) {
  if (!n_words) return;
  from_shares_epilogue_kernel<<<(unsigned)((n_words + 255) / 256), 256, 0, st>>>(v, n_words, q0, T);
  g_launches++;
}

void launch_center(u64* x, size_t n_words, u64 t, cudaStream_t st) {
  if (!n_words) return;
  center_kernel<<<(unsigned)((n_words + 255) / 256), 256, 0, st>>>(x, n_words, t);
  g_launches++;
}

void launch_noise(const u64* x, u32* out, u32 cts, u32 L, const u64* garner, const u64* q_words, u32 W,
                  const LimbDev* limbs, u32 logn, cudaStream_t st) {
  if (!cts) return;
  NoiseArgs A;
  A.x = x; A.out = out; A.garner = garner; A.q_words = q_words; A.L = L; A.W = W; A.logn = logn; A.limbs = limbs;
  const u32 N = 1u << logn;
  noise_kernel<<<dim3((N + 255) / 256, cts), 256, 0, st>>>(A);
  g_launches++;
}

void launch_encrypt_sk(const u64* s, const u64* e, u64* out, u32 cts, u32 ct_base, const EncSeed& K, const RowIds& ids,
                       const LimbDev* limbs, u32 logn, cudaStream_t st) {
  EncSkArgs A;
  A.s = s; A.e = e; A.out = out; A.K = K; A.cts = cts; A.ct_base = ct_base; A.logn = logn;
  A.limbs_per_poly = ids.limbs_per_poly; A.limbs = limbs;
  copy_ids(A.ids, ids);
  const size_t total = ((size_t)cts * ids.limbs_per_poly) << (logn - 2);
  if (!total) return;
  encrypt_sk_kernel<<<(unsigned)((total + 127) / 128), 128, 0, st>>>(A);
  g_launches++;
}

void launch_cbd(u64* out, u32 cts, u32 ct_base, u32 role0, u32 n_roles, u32 variance, const EncSeed& K,
                const RowIds& ids, const LimbDev* limbs, u32 logn, cudaStream_t st, u32 digits) {
  CbdArgs A;
  const u128 add = (((u128)1) << (2 * variance)) - 1;   // variance <= 32: 2 variance <= 64 bits each
  const u128 sub = add << (2 * variance);
  A.add_lo = (u64)add; A.add_hi = (u64)(add >> 64); A.sub_lo = (u64)sub; A.sub_hi = (u64)(sub >> 64);
  A.out = out; A.K = K; A.cts = cts; A.ct_base = ct_base; A.role0 = role0; A.n_roles = n_roles; A.logn = logn;
  A.digits = digits; A.limbs_per_poly = ids.limbs_per_poly; A.limbs = limbs;
  copy_ids(A.ids, ids);
  const size_t total = ((size_t)cts * n_roles) << (logn - 2);
  if (!total) return;
  cbd_kernel<<<(unsigned)((total + 127) / 128), 128, 0, st>>>(A);
  g_launches++;
}

void launch_encrypt_pk(const u64* uee, const u64* pk, u64* out, u32 cts, const RowIds& ids, const LimbDev* limbs,
                       u32 logn, cudaStream_t st) {
  EncPkArgs A;
  A.uee = uee; A.pk = pk; A.out = out; A.cts = cts; A.logn = logn; A.limbs_per_poly = ids.limbs_per_poly;
  A.limbs = limbs;
  copy_ids(A.ids, ids);
  const size_t total = ((size_t)cts * ids.limbs_per_poly) << logn;
  if (!total) return;
  encrypt_pk_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(A);
  g_launches++;
}

void launch_ksk_gen(const u64* s, const u64* e, const u64* x, u64* k0, u64* k1, u32 key, u32 digit0, u32 digits,
                    u32 n_dig, const KskG& G, const EncSeed& K, const RowIds& ids, const LimbDev* limbs, u32 logn,
                    cudaStream_t st) {
  KskGenArgs A;
  A.s = s; A.e = e; A.x = x; A.k0 = k0; A.k1 = k1; A.K = K; A.key = key; A.digit0 = digit0; A.digits = digits;
  A.n_dig = n_dig; A.logn = logn; A.limbs_per_poly = ids.limbs_per_poly; A.decomp = G.decomp; A.limbs = limbs;
  for (int i = 0; i < kMaxPos; i++) { A.g[i] = G.g[i]; A.g_s[i] = G.g_s[i]; }
  copy_ids(A.ids, ids);
  const size_t total = ((size_t)digits * ids.limbs_per_poly) << (logn - 2);
  if (!total) return;
  ksk_gen_kernel<<<(unsigned)((total + 127) / 128), 128, 0, st>>>(A);
  g_launches++;
}

void launch_ew(EwOp op, u64* a, const u64* b, size_t n_rows, const RowIds& ids, const LimbDev* limbs, u32 logn,
               cudaStream_t st) {
  EwArgs A;
  A.a = a;
  A.b = b;
  A.n_words = n_rows << logn;
  A.logn = logn;
  A.limbs_per_poly = ids.limbs_per_poly;
  A.limbs = limbs;
  copy_ids(A.ids, ids);
  if (A.n_words == 0) return;
  const u32 threads = 256;
  const size_t blocks = (A.n_words / 2 + threads - 1) / threads;
  if (op == EW_ADD) ew_kernel<EW_ADD><<<(unsigned)blocks, threads, 0, st>>>(A);
  else if (op == EW_SUB) ew_kernel<EW_SUB><<<(unsigned)blocks, threads, 0, st>>>(A);
  else ew_kernel<EW_NEG><<<(unsigned)blocks, threads, 0, st>>>(A);
  g_launches++;
}

void launch_mul_plain(u64* a, const u64* pt, u32 cts, u32 parts, u32 n_pt, const RowIds& ids, const LimbDev* limbs,
                      u32 logn, cudaStream_t st, u32 op) {
  MulPlainArgs A;
  A.a = a; A.pt = pt; A.cts = cts; A.parts = parts; A.n_pt = n_pt; A.logn = logn; A.op = op;
  A.limbs_per_poly = ids.limbs_per_poly; A.limbs = limbs;
  copy_ids(A.ids, ids);
  size_t total = ((size_t)cts * parts * ids.limbs_per_poly) << logn;
  if (!total) return;
  mul_plain_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(A);
  g_launches++;
}

void launch_expand_butterfly(u64* lo, u64* hi, const u64* spill, u32 pairs, u32 n_hi, const ulonglong2* mono,
                             const RowIds& ids, const LimbDev* limbs, u32 logn, cudaStream_t st) {
  ExpandArgs A;
  const size_t ct_words = ((size_t)2 * ids.limbs_per_poly) << logn;
  A.lo = lo; A.hi = hi; A.spill = spill; A.mono = mono;
  A.n_words = pairs * ct_words;
  A.hi_words = n_hi * ct_words;
  A.logn = logn; A.limbs_per_poly = ids.limbs_per_poly; A.limbs = limbs;
  copy_ids(A.ids, ids);
  if (!A.n_words) return;
  const u32 threads = 256;
  expand_butterfly_kernel<<<(unsigned)((A.n_words / 2 + threads - 1) / threads), threads, 0, st>>>(A);
  g_launches++;
}

void launch_dot(const u64* ct, const u64* pt, u64* out, u32 groups, u32 n_terms, u32 parts, u32 ct_count,
                u32 pt_count, const RowIds& ids, const LimbDev* limbs, u32 logn, cudaStream_t st) {
  DotArgs A;
  A.ct = ct; A.pt = pt; A.out = out; A.groups = groups; A.n_terms = n_terms; A.parts = parts;
  A.ct_count = ct_count; A.pt_count = pt_count; A.logn = logn;
  A.limbs_per_poly = ids.limbs_per_poly; A.limbs = limbs;
  copy_ids(A.ids, ids);
  size_t total = ((size_t)groups * parts * ids.limbs_per_poly) << logn;
  if (!total) return;
  dot_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(A);
  g_launches++;
}

void launch_tensor(const u64* a, const u64* b, const u64* xa, const u64* xb, u64* out, u32 cts, u32 L, u32 nca,
                   u32 ncb, u32 K, const RowIds& mul_ids, const LimbDev* limbs, u32 logn, cudaStream_t st) {
  TensorArgs A;
  A.a = a; A.b = b; A.xa = xa; A.xb = xb; A.out = out;
  A.cts = cts; A.L = L; A.nca = nca; A.ncb = ncb; A.K = K; A.logn = logn;
  A.limbs = limbs;
  copy_ids(A.ids, mul_ids);
  size_t total = ((size_t)cts * K) << logn;
  if (!total) return;
  tensor_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(A);
  g_launches++;
}

void launch_tensor_nm(const u64* a, const u64* b, const u64* xa, const u64* xb, u64* out, u32 cts, u32 L, u32 E, u32 na,
                      u32 nb, const RowIds& mul_ids, const LimbDev* limbs, u32 logn, cudaStream_t st) {
  TensorNmArgs A;
  A.a = a; A.b = b; A.xa = xa; A.xb = xb; A.out = out;
  A.cts = cts; A.L = L; A.E = E; A.na = na; A.nb = nb; A.logn = logn;
  A.limbs = limbs;
  copy_ids(A.ids, mul_ids);
  size_t total = ((size_t)cts * (na + nb - 1) * (L + E)) << logn;
  if (!total) return;
  tensor_nm_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(A);
  g_launches++;
}

// The persistent TMA-fed kernel serves N >= 128 when every output limb is a Solinas prime (all 62-bit primes the
// reference's parameter builder generates are); FHE_B200_SCALER=classic keeps the per-tile kernel.
static bool launch_scale_tma(const ScalerDev& S, const LimbDev* limbs, const u64* in, u64* out0, u64* out1, u32 polys,
                             u32 out_rows_per_poly, u32 start, u32 n_out, int split3, u32 logn, cudaStream_t st) {
  if (switches().classic_scaler || !tensor_map_encoder() || logn < 7 || (reinterpret_cast<uintptr_t>(in) & 127))
    return false;
  const u32 N = 1u << logn, nf = S.n_from;
  if (nf > 64 || (u64)polys * nf >= (1ull << 31)) return false;
  CUtensorMap tm;
  if (!box_map(&tm, in, (u64)polys * nf, logn, kScaleTC, nf)) return false;
  ScaleTmaArgs A;
  A.S = S; A.limbs = limbs; A.out0 = out0; A.out1 = out1;
  A.polys = polys; A.out_rows_per_poly = out_rows_per_poly; A.start = start; A.n_out = n_out;
  A.split3 = split3; A.logn = logn;
  A.tiles_total = polys * (N / kScaleTC);
  const size_t n_out4 = (n_out + 3) & ~(size_t)3;
  const size_t smem = (nf * kScaleTC + 3 * n_out4 + 4 * nf) * sizeof(u64) + nf * 3 * n_out4 * sizeof(u32) +
                      ((nf + 1) & ~(size_t)1) * 4 + 16;
  // persistent grid = exactly the CTAs that are resident at once (registers and shared memory both limit it)
  auto resident = [&](const void* k) {
    ensure_dynamic_smem(k, smem);
    int per_sm = 0;
    FHE_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k, kScaleTC, smem));
    return (u32)std::min<u64>(A.tiles_total, (u64)sm_count() * std::max(per_sm, 1));
  };
  if (switches().scale_unroll == 4) {
    if (S.is_one) scale_tma_kernel<true, 4><<<resident((const void*)scale_tma_kernel<true, 4>), kScaleTC, smem, st>>>(tm, A);
    else scale_tma_kernel<false, 4><<<resident((const void*)scale_tma_kernel<false, 4>), kScaleTC, smem, st>>>(tm, A);
  } else {
    if (S.is_one) scale_tma_kernel<true, 2><<<resident((const void*)scale_tma_kernel<true, 2>), kScaleTC, smem, st>>>(tm, A);
    else scale_tma_kernel<false, 2><<<resident((const void*)scale_tma_kernel<false, 2>), kScaleTC, smem, st>>>(tm, A);
  }
  g_launches++;
  return true;
}

void launch_scale(const ScalerDev& S, const LimbDev* limbs, const u64* in, u64* out0, u64* out1, u32 polys,
                  u32 out_rows_per_poly, u32 start, u32 n_out, int split3, u32 logn, cudaStream_t st) {
  if (!polys || !n_out) return;
  if (S.all_solinas &&
      launch_scale_tma(S, limbs, in, out0, out1, polys, out_rows_per_poly, start, n_out, split3, logn, st))
    return;
  ScaleArgs A;
  A.S = S; A.limbs = limbs; A.in = in; A.out0 = out0; A.out1 = out1;
  A.polys = polys; A.out_rows_per_poly = out_rows_per_poly; A.start = start; A.n_out = n_out;
  A.split3 = split3; A.logn = logn;
  const u32 N = 1u << logn;
  if (N < (u32)kScaleTC) {
    const u32 total = polys * N;
    scale_small_kernel<<<(total + 63) / 64, 64, 0, st>>>(A);
    g_launches++;
    return;
  }
  const size_t n_out4 = (n_out + 3) & ~(size_t)3, nf = S.n_from;
  const size_t smem = (nf * kScaleTC + n_out4 + 5 * nf) * sizeof(u64) + nf * 3 * n_out4 * sizeof(u32);
  ensure_dynamic_smem((const void*)scale_kernel, smem);
  scale_kernel<<<polys * (N / kScaleTC), kScaleTC, smem, st>>>(A);
  g_launches++;
}

void launch_ksmac(const u64* inter, const std::vector<KeyRange>& ranges, const u64* base0, const u64* base1, u64* out0,
                  u64* out1, u32 n_dig, u32 Lk, u32 out_ct_rows, const RowIds& ids, const LimbDev* limbs, u32 logn,
                  cudaStream_t st, bool adjacent) {
  const bool classic = switches().ksmac == Switches::KSMAC_CLASSIC;
  // ring depth: 2 buffers -> 4 resident CTAs per SM at set C: the kernel needs warps more than prefetch depth.
  // FHE_B200_KS_STAGES = 2 | 3 | 4.
  const int stages = (int)switches().ks_stages;
  const size_t smem_tma = ((size_t)(2 + stages) * n_dig * kKsTC + stages + 1) * sizeof(u64);
  bool tma = adjacent && !classic && tensor_map_encoder() && logn >= 7 && n_dig <= 256 && smem_tma <= 200 * 1024 &&
             !(reinterpret_cast<uintptr_t>(inter) & 127);
  for (const KeyRange& r : ranges) {
    tma = tma && (u64)r.cts * Lk * n_dig < (1ull << 31);
    for (u32 s = 0; s < r.keys.n; s++)
      tma = tma && !((reinterpret_cast<uintptr_t>(r.keys.k0[s]) | reinterpret_cast<uintptr_t>(r.keys.k1[s])) & 127);
  }
  // every tensor map first: a shape the TMA cannot describe takes the classic kernel for the whole call
  std::vector<CUtensorMap> mt(ranges.size());
  for (size_t r = 0; tma && r < ranges.size(); r++)
    tma = box_map(&mt[r], inter + (((size_t)ranges[r].ct0 * Lk * n_dig) << logn), (u64)ranges[r].cts * Lk * n_dig,
                  logn, kKsTC, n_dig);
  for (size_t r = 0; r < ranges.size(); r++) {
    const KeyRange& R = ranges[r];
    const size_t total = ((size_t)R.cts * Lk) << logn;
    if (!total) continue;
    const size_t o = ((size_t)R.ct0 * out_ct_rows) << logn;
    if (tma) {
      KsTmaArgs T;
      T.keys = R.keys;
      T.base0 = base0 ? base0 + o : nullptr; T.base1 = base1 ? base1 + o : nullptr;
      T.out0 = out0 + o; T.out1 = out1 + o;
      T.cts = R.cts; T.n_dig = n_dig; T.Lk = Lk; T.out_ct_rows = out_ct_rows; T.logn = logn;
      T.items_total = Lk * ((1u << logn) / kKsTC) * R.cts;
      T.limbs = limbs;
      copy_ids(T.ids, ids);
      auto go = [&](auto kern) {
        ensure_dynamic_smem((const void*)kern, smem_tma);
        int per_sm = 0;
        FHE_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, (const void*)kern, kKsTC, smem_tma));
        const u32 grid = (u32)std::min<u64>(T.items_total, (u64)sm_count() * std::max(per_sm, 1));
        kern<<<grid, kKsTC, smem_tma, st>>>(mt[r], T);
      };
      if (stages == 2) go(ksmac_tma_kernel<2>);
      else if (stages == 3) go(ksmac_tma_kernel<3>);
      else go(ksmac_tma_kernel<4>);
      g_launches++;
      continue;
    }
    KsMacArgs A;
    A.keys = R.keys;
    A.adjacent = adjacent ? 1 : 0;
    A.inter = inter + ((((size_t)R.ct0 * Lk) * n_dig) << logn);
    A.base0 = base0 ? base0 + o : nullptr; A.base1 = base1 ? base1 + o : nullptr;
    A.out0 = out0 + o; A.out1 = out1 + o;
    A.cts = R.cts; A.n_dig = n_dig; A.Lk = Lk; A.out_ct_rows = out_ct_rows; A.logn = logn;
    A.limbs = limbs;
    copy_ids(A.ids, ids);
    ksmac_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(A);
    g_launches++;
  }
}

void launch_decompose(const u64* in, u64* out, size_t polys, u32 n_dig, u32 log_base, u32 logn, cudaStream_t st) {
  const size_t n_words = polys << logn;
  if (!n_words) return;
  decompose_kernel<<<(unsigned)((n_words + 255) / 256), 256, 0, st>>>(in, out, n_words, n_dig, log_base, logn);
  g_launches++;
}

void launch_gather(const u64* in, u64* out, size_t n_rows, const int* perm, u32 logn, cudaStream_t st) {
  size_t n = n_rows << logn;
  if (!n) return;
  gather_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(in, out, n, perm, logn);
  g_launches++;
}

void launch_substitute_ntt(const u64* in, size_t in_stride, u64* out0, size_t out0_stride, u64* out1,
                           size_t out1_stride, const u32* exponent, const u32* source, u32 cts, u32 L, bool sum,
                           const RowIds& ids, const LimbDev* limbs, u32 logn, cudaStream_t st) {
  const size_t words = (size_t)L << logn;
  if (!words || !cts) return;
  SubstArgs A;
  std::memset(&A, 0, sizeof(A));
  A.in = in; A.in_stride = in_stride;
  A.out1 = out1; A.out0_stride = out0_stride; A.out1_stride = out1_stride;
  A.L = L; A.logn = logn; A.sum = sum ? 1 : 0; A.limbs = limbs;
  copy_ids(A.ids, ids);
  const dim3 block(256);
  u32 c0 = 0;   // first ciphertext of the pending launch
  auto flush = [&](u32 end) {
    A.out0 = out0 + (size_t)c0 * out0_stride;
    A.out1 = out1 ? out1 + (size_t)c0 * out1_stride : nullptr;
    subst_kernel<<<dim3((unsigned)((words + 255) / 256), end - c0), block, 0, st>>>(A);
    g_launches++;
    A.T.n = 0;
    c0 = end;
  };
  for (u32 c = 0; c < cts; c++) {
    if (c - c0 == 65535) flush(c);   // gridDim.y
    const u32 e = exponent[c], s = source ? source[c] : c;
    const u32 r = A.T.n;
    if (r && A.T.exponent[r - 1] == e && A.T.src0[r - 1] + (c - c0 - A.T.ct0[r - 1]) == s) continue;   // extends run r-1
    if (r == kSubstRuns) flush(c);
    A.T.ct0[A.T.n] = c - c0;
    A.T.exponent[A.T.n] = e;
    A.T.src0[A.T.n] = s;
    A.T.n++;
  }
  flush(cts);
}

void launch_substitute_power(const u64* in, u64* out, size_t n_rows, u32 exponent, const RowIds& ids,
                             const LimbDev* limbs, u32 logn, cudaStream_t st) {
  SubstPowerArgs A;
  A.in = in; A.out = out; A.n_words = n_rows << logn; A.logn = logn; A.limbs_per_poly = ids.limbs_per_poly;
  A.exponent = exponent; A.limbs = limbs;
  copy_ids(A.ids, ids);
  if (!A.n_words) return;
  substitute_power_kernel<<<(unsigned)((A.n_words + 255) / 256), 256, 0, st>>>(A);
  g_launches++;
}

// the outputs [i0, i0 + T.n) of `outs` as a launch table
static void hoist_table(HoistTable& T, const HoistOut* outs, u32 i0, u32 n) {
  std::memset(&T, 0, sizeof(T));
  T.n = n;
  for (u32 i = 0; i < n; i++) {
    const HoistOut& h = outs[i0 + i];
    T.exponent[i] = h.exponent;
    T.src_ct[i] = h.src_ct;
    T.dst[i] = h.dst;
    T.src[i] = (unsigned short)h.src;
    T.mrow[i] = (unsigned short)h.mrow;
  }
}

void launch_hoist_zero(const HoistOut* outs, u32 n, const u64* x, u32* flags, u32 L, u32 logn, cudaStream_t st) {
  const u32 N = 1u << logn;
  HoistTable T;
  for (u32 i0 = 0; i0 < n; i0 += kHoistOuts) {
    hoist_table(T, outs, i0, std::min(kHoistOuts, n - i0));
    hoist_zero_kernel<<<dim3((N + 255) / 256, T.n), 256, 0, st>>>(T, x, flags + i0, L, logn);
    g_launches++;
  }
}

void launch_negation_rows(u64* out, const u32* exps, u32 n_exp, u32 Lk, u32 logn, cudaStream_t st) {
  const u32 N = 1u << logn;
  HoistTable T;
  for (u32 m0 = 0; m0 < n_exp; m0 += kHoistOuts) {
    std::memset(&T, 0, sizeof(T));
    T.n = std::min(kHoistOuts, n_exp - m0);
    for (u32 m = 0; m < T.n; m++) T.exponent[m] = exps[m0 + m];
    negation_rows_kernel<<<dim3((N + 255) / 256, T.n), 256, 0, st>>>(T, out + (((size_t)m0 * Lk) << logn), Lk, logn);
    g_launches++;
  }
}

void launch_hoist_mac(const HoistOut* outs, u32 n, const u64* D, bool adjacent, const u64* mrows, const u64* c0,
                      size_t c0_stride, u64* out, size_t out_stride, u32 L, u32 Lk, const RowIds& ids,
                      const LimbDev* limbs, u32 logn, cudaStream_t st) {
  const u32 N = 1u << logn;
  HoistMacArgs A;
  std::memset(&A, 0, sizeof(A));
  A.D = D; A.mrows = mrows; A.c0 = c0; A.out = out; A.c0_stride = c0_stride; A.out_stride = out_stride;
  A.L = L; A.Lk = Lk; A.logn = logn; A.adjacent = adjacent ? 1 : 0; A.limbs = limbs;
  copy_ids(A.ids, ids);
  // one launch per run of at most kHoistOuts outputs and kKeyPairs distinct keys
  u32 i0 = 0;
  auto flush = [&](u32 end) {
    hoist_table(A.T, outs, i0, end - i0);
    hoist_mac_kernel<<<dim3((N + 255) / 256, A.T.n, Lk), 256, 0, st>>>(A);
    g_launches++;
    std::memset(&A.keys, 0, sizeof(A.keys));
    i0 = end;
  };
  for (u32 i = 0; i < n; i++) {
    u32 s = 0;
    while (s < A.keys.n && A.keys.k0[s] != outs[i].k0) s++;
    if (i - i0 == kHoistOuts || (s == A.keys.n && s == kKeyPairs)) {
      flush(i);
      s = 0;
    }
    if (s == A.keys.n) {
      A.keys.k0[s] = outs[i].k0;
      A.keys.k1[s] = outs[i].k1;
      A.keys.n++;
    }
    A.keys.slot[i - i0] = (unsigned char)s;
  }
  if (n > i0) flush(n);
}

void launch_hoist_dot(const LtStep* steps, const int* fallback, const u64* fb, const u64* D, bool adjacent,
                      const u64* mrows, const u64* ct, size_t ct_stride, u32 cts, const u64* diag, u32 diag_ct0,
                      bool per_ct, u32 n_diags, u32 baby, u32 g0, u32 n_groups, u64* out, u32 L, const RowIds& ids,
                      const LimbDev* limbs, u32 logn, cudaStream_t st) {
  if (!cts || !n_groups) return;
  const u32 N = 1u << logn, threads = std::min(256u, N);
  HoistDotArgs A;
  std::memset(&A, 0, sizeof(A));
  A.steps = steps; A.fallback = fallback; A.fb = fb; A.D = D; A.mrows = mrows; A.ct = ct; A.diag = diag; A.out = out;
  A.ct_stride = ct_stride; A.cts = cts; A.ct_tiles = (cts + kDotCts - 1) / kDotCts; A.diag_ct0 = diag_ct0;
  A.per_ct = per_ct ? 1 : 0; A.n_diags = n_diags; A.baby = baby; A.g0 = g0; A.n_groups = n_groups; A.L = L;
  A.logn = logn; A.adjacent = adjacent ? 1 : 0; A.limbs = limbs;
  copy_ids(A.ids, ids);
  const u32 group_tiles = (n_groups + kDotGroups - 1) / kDotGroups;
  hoist_dot_kernel<<<dim3(group_tiles * A.ct_tiles, (N + threads - 1) / threads, L), threads, 0, st>>>(A);
  g_launches++;
}

void launch_pack(const PackDev& P, const u64* words, unsigned char* bytes, size_t n_rows, u32 logn, cudaStream_t st) {
  const size_t groups = n_rows << (logn - 3);
  if (!groups) return;
  pack_kernel<<<(unsigned)((groups + 127) / 128), 128, 0, st>>>(P, words, bytes, groups, logn);
  g_launches++;
}
void launch_unpack(const PackDev& P, const unsigned char* bytes, u64* words, size_t n_rows, u32 logn, cudaStream_t st) {
  const size_t groups = n_rows << (logn - 3);
  if (!groups) return;
  unpack_kernel<<<(unsigned)((groups + 127) / 128), 128, 0, st>>>(P, bytes, words, groups, logn);
  g_launches++;
}

void launch_transcode(const TranscodeRows& T, size_t n_rows, cudaStream_t st) {
  const size_t n = n_rows * T.out_len;
  if (!n) return;
  const unsigned blocks = (unsigned)std::min<size_t>((n + 255) / 256, 1u << 20);
  if (T.in_elem == 8 && T.out_elem == 8) transcode_kernel<u64, u64><<<blocks, 256, 0, st>>>(T, n);
  else if (T.in_elem == 8) transcode_kernel<u64, unsigned char><<<blocks, 256, 0, st>>>(T, n);
  else if (T.out_elem == 8) transcode_kernel<unsigned char, u64><<<blocks, 256, 0, st>>>(T, n);
  else transcode_kernel<unsigned char, unsigned char><<<blocks, 256, 0, st>>>(T, n);
  g_launches++;
}

void launch_fold_stage(const u64* ct, u32 n_ct, u32 parts, size_t row_words, u32 in_bits, u32 out_bits, u32 P,
                       u64* coeffs, u32 logn, cudaStream_t st) {
  const size_t n = ((size_t)P * n_ct) << logn;
  if (!n) return;
  const u64 E = ((u64)row_words * in_bits + out_bits - 1) / out_bits;
  fold_stage_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(ct, n_ct, parts, row_words, in_bits, out_bits, E,
                                                                 coeffs, n, logn);
  g_launches++;
}

void launch_switch_down(const SwitchDownDev& S, const u64* in, u64* out, u32 polys, u32 L, const RowIds& ids,
                        const LimbDev* limbs, u32 logn, cudaStream_t st) {
  SwitchDownArgs A;
  A.S = S; A.in = in; A.out = out; A.polys = polys; A.L = L; A.logn = logn; A.limbs = limbs;
  copy_ids(A.ids, ids);
  size_t total = (size_t)polys << logn;
  if (!total) return;
  switch_down_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(A);
  g_launches++;
}

}  // namespace fhe_b200
