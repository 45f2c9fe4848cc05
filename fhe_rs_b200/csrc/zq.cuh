// Device-side arithmetic modulo one <=62-bit prime (sm_90a).
// Mirrors the semantics of zq::Modulus in the reference
// (crates/fhe-math/src/zq/mod.rs): Barrett with a 128-bit constant (:693),
// Shoup multiplication (:224) and the single conditional subtraction (:659).
// All API-visible results are canonical residues, so any correct reduction
// strategy is bit-exact with the reference.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

namespace fhe_b200 {

typedef unsigned long long u64;
typedef unsigned int u32;

// Per-limb constants + NTT tables; one entry per distinct prime of a parameter set.
struct LimbDev {
  u64 p;       // modulus
  u64 p2;      // 2p
  u64 bhi;     // floor(2^128 / p) >> 64          (zq/mod.rs:87-91)
  u64 blo;     // floor(2^128 / p) & (2^64-1)
  u64 ninv;    // N^-1 mod p                      (ntt/native.rs:39)
  u64 ninv_s;  // shoup(N^-1)
  u64 zn;      // zetas_inv[N-2] * N^-1 mod p  (last inverse stage fused with the N^-1 scaling)
  u64 zn_s;    // shoup(zn)
  u64 c128;    // 2^128 mod p (folds the third accumulator word of lazy sums)
  u64 sol_c;   // c if p = 2^62 - c with c < 2^28 ("Solinas" limb: lazy sums / products fold with 2^62 == c), else 0
  u64 sol_ntt; // 1: twiddle pairs are (w, w*2^32 mod p) and the butterflies use mul_solinas_lazy; 0: Shoup pairs
  // twiddle tables as (value, companion) pairs so one 128-bit load fetches both words:
  const ulonglong2* om;  // omegas[N]    = psi^{bitrev(i)}       (ntt/native.rs:50-56) + Shoup quotient | w*2^32 mod p
  const ulonglong2* zi;  // zetas_inv[N] = psi^{-(bitrev(i)+1)}  + companion
};

__device__ __forceinline__ u64 csub(u64 x, u64 p) { return x >= p ? x - p : x; }

// lazy Shoup product: a*w mod p in [0,2p) for any 64-bit a (zq/mod.rs:224-234)
__device__ __forceinline__ u64 mul_shoup_lazy(u64 a, u64 w, u64 ws, u64 p) {
  const u64 q = __umul64hi(a, ws);
  // a*w - q*p (mod 2^64) as a*w + q*(-p): one accumulating chain of two IMAD.WIDE and four IMAD, no separate
  // negation/subtraction (four ALU-pipe instructions fewer per butterfly than the two-product form)
  const u64 np = 0 - p;
  u64 r;
  asm("{\n\t"
      ".reg .u32 a0, a1, w0, w1, q0, q1, n0, n1, lo, hi;\n\t"
      ".reg .u64 W;\n\t"
      "mov.b64 {a0, a1}, %1;\n\t"
      "mov.b64 {w0, w1}, %2;\n\t"
      "mov.b64 {q0, q1}, %3;\n\t"
      "mov.b64 {n0, n1}, %4;\n\t"
      "mul.wide.u32 W, q0, n0;\n\t"
      "mad.wide.u32 W, a0, w0, W;\n\t"
      "mov.b64 {lo, hi}, W;\n\t"
      "mad.lo.u32 hi, q0, n1, hi;\n\t"
      "mad.lo.u32 hi, q1, n0, hi;\n\t"
      "mad.lo.u32 hi, a0, w1, hi;\n\t"
      "mad.lo.u32 hi, a1, w0, hi;\n\t"
      "mov.b64 %0, {lo, hi};\n\t"
      "}"
      : "=l"(r)
      : "l"(a), "l"(w), "l"(q), "l"(np));
  return r;
}
__device__ __forceinline__ u64 mul_shoup(u64 a, u64 w, u64 ws, u64 p) {
  return csub(mul_shoup_lazy(a, w, ws, p), p);
}

// Multiplication of any 64-bit y by a precomputed constant w modulo p = 2^62 - c, c < 2^28,
// result in [0,2p) -- the same contract as the reference's lazy_mul_shoup (zq/mod.rs:224), so it can
// replace it inside the Harvey butterflies without changing any canonical output.
//   y = y1*2^32 + y0 ;  w0 = w, w1 = w*2^32 mod p  (both < 2^62, precomputed)
//   S = y0*w0 + y1*w1  (== y*w mod p, S < 2^95)   -- four 32x32->64 products, no 64x64 high product
//   S = Shi*2^62 + Slo ;  2^62 == c (mod p)  =>  y*w == Shi*c + Slo < 2^33*2^28 + 2^62 < 2p
// Five IMAD.WIDE against six IMAD.WIDE + four IMAD for the Shoup form; the integer multiplier pipe is the
// binding resource of the NTT.
__device__ __forceinline__ u64 mul_solinas_lazy(u64 y, u64 w0, u64 w1, u32 c) {
  u64 r;
  // two word-serial 32x64 products (the high IMAD.WIDE takes the low one's top word as addend, so the
  // FMA pipe does those additions), one 96-bit addition, one fold:
  //   y0*w0 = PH*2^32 + p0 ,  y1*w1 = QH*2^32 + q0 ,  S = (PH + QH + carry(p0+q0))*2^32 + (p0+q0 mod 2^32)
  //   H = S >> 32 < 2^63 ;  Shi = H >> 30 = hh + tt*2^32 ;  Slo = (H mod 2^30)*2^32 + s0 ;  r = Shi*c + Slo
  asm("{\n\t"
      ".reg .u32 y0, y1, a0, a1, b0, b1, p0, pc, q0, qc, s0, h0, h1, hh, tt, sl, r0, r1;\n\t"
      ".reg .u64 P, Q, PH, QH, PC, QC, S, R;\n\t"
      "mov.b64 {y0, y1}, %1;\n\t"
      "mov.b64 {a0, a1}, %2;\n\t"
      "mov.b64 {b0, b1}, %3;\n\t"
      "mul.wide.u32 P, y0, a0;\n\t"
      "mul.wide.u32 Q, y1, b0;\n\t"
      "mov.b64 {p0, pc}, P;\n\t"
      "mov.b64 {q0, qc}, Q;\n\t"
      "cvt.u64.u32 PC, pc;\n\t"
      "cvt.u64.u32 QC, qc;\n\t"
      "mad.wide.u32 PH, y0, a1, PC;\n\t"
      "mad.wide.u32 QH, y1, b1, QC;\n\t"
      "add.cc.u32 s0, p0, q0;\n\t"
      "mov.b64 {h0, h1}, PH;\n\t"
      "mov.b64 {r0, r1}, QH;\n\t"
      "addc.cc.u32 h0, h0, r0;\n\t"
      "addc.u32 h1, h1, r1;\n\t"
      "shf.r.wrap.b32 hh, h0, h1, 30;\n\t"
      "shr.u32 tt, h1, 30;\n\t"
      "and.b32 sl, h0, 0x3fffffff;\n\t"
      "mov.b64 S, {s0, sl};\n\t"
      "mad.wide.u32 R, hh, %4, S;\n\t"
      "mov.b64 {r0, r1}, R;\n\t"
      "mad.lo.u32 r1, tt, %4, r1;\n\t"
      "mov.b64 %0, {r0, r1};\n\t"
      "}"
      : "=l"(r)
      : "l"(y), "l"(w0), "l"(w1), "r"(c));
  return r;
}

// alternative instruction selection of the same product (kept for bench_micro/bf_bench.cu): four plain
// products, M = y0*a1 + y1*b1 accumulated by the FMA pipe, five carry adds
__device__ __forceinline__ u64 mul_solinas_lazy_v1(u64 y, u64 w0, u64 w1, u32 c) {
  u64 r;
  asm("{\n\t"
      ".reg .u32 y0, y1, a0, a1, b0, b1, pl, ph, ql, qh, m0, m1, s0, h0, h1, hh, tt, sl, r0, r1;\n\t"
      ".reg .u64 P, Q, M, S, R;\n\t"
      "mov.b64 {y0, y1}, %1;\n\t"
      "mov.b64 {a0, a1}, %2;\n\t"
      "mov.b64 {b0, b1}, %3;\n\t"
      "mul.wide.u32 P, y0, a0;\n\t"
      "mul.wide.u32 Q, y1, b0;\n\t"
      "mul.wide.u32 M, y0, a1;\n\t"
      "mad.wide.u32 M, y1, b1, M;\n\t"
      "mov.b64 {pl, ph}, P;\n\t"
      "mov.b64 {ql, qh}, Q;\n\t"
      "mov.b64 {m0, m1}, M;\n\t"
      "add.cc.u32 s0, pl, ql;\n\t"
      "addc.cc.u32 h0, ph, qh;\n\t"
      "addc.u32 h1, m1, 0;\n\t"
      "add.cc.u32 h0, h0, m0;\n\t"
      "addc.u32 h1, h1, 0;\n\t"
      "shf.r.wrap.b32 hh, h0, h1, 30;\n\t"
      "shr.u32 tt, h1, 30;\n\t"
      "and.b32 sl, h0, 0x3fffffff;\n\t"
      "mov.b64 S, {s0, sl};\n\t"
      "mad.wide.u32 R, hh, %4, S;\n\t"
      "mov.b64 {r0, r1}, R;\n\t"
      "mad.lo.u32 r1, tt, %4, r1;\n\t"
      "mov.b64 %0, {r0, r1};\n\t"
      "}"
      : "=l"(r)
      : "l"(y), "l"(w0), "l"(w1), "r"(c));
  return r;
}

// x (any 64-bit value) -> x - 2p*[x >= 2^63]  in [0, 2^63 + 2c), using 2^64 - 2p = 2^63 + 2c:
// clear bit 63 and add bit63 * 2c (one IMAD.WIDE instead of compare + select on the busy ALU pipe)
__device__ __forceinline__ u64 fold63_solinas(u64 x, u32 c2) {
  u64 r;
  asm("{\n\t"
      ".reg .u32 lo, hi, b;\n\t"
      ".reg .u64 M;\n\t"
      "mov.b64 {lo, hi}, %1;\n\t"
      "shr.u32 b, hi, 31;\n\t"
      "and.b32 hi, hi, 0x7fffffff;\n\t"
      "mov.b64 M, {lo, hi};\n\t"
      "mad.wide.u32 %0, b, %2, M;\n\t"
      "}"
      : "=l"(r)
      : "l"(x), "r"(c2));
  return r;
}
// t in (-2p, 2p) as two's complement -> t + 2p*[t < 0]  (conditional add-back on the FMA pipe)
__device__ __forceinline__ u64 addback2p(u64 t, u64 p2) {
  u64 r;
  asm("{\n\t"
      ".reg .u32 lo, hi, b, pl, ph;\n\t"
      ".reg .u64 R;\n\t"
      "mov.b64 {lo, hi}, %1;\n\t"
      "mov.b64 {pl, ph}, %2;\n\t"
      "shr.u32 b, hi, 31;\n\t"
      "mad.wide.u32 R, b, pl, %1;\n\t"
      "mov.b64 {lo, hi}, R;\n\t"
      "mad.lo.u32 hi, b, ph, hi;\n\t"
      "mov.b64 %0, {lo, hi};\n\t"
      "}"
      : "=l"(r)
      : "l"(t), "l"(p2));
  return r;
}

// lazy product by a precomputed constant pair (a, b) in the limb's mode
template <bool SOL>
__device__ __forceinline__ u64 mul_const_lazy(u64 y, u64 a, u64 b, u64 p, u32 c) {
  return SOL ? mul_solinas_lazy(y, a, b, c) : mul_shoup_lazy(y, a, b, p);
}

// device shoup(a) = floor(a * 2^64 / p), a < p (zq/mod.rs:195).  Uses the Barrett
// constant: q ~ floor(a * floor(2^128/p) / 2^64), then fix up by at most 2.
__device__ __forceinline__ u64 shoup_of(u64 a, u64 p, u64 bhi, u64 blo) {
  // a * 2^64 / p: estimate with the 128-bit reciprocal
  u64 q = a * bhi + __umul64hi(a, blo);  // floor(a*B / 2^64) low 64 bits, B = bhi*2^64+blo (a*bhi < 2^64 since a<p, bhi<=2^64/p*...)
  // remainder r = a*2^64 - q*p (mod 2^64 arithmetic on the low word suffices: true r < 3p < 2^64)
  u64 r = 0ull - q * p;  // low 64 bits of a*2^64 are 0
  // r is in [0, 3p): correct q upward
  if (r >= p) { r -= p; q++; }
  if (r >= p) { r -= p; q++; }
  return q;
}

// Barrett reduction of a 128-bit value (lo,hi) to [0,2p)  (zq/mod.rs:693-707)
__device__ __forceinline__ u64 barrett128_lazy(u64 lo, u64 hi, u64 p, u64 bhi, u64 blo) {
  // q = floor(((lo*bhi + hi*blo + (lo*blo >> 64)) >> 64) + hi*bhi
  u64 t0 = __umul64hi(lo, blo);
  u64 a_lo = lo * bhi, a_hi = __umul64hi(lo, bhi);
  u64 b_lo = hi * blo, b_hi = __umul64hi(hi, blo);
  // sum = a + b + t0 (up to 130 bits; we only need bits 64.. of the sum)
  u64 s = a_lo + b_lo;
  u64 c = s < a_lo;
  u64 s2 = s + t0;
  c += s2 < s;
  u64 q = a_hi + b_hi + c + hi * bhi;  // low 64 bits of the quotient are all that matter
  return lo - q * p;
}
__device__ __forceinline__ u64 barrett128(u64 lo, u64 hi, u64 p, u64 bhi, u64 blo) {
  return csub(barrett128_lazy(lo, hi, p, bhi, blo), p);
}
// Barrett reduction of a 64-bit value to [0,p) (zq/mod.rs:712 + :659)
__device__ __forceinline__ u64 barrett64(u64 a, u64 p, u64 bhi, u64 blo) {
  // q = (a*bhi + (a*blo >> 64)) >> 64
  u64 t0 = __umul64hi(a, blo);
  u64 a_lo = a * bhi, a_hi = __umul64hi(a, bhi);
  u64 s = a_lo + t0;
  u64 q = a_hi + (s < a_lo);
  return csub(a - q * p, p);
}
// a*b mod p, canonical
__device__ __forceinline__ u64 mulmod(u64 a, u64 b, u64 p, u64 bhi, u64 blo) {
  return barrett128(a * b, __umul64hi(a, b), p, bhi, blo);
}

// Full 128-bit product of two operands < 2^62 (four IMAD.WIDE; the middle sum a0*b1 + a1*b0 < 2^63
// cannot overflow because both high words are < 2^30).
__device__ __forceinline__ void mul128_62(u64 a, u64 b, u64& lo, u64& hi) {
  asm("{\n\t"
      ".reg .u32 a0, a1, b0, b1, p0, p1, m0, m1, q0, q1, t1, t2, t3;\n\t"
      ".reg .u64 P, M, Q;\n\t"
      "mov.b64 {a0, a1}, %2;\n\t"
      "mov.b64 {b0, b1}, %3;\n\t"
      "mul.wide.u32 P, a0, b0;\n\t"
      "mul.wide.u32 M, a0, b1;\n\t"
      "mad.wide.u32 M, a1, b0, M;\n\t"
      "mul.wide.u32 Q, a1, b1;\n\t"
      "mov.b64 {p0, p1}, P;\n\t"
      "mov.b64 {m0, m1}, M;\n\t"
      "mov.b64 {q0, q1}, Q;\n\t"
      "add.cc.u32 t1, p1, m0;\n\t"
      "addc.cc.u32 t2, q0, m1;\n\t"
      "addc.u32 t3, q1, 0;\n\t"
      "mov.b64 %0, {p0, t1};\n\t"
      "mov.b64 %1, {t2, t3};\n\t"
      "}"
      : "=l"(lo), "=l"(hi)
      : "l"(a), "l"(b));
}

// One fold of 2^62 == c (mod p = 2^62 - c, c < 2^28) on a 128-bit value (hi:lo) with an extra
// addend `top` for the word above (bits >= 126 of the quotient):  returns (hi':lo') == value (mod p),
// (hi':lo') < 2^92 + top*c*2^64.  64-bit operations only (IMAD.WIDE + shifts).
__device__ __forceinline__ void fold_step_solinas(u64& lo, u64& hi, u64 top, u32 c) {
  const u64 mask = (1ull << 62) - 1;
  const u64 x = (lo >> 62) | (hi << 2);                 // quotient bits 62..125
  const u64 t0 = (u64)c * (u32)x + (lo & mask);         // < 2^60 + 2^62
  const u64 t1 = (u64)c * (u32)(x >> 32) + (t0 >> 32);  // < 2^60 + 2^31
  lo = (t1 << 32) | (u32)t0;
  hi = (t1 >> 32) + top * c;
}
// value (hi:lo) < 2^94 (hi < 2^30) -> [0,2p)
__device__ __forceinline__ u64 fold94_solinas(u64 lo, u64 hi, u32 c) {
  const u32 x = (u32)((lo >> 62) | (hi << 2));
  return (u64)c * x + (lo & ((1ull << 62) - 1));         // < 2^60 + 2^62 < 2p
}
// Reduction of a lazy sum V = hi*2^128 + mid*2^64 + lo, hi < 2^32 (every sum an Acc192 holds, up to 2^160), modulo
// p = 2^62 - c to [0,2p): top*c < 2^34 * 2^28 keeps the first fold's high word below 2^62, so
// 192 -> <2^126 -> <2^93 -> <2^62 + 2^59 bits (tests/test_gpu_zq_probe.py checks hi = 2^32 - 1).
__device__ __forceinline__ u64 fold192_solinas(u64 lo, u64 mid, u64 hi, u32 c) {
  u64 top = (mid >> 62) | (hi << 2);                     // quotient bits 126.. (< 2^34)
  fold_step_solinas(lo, mid, top, c);                    // < 2^126
  fold_step_solinas(lo, mid, 0, c);                      // < 2^93
  return fold94_solinas(lo, mid, c);
}
// residue in [0,2p) of a lazy sum hi*2^128 + mid*2^64 + lo < 2^160 in the limb's mode (Solinas fold or Barrett)
__device__ __forceinline__ u64 reduce160_lazy(u64 lo, u64 mid, u64 hi, const LimbDev& m) {
  if (m.sol_c) return fold192_solinas(lo, mid, hi, (u32)m.sol_c);
  u64 r1 = barrett128_lazy(lo, mid, m.p, m.bhi, m.blo);  // [0,2p)
  u64 hl = hi * m.c128, hh = __umul64hi(hi, m.c128);
  u64 r2 = barrett128_lazy(hl, hh, m.p, m.bhi, m.blo);   // [0,2p)
  return csub(r1 + r2, m.p2);
}

// Lazy multiply-accumulate register: sum of 64x64-bit products, exact up to 2^160, reduced once at the end
// (used by the key-switch inner product, the tensor and the scaler of rings below one tile; replaces the reference's per-term Shoup
// reduction, rns/scaler.rs:340-347 and rq/ops.rs:208).
// The four 32x32 partial products of a term go to two column sets that are never added to each other inside the
// loop: the even one (e0..e4, products aligned at words 0 and 2) and the odd one (o1..o3, aligned at word 1).
// Each mad.lo.cc/madc.hi.cc pair is ONE IMAD.WIDE.U32 with carry-out (and carry-in for the second of a chain), so
// a term costs 4 IMAD.WIDE + 2 IADD3.X -- the minimum of the schoolbook product (AccKara below takes three products
// when both operands are < 2^62) -- instead of 4 IMAD.WIDE + 9 carry-chain adds of
// the 128-bit-product-then-192-bit-add form, whose carry-chain adds load the ALU pipe more than its multiplies do.
struct Acc192 {
  u32 e0, e1, e2, e3, e4, o1, o2, o3;
  __device__ __forceinline__ void clear() { e0 = e1 = e2 = e3 = e4 = o1 = o2 = o3 = 0; }
  __device__ __forceinline__ void mac(u64 a, u64 b) {
    asm("{\n\t"
        ".reg .u32 a0, a1, b0, b1;\n\t"
        "mov.b64 {a0, a1}, %8;\n\t"
        "mov.b64 {b0, b1}, %9;\n\t"
        "mad.lo.cc.u32 %0, a0, b0, %0;\n\t"
        "madc.hi.cc.u32 %1, a0, b0, %1;\n\t"
        "madc.lo.cc.u32 %2, a1, b1, %2;\n\t"
        "madc.hi.cc.u32 %3, a1, b1, %3;\n\t"
        "addc.u32 %4, %4, 0;\n\t"
        "mad.lo.cc.u32 %5, a0, b1, %5;\n\t"
        "madc.hi.cc.u32 %6, a0, b1, %6;\n\t"
        "addc.u32 %7, %7, 0;\n\t"
        "mad.lo.cc.u32 %5, a1, b0, %5;\n\t"
        "madc.hi.cc.u32 %6, a1, b0, %6;\n\t"
        "addc.u32 %7, %7, 0;\n\t"
        "}"
        : "+r"(e0), "+r"(e1), "+r"(e2), "+r"(e3), "+r"(e4), "+r"(o1), "+r"(o2), "+r"(o3)
        : "l"(a), "l"(b));
  }
  __device__ __forceinline__ void add64(u64 v) {
    asm("{\n\t"
        ".reg .u32 v0, v1;\n\t"
        "mov.b64 {v0, v1}, %5;\n\t"
        "add.cc.u32 %0, %0, v0;\n\t"
        "addc.cc.u32 %1, %1, v1;\n\t"
        "addc.cc.u32 %2, %2, 0;\n\t"
        "addc.cc.u32 %3, %3, 0;\n\t"
        "addc.u32 %4, %4, 0;\n\t"
        "}"
        : "+r"(e0), "+r"(e1), "+r"(e2), "+r"(e3), "+r"(e4)
        : "l"(v));
  }
  // value = hi * 2^128 + mid * 2^64 + lo
  __device__ __forceinline__ void merged(u64& lo, u64& mid, u32& hi) const {
    u32 w1, w2, w3;
    asm("add.cc.u32 %0, %4, %8;\n\t"
        "addc.cc.u32 %1, %5, %9;\n\t"
        "addc.cc.u32 %2, %6, %10;\n\t"
        "addc.u32 %3, %7, 0;"
        : "=r"(w1), "=r"(w2), "=r"(w3), "=r"(hi)
        : "r"(e1), "r"(e2), "r"(e3), "r"(e4), "r"(o1), "r"(o2), "r"(o3));
    lo = ((u64)w1 << 32) | e0;
    mid = ((u64)w3 << 32) | w2;
  }
  // residue in [0,2p) of the accumulated value (which must be < 2^160)
  __device__ __forceinline__ u64 reduce_lazy(const LimbDev& m) const {
    u64 lo, mid;
    u32 hi;
    merged(lo, mid, hi);
    return reduce160_lazy(lo, mid, hi, m);
  }
  // canonical residue of the accumulated value (which must be < 2^160)
  __device__ __forceinline__ u64 reduce(const LimbDev& m) const {
    u64 lo, mid;
    u32 hi;
    merged(lo, mid, hi);
    return csub(reduce160_lazy(lo, mid, hi, m), m.p);
  }
};

// Lazy multiply-accumulate of terms r*w with BOTH operands < 2^62, three 32x32 products per term instead of four.
// The caller splits each operand at bit 31 (split31: r = r1*2^31 + r0, halves < 2^31, half sum rs = r0 + r1 < 2^32),
// and Karatsuba gives
//   r*w = r0*w0 + 2^31*[(r0+r1)(w0+w1) - r0*w0 - r1*w1] + 2^62*r1*w1 .
// The three products go to three 96-bit column sums L = sum r0*w0, M = sum rs*ws, H = sum r1*w1, each its own
// mad.lo.cc/madc.hi.cc/addc chain (one IMAD.WIDE with carry + one IADD3.X), no carry crossing between them; merged()
// combines them once.  Bounds for n terms and k add64 addends: r0*w0, r1*w1 < 2^62 and rs*ws < 2^64, so the sums are
// exact while n + k < 2^32; M - L - H = sum (r0*w1 + r1*w0) >= 0 because add64 adds to L and M alike; the value
// V = sum r*w + sum addends < n*2^124 + k*2^64 < 2^160, the contract of Acc192::merged (the scaler: n <= 65, k <= 1).
// An operand of 2^62 or more breaks the split (r1 or rs no longer fits its word): such terms go through Acc192.
struct Split31 {
  u32 lo, hi, sum;
};
__device__ __forceinline__ Split31 split31(u64 x) {
  const u32 lo = (u32)x & 0x7fffffffu, hi = (u32)(x >> 31);
  return {lo, hi, lo + hi};
}
struct AccKara {
  // the low two words of each sum are one 64-bit register, so the pair an IMAD.WIDE adds into stays in place
  u64 l, m, h;
  u32 l2, m2, h2;
  __device__ __forceinline__ void clear() { l = m = h = 0; l2 = m2 = h2 = 0; }
  __device__ __forceinline__ void mac(u32 r0, u32 r1, u32 rs, u32 w0, u32 w1, u32 ws) {
    asm("{\n\t"
        ".reg .u32 x0, x1, y0, y1, z0, z1;\n\t"
        "mov.b64 {x0, x1}, %0;\n\t"
        "mov.b64 {y0, y1}, %1;\n\t"
        "mov.b64 {z0, z1}, %2;\n\t"
        "mad.lo.cc.u32 x0, %6, %9, x0;\n\t"
        "madc.hi.cc.u32 x1, %6, %9, x1;\n\t"
        "addc.u32 %3, %3, 0;\n\t"
        "mad.lo.cc.u32 y0, %8, %11, y0;\n\t"
        "madc.hi.cc.u32 y1, %8, %11, y1;\n\t"
        "addc.u32 %4, %4, 0;\n\t"
        "mad.lo.cc.u32 z0, %7, %10, z0;\n\t"
        "madc.hi.cc.u32 z1, %7, %10, z1;\n\t"
        "addc.u32 %5, %5, 0;\n\t"
        "mov.b64 %0, {x0, x1};\n\t"
        "mov.b64 %1, {y0, y1};\n\t"
        "mov.b64 %2, {z0, z1};\n\t"
        "}"
        : "+l"(l), "+l"(m), "+l"(h), "+r"(l2), "+r"(m2), "+r"(h2)
        : "r"(r0), "r"(r1), "r"(rs), "r"(w0), "r"(w1), "r"(ws));
  }
  __device__ __forceinline__ void mac(const Split31& r, const Split31& w) { mac(r.lo, r.hi, r.sum, w.lo, w.hi, w.sum); }
  __device__ __forceinline__ void add64(u64 v) {
    asm("add.cc.u64 %0, %0, %4;\n\t"
        "addc.u32 %1, %1, 0;\n\t"
        "add.cc.u64 %2, %2, %4;\n\t"
        "addc.u32 %3, %3, 0;"
        : "+l"(l), "+r"(l2), "+l"(m), "+r"(m2)
        : "l"(v));
  }
  // value = hi * 2^128 + mid * 2^64 + lo = L + 2^31 * (M - L - H) + 2^62 * H
  __device__ __forceinline__ void merged(u64& lo, u64& mid, u32& hi) const {
    const u32 l0 = (u32)l, l1 = (u32)(l >> 32), h0 = (u32)h, h1 = (u32)(h >> 32);
    u32 d0, d1, d2;
    asm("sub.cc.u32 %0, %3, %6;\n\t"
        "subc.cc.u32 %1, %4, %7;\n\t"
        "subc.u32 %2, %5, %8;\n\t"
        "sub.cc.u32 %0, %0, %9;\n\t"
        "subc.cc.u32 %1, %1, %10;\n\t"
        "subc.u32 %2, %2, %11;"
        : "=r"(d0), "=r"(d1), "=r"(d2)
        : "r"((u32)m), "r"((u32)(m >> 32)), "r"(m2), "r"(l0), "r"(l1), "r"(l2), "r"(h0), "r"(h1), "r"(h2));
    // D * 2^31 and H * 2^62 as five little-endian words (H * 2^62 has none at word 0)
    const u32 a0 = d0 << 31, a1 = __funnelshift_l(d0, d1, 31), a2 = __funnelshift_l(d1, d2, 31), a3 = d2 >> 1;
    const u32 b1 = h0 << 30, b2 = __funnelshift_l(h0, h1, 30), b3 = __funnelshift_l(h1, h2, 30), b4 = h2 >> 2;
    u32 w0, w1, w2, w3;
    asm("add.cc.u32 %0, %5, %8;\n\t"
        "addc.cc.u32 %1, %6, %9;\n\t"
        "addc.cc.u32 %2, %7, %10;\n\t"
        "addc.cc.u32 %3, %11, 0;\n\t"
        "addc.u32 %4, %15, 0;\n\t"
        "add.cc.u32 %1, %1, %12;\n\t"
        "addc.cc.u32 %2, %2, %13;\n\t"
        "addc.cc.u32 %3, %3, %14;\n\t"
        "addc.u32 %4, %4, 0;"
        : "=r"(w0), "=r"(w1), "=r"(w2), "=r"(w3), "=r"(hi)
        : "r"(l0), "r"(l1), "r"(l2), "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b1), "r"(b2), "r"(b3), "r"(b4));
    lo = ((u64)w1 << 32) | w0;
    mid = ((u64)w3 << 32) | w2;
  }
  // canonical residue of the accumulated value
  __device__ __forceinline__ u64 reduce(const LimbDev& m) const {
    u64 lo, mid;
    u32 hi;
    merged(lo, mid, hi);
    return csub(reduce160_lazy(lo, mid, hi, m), m.p);
  }
};

// canonical residue of a 128-bit value
__device__ __forceinline__ u64 reduce128_limb(u64 lo, u64 hi, const LimbDev& m) {
  if (m.sol_c) return csub(fold192_solinas(lo, hi, 0, (u32)m.sol_c), m.p);
  return barrett128(lo, hi, m.p, m.bhi, m.blo);
}
// canonical residue of a value < 2^94 (the fixed-point quotients v, w of the scaler are < 2^70)
__device__ __forceinline__ u64 reduce94_limb(u64 lo, u64 hi, const LimbDev& m) {
  if (m.sol_c) return csub(fold94_solinas(lo, hi, (u32)m.sol_c), m.p);
  return barrett128(lo, hi, m.p, m.bhi, m.blo);
}

// acc (7 x 32-bit words, little endian) += r * theta, r = r1*2^32 + r0 (any 64-bit), theta = 128-bit
// (t3:t2:t1:t0).  Two word-serial 32x128 products (IMAD.WIDE with the running carry as addend:
// 32x32 + 32 < 2^64, no overflow) added at word offsets 0 and 1.  Used for the fixed-point sums of
// RnsScaler::scale (rns/scaler.rs:260-298), whose U256 accumulator never exceeds 2^200 here.
__device__ __forceinline__ void mac_theta(u32 (&a)[7], u64 r, u64 tlo, u64 thi) {
  asm("{\n\t"
      ".reg .u32 r0, r1, t0, t1, t2, t3, u0, u1, u2, u3, u4, c;\n\t"
      ".reg .u64 P, C;\n\t"
      "mov.b64 {r0, r1}, %7;\n\t"
      "mov.b64 {t0, t1}, %8;\n\t"
      "mov.b64 {t2, t3}, %9;\n\t"
      // U = r0 * theta
      "mul.wide.u32 P, r0, t0;\n\t"
      "mov.b64 {u0, c}, P;\n\t"
      "cvt.u64.u32 C, c;\n\t"
      "mad.wide.u32 P, r0, t1, C;\n\t"
      "mov.b64 {u1, c}, P;\n\t"
      "cvt.u64.u32 C, c;\n\t"
      "mad.wide.u32 P, r0, t2, C;\n\t"
      "mov.b64 {u2, c}, P;\n\t"
      "cvt.u64.u32 C, c;\n\t"
      "mad.wide.u32 P, r0, t3, C;\n\t"
      "mov.b64 {u3, u4}, P;\n\t"
      "add.cc.u32 %0, %0, u0;\n\t"
      "addc.cc.u32 %1, %1, u1;\n\t"
      "addc.cc.u32 %2, %2, u2;\n\t"
      "addc.cc.u32 %3, %3, u3;\n\t"
      "addc.cc.u32 %4, %4, u4;\n\t"
      "addc.cc.u32 %5, %5, 0;\n\t"
      "addc.u32 %6, %6, 0;\n\t"
      // V = r1 * theta, one word up
      "mul.wide.u32 P, r1, t0;\n\t"
      "mov.b64 {u0, c}, P;\n\t"
      "cvt.u64.u32 C, c;\n\t"
      "mad.wide.u32 P, r1, t1, C;\n\t"
      "mov.b64 {u1, c}, P;\n\t"
      "cvt.u64.u32 C, c;\n\t"
      "mad.wide.u32 P, r1, t2, C;\n\t"
      "mov.b64 {u2, c}, P;\n\t"
      "cvt.u64.u32 C, c;\n\t"
      "mad.wide.u32 P, r1, t3, C;\n\t"
      "mov.b64 {u3, u4}, P;\n\t"
      "add.cc.u32 %1, %1, u0;\n\t"
      "addc.cc.u32 %2, %2, u1;\n\t"
      "addc.cc.u32 %3, %3, u2;\n\t"
      "addc.cc.u32 %4, %4, u3;\n\t"
      "addc.cc.u32 %5, %5, u4;\n\t"
      "addc.u32 %6, %6, 0;\n\t"
      "}"
      : "+r"(a[0]), "+r"(a[1]), "+r"(a[2]), "+r"(a[3]), "+r"(a[4]), "+r"(a[5]), "+r"(a[6])
      : "l"(r), "l"(tlo), "l"(thi));
}

// The same sum as repeated mac_theta calls, restructured like Acc192: r0*theta and r1*theta each go to an even
// and an odd column set (words 0/2 and 1/3 of the product), four independent carry chains of two IMAD.WIDE and
// one IADD3.X each, no dependence between the eight multiplies of a term.  value = A + (B + C) * 2^32 + D * 2^64.
struct AccTheta {
  u32 a[5], b[5], c[5], d[5];
  __device__ __forceinline__ void clear() {
#pragma unroll
    for (int i = 0; i < 5; i++) a[i] = b[i] = c[i] = d[i] = 0;
  }
  __device__ __forceinline__ void mac(u64 r, u64 tlo, u64 thi) {
    asm("{\n\t"
        ".reg .u32 r0, r1, t0, t1, t2, t3;\n\t"
        "mov.b64 {r0, r1}, %20;\n\t"
        "mov.b64 {t0, t1}, %21;\n\t"
        "mov.b64 {t2, t3}, %22;\n\t"
        "mad.lo.cc.u32 %0, r0, t0, %0;\n\t"
        "madc.hi.cc.u32 %1, r0, t0, %1;\n\t"
        "madc.lo.cc.u32 %2, r0, t2, %2;\n\t"
        "madc.hi.cc.u32 %3, r0, t2, %3;\n\t"
        "addc.u32 %4, %4, 0;\n\t"
        "mad.lo.cc.u32 %5, r0, t1, %5;\n\t"
        "madc.hi.cc.u32 %6, r0, t1, %6;\n\t"
        "madc.lo.cc.u32 %7, r0, t3, %7;\n\t"
        "madc.hi.cc.u32 %8, r0, t3, %8;\n\t"
        "addc.u32 %9, %9, 0;\n\t"
        "mad.lo.cc.u32 %10, r1, t0, %10;\n\t"
        "madc.hi.cc.u32 %11, r1, t0, %11;\n\t"
        "madc.lo.cc.u32 %12, r1, t2, %12;\n\t"
        "madc.hi.cc.u32 %13, r1, t2, %13;\n\t"
        "addc.u32 %14, %14, 0;\n\t"
        "mad.lo.cc.u32 %15, r1, t1, %15;\n\t"
        "madc.hi.cc.u32 %16, r1, t1, %16;\n\t"
        "madc.lo.cc.u32 %17, r1, t3, %17;\n\t"
        "madc.hi.cc.u32 %18, r1, t3, %18;\n\t"
        "addc.u32 %19, %19, 0;\n\t"
        "}"
        : "+r"(a[0]), "+r"(a[1]), "+r"(a[2]), "+r"(a[3]), "+r"(a[4]), "+r"(b[0]), "+r"(b[1]), "+r"(b[2]), "+r"(b[3]),
          "+r"(b[4]), "+r"(c[0]), "+r"(c[1]), "+r"(c[2]), "+r"(c[3]), "+r"(c[4]), "+r"(d[0]), "+r"(d[1]), "+r"(d[2]),
          "+r"(d[3]), "+r"(d[4])
        : "l"(r), "l"(tlo), "l"(thi));
  }
  // the 7 little-endian words of the sum (which must be < 2^224)
  __device__ __forceinline__ void words(u32 (&w)[7]) const {
    u64 t = (u64)a[1] + b[0] + c[0];
    w[0] = a[0];
    w[1] = (u32)t;
    t = (t >> 32) + a[2] + b[1] + c[1] + d[0];
    w[2] = (u32)t;
    t = (t >> 32) + a[3] + b[2] + c[2] + d[1];
    w[3] = (u32)t;
    t = (t >> 32) + a[4] + b[3] + c[3] + d[2];
    w[4] = (u32)t;
    t = (t >> 32) + b[4] + c[4] + d[3];
    w[5] = (u32)t;
    t = (t >> 32) + d[4];
    w[6] = (u32)t;
  }
};

// a*b mod p in [0,2p) for canonical a, b: for consumers that accept lazy operands (the inverse butterflies)
__device__ __forceinline__ u64 mulmod_limb_lazy(u64 a, u64 b, const LimbDev& m) {
  if (m.sol_c) {
    u64 lo, hi;
    mul128_62(a, b, lo, hi);
    return fold192_solinas(lo, hi, 0, (u32)m.sol_c);
  }
  return barrett128_lazy(a * b, __umul64hi(a, b), m.p, m.bhi, m.blo);
}

// canonical a*b mod p for canonical a, b (Modulus::mul / mul_opt, zq/mod.rs:131-156)
__device__ __forceinline__ u64 mulmod_limb(u64 a, u64 b, const LimbDev& m) {
  if (m.sol_c) {
    u64 lo, hi;
    mul128_62(a, b, lo, hi);
    return csub(fold192_solinas(lo, hi, 0, (u32)m.sol_c), m.p);
  }
  return mulmod(a, b, m.p, m.bhi, m.blo);
}

}  // namespace fhe_b200
