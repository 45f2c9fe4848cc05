// TMA-fed persistent NTT tile kernels for N >= 2^13 (sm_90a).  Same transform, tables and canonical outputs as
// ntt.cuh / ntt_fast.cuh (NttOperator::{forward,backward}, crates/fhe-math/src/ntt/native.rs:77-233); what changes
// is who moves the data and how often the constants are fetched:
//
//   * every tile travels HBM -> shared memory -> HBM by TMA (cp.async.bulk.tensor, SASS UTMALDG / UTMASTG) issued by
//     one producer thread per CTA and tracked with mbarriers; the compute warps execute no global load / store and
//     no 64-bit address arithmetic at all -- those instructions compete with the butterflies for the integer
//     multiplier pipe, which (not HBM) bounds this transform (DESIGN.md section 3);
//   * CTAs are persistent: each one walks a contiguous range of the launch's tiles through a ring of STAGES
//     shared-memory buffers, so tiles k+1 .. k+STAGES-1 are already in flight (or landed) while tile k's butterflies run;
//   * the tiles of a launch are ordered limb-major, polynomial-minor, so consecutive tiles of a CTA use the SAME
//     twiddles: they are staged in shared memory once per (limb, tile position) and read from there with
//     `base + immediate` 128-bit loads (the rows pass used to fetch 16 KiB of twiddles from L2 per 8 KiB of data);
//   * butterflies update the tile in place (one CTA barrier per radix-8 round, none for the tile hand-over); the rows
//     pass handles two polynomials per iteration, so one twiddle fetch, one hand-over and one barrier serve 48
//     butterflies per thread.
//
// Layouts.  cols tile: [N1 points][16 columns] u64, 128-byte box rows, no swizzle: every radix-8 access of a warp is
// 256 contiguous bytes (or two 128-byte rows 1 KiB apart).  rows tile: [R rows][64 points] seen as 128-byte box rows
// with the TMA 128-byte swizzle (16-byte chunk c of box row r sits at chunk c ^ (r & 7)): the stride-8 round reads
// 64-bit words, the unit-stride round 128-bit pairs, both without bank conflicts.
#pragma once
#include <cuda.h>
#include <type_traits>

#include "engine.hpp"
#include "ntt.cuh"

namespace fhe_b200 {

struct NttTmaArgs {
  const LimbDev* limbs;
  u32 n_polys;         // polynomials (ciphertext x part, or ciphertext x digit)
  u32 lpp;             // limbs per polynomial of the output: limb position j = 0 .. lpp-1
  u32 in_bcast;        // 1: the source row of (p, j) is p (digit broadcast, rq/mod.rs:563-586); 0: it is the output row
  u32 digit_adjacent;  // output row of (p, j): 0: p*lpp + j ; 1: ((p / n_dig)*lpp + j)*n_dig + p % n_dig
  u32 n_dig;
  u32 reduce_on_load;  // forward first pass only: reduce source words modulo the row's prime
  u32 lazy_out;        // forward last pass only: leave outputs in [0,4p)
  u32 logn;
  u32 tiles_per_row;
  u32 tiles_total;     // lpp * tiles_per_row * n_polys; tile index = (j*tiles_per_row + tau)*n_polys + p
  u32 limb_inner;      // = in_bcast (cols pass): tile index = (tau*n_polys + p)*lpp + j instead (see cols_tile)
  unsigned short ids[kMaxPos];
};

namespace tma {

__device__ __forceinline__ u32 smem_u32(const void* p) { return (u32)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(u32 bar, u32 count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(u32 bar, u32 bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(u32 bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
// one bounded wait: the hardware may suspend the thread for up to `ns` nanoseconds while the phase is incomplete
__device__ __forceinline__ u32 mbar_try_wait(u32 bar, u32 parity, u32 ns) {
  u32 ok;
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t"
      "}"
      : "=r"(ok)
      : "r"(bar), "r"(parity), "r"(ns)
      : "memory");
  return ok;
}
// a wait that cannot hang the device: a protocol error traps after a few seconds instead of spinning forever.  The
// waiter sleeps inside try_wait (no instruction stream of polls competing with the butterflies for issue slots).
__device__ __forceinline__ void mbar_wait(u32 bar, u32 parity) {
  u32 tries = 0;
  while (!mbar_try_wait(bar, parity, 100000u)) {
    if (++tries > 4000000u) __trap();
  }
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void bulk_wait_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
__device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
template <int NT>
__device__ __forceinline__ void consumer_sync() {
  asm volatile("bar.sync 1, %0;" ::"n"(NT) : "memory");
}

__device__ __forceinline__ void load_2d(u32 dst, const CUtensorMap* tm, u32 c0, u32 c1, u32 bar) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
      ::"r"(dst), "l"(tm), "r"(c0), "r"(c1), "r"(bar)
      : "memory");
}
// a contiguous global -> shared copy (16-byte aligned, a multiple of 16 bytes) completing on mbarrier `bar`
__device__ __forceinline__ void load_1d(u32 dst, const void* src, u32 bytes, u32 bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(dst), "l"(src), "r"(bytes), "r"(bar)
               : "memory");
}
// the key tiles of (limb j, TC-coefficient tile tau) of a key pair [limb][digit][N]: digit d of k0 / k1 lands at
// dst0 / dst1 + d * TC * 8.  2 * nd row segments of TC words, all completing on `bar`.
template <u32 TC>
__device__ __forceinline__ void load_key_tiles(u32 dst0, u32 dst1, const u64* k0, const u64* k1, u32 j, u32 tau,
                                               u32 nd, u32 logn, u32 bar) {
  mbar_expect_tx(bar, 2 * nd * TC * 8);
  const size_t row0 = ((size_t)j * nd << logn) + (size_t)tau * TC;
  for (u32 d = 0; d < nd; d++) {
    const size_t off = row0 + ((size_t)d << logn);
    load_1d(dst0 + d * TC * 8, k0 + off, TC * 8, bar);
    load_1d(dst1 + d * TC * 8, k1 + off, TC * 8, bar);
  }
}
__device__ __forceinline__ void store_2d(const CUtensorMap* tm, u32 c0, u32 c1, u32 src) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.tile.bulk_group [%0, {%1, %2}], [%3];" ::"l"(tm), "r"(c0),
               "r"(c1), "r"(src)
               : "memory");
}
__device__ __forceinline__ void load_3d(u32 dst, const CUtensorMap* tm, u32 c0, u32 c1, u32 c2, u32 bar) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], "
      "[%5];" ::"r"(dst),
      "l"(tm), "r"(c0), "r"(c1), "r"(c2), "r"(bar)
      : "memory");
}
__device__ __forceinline__ void store_3d(const CUtensorMap* tm, u32 c0, u32 c1, u32 c2, u32 src) {
  asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.tile.bulk_group [%0, {%1, %2, %3}], [%4];" ::"l"(tm),
               "r"(c0), "r"(c1), "r"(c2), "r"(src)
               : "memory");
}
__device__ __forceinline__ void prefetch_map(const CUtensorMap* tm) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(tm) : "memory");
}

__device__ __forceinline__ u64 lds64(u32 a) {
  u64 v;
  asm volatile("ld.shared.u64 %0, [%1];" : "=l"(v) : "r"(a));
  return v;
}
__device__ __forceinline__ void sts64(u32 a, u64 v) { asm volatile("st.shared.u64 [%0], %1;" ::"r"(a), "l"(v) : "memory"); }
__device__ __forceinline__ ulonglong2 lds128(u32 a) {
  ulonglong2 v;
  asm volatile("ld.shared.v2.u64 {%0, %1}, [%2];" : "=l"(v.x), "=l"(v.y) : "r"(a));
  return v;
}
__device__ __forceinline__ void sts128(u32 a, u64 x, u64 y) {
  asm volatile("st.shared.v2.u64 [%0], {%1, %2};" ::"r"(a), "l"(x), "l"(y) : "memory");
}

// NS Cooley-Tukey stages on a radix-2^NS group (ntt/native.rs:160-176), tw[(1<<u)-1+m] = twiddle of stage u, block m
template <int NS>
__device__ __forceinline__ void fwd_stages(u64* v, const ulonglong2* tw, u64 p, u64 p2) {
  constexpr int R = 1 << NS;
#pragma unroll
  for (int u = 0; u < NS; u++) {
    const int half = R >> (u + 1);
#pragma unroll
    for (int m = 0; m < (1 << u); m++) {
      const ulonglong2 w = tw[(1 << u) - 1 + m];
#pragma unroll
      for (int e = 0; e < half; e++) {
        const int jj = m * 2 * half + e;
        bf_fwd<false>(v[jj], v[jj + half], w.x, w.y, p, p2, 0);
      }
    }
  }
}
// fwd_stages<3> with the twiddle pair of (stage u, block m) fetched by tw(u, m) right before the stage that uses it
template <class TW>
__device__ __forceinline__ void fwd_stages3_staged(u64* v, u64 p, u64 p2, const TW& tw) {
#pragma unroll
  for (int u = 0; u < 3; u++) {
    const int half = 8 >> (u + 1);
    ulonglong2 w[4];
#pragma unroll
    for (int m = 0; m < (1 << u); m++) w[m] = tw(u, m);
#pragma unroll
    for (int m = 0; m < (1 << u); m++) {
#pragma unroll
      for (int e = 0; e < half; e++) {
        const int jj = m * 2 * half + e;
        bf_fwd<false>(v[jj], v[jj + half], w[m].x, w[m].y, p, p2, 0);
      }
    }
  }
}
// constants of the last inverse stage (N^-1 and zetas_inv[N-2] * N^-1 with their Shoup companions), held in
// registers by the kernels that reach it
struct LastStage {
  u64 ninv, ninv_s, zn, zn_s;
};
// NS Gentleman-Sande stages, innermost stage first (ntt/native.rs:120-136); `last`: stage u == 0 is the transform's
// final stage, fused with the N^-1 scaling (native.rs:230-232)
template <int NS, typename LS>
__device__ __forceinline__ void inv_stages(u64* v, const ulonglong2* tz, u64 p, u64 p2, bool last, const LS& L) {
  constexpr int R = 1 << NS;
#pragma unroll
  for (int u = NS - 1; u >= 0; u--) {
    const int half = R >> (u + 1);
    if (u == 0 && last) {
#pragma unroll
      for (int e = 0; e < half; e++) {
        const u64 a = v[e], b2 = v[e + half];
        v[e] = csub(mul_shoup_lazy(a + b2, L.ninv, L.ninv_s, p), p);
        v[e + half] = csub(mul_shoup_lazy(p2 + a - b2, L.zn, L.zn_s, p), p);
      }
    } else {
#pragma unroll
      for (int m = 0; m < (1 << u); m++) {
        const ulonglong2 z = tz[(1 << u) - 1 + m];
#pragma unroll
        for (int e = 0; e < half; e++) {
          const int jj = m * 2 * half + e;
          bf_inv<false>(v[jj], v[jj + half], z.x, z.y, p, p2, 0);
        }
      }
    }
  }
}

// tile walk shared by producer and consumers: tile index -> (jt = j*tiles_per_row + tau, p)
struct TileWalk {
  u32 jt, p, n_polys;
  __device__ __forceinline__ void init(u32 idx, u32 np) {
    n_polys = np;
    jt = idx / np;
    p = idx - jt * np;
  }
  __device__ __forceinline__ bool next() {   // true when jt changed
    if (++p == n_polys) {
      p = 0;
      jt++;
      return true;
    }
    return false;
  }
};

__device__ __forceinline__ u32 out_row_of(const NttTmaArgs& A, u32 p, u32 j) {
  if (A.digit_adjacent) {
    const u32 ct = p / A.n_dig, d = p - ct * A.n_dig;
    return (ct * A.lpp + j) * A.n_dig + d;
  }
  return p * A.lpp + j;
}

}  // namespace tma

// ------------------------------------------------------------------------------------------------ rows pass
// The 6 unit-stride-side stages on tiles of R = 2^RLOG matrix rows of 64 points (one contiguous 512*R-byte chunk).
// 8R consumer threads (8 words each) + one producer warp.  Tensor map: the whole buffer as [..][16] u64 (128-byte
// rows), box {16, 4R}, 128-byte swizzle.
template <int RLOG, int STAGES>
struct RowsCfg {
  static constexpr u32 R = 1u << RLOG;
  static constexpr u32 NT = 8 * R;                 // consumer threads
  static constexpr u32 TILE_BYTES = 512 * R;
  static constexpr u32 TW_PAIRS = 63 * R;          // twiddle pairs of one tile position
  static constexpr u32 SMEM = STAGES * TILE_BYTES + TW_PAIRS * 16 + 2 * STAGES * 8 + 1024;   // + alignment slack
};

// LAZY (forward only): leave the outputs in [0,4p) (forward_vt_lazy, native.rs:142-181)
template <bool INV, int RLOG, int STAGES, int MINB, bool LAZY>
__global__ void __launch_bounds__(RowsCfg<RLOG, STAGES>::NT + 32, MINB)
    ntt_tma_rows_kernel(const __grid_constant__ CUtensorMap tm_in, const __grid_constant__ CUtensorMap tm_out,
                        const NttTmaArgs A) {
  using namespace tma;
  using Cfg = RowsCfg<RLOG, STAGES>;
  constexpr u32 R = Cfg::R, NT = Cfg::NT, TILE_BYTES = Cfg::TILE_BYTES;
  extern __shared__ unsigned char smem_raw[];
  const u32 base = (smem_u32(smem_raw) + 1023u) & ~1023u;   // the 128-byte swizzle works on absolute address bits
  const u32 tw_base = base + STAGES * TILE_BYTES;
  const u32 bar_full = tw_base + Cfg::TW_PAIRS * 16;
  const u32 bar_done = bar_full + STAGES * 8;

  if (threadIdx.x == 0) {
#pragma unroll
    for (int s = 0; s < STAGES; s++) {
      mbar_init(bar_full + 8 * s, 1);
      mbar_init(bar_done + 8 * s, NT);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  const u32 lo = (u32)(((u64)A.tiles_total * blockIdx.x) / gridDim.x);
  const u32 hi = (u32)(((u64)A.tiles_total * (blockIdx.x + 1)) / gridDim.x);
  const u32 n = hi - lo;
  const u32 box_rows_per_row = (1u << A.logn) >> 4;   // 128-byte box rows per polynomial row

  if (threadIdx.x >= NT) {
    // ---------------- producer: one thread moves every tile of this CTA in and out
    if (threadIdx.x != NT) return;
    prefetch_map(&tm_in);
    prefetch_map(&tm_out);
    TileWalk wl, ws;   // load cursor, store cursor
    wl.init(lo, A.n_polys);
    ws.init(lo, A.n_polys);
    auto coord = [&](const TileWalk& w, bool input) -> u32 {
      const u32 j = w.jt / A.tiles_per_row, tau = w.jt - j * A.tiles_per_row;
      const u32 row = (input && A.in_bcast) ? w.p : out_row_of(A, w.p, j);
      return row * box_rows_per_row + tau * (4 * R);
    };
    u32 loaded = 0;
    auto load_next = [&]() {
      const u32 s = loaded % STAGES;
      mbar_expect_tx(bar_full + 8 * s, TILE_BYTES);
      load_2d(base + s * TILE_BYTES, &tm_in, 0, coord(wl, true), bar_full + 8 * s);
      wl.next();
      loaded++;
    };
    while (loaded < n && loaded < (u32)STAGES) load_next();  // every buffer starts full
    for (u32 i = 0; i < n; i++) {
      const u32 s = i % STAGES;
      mbar_wait(bar_done + 8 * s, (i / STAGES) & 1);         // the consumers have finished tile i (in place)
      store_2d(&tm_out, 0, coord(ws, false), base + s * TILE_BYTES);
      bulk_commit();
      ws.next();
      if (loaded < n) {
        bulk_wait_read<0>();                                 // the store has left shared memory: its buffer takes
        load_next();                                         // tile i+STAGES while tiles i+1 .. are being computed
      }
    }
    bulk_wait_all();
    return;
  }

  // ---------------- consumers
  const u32 tid = threadIdx.x;
  const u32 x = tid & 7, b = tid >> 3;   // both rounds: b = matrix row inside the tile, x = a_lo (round 0) / a_hi (round 1)
  // byte offsets inside a (1024-byte aligned) tile buffer, TMA 128-byte swizzle: word i lives in 16-byte chunk
  // ((i>>1)&7) ^ ((i>>4)&7) of 128-byte row i>>4
  u32 off0[8];   // round 0: words 64b + x + 8e (64-bit accesses)
#pragma unroll
  for (int e = 0; e < 8; e++) {
    const u32 i = 64 * b + x + 8 * e;
    off0[e] = ((i >> 4) << 7) | ((((i >> 1) & 7) ^ ((i >> 4) & 7)) << 4) | ((i & 1) << 3);
  }
  u32 off1[4];   // round 1: pairs (64b + 8x + 2k, +1) (128-bit accesses)
#pragma unroll
  for (int k = 0; k < 4; k++) {
    const u32 i = 64 * b + 8 * x + 2 * k;
    off1[k] = ((i >> 4) << 7) | ((((i >> 1) & 7) ^ ((i >> 4) & 7)) << 4);
  }
  // twiddle pair addresses: region tl starts at pair R*(2^tl - 1); stages 0..2 index (b << tl) + m, stages 3..5 are
  // stored as 2^u planes of 8R pairs so that lane `tid` reads pair `tid` of plane m (unit stride across the warp)
  const u32 tw0 = tw_base + 16 * (b);                       // tl = 0: region offset 0
  const u32 tw1 = tw_base + 16 * (R * 1 + (b << 1));        // tl = 1
  const u32 tw2 = tw_base + 16 * (R * 3 + (b << 2));        // tl = 2
  const u32 tw3 = tw_base + 16 * (R * 7 + tid);             // tl = 3: 1 plane
  const u32 tw4 = tw_base + 16 * (R * 15 + tid);            // tl = 4: 2 planes of 8R
  const u32 tw5 = tw_base + 16 * (R * 31 + tid);            // tl = 5: 4 planes of 8R

  TileWalk w;
  w.init(lo, A.n_polys);
  bool fresh = true;
  u64 p = 0, p2 = 0;
  const u32 logn1 = A.logn - 6;
  for (u32 i = 0; i < n; i++) {
    if (fresh) {
      // new (limb, tile position): stage its 63R twiddle pairs (omegas[(1<<s) + (row0<<tl) + k] forward,
      // zetas_inv[N - (2<<s) + (row0<<tl) + k] inverse, s = logn1 + tl; ntt/native.rs:44-56)
      const u32 j = w.jt / A.tiles_per_row, tau = w.jt - j * A.tiles_per_row;
      const LimbDev& L = A.limbs[A.ids[j]];
      p = L.p;
      p2 = L.p2;
      const ulonglong2* tab = INV ? L.zi : L.om;
      const u32 row0 = tau * R;
      if (i) consumer_sync<NT>();   // nobody still reads the previous twiddles
#pragma unroll
      for (int tl = 0; tl < 6; tl++) {
        const u32 s = logn1 + tl;
        const u32 g0 = (INV ? ((1u << A.logn) - (2u << s)) : (1u << s)) + (row0 << tl);
        for (u32 k = tid; k < (R << tl); k += NT) {
          const ulonglong2 v = __ldg(tab + g0 + k);
          const u32 dst = tl < 3 ? k : (k & ((1u << (tl >= 3 ? tl - 3 : 0)) - 1)) * (8 * R) + (k >> (tl >= 3 ? tl - 3 : 0));
          sts128(tw_base + 16 * (R * ((1u << tl) - 1) + dst), v.x, v.y);
        }
      }
      consumer_sync<NT>();
    }
    const u32 s = i % STAGES;
    const u32 buf = base + s * TILE_BYTES;
    mbar_wait(bar_full + 8 * s, (i / STAGES) & 1);
    u64 v[8];
    ulonglong2 tw[7];
    if (!INV) {
      // round 0: stages logn1 .. logn1+2 (strides 32, 16, 8)
#pragma unroll
      for (int e = 0; e < 8; e++) v[e] = lds64(buf + off0[e]);
      tw[0] = lds128(tw0);
      tw[1] = lds128(tw1);
      tw[2] = lds128(tw1 + 16);
#pragma unroll
      for (int m = 0; m < 4; m++) tw[3 + m] = lds128(tw2 + 16 * m);
      fwd_stages<3>(v, tw, p, p2);
#pragma unroll
      for (int e = 0; e < 8; e++) sts64(buf + off0[e], v[e]);
      consumer_sync<NT>();
      // round 1: stages logn1+3 .. logn-1 (strides 4, 2, 1), then reduce3 unless lazy (native.rs:178-180, :238)
#pragma unroll
      for (int k = 0; k < 4; k++) {
        const ulonglong2 t = lds128(buf + off1[k]);
        v[2 * k] = t.x;
        v[2 * k + 1] = t.y;
      }
      tw[0] = lds128(tw3);
      tw[1] = lds128(tw4);
      tw[2] = lds128(tw4 + 16 * 8 * R);
#pragma unroll
      for (int m = 0; m < 4; m++) tw[3 + m] = lds128(tw5 + 16 * 8 * R * m);
      fwd_stages<3>(v, tw, p, p2);
      if (!LAZY) {
#pragma unroll
        for (int e = 0; e < 8; e++) v[e] = fwd_final<false>(v[e], p, p2, 0);
      }
#pragma unroll
      for (int k = 0; k < 4; k++) sts128(buf + off1[k], v[2 * k], v[2 * k + 1]);
    } else {
      // inverse: round 1 first (strides 1, 2, 4), then round 0 (strides 8, 16, 32)
#pragma unroll
      for (int k = 0; k < 4; k++) {
        const ulonglong2 t = lds128(buf + off1[k]);
        v[2 * k] = t.x;
        v[2 * k + 1] = t.y;
      }
      tw[0] = lds128(tw3);
      tw[1] = lds128(tw4);
      tw[2] = lds128(tw4 + 16 * 8 * R);
#pragma unroll
      for (int m = 0; m < 4; m++) tw[3 + m] = lds128(tw5 + 16 * 8 * R * m);
      inv_stages<3>(v, tw, p, p2, false, A.limbs[0]);
#pragma unroll
      for (int k = 0; k < 4; k++) sts128(buf + off1[k], v[2 * k], v[2 * k + 1]);
      consumer_sync<NT>();
#pragma unroll
      for (int e = 0; e < 8; e++) v[e] = lds64(buf + off0[e]);
      tw[0] = lds128(tw0);
      tw[1] = lds128(tw1);
      tw[2] = lds128(tw1 + 16);
#pragma unroll
      for (int m = 0; m < 4; m++) tw[3 + m] = lds128(tw2 + 16 * m);
      inv_stages<3>(v, tw, p, p2, false, A.limbs[0]);
#pragma unroll
      for (int e = 0; e < 8; e++) sts64(buf + off0[e], v[e]);
    }
    fence_proxy_async();            // the tile is read next by the TMA store (async proxy)
    mbar_arrive(bar_done + 8 * s);
    fresh = w.next();
  }
}

// The same pass on TWO polynomials per iteration (tiles (p, p+1) of the same limb and tile position): one twiddle fetch,
// one tile hand-over and one CTA barrier serve 48 butterflies per thread instead of 24.  A.n_polys counts PAIRS.
template <bool INV, int RLOG, int STAGES, int MINB, bool LAZY>
__global__ void __launch_bounds__(RowsCfg<RLOG, STAGES>::NT + 32, MINB)
    ntt_tma_rows_pair_kernel(const __grid_constant__ CUtensorMap tm_in, const __grid_constant__ CUtensorMap tm_out,
                        const NttTmaArgs A) {
  using namespace tma;
  using Cfg = RowsCfg<RLOG, STAGES>;
  constexpr u32 R = Cfg::R, NT = Cfg::NT, TILE_BYTES = Cfg::TILE_BYTES, STAGE_BYTES = 2 * TILE_BYTES;
  extern __shared__ unsigned char smem_raw[];
  const u32 base = (smem_u32(smem_raw) + 1023u) & ~1023u;   // the 128-byte swizzle works on absolute address bits
  const u32 tw_base = base + STAGES * STAGE_BYTES;
  const u32 bar_full = tw_base + Cfg::TW_PAIRS * 16;
  const u32 bar_done = bar_full + STAGES * 8;

  if (threadIdx.x == 0) {
#pragma unroll
    for (int s = 0; s < STAGES; s++) {
      mbar_init(bar_full + 8 * s, 1);
      mbar_init(bar_done + 8 * s, NT);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  const u32 lo = (u32)(((u64)A.tiles_total * blockIdx.x) / gridDim.x);
  const u32 hi = (u32)(((u64)A.tiles_total * (blockIdx.x + 1)) / gridDim.x);
  const u32 n = hi - lo;
  const u32 box_rows_per_row = (1u << A.logn) >> 4;   // 128-byte box rows per polynomial row

  if (threadIdx.x >= NT) {
    // ---------------- producer: one thread moves every tile of this CTA in and out
    if (threadIdx.x != NT) return;
    prefetch_map(&tm_in);
    prefetch_map(&tm_out);
    TileWalk wl, ws;   // load cursor, store cursor
    wl.init(lo, A.n_polys);
    ws.init(lo, A.n_polys);
    auto coord = [&](const TileWalk& w, bool input, u32 h) -> u32 {
      const u32 j = w.jt / A.tiles_per_row, tau = w.jt - j * A.tiles_per_row;
      const u32 poly = 2 * w.p + h;
      const u32 row = (input && A.in_bcast) ? poly : out_row_of(A, poly, j);
      return row * box_rows_per_row + tau * (4 * R);
    };
    u32 loaded = 0;
    auto load_next = [&]() {
      const u32 s = loaded % STAGES;
      mbar_expect_tx(bar_full + 8 * s, STAGE_BYTES);
      load_2d(base + s * STAGE_BYTES, &tm_in, 0, coord(wl, true, 0), bar_full + 8 * s);
      load_2d(base + s * STAGE_BYTES + TILE_BYTES, &tm_in, 0, coord(wl, true, 1), bar_full + 8 * s);
      wl.next();
      loaded++;
    };
    while (loaded < n && loaded < (u32)STAGES) load_next();  // every buffer starts full
    for (u32 i = 0; i < n; i++) {
      const u32 s = i % STAGES;
      mbar_wait(bar_done + 8 * s, (i / STAGES) & 1);         // the consumers have finished tile i (in place)
      store_2d(&tm_out, 0, coord(ws, false, 0), base + s * STAGE_BYTES);
      store_2d(&tm_out, 0, coord(ws, false, 1), base + s * STAGE_BYTES + TILE_BYTES);
      bulk_commit();
      ws.next();
      if (loaded < n) {
        bulk_wait_read<0>();                                 // the store has left shared memory: its buffer takes
        load_next();                                         // tile i+STAGES while tiles i+1 .. are being computed
      }
    }
    bulk_wait_all();
    return;
  }

  // ---------------- consumers
  const u32 tid = threadIdx.x;
  const u32 x = tid & 7, b = tid >> 3;   // both rounds: b = matrix row inside the tile, x = a_lo (round 0) / a_hi (round 1)
  // byte offsets inside a (1024-byte aligned) tile buffer, TMA 128-byte swizzle: word i lives in 16-byte chunk
  // ((i>>1)&7) ^ ((i>>4)&7) of 128-byte row i>>4
  u32 off0[8];   // round 0: words 64b + x + 8e (64-bit accesses)
#pragma unroll
  for (int e = 0; e < 8; e++) {
    const u32 i = 64 * b + x + 8 * e;
    off0[e] = ((i >> 4) << 7) | ((((i >> 1) & 7) ^ ((i >> 4) & 7)) << 4) | ((i & 1) << 3);
  }
  u32 off1[4];   // round 1: pairs (64b + 8x + 2k, +1) (128-bit accesses)
#pragma unroll
  for (int k = 0; k < 4; k++) {
    const u32 i = 64 * b + 8 * x + 2 * k;
    off1[k] = ((i >> 4) << 7) | ((((i >> 1) & 7) ^ ((i >> 4) & 7)) << 4);
  }
  // twiddle pair addresses: region tl starts at pair R*(2^tl - 1); stages 0..2 index (b << tl) + m, stages 3..5 are
  // stored as 2^u planes of 8R pairs so that lane `tid` reads pair `tid` of plane m (unit stride across the warp)
  const u32 tw0 = tw_base + 16 * (b);                       // tl = 0: region offset 0
  const u32 tw1 = tw_base + 16 * (R * 1 + (b << 1));        // tl = 1
  const u32 tw2 = tw_base + 16 * (R * 3 + (b << 2));        // tl = 2
  const u32 tw3 = tw_base + 16 * (R * 7 + tid);             // tl = 3: 1 plane
  const u32 tw4 = tw_base + 16 * (R * 15 + tid);            // tl = 4: 2 planes of 8R
  const u32 tw5 = tw_base + 16 * (R * 31 + tid);            // tl = 5: 4 planes of 8R

  TileWalk w;
  w.init(lo, A.n_polys);
  bool fresh = true;
  u64 p = 0, p2 = 0;
  const u32 logn1 = A.logn - 6;
  for (u32 i = 0; i < n; i++) {
    if (fresh) {
      // new (limb, tile position): stage its 63R twiddle pairs (omegas[(1<<s) + (row0<<tl) + k] forward,
      // zetas_inv[N - (2<<s) + (row0<<tl) + k] inverse, s = logn1 + tl; ntt/native.rs:44-56)
      const u32 j = w.jt / A.tiles_per_row, tau = w.jt - j * A.tiles_per_row;
      const LimbDev& L = A.limbs[A.ids[j]];
      p = L.p;
      p2 = L.p2;
      const ulonglong2* tab = INV ? L.zi : L.om;
      const u32 row0 = tau * R;
      if (i) consumer_sync<NT>();   // nobody still reads the previous twiddles
#pragma unroll
      for (int tl = 0; tl < 6; tl++) {
        const u32 s = logn1 + tl;
        const u32 g0 = (INV ? ((1u << A.logn) - (2u << s)) : (1u << s)) + (row0 << tl);
        for (u32 k = tid; k < (R << tl); k += NT) {
          const ulonglong2 v = __ldg(tab + g0 + k);
          const u32 dst = tl < 3 ? k : (k & ((1u << (tl >= 3 ? tl - 3 : 0)) - 1)) * (8 * R) + (k >> (tl >= 3 ? tl - 3 : 0));
          sts128(tw_base + 16 * (R * ((1u << tl) - 1) + dst), v.x, v.y);
        }
      }
      consumer_sync<NT>();
    }
    const u32 s = i % STAGES;
    const u32 buf0 = base + s * STAGE_BYTES;
    mbar_wait(bar_full + 8 * s, (i / STAGES) & 1);
    u64 v[8];
    ulonglong2 tw[7];
    // first round of the pass on both tiles (twiddles fetched once), barrier, second round on both tiles
    if (!INV) {
      tw[0] = lds128(tw0);
      tw[1] = lds128(tw1);
      tw[2] = lds128(tw1 + 16);
#pragma unroll
      for (int m = 0; m < 4; m++) tw[3 + m] = lds128(tw2 + 16 * m);
    } else {
      tw[0] = lds128(tw3);
      tw[1] = lds128(tw4);
      tw[2] = lds128(tw4 + 16 * 8 * R);
#pragma unroll
      for (int m = 0; m < 4; m++) tw[3 + m] = lds128(tw5 + 16 * 8 * R * m);
    }
#pragma unroll
    for (u32 h = 0; h < 2; h++) {
      const u32 buf = buf0 + h * TILE_BYTES;
      if (!INV) {   // round 0: strides 32, 16, 8
#pragma unroll
        for (int e = 0; e < 8; e++) v[e] = lds64(buf + off0[e]);
        fwd_stages<3>(v, tw, p, p2);
#pragma unroll
        for (int e = 0; e < 8; e++) sts64(buf + off0[e], v[e]);
      } else {      // inverse starts with round 1: strides 1, 2, 4
#pragma unroll
        for (int k = 0; k < 4; k++) {
          const ulonglong2 t = lds128(buf + off1[k]);
          v[2 * k] = t.x;
          v[2 * k + 1] = t.y;
        }
        inv_stages<3>(v, tw, p, p2, false, A.limbs[0]);
#pragma unroll
        for (int k = 0; k < 4; k++) sts128(buf + off1[k], v[2 * k], v[2 * k + 1]);
      }
    }
    consumer_sync<NT>();
    if (!INV) {
      tw[0] = lds128(tw3);
      tw[1] = lds128(tw4);
      tw[2] = lds128(tw4 + 16 * 8 * R);
#pragma unroll
      for (int m = 0; m < 4; m++) tw[3 + m] = lds128(tw5 + 16 * 8 * R * m);
    } else {
      tw[0] = lds128(tw0);
      tw[1] = lds128(tw1);
      tw[2] = lds128(tw1 + 16);
#pragma unroll
      for (int m = 0; m < 4; m++) tw[3 + m] = lds128(tw2 + 16 * m);
    }
#pragma unroll
    for (u32 h = 0; h < 2; h++) {
      const u32 buf = buf0 + h * TILE_BYTES;
      if (!INV) {   // round 1: strides 4, 2, 1, then reduce3 unless lazy (native.rs:178-180, :238)
#pragma unroll
        for (int k = 0; k < 4; k++) {
          const ulonglong2 t = lds128(buf + off1[k]);
          v[2 * k] = t.x;
          v[2 * k + 1] = t.y;
        }
        fwd_stages<3>(v, tw, p, p2);
        if (!LAZY) {
#pragma unroll
          for (int e = 0; e < 8; e++) v[e] = fwd_final<false>(v[e], p, p2, 0);
        }
#pragma unroll
        for (int k = 0; k < 4; k++) sts128(buf + off1[k], v[2 * k], v[2 * k + 1]);
      } else {      // round 0: strides 8, 16, 32
#pragma unroll
        for (int e = 0; e < 8; e++) v[e] = lds64(buf + off0[e]);
        inv_stages<3>(v, tw, p, p2, false, A.limbs[0]);
#pragma unroll
        for (int e = 0; e < 8; e++) sts64(buf + off0[e], v[e]);
      }
    }
    fence_proxy_async();            // the tile is read next by the TMA store (async proxy)
    mbar_arrive(bar_done + 8 * s);
    fresh = w.next();
  }
}

// ------------------------------------------------------------------------------------------------ tensor + inverse rows
// The tensor product of two 2-part ciphertexts over the multiplication basis (c0 = a0*b0, c1 = a0*b1 + a1*b0,
// c2 = a1*b1; bfv/ops/mul.rs:198-201, Modulus::mul_vec zq/mod.rs:332) fused with the FIRST pass of the inverse
// transform that always follows it (mul.rs:204: the scaler takes power-basis input).  The product is point-wise and the
// inverse rows pass starts from the same 1024-word tile of every row, so one work item = (limb j, tile tau,
// ciphertext ct): four source tiles in (a0, a1, b0, b1 -- from the ciphertexts themselves for the common-prefix
// limbs, from the extended rows otherwise), three transformed tiles out.  The 3K product rows never travel to HBM
// and back between the two steps, and the stand-alone tensor kernel disappears from the path.
struct TensorRowsArgs {
  const LimbDev* limbs;
  u32 cts, L, K, logn;
  u32 tiles_per_row;
  u32 items_total;     // K * tiles_per_row * cts; item = (j*tiles_per_row + tau)*cts + ct
  unsigned short ids[kMaxPos];   // multiplication-basis position -> limb
};

template <int RLOG, int STAGES>
struct TensorRowsCfg {
  static constexpr u32 R = 1u << RLOG;
  static constexpr u32 NT = 8 * R;
  static constexpr u32 TILE_BYTES = 512 * R;
  static constexpr u32 STAGE_BYTES = 4 * TILE_BYTES;
  static constexpr u32 TW_PAIRS = 63 * R;
  static constexpr u32 SMEM = STAGES * STAGE_BYTES + TW_PAIRS * 16 + 2 * STAGES * 8 + 1024;
};

template <int RLOG, int STAGES, int MINB>
__global__ void __launch_bounds__(TensorRowsCfg<RLOG, STAGES>::NT + 32, MINB)
    ntt_tma_tensor_rows_kernel(const __grid_constant__ CUtensorMap tm_a, const __grid_constant__ CUtensorMap tm_b,
                               const __grid_constant__ CUtensorMap tm_xa, const __grid_constant__ CUtensorMap tm_xb,
                               const __grid_constant__ CUtensorMap tm_out, const TensorRowsArgs A) {
  using namespace tma;
  using Cfg = TensorRowsCfg<RLOG, STAGES>;
  constexpr u32 R = Cfg::R, NT = Cfg::NT, TILE_BYTES = Cfg::TILE_BYTES, STAGE_BYTES = Cfg::STAGE_BYTES;
  extern __shared__ unsigned char smem_raw[];
  const u32 base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const u32 tw_base = base + STAGES * STAGE_BYTES;
  const u32 bar_full = tw_base + Cfg::TW_PAIRS * 16;
  const u32 bar_done = bar_full + STAGES * 8;
  if (threadIdx.x == 0) {
#pragma unroll
    for (int s = 0; s < STAGES; s++) {
      mbar_init(bar_full + 8 * s, 1);
      mbar_init(bar_done + 8 * s, NT);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  const u32 lo = (u32)(((u64)A.items_total * blockIdx.x) / gridDim.x);
  const u32 hi = (u32)(((u64)A.items_total * (blockIdx.x + 1)) / gridDim.x);
  const u32 n = hi - lo;
  const u32 box_rows_per_row = (1u << A.logn) >> 4;
  const u32 E = A.K - A.L;

  if (threadIdx.x >= NT) {
    if (threadIdx.x != NT) return;
    prefetch_map(&tm_a);
    prefetch_map(&tm_b);
    prefetch_map(&tm_xa);
    prefetch_map(&tm_xb);
    prefetch_map(&tm_out);
    TileWalk wl, ws;
    wl.init(lo, A.cts);
    ws.init(lo, A.cts);
    u32 loaded = 0;
    auto load_next = [&]() {
      const u32 s = loaded % STAGES;
      const u32 j = wl.jt / A.tiles_per_row, tau = wl.jt - j * A.tiles_per_row;
      const u32 ct = wl.p;
      const bool pre = j < A.L;                       // common-prefix limb: the operands themselves
      const u32 rows = pre ? A.L : E, jj = pre ? j : j - A.L;
      const CUtensorMap* ma = pre ? &tm_a : &tm_xa;
      const CUtensorMap* mb = pre ? &tm_b : &tm_xb;
      const u32 r0 = ((ct * 2) * rows + jj) * box_rows_per_row + tau * (4 * R);
      const u32 r1 = ((ct * 2 + 1) * rows + jj) * box_rows_per_row + tau * (4 * R);
      const u32 dst = base + s * STAGE_BYTES, bar = bar_full + 8 * s;
      mbar_expect_tx(bar, STAGE_BYTES);
      load_2d(dst, ma, 0, r0, bar);
      load_2d(dst + TILE_BYTES, ma, 0, r1, bar);
      load_2d(dst + 2 * TILE_BYTES, mb, 0, r0, bar);
      load_2d(dst + 3 * TILE_BYTES, mb, 0, r1, bar);
      wl.next();
      loaded++;
    };
    while (loaded < n && loaded < (u32)STAGES) load_next();
    for (u32 i = 0; i < n; i++) {
      const u32 s = i % STAGES;
      mbar_wait(bar_done + 8 * s, (i / STAGES) & 1);
      const u32 j = ws.jt / A.tiles_per_row, tau = ws.jt - j * A.tiles_per_row;
      const u32 ct = ws.p;
      const u32 src = base + s * STAGE_BYTES;
      // transformed c0 sits in the a0 buffer, c1 in the b0 buffer, c2 in the a1 buffer
      store_2d(&tm_out, 0, ((ct * 3 + 0) * A.K + j) * box_rows_per_row + tau * (4 * R), src);
      store_2d(&tm_out, 0, ((ct * 3 + 1) * A.K + j) * box_rows_per_row + tau * (4 * R), src + 2 * TILE_BYTES);
      store_2d(&tm_out, 0, ((ct * 3 + 2) * A.K + j) * box_rows_per_row + tau * (4 * R), src + TILE_BYTES);
      bulk_commit();
      ws.next();
      if (loaded < n) {
        bulk_wait_read<0>();
        load_next();
      }
    }
    bulk_wait_all();
    return;
  }

  const u32 tid = threadIdx.x;
  const u32 x = tid & 7, b = tid >> 3;
  u32 off0[8];
#pragma unroll
  for (int e = 0; e < 8; e++) {
    const u32 i = 64 * b + x + 8 * e;
    off0[e] = ((i >> 4) << 7) | ((((i >> 1) & 7) ^ ((i >> 4) & 7)) << 4) | ((i & 1) << 3);
  }
  u32 off1[4];
#pragma unroll
  for (int k = 0; k < 4; k++) {
    const u32 i = 64 * b + 8 * x + 2 * k;
    off1[k] = ((i >> 4) << 7) | ((((i >> 1) & 7) ^ ((i >> 4) & 7)) << 4);
  }
  const u32 tw0 = tw_base + 16 * (b);
  const u32 tw1 = tw_base + 16 * (R * 1 + (b << 1));
  const u32 tw2 = tw_base + 16 * (R * 3 + (b << 2));
  const u32 tw3 = tw_base + 16 * (R * 7 + tid);
  const u32 tw4 = tw_base + 16 * (R * 15 + tid);
  const u32 tw5 = tw_base + 16 * (R * 31 + tid);

  TileWalk w;
  w.init(lo, A.cts);
  bool fresh = true;
  LimbDev M = A.limbs[0];
  const u32 logn1 = A.logn - 6;
  for (u32 i = 0; i < n; i++) {
    if (fresh) {
      const u32 j = w.jt / A.tiles_per_row, tau = w.jt - j * A.tiles_per_row;
      M = A.limbs[A.ids[j]];
      const ulonglong2* tab = M.zi;
      const u32 row0 = tau * R;
      if (i) consumer_sync<NT>();
#pragma unroll
      for (int tl = 0; tl < 6; tl++) {
        const u32 s = logn1 + tl;
        const u32 g0 = ((1u << A.logn) - (2u << s)) + (row0 << tl);
        for (u32 k = tid; k < (R << tl); k += NT) {
          const ulonglong2 v = __ldg(tab + g0 + k);
          const u32 dst = tl < 3 ? k : (k & ((1u << (tl >= 3 ? tl - 3 : 0)) - 1)) * (8 * R) + (k >> (tl >= 3 ? tl - 3 : 0));
          sts128(tw_base + 16 * (R * ((1u << tl) - 1) + dst), v.x, v.y);
        }
      }
      consumer_sync<NT>();
    }
    const u64 p = M.p, p2 = M.p2;
    const u32 s = i % STAGES;
    const u32 buf = base + s * STAGE_BYTES;
    mbar_wait(bar_full + 8 * s, (i / STAGES) & 1);
    // Phase 1: point-wise products of this thread's 8 consecutive positions, two per trip, deposited over the
    // consumed operands (c0 -> a0 buffer, c1 -> b0 buffer, c2 -> a1 buffer; only this thread touches those words).
    // The loops over trips and tiles are rolled on purpose: fully unrolled the kernel was ~64 KB of code and lost
    // a large share of its issue slots to instruction fetch.
#pragma unroll 1
    for (u32 k = 0; k < 4; k++) {
      const u32 i = 64 * b + 8 * x + 2 * k;
      const u32 o = buf + (((i >> 4) << 7) | ((((i >> 1) & 7) ^ ((i >> 4) & 7)) << 4));
      const ulonglong2 a0 = lds128(o), a1 = lds128(o + TILE_BYTES);
      const ulonglong2 b0 = lds128(o + 2 * TILE_BYTES), b1 = lds128(o + 3 * TILE_BYTES);
      // (residues in [0,2p): the inverse butterflies that consume them take lazy operands, native.rs:303-316)
      const u64 c0x = mulmod_limb_lazy(a0.x, b0.x, M), c0y = mulmod_limb_lazy(a0.y, b0.y, M);
      const u64 c2x = mulmod_limb_lazy(a1.x, b1.x, M), c2y = mulmod_limb_lazy(a1.y, b1.y, M);
      Acc192 sx, sy;                               // a0*b1 + a1*b0 < 2^125, one reduction
      sx.clear();
      sy.clear();
      sx.mac(a0.x, b1.x);
      sx.mac(a1.x, b0.x);
      sy.mac(a0.y, b1.y);
      sy.mac(a1.y, b0.y);
      const u64 c1x = sx.reduce_lazy(M), c1y = sy.reduce_lazy(M);
      sts128(o, c0x, c0y);
      sts128(o + 2 * TILE_BYTES, c1x, c1y);
      sts128(o + TILE_BYTES, c2x, c2y);
    }
    // Phase 2: inverse round 1 (strides 1, 2, 4) of the three product tiles: the same 8 positions, same thread
    u64 v[8];
    ulonglong2 tw[7];
    tw[0] = lds128(tw3);
    tw[1] = lds128(tw4);
    tw[2] = lds128(tw4 + 16 * 8 * R);
#pragma unroll
    for (int m = 0; m < 4; m++) tw[3 + m] = lds128(tw5 + 16 * 8 * R * m);
#pragma unroll 1
    for (u32 t = 0; t < 3; t++) {
      const u32 tb = buf + t * TILE_BYTES;
#pragma unroll
      for (int k = 0; k < 4; k++) {
        const ulonglong2 q = lds128(tb + off1[k]);
        v[2 * k] = q.x;
        v[2 * k + 1] = q.y;
      }
      inv_stages<3>(v, tw, p, p2, false, M);
#pragma unroll
      for (int k = 0; k < 4; k++) sts128(tb + off1[k], v[2 * k], v[2 * k + 1]);
    }
    consumer_sync<NT>();
    // Phase 3: inverse round 0 (strides 8, 16, 32) of each product tile
    tw[0] = lds128(tw0);
    tw[1] = lds128(tw1);
    tw[2] = lds128(tw1 + 16);
#pragma unroll
    for (int m = 0; m < 4; m++) tw[3 + m] = lds128(tw2 + 16 * m);
#pragma unroll 1
    for (u32 t = 0; t < 3; t++) {
      const u32 tb = buf + t * TILE_BYTES;
#pragma unroll
      for (int e = 0; e < 8; e++) v[e] = lds64(tb + off0[e]);
      inv_stages<3>(v, tw, p, p2, false, M);
#pragma unroll
      for (int e = 0; e < 8; e++) sts64(tb + off0[e], v[e]);
    }
    fence_proxy_async();
    mbar_arrive(bar_done + 8 * s);
    fresh = w.next();
  }
}

// ------------------------------------------------------------------------------------------------ key-switch rows + inner product
// The last pass of the digit transforms of a key switch fused with the inner product that consumes them
// (key_switching_key.rs:256-268: out{0,1} = base{0,1} + sum_d NTT_j(digit_d) * k{0,1}[j][d]).  Every digit of one
// (ciphertext, limb j) is transformed modulo the same q_j, so all of them share the rows-pass twiddles of (j, tau) and
// the key tiles of (j, tau); the cols pass has left them in adjacent rows (digit-adjacent layout, [ct][j][d][N]).
//   work item = (limb j, 128-coefficient tile tau, ciphertext ct), ct innermost: twiddles are staged once per (j, tau)
//   and the two key tiles of (j, tau) (2 n_dig row segments of 1 KiB, from the key pair the ciphertext's slot names)
//   once per run of ciphertexts with the same (j, tau) and the same key (Keys = OneKey: the {128, n_dig} boxes of the
//   key's tensor maps; Keys = KeyTable: the pair the ciphertext's slot names); the n_dig digit tiles of each item arrive
//   through a ring of STAGES buffers.  Per item: the six small-stride forward stages on each digit tile (16 threads per
//   tile, 16 tiles side by side, lazy outputs in [0,4q_j) as the unfused pass leaves them), a CTA barrier, then one
//   thread per (output, coefficient) accumulates sum_d digit_d * key_d with Acc192, adds the base and reduces once.
// The transformed digits never travel to HBM and back: the unfused chain wrote and re-read all of them.
struct KsRowsArgs {
  const LimbDev* limbs;
  const u64 *base0, *base1;   // nullable, indexed like out0 / out1
  u64 *out0, *out1;           // row (ct, j) at (ct*out_ct_rows + j)*N
  u32 cts, n_dig, Lk, out_ct_rows, logn;
  u32 tiles_per_row;
  u32 items_total;            // Lk * tiles_per_row * cts; item = (j*tiles_per_row + tau)*cts + ct
  unsigned short ids[kMaxPos];
};

template <int STAGES>
struct KsRowsCfg {
  static constexpr u32 R = 2;                 // matrix rows of 64 points per tile: 128 coefficients
  static constexpr u32 TC = 64 * R;
  static constexpr u32 TILE_BYTES = 512 * R;  // one digit tile, 1024-byte aligned for the 128-byte swizzle
  static constexpr u32 GROUPS = 16;           // digit tiles transformed side by side (8R = 16 threads each)
  static constexpr u32 NT = GROUPS * 8 * R;   // 256 consumers = one per (output, coefficient) of the inner product
  static constexpr u32 TW_PAIRS = 63 * R;
  static constexpr size_t smem(u32 nd) {
    return (size_t)STAGES * nd * TILE_BYTES + 2 * (size_t)nd * TC * 8 + TW_PAIRS * 16 + 2 * STAGES * 8 + 8 + 1024;
  }
};

// the keys of a launch with one key: its tensor maps (tm_k0, tm_k1), every ciphertext in slot 0
struct OneKey {};
__device__ __forceinline__ u32 key_slot(const OneKey&, u32) { return 0; }

template <int STAGES, int MINB, class Keys>
__global__ void __launch_bounds__(KsRowsCfg<STAGES>::NT + 32, MINB)
    ks_rows_mac_tma_kernel(const __grid_constant__ CUtensorMap tm_in, const __grid_constant__ CUtensorMap tm_k0,
                           const __grid_constant__ CUtensorMap tm_k1, const KsRowsArgs A,
                           const __grid_constant__ Keys K) {
  using namespace tma;
  using Cfg = KsRowsCfg<STAGES>;
  constexpr u32 R = Cfg::R, TC = Cfg::TC, NT = Cfg::NT, TILE_BYTES = Cfg::TILE_BYTES, GROUPS = Cfg::GROUPS;
  extern __shared__ unsigned char smem_raw[];
  const u32 nd = A.n_dig;
  const u32 base = (smem_u32(smem_raw) + 1023u) & ~1023u;   // the 128-byte swizzle works on absolute address bits
  const u32 stage_bytes = nd * TILE_BYTES;
  const u32 k0_base = base + STAGES * stage_bytes;         // [n_dig][TC] u64, no swizzle
  const u32 k1_base = k0_base + nd * TC * 8;
  const u32 tw_base = k1_base + nd * TC * 8;
  const u32 bar_full = tw_base + Cfg::TW_PAIRS * 16;
  const u32 bar_done = bar_full + STAGES * 8;
  const u32 bar_key = bar_done + STAGES * 8;

  if (threadIdx.x == 0) {
#pragma unroll
    for (int s = 0; s < STAGES; s++) {
      mbar_init(bar_full + 8 * s, 1);
      mbar_init(bar_done + 8 * s, NT);
    }
    mbar_init(bar_key, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  const u32 lo = (u32)(((u64)A.items_total * blockIdx.x) / gridDim.x);
  const u32 hi = (u32)(((u64)A.items_total * (blockIdx.x + 1)) / gridDim.x);
  const u32 n = hi - lo;
  const u32 box_rows_per_row = (1u << A.logn) >> 4;   // 128-byte box rows per polynomial row

  if (threadIdx.x >= NT) {
    // ---------------- producer: the digit tiles of every item of this CTA, STAGES items ahead of the consumers
    if (threadIdx.x != NT) return;
    prefetch_map(&tm_in);
    TileWalk wl;
    wl.init(lo, A.cts);
    for (u32 i = 0; i < n; i++) {
      const u32 s = i % STAGES;
      if (i >= (u32)STAGES) mbar_wait(bar_done + 8 * s, (i / STAGES - 1) & 1);   // item i - STAGES consumed
      const u32 j = wl.jt / A.tiles_per_row, tau = wl.jt - j * A.tiles_per_row;
      const u32 row0 = (wl.p * A.Lk + j) * nd;
      mbar_expect_tx(bar_full + 8 * s, stage_bytes);
      for (u32 d = 0; d < nd; d++)
        load_2d(base + s * stage_bytes + d * TILE_BYTES, &tm_in, 0, (row0 + d) * box_rows_per_row + tau * (4 * R),
                bar_full + 8 * s);
      wl.next();
    }
    return;
  }

  // ---------------- consumers
  const u32 tid = threadIdx.x;
  const u32 g = tid >> 4, lt = tid & 15;            // transform: digit group, thread inside the digit tile
  const u32 hmask = 0xffffu << (tid & 16);          // the half warp that owns one digit tile
  const u32 x = lt & 7, b = lt >> 3;
  // Offsets inside a (1024-byte aligned) digit tile with the TMA 128-byte swizzle, as in the rows pass.  With two
  // matrix rows per tile the offset of word e differs from that of word 0 by a compile-time XOR mask, so only word 0's
  // offset is kept in a register: round 0 reads words 64b + x + 8e, round 1 the pairs (64b + 8x + 2k, +1).
  const u32 off0 = ((4 * b) << 7) | ((((x >> 1) & 7) ^ (4 * b)) << 4) | ((x & 1) << 3);
  const u32 off1 = ((4 * b + (x >> 1)) << 7) | (((4 * (x & 1)) ^ (4 * b + (x >> 1))) << 4);
  auto x0 = [](int e) -> u32 { return ((u32)(e >> 1) << 7) | ((u32)((e >> 1) ^ (4 * (e & 1))) << 4); };
  const u32 tw0 = tw_base + 16 * (b);
  const u32 tw1 = tw_base + 16 * (R * 1 + (b << 1));
  const u32 tw2 = tw_base + 16 * (R * 3 + (b << 2));
  const u32 tw3 = tw_base + 16 * (R * 7 + lt);
  const u32 tw4 = tw_base + 16 * (R * 15 + lt);
  const u32 tw5 = tw_base + 16 * (R * 31 + lt);
  // inner product: coefficient c of output o
  const u32 c = tid & (TC - 1), o = tid / TC;
  const u32 offc = ((c >> 4) << 7) | ((((c >> 1) & 7) ^ ((c >> 4) & 7)) << 4) | ((c & 1) << 3);
  const u32 key_c = (o ? k1_base : k0_base) + 8 * c;
  const u64* bsrc = o ? A.base1 : A.base0;
  u64* dst = o ? A.out1 : A.out0;

  TileWalk w;
  w.init(lo, A.cts);
  bool fresh = true;
  u32 key_phase = 0, cur_slot = 0;
  const LimbDev* Mp = A.limbs;
  u64 p = 0, p2 = 0;
  const u32 logn1 = A.logn - 6;
  for (u32 i = 0; i < n; i++) {
    const u32 j = w.jt / A.tiles_per_row, tau = w.jt - j * A.tiles_per_row;
    const u32 slot = key_slot(K, w.p);
    const bool new_keys = fresh || slot != cur_slot;
    if (new_keys) {
      // new (limb, tile position) or new key: the key tiles replace the previous ones
      cur_slot = slot;
      if (i) consumer_sync<NT>();   // nobody still reads the previous twiddles or key tiles
      if (tid == 0) {
        if constexpr (std::is_same<Keys, OneKey>::value) {
          mbar_expect_tx(bar_key, 2 * nd * TC * 8);
          load_2d(k0_base, &tm_k0, tau * TC, j * nd, bar_key);
          load_2d(k1_base, &tm_k1, tau * TC, j * nd, bar_key);
        } else {
          load_key_tiles<TC>(k0_base, k1_base, K.k0[slot], K.k1[slot], j, tau, nd, A.logn, bar_key);
        }
      }
    }
    if (fresh) {
      // new (limb, tile position): its 63R twiddle pairs replace the previous ones
      Mp = A.limbs + A.ids[j];
      p = Mp->p;
      p2 = Mp->p2;
      const u32 row0 = tau * R;
#pragma unroll
      for (int tl = 0; tl < 6; tl++) {
        const u32 s = logn1 + tl;
        const u32 g0 = (1u << s) + (row0 << tl);
        if (tid < (R << tl)) {
          const ulonglong2 v = __ldg(Mp->om + g0 + tid);
          const u32 k = tid;
          const u32 dst_pair = tl < 3 ? k : (k & ((1u << (tl >= 3 ? tl - 3 : 0)) - 1)) * (8 * R) + (k >> (tl >= 3 ? tl - 3 : 0));
          sts128(tw_base + 16 * (R * ((1u << tl) - 1) + dst_pair), v.x, v.y);
        }
      }
      consumer_sync<NT>();
    }
    const size_t oi = (((size_t)w.p * A.out_ct_rows + j) << A.logn) + tau * TC + c;
    const u64 bv = bsrc ? bsrc[oi] : 0;   // in flight while the digits are transformed
    const u32 s = i % STAGES;
    const u32 ring = base + s * stage_bytes;
    mbar_wait(bar_full + 8 * s, (i / STAGES) & 1);
    // the six small-stride forward stages of every digit tile, outputs lazy in [0, 4q_j) (forward_vt_lazy)
    // (each stage's twiddles are read from shared memory just before it: holding all seven pairs of a round spilled
    // at the 72 registers that three 288-thread CTAs per SM leave)
    for (u32 d = g; d < nd; d += GROUPS) {
      const u32 a0 = ring + d * TILE_BYTES + off0, a1 = ring + d * TILE_BYTES + off1;
      u64 v[8];
#pragma unroll
      for (int e = 0; e < 8; e++) v[e] = lds64(a0 ^ x0(e));
      fwd_stages3_staged(v, p, p2, [&](int u, int m) {
        return lds128(u == 0 ? tw0 : u == 1 ? tw1 + 16 * m : tw2 + 16 * m);
      });
#pragma unroll
      for (int e = 0; e < 8; e++) sts64(a0 ^ x0(e), v[e]);
      __syncwarp(hmask);
#pragma unroll
      for (int k = 0; k < 4; k++) {
        const ulonglong2 t = lds128(a1 ^ (k << 4));
        v[2 * k] = t.x;
        v[2 * k + 1] = t.y;
      }
      fwd_stages3_staged(v, p, p2, [&](int u, int m) {
        return lds128(u == 0 ? tw3 : u == 1 ? tw4 + 16 * 8 * R * m : tw5 + 16 * 8 * R * m);
      });
#pragma unroll
      for (int k = 0; k < 4; k++) sts128(a1 ^ (k << 4), v[2 * k], v[2 * k + 1]);
    }
    if (new_keys) {
      mbar_wait(bar_key, key_phase);
      key_phase ^= 1;
    }
    consumer_sync<NT>();   // every digit tile of the item is transformed
    Acc192 acc;
    acc.clear();
#pragma unroll 2
    for (u32 d = 0; d < nd; d++) acc.mac(lds64(ring + d * TILE_BYTES + offc), lds64(key_c + d * TC * 8));
    acc.add64(bv);
    dst[oi] = acc.reduce(*Mp);
    mbar_arrive(bar_done + 8 * s);   // the ring stage may take the item STAGES ahead
    fresh = w.next();
  }
}

// ------------------------------------------------------------------------------------------------ cols pass
// The log2(N1) large-stride stages on tiles of all N1 = 2^LOGP points x 16 adjacent columns (128-byte segments at
// stride 512 bytes).  2^LOGP consumer threads + one producer warp; radix-8 rounds in place, 16 / 8 words per thread
// per round.  Tensor map: the buffer as [rows][N1][64] u64, box {16, min(N1, 256), 1}, no swizzle.
template <int LOGP, int STAGES>
struct ColsCfg {
  static constexpr u32 P = 1u << LOGP;
  static constexpr u32 NT = P;                      // consumer threads
  static constexpr u32 TILE_BYTES = P * 128;
  static constexpr u32 BOX_ROWS = P < 256 ? P : 256;
  static constexpr u32 BOXES = P / BOX_ROWS;
  static constexpr u32 SMEM = STAGES * TILE_BYTES + P * 16 + 2 * STAGES * 8 + 1024;
  static constexpr int NR = (LOGP + 2) / 3;
  static constexpr int REM = LOGP - 3 * (NR - 1);
};

// one radix-2^NS round (stages t .. t+NS-1 of the in-tile transform) over the whole tile, in place
// The radix groups of a thread differ by compile-time address / twiddle offsets.  ROLL keeps the loop over them rolled
// (half the code); measured slower than the unrolled form, which stays the default.
template <int LOGP, bool INV, int NS, int T, bool REDUCE, bool ROLL = false>
__device__ __forceinline__ void cols_round(u32 buf, u32 tw_base, u64 p, u64 p2, const tma::LastStage& L, u64 bhi, u64 blo) {
  using namespace tma;
  constexpr int t = T;
  constexpr u32 NT = 1u << LOGP;
  constexpr int R = 1 << NS;
  constexpr u32 UNITS = (1u << (LOGP + 4 - NS)) / NT;   // radix groups per thread: 2 (NS=3), 4, 8
  constexpr int logstride = LOGP - t - NS;
  constexpr u32 stride_bytes = 128u << logstride;
  // group q+1 of a thread is group q shifted by NT/16 positions of `rest`
  constexpr bool HI = (LOGP - 4) >= logstride;                                   // the shift lands in a_hi
  constexpr u32 D_AHI = HI ? (1u << (LOGP - 4 - logstride)) : 0;
  constexpr u32 D_ADDR = (HI ? (D_AHI << (LOGP - t)) : (1u << (LOGP - 4))) * 128;
  const u32 bcol = threadIdx.x & 15, rest = threadIdx.x >> 4;
  const u32 a_lo = rest & ((1u << logstride) - 1);
  u32 a_hi = rest >> logstride;
  u32 addr = buf + ((a_hi << (LOGP - t)) + a_lo) * 128 + bcol * 8;
#pragma unroll(ROLL ? 1 : 8)
  for (u32 q = 0; q < UNITS; q++) {
    u64 v[R];
#pragma unroll
    for (int e = 0; e < R; e++) {
      v[e] = lds64(addr + e * stride_bytes);
      if (REDUCE) v[e] = barrett64(v[e], p, bhi, blo);
    }
    ulonglong2 tw[R - 1];
#pragma unroll
    for (int u = 0; u < NS; u++) {
      const int tl = t + u;
      if (INV && tl == 0) continue;   // the fused last stage has no table entry
      // forward: omegas[(1<<tl) + (a_hi<<u) + m]; inverse: zetas_inv[N - (2<<tl) + (a_hi<<u) + m], staged at
      // table index  P - (2<<tl) + ...
      const u32 idx = (INV ? ((1u << LOGP) - (2u << tl)) : (1u << tl)) + (a_hi << u);
#pragma unroll
      for (int m = 0; m < (1 << u); m++) tw[(1 << u) - 1 + m] = lds128(tw_base + 16 * (idx + m));
    }
    if (!INV) fwd_stages<NS>(v, tw, p, p2);
    else inv_stages<NS>(v, tw, p, p2, t == 0, L);
#pragma unroll
    for (int e = 0; e < R; e++) sts64(addr + e * stride_bytes, v[e]);
    addr += D_ADDR;
    a_hi += D_AHI;
  }
}

// tile index -> (limb j, tile position tau, polynomial p).  Limb-major by default: consecutive tiles of a CTA share
// the limb's twiddles.  A.limb_inner (set with in_bcast) puts the limb innermost, for the digit broadcast: there the Lk tiles
// (tau, p, j = 0 .. Lk-1) read the SAME source tile, so back to back only the first read reaches DRAM and the rest
// hit L2 (limb-major, one limb's pass over a chunk's c2 is far larger than L2 and every limb refetches it), for the
// price of restaging the 2^LOGP twiddle pairs per tile.
__device__ __forceinline__ void cols_tile(const NttTmaArgs& A, u32 idx, u32& j, u32& tau, u32& p) {
  if (A.limb_inner) {
    const u32 r = idx / A.lpp;
    j = idx - r * A.lpp;
    tau = r / A.n_polys;
    p = r - tau * A.n_polys;
  } else {
    const u32 jt = idx / A.n_polys;
    p = idx - jt * A.n_polys;
    j = jt / A.tiles_per_row;
    tau = jt - j * A.tiles_per_row;
  }
}

template <int LOGP, bool INV, int STAGES, int MINB, bool REDUCE, bool ROLL = false>
__global__ void __launch_bounds__(ColsCfg<LOGP, STAGES>::NT + 32, MINB)
    ntt_tma_cols_kernel(const __grid_constant__ CUtensorMap tm_in, const __grid_constant__ CUtensorMap tm_out,
                        const NttTmaArgs A) {
  using namespace tma;
  using Cfg = ColsCfg<LOGP, STAGES>;
  constexpr u32 NT = Cfg::NT, TILE_BYTES = Cfg::TILE_BYTES, P = Cfg::P;
  constexpr int NR = Cfg::NR, REM = Cfg::REM;
  extern __shared__ unsigned char smem_raw[];
  const u32 base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const u32 tw_base = base + STAGES * TILE_BYTES;
  const u32 bar_full = tw_base + P * 16;
  const u32 bar_done = bar_full + STAGES * 8;

  if (threadIdx.x == 0) {
#pragma unroll
    for (int s = 0; s < STAGES; s++) {
      mbar_init(bar_full + 8 * s, 1);
      mbar_init(bar_done + 8 * s, NT);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  const u32 lo = (u32)(((u64)A.tiles_total * blockIdx.x) / gridDim.x);
  const u32 hi = (u32)(((u64)A.tiles_total * (blockIdx.x + 1)) / gridDim.x);
  const u32 n = hi - lo;

  if (threadIdx.x >= NT) {
    if (threadIdx.x != NT) return;
    prefetch_map(&tm_in);
    prefetch_map(&tm_out);
    u32 loaded = 0;
    auto load_next = [&]() {
      const u32 s = loaded % STAGES;
      u32 j, tau, pp;
      cols_tile(A, lo + loaded, j, tau, pp);
      const u32 row = A.in_bcast ? pp : out_row_of(A, pp, j);
      mbar_expect_tx(bar_full + 8 * s, TILE_BYTES);
#pragma unroll
      for (u32 h = 0; h < Cfg::BOXES; h++)
        load_3d(base + s * TILE_BYTES + h * Cfg::BOX_ROWS * 128, &tm_in, tau * 16, h * Cfg::BOX_ROWS, row,
                bar_full + 8 * s);
      loaded++;
    };
    while (loaded < n && loaded < (u32)STAGES) load_next();
    for (u32 i = 0; i < n; i++) {
      const u32 s = i % STAGES;
      mbar_wait(bar_done + 8 * s, (i / STAGES) & 1);
      u32 j, tau, pp;
      cols_tile(A, lo + i, j, tau, pp);
      const u32 row = out_row_of(A, pp, j);
#pragma unroll
      for (u32 h = 0; h < Cfg::BOXES; h++)
        store_3d(&tm_out, tau * 16, h * Cfg::BOX_ROWS, row, base + s * TILE_BYTES + h * Cfg::BOX_ROWS * 128);
      bulk_commit();
      if (loaded < n) {
        bulk_wait_read<0>();
        load_next();
      }
    }
    bulk_wait_all();
    return;
  }

  const u32 tid = threadIdx.x;
  u32 cur_j = 0xffffffffu;
  const LimbDev* Lp = A.limbs;
  u64 p = 0, p2 = 0, bhi = 0, blo = 0;
  LastStage ls = {0, 0, 0, 0};
  for (u32 i = 0; i < n; i++) {
    u32 j, tau_unused, p_unused;
    cols_tile(A, lo + i, j, tau_unused, p_unused);
    if (j != cur_j) {
      // new limb: stage the 2^LOGP - 1 twiddle pairs of the large-stride stages (the same for every tile of the limb)
      Lp = A.limbs + A.ids[j];
      p = Lp->p;
      p2 = Lp->p2;
      if (INV) ls = LastStage{Lp->ninv, Lp->ninv_s, Lp->zn, Lp->zn_s};   // loop-invariant per limb: out of the hot loop
      if (REDUCE) {
        bhi = Lp->bhi;
        blo = Lp->blo;
      }
      const ulonglong2* tab = INV ? Lp->zi + ((1u << A.logn) - P) : Lp->om;
      if (cur_j != 0xffffffffu) consumer_sync<NT>();
      for (u32 k = tid; k < P; k += NT) {
        const ulonglong2 v = __ldg(tab + k);
        sts128(tw_base + 16 * k, v.x, v.y);
      }
      consumer_sync<NT>();
      cur_j = j;
    }
    const u32 s = i % STAGES;
    const u32 buf = base + s * TILE_BYTES;
    mbar_wait(bar_full + 8 * s, (i / STAGES) & 1);
    if (!INV) {
#pragma unroll
      for (int r = 0; r < NR; r++) {
        if (r == 0) cols_round<LOGP, false, 3, 0, REDUCE, ROLL>(buf, tw_base, p, p2, ls, bhi, blo);
        else if (r == 1 && NR > 2) cols_round<LOGP, false, 3, 3, false, ROLL>(buf, tw_base, p, p2, ls, bhi, blo);
        else cols_round<LOGP, false, REM, 3 * (NR - 1), false, ROLL>(buf, tw_base, p, p2, ls, bhi, blo);
        if (r < NR - 1) consumer_sync<NT>();
      }
    } else {
#pragma unroll
      for (int r = NR - 1; r >= 0; r--) {
        if (r == 0) cols_round<LOGP, true, 3, 0, false, ROLL>(buf, tw_base, p, p2, ls, bhi, blo);
        else if (r == 1 && NR > 2) cols_round<LOGP, true, 3, 3, false, ROLL>(buf, tw_base, p, p2, ls, bhi, blo);
        else cols_round<LOGP, true, REM, 3 * (NR - 1), false, ROLL>(buf, tw_base, p, p2, ls, bhi, blo);
        if (r > 0) consumer_sync<NT>();
      }
    }
    fence_proxy_async();
    mbar_arrive(bar_done + 8 * s);
  }
}

}  // namespace fhe_b200
