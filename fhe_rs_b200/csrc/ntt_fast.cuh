// Register-resident variant of the two tile kernels of ntt.cuh for N >= 2^13 (2^TLOG-word tiles,
// 2^(TLOG-3) threads, 8 words per thread; TLOG = 10 for the rows pass, 11 for the cols pass (12 at N = 2^16), see ntt.cu).  Same transform, same tables, same outputs; what changes is
// the data movement, tuned to the issue limits (the ALU pipe -- address arithmetic, selects, carries --
// not HBM, bounds the NTT):
//   * the first round reads its 8 words straight from global memory into registers and the last
//     round writes them straight back (one shared-memory round trip less per pass);
//   * every shared-memory access is `base + compile-time offset` (the i + i/32 padding is affine
//     over the disjoint bit fields of a radix group), every twiddle fetch is a run of 1/2/4
//     consecutive 16-byte (value, companion) pairs;
//   * two tile buffers, so one __syncthreads per exchange.
#pragma once
#include "ntt.cuh"

namespace fhe_b200 {

// offset of element `je` (stride S words) of a radix group relative to the padded base
__host__ __device__ constexpr u32 pad_delta(u32 je, u32 S) { return je * S + ((je * S) >> 5); }

// LOGP: log2 points of the in-tile transform; TLOG: log2 words per tile (8 words per thread, 2^(TLOG-3) threads);
// LOGB = TLOG - LOGP batch lanes; COLS layout as in ntt.cuh.
template <int LOGP, bool COLS, bool INV, int TLOG>
struct FastTile {
  static constexpr int LOGB = TLOG - LOGP;
  static constexpr u32 NT = 1u << (TLOG - 3);
  static constexpr u32 P = 1u << LOGP, B = 1u << LOGB;
  static constexpr int NR = (LOGP + 2) / 3;
  static constexpr int REM = LOGP - 3 * (NR - 1);
  static constexpr u32 TW = (1u << TLOG) + (1u << (TLOG - 3)) + 64;  // padded words per tile buffer (4672 for 4096)
  // Shared-memory padding.  cols layout: i + i/32.  rows layout with 64-point rows: i + 8*(i/64) + (i/8)%8, which makes
  // both exchange patterns of the pass (8 lanes x 4 rows at stride 8, and 8-word runs) hit 16 distinct bank pairs
  // (the i + i/32 padding left the stride-8 pattern 4-way conflicted: millions of conflicts per launch).
  static constexpr bool ROWS6 = !COLS && LOGP == 6;
  static __device__ __forceinline__ u32 phys(u32 i) {
    return ROWS6 ? i + ((i >> 6) << 3) + ((i >> 3) & 7) : i + (i >> 5);
  }
  // offset of element e (stride S words) of a radix group relative to phys(group base); the group's bit field is
  // zero in the base index, so the padding terms add without carries
  static __host__ __device__ constexpr u32 delta(u32 e, u32 S) {
    return ROWS6 ? (S == 8 ? 9 * e : e) : e * S + ((e * S) >> 5);
  }

  // geometry of round r for this thread: NS stages starting at local stage t = 3r
  template <int NS>
  struct Geo {
    u32 b[8 >> NS], a_hi[8 >> NS], a0[8 >> NS];
  };

  template <int NS>
  static __device__ __forceinline__ void decode(int t, Geo<NS>& g) {
    const int logstride = LOGP - t - NS;
#pragma unroll
    for (int q = 0; q < (8 >> NS); q++) {
      const u32 gid = threadIdx.x + q * NT;
      u32 b, a_lo, a_hi;
      if (COLS) {
        b = gid & (B - 1);
        const u32 rest = gid >> LOGB;
        a_lo = rest & ((1u << logstride) - 1);
        a_hi = rest >> logstride;
      } else {
        a_lo = gid & ((1u << logstride) - 1);
        const u32 rest = gid >> logstride;
        a_hi = rest & ((1u << t) - 1);
        b = rest >> t;
      }
      g.b[q] = b;
      g.a_hi[q] = a_hi;
      g.a0[q] = (a_hi << (LOGP - t)) + a_lo;
    }
  }

  // butterflies of one round on the thread's 8 registers
  template <int NS>
  static __device__ __forceinline__ void compute(u64 (&x)[8], const Geo<NS>& g, const LimbDev& L, int t, int s_base,
                                                 u32 logn, u32 row0, bool first_pass) {
    constexpr int R = 1 << NS;
    const u64 p = L.p, p2 = L.p2;
#pragma unroll
    for (int q = 0; q < (8 >> NS); q++) {
      const u32 root0 = COLS ? 0u : (row0 + g.b[q]);
      u64* v = &x[q * R];
      if (!INV) {
        // all twiddle pairs of the round are requested before the first butterfly: in the rows pass they come from
        // L2 (each tile has its own 63 KB of them) and ptxas otherwise leaves half of the loads in mid-round
        ulonglong2 tw[R - 1];
#pragma unroll
        for (int u = 0; u < NS; u++) {
          const int tl = t + u, s = s_base + tl;
          const ulonglong2* tp = L.om + ((1u << s) + (root0 << tl) + (g.a_hi[q] << u));
#pragma unroll
          for (int m = 0; m < (1 << u); m++) tw[(1 << u) - 1 + m] = __ldg(tp + m);
        }
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
        if (s_base + t + NS == (int)logn) {
#pragma unroll
          for (int j = 0; j < R; j++) v[j] = fwd_final<false>(v[j], p, p2, 0);
        }
      } else {
        // twiddles of the round up front as in the forward branch
        constexpr bool PF = true;
        ulonglong2 tz[PF ? R - 1 : 1];
        if (PF) {
#pragma unroll
          for (int u = 0; u < NS; u++) {
            const int tl = t + u, s = s_base + tl;
            if (!(s == 0 && first_pass)) {
              const ulonglong2* tp = L.zi + ((1u << logn) - (2u << s) + (root0 << tl) + (g.a_hi[q] << u));
#pragma unroll
              for (int m = 0; m < (1 << u); m++) tz[(1 << u) - 1 + m] = __ldg(tp + m);
            }
          }
        }
#pragma unroll
        for (int u = NS - 1; u >= 0; u--) {
          const int half = R >> (u + 1), tl = t + u, s = s_base + tl;
          if (s == 0 && first_pass) {
#pragma unroll
            for (int e = 0; e < half; e++) {
              u64 a = v[e], b2 = v[e + half];
              v[e] = csub(mul_const_lazy<false>(a + b2, L.ninv, L.ninv_s, p, 0), p);
              v[e + half] = csub(mul_const_lazy<false>(p2 + a - b2, L.zn, L.zn_s, p, 0), p);
            }
          } else {
            const ulonglong2* tp = L.zi + ((1u << logn) - (2u << s) + (root0 << tl) + (g.a_hi[q] << u));
#pragma unroll
            for (int m = 0; m < (1 << u); m++) {
              const ulonglong2 z = PF ? tz[(1 << u) - 1 + m] : __ldg(tp + m);
#pragma unroll
              for (int e = 0; e < half; e++) {
                const int jj = m * 2 * half + e;
                bf_inv<false>(v[jj], v[jj + half], z.x, z.y, p, p2, 0);
              }
            }
          }
        }
      }
    }
  }

  template <int NS>
  static __device__ __forceinline__ u32 tile_index(const Geo<NS>& g, int q) {
    return COLS ? (g.a0[q] << LOGB) + g.b[q] : (g.b[q] << LOGP) + g.a0[q];
  }

  // One round: fetch (global or shared), compute, deposit (global or shared).
  template <int NS>
  static __device__ __forceinline__ void round(u64 (&x)[8], int r, const u64* __restrict__ src, u64* __restrict__ dst,
                                               u32 gstride_a, u64* sm_in, u64* sm_out, bool from_global,
                                               bool to_global, bool reduce_on_load, const LimbDev& L, int s_base,
                                               u32 logn, u32 row0, bool first_pass) {
    constexpr int R = 1 << NS;
    const int t = 3 * r;
    const int logstride = LOGP - t - NS;
    const u32 S = (1u << logstride) * (COLS ? B : 1u);  // word stride between group elements inside the tile
    Geo<NS> g;
    decode<NS>(t, g);
#pragma unroll
    for (int q = 0; q < (8 >> NS); q++) {
      if (from_global) {
        // cols: word (a, b) of the tile lives at a*gstride_a + b ; rows: the tile is one contiguous chunk
        const u64* ptr = COLS ? src + (size_t)g.a0[q] * gstride_a + g.b[q] : src + tile_index<NS>(g, q);
        const size_t gs = COLS ? ((size_t)gstride_a << logstride) : ((size_t)1 << logstride);
#pragma unroll
        for (int e = 0; e < R; e++) {
          u64 v = ptr[e * gs];
          if (reduce_on_load) v = barrett64(v, L.p, L.bhi, L.blo);
          x[q * R + e] = v;
        }
      } else {
        const u64* ptr = sm_in + phys(tile_index<NS>(g, q));
#pragma unroll
        for (int e = 0; e < R; e++) x[q * R + e] = ptr[delta(e, S)];
      }
    }
    compute<NS>(x, g, L, t, s_base, logn, row0, first_pass);
#pragma unroll
    for (int q = 0; q < (8 >> NS); q++) {
      if (to_global) {
        u64* ptr = COLS ? dst + (size_t)g.a0[q] * gstride_a + g.b[q] : dst + tile_index<NS>(g, q);
        const size_t gs = COLS ? ((size_t)gstride_a << logstride) : ((size_t)1 << logstride);
#pragma unroll
        for (int e = 0; e < R; e++) ptr[e * gs] = x[q * R + e];
      } else {
        u64* ptr = sm_out + phys(tile_index<NS>(g, q));
#pragma unroll
        for (int e = 0; e < R; e++) ptr[delta(e, S)] = x[q * R + e];
      }
    }
  }

  // The rows layout (one contiguous 4096-word chunk) reaches its unit-stride round with 8 consecutive
  // words per thread: touching global memory directly there spreads one warp request over many sectors.
  // That end of the pass is therefore staged through
  // shared memory with fully coalesced 128-bit global accesses; every other global access pattern
  // (64-byte segments) stays register-direct.
  static __device__ __forceinline__ void stage_in(const u64* __restrict__ src, u64* buf, bool reduce_on_load,
                                                  const LimbDev& L) {
#pragma unroll
    for (int k = 0; k < 8; k++) {
      const u32 i = k * NT + threadIdx.x;   // consecutive lanes -> consecutive words: 256 B per request, no conflicts
      u64 v = src[i];
      if (reduce_on_load) v = barrett64(v, L.p, L.bhi, L.blo);
      buf[phys(i)] = v;
    }
  }
  static __device__ __forceinline__ void stage_out(u64* __restrict__ dst, const u64* buf) {
#pragma unroll
    for (int k = 0; k < 8; k++) {
      const u32 i = k * NT + threadIdx.x;
      dst[i] = buf[phys(i)];
    }
  }

  static __device__ __forceinline__ void run(const u64* src, u64* dst, u32 gstride_a, u64* sm, bool reduce_on_load,
                                             const LimbDev& L, int s_base, u32 logn, u32 row0, bool first_pass) {
    u64 x[8];
    u64* buf[2] = {sm, sm + TW};
    constexpr bool STAGE = !COLS;  // stage the unit-stride end of a rows pass
    if (!INV) {
#pragma unroll
      for (int r = 0; r < NR; r++) {
        u64* in = buf[(r + 1) & 1];
        u64* out = buf[r & 1];
        if (r < NR - 1)
          round<3>(x, r, src, dst, gstride_a, in, out, r == 0, false, reduce_on_load, L, s_base, logn, row0, first_pass);
        else
          round<REM>(x, r, src, dst, gstride_a, in, out, r == 0, !STAGE, reduce_on_load, L, s_base, logn, row0, first_pass);
        if (r < NR - 1 || STAGE) __syncthreads();
      }
      if (STAGE) stage_out(dst, buf[(NR - 1) & 1]);
    } else {
      if (STAGE) {
        stage_in(src, buf[NR & 1], reduce_on_load, L);  // the buffer round NR-1 reads from
        __syncthreads();
      }
#pragma unroll
      for (int r = NR - 1; r >= 0; r--) {
        u64* in = buf[(r + 1) & 1];
        u64* out = buf[r & 1];
        if (r < NR - 1)
          round<3>(x, r, src, dst, gstride_a, in, out, false, r == 0, reduce_on_load, L, s_base, logn, row0, first_pass);
        else
          round<REM>(x, r, src, dst, gstride_a, in, out, !STAGE, r == 0, reduce_on_load, L, s_base, logn, row0, first_pass);
        if (r > 0) __syncthreads();
      }
    }
  }
};

// blockIdx -> (row, tile), row-major: consecutive CTAs sweep one 8N-byte row.  (A polynomial-minor order, which
// lets co-resident CTAs share a twiddle block in L1, scatters the HBM accesses over many rows at once.)
__device__ __forceinline__ void decode_block(const NttArgs& A, u32 tiles, u32& row, u32& tile) {
  row = blockIdx.x / tiles;
  tile = blockIdx.x % tiles;
}

template <int LOGP, bool COLS, bool INV, int TLOG>
__global__ void __launch_bounds__(1 << (TLOG - 3), 2 << (12 - TLOG)) ntt_fast_kernel(NttArgs A) {
  extern __shared__ u64 sm[];
  constexpr int LOGB = TLOG - LOGP;
  u32 row, tile;
  const u64* src;
  u64* dst;
  u32 gstride_a = 0, row0 = 0;
  int s_base;
  if (COLS) {
    const u32 logn2 = A.logn - LOGP;
    const u32 tiles = (1u << logn2) >> LOGB;
    decode_block(A, tiles, row, tile);
    src = A.in + ((size_t)(row / A.in_div) << A.logn) + (tile << LOGB);
    dst = A.out + ((size_t)row << A.logn) + (tile << LOGB);
    gstride_a = 1u << logn2;
    s_base = 0;
  } else {
    const u32 tiles = (1u << A.logn1) >> LOGB;
    decode_block(A, tiles, row, tile);
    src = A.in + ((size_t)(row / A.in_div) << A.logn) + ((size_t)tile << TLOG);
    dst = A.out + ((size_t)row << A.logn) + ((size_t)tile << TLOG);
    row0 = tile << LOGB;
    s_base = (int)A.logn1;
  }
  const LimbDev& L = A.limbs[A.ids[row % A.limbs_per_poly]];
  const bool first_pass = COLS || A.logn1 == 0;
  // (a lazy forward transform never meets the `stage == logn` test that selects the fully reducing last stage)
  FastTile<LOGP, COLS, INV, TLOG>::run(src, dst, gstride_a, sm, A.reduce_on_load != 0, L, s_base,
                                 (!INV && A.lazy_out) ? 0xffu : A.logn, row0, first_pass);
}

}  // namespace fhe_b200
