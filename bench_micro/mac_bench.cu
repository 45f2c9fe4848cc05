// Throughput of the 64x64 multiply-accumulate forms on one SM sub-partition (clk per MAC per warp):
//  V0: four plain IMAD.WIDE (no carries; lower bound)   V1: even/odd carry chains (Acc192 in zq.cuh)
//  V2: 128-bit product then 192-bit add (the r1a form)
//  V3: three products per term, operands < 2^62 split at bit 31 (AccKara in zq.cuh), at the scaler loop's shape: the
//      split of r is shared by the NACC outputs, the omega halves and their sums are precomputed
#include <cstdio>
#include <cuda_runtime.h>
#include "device.cuh"
#include "../fhe_rs_b200/csrc/zq.cuh"
typedef unsigned long long u64;
typedef unsigned int u32;

template <int V>
struct Acc {
  u32 e0, e1, e2, e3, e4, o1, o2, o3;
  u64 lo, mid, hi;
  fhe_b200::AccKara kara;
  __device__ __forceinline__ void clear() { e0 = e1 = e2 = e3 = e4 = o1 = o2 = o3 = 0; lo = mid = hi = 0; kara.clear(); }
  __device__ __forceinline__ void mac(const fhe_b200::Split31& r, const fhe_b200::Split31& w) { kara.mac(r, w); }
  __device__ __forceinline__ void mac(u64 a, u64 b) {
    if (V == 0) {
      asm volatile("{\n\t.reg .u32 a0,a1,b0,b1;\n\tmov.b64 {a0,a1}, %3;\n\tmov.b64 {b0,b1}, %4;\n\t"
          "mad.wide.u32 %0, a0, b0, %0;\n\tmad.wide.u32 %1, a0, b1, %1;\n\tmad.wide.u32 %1, a1, b0, %1;\n\tmad.wide.u32 %2, a1, b1, %2;\n\t}"
          : "+l"(lo), "+l"(mid), "+l"(hi) : "l"(a), "l"(b));
    } else if (V == 1) {
      asm volatile("{\n\t.reg .u32 a0, a1, b0, b1;\n\tmov.b64 {a0, a1}, %8;\n\tmov.b64 {b0, b1}, %9;\n\t"
          "mad.lo.cc.u32 %0, a0, b0, %0;\n\tmadc.hi.cc.u32 %1, a0, b0, %1;\n\tmadc.lo.cc.u32 %2, a1, b1, %2;\n\t"
          "madc.hi.cc.u32 %3, a1, b1, %3;\n\taddc.u32 %4, %4, 0;\n\t"
          "mad.lo.cc.u32 %5, a0, b1, %5;\n\tmadc.hi.cc.u32 %6, a0, b1, %6;\n\taddc.u32 %7, %7, 0;\n\t"
          "mad.lo.cc.u32 %5, a1, b0, %5;\n\tmadc.hi.cc.u32 %6, a1, b0, %6;\n\taddc.u32 %7, %7, 0;\n\t}"
          : "+r"(e0), "+r"(e1), "+r"(e2), "+r"(e3), "+r"(e4), "+r"(o1), "+r"(o2), "+r"(o3) : "l"(a), "l"(b));
    } else {
      u64 pl, ph;
      asm volatile("{\n\t.reg .u32 a0, a1, b0, b1, p0, p1, m0, m1, q0, q1, t1, t2, t3;\n\t.reg .u64 P, M, Q;\n\t"
          "mov.b64 {a0, a1}, %2;\n\tmov.b64 {b0, b1}, %3;\n\tmul.wide.u32 P, a0, b0;\n\tmul.wide.u32 M, a0, b1;\n\t"
          "mad.wide.u32 M, a1, b0, M;\n\tmul.wide.u32 Q, a1, b1;\n\tmov.b64 {p0, p1}, P;\n\tmov.b64 {m0, m1}, M;\n\t"
          "mov.b64 {q0, q1}, Q;\n\tadd.cc.u32 t1, p1, m0;\n\taddc.cc.u32 t2, q0, m1;\n\taddc.u32 t3, q1, 0;\n\t"
          "mov.b64 %0, {p0, t1};\n\tmov.b64 %1, {t2, t3};\n\t}" : "=l"(pl), "=l"(ph) : "l"(a), "l"(b));
      asm volatile("add.cc.u64 %0, %0, %3;\n\taddc.cc.u64 %1, %1, %4;\n\taddc.u64 %2, %2, 0;" : "+l"(lo), "+l"(mid), "+l"(hi) : "l"(pl), "l"(ph));
    }
  }
  __device__ __forceinline__ u64 fin() const {
    u64 a, b;
    u32 c;
    kara.merged(a, b, c);
    return lo ^ mid ^ hi ^ e0 ^ e1 ^ e2 ^ e3 ^ e4 ^ o1 ^ o2 ^ o3 ^ (V == 3 ? a ^ b ^ c : 0);
  }
};

template <int V, int NACC>
__global__ void k(u64* out, u64 seed, int iters) {
  Acc<V> acc[NACC];
  u64 w[8];
  fhe_b200::Split31 ws[8];
#pragma unroll
  for (int i = 0; i < NACC; i++) acc[i].clear();
#pragma unroll
  for (int i = 0; i < 8; i++) {
    w[i] = (seed * (threadIdx.x + 17 + i)) & 0x3fffffffffffffffull;
    ws[i] = fhe_b200::split31(w[i]);
  }
  u64 r = (seed ^ threadIdx.x) & 0x3fffffffffffffffull;
  for (int it = 0; it < iters; it++) {
#pragma unroll
    for (int u = 0; u < 8 / NACC * 1; u++) {
      if (V == 3) {
        const fhe_b200::Split31 rs = fhe_b200::split31(r);
#pragma unroll
        for (int a = 0; a < NACC; a++) acc[a].mac(rs, ws[(u * NACC + a) & 7]);
      } else {
#pragma unroll
        for (int a = 0; a < NACC; a++) acc[a].mac(r, w[(u * NACC + a) & 7]);
      }
      r = (r + 0x9e3779b97f4a7c15ull) & 0x3fffffffffffffffull;
    }
  }
  u64 x = 0;
#pragma unroll
  for (int i = 0; i < NACC; i++) x ^= acc[i].fin();
  out[blockIdx.x * blockDim.x + threadIdx.x] = x;
}
template <int V, int NACC>
void run(int warps_per_smsp) {
  u64* out;
  int threads = 128, blocks = dev_sms() * warps_per_smsp, iters = 2000;   // 128 threads = one warp per SMSP per block
  cudaMalloc(&out, sizeof(u64) * blocks * threads);
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0); cudaEventCreate(&e1);
  k<V, NACC><<<blocks, threads>>>(out, 12345, 10);
  cudaDeviceSynchronize();
  cudaEventRecord(e0);
  k<V, NACC><<<blocks, threads>>>(out, 12345, iters);
  cudaEventRecord(e1);
  cudaEventSynchronize(e1);
  float ms; cudaEventElapsedTime(&ms, e0, e1);
  int dev_clk; cudaDeviceGetAttribute(&dev_clk, cudaDevAttrClockRate, 0);
  double macs_per_warp = 8.0 * iters;
  double clk = ms * 1e-3 * (dev_clk * 1e3) / (macs_per_warp * warps_per_smsp);
  printf("V%d NACC=%d warps/SMSP=%2d : %7.3f ms -> %5.1f clk per MAC per warp (at %d MHz nominal)\n", V, NACC, warps_per_smsp, ms, clk, dev_clk / 1000);
  cudaFree(out);
}
int main() {
  for (int w : {1, 2, 4, 6, 12}) {
    run<0, 4>(w); run<1, 4>(w); run<2, 4>(w); run<3, 4>(w);
  }
  run<1, 1>(6); run<1, 2>(6); run<1, 8>(6); run<2, 2>(6); run<2, 1>(6);
  return 0;
}
