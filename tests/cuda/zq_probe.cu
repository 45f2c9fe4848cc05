// Test-only probe of the device arithmetic in fhe_rs_b200/csrc/zq.cuh (never linked into libfhe_b200.so).
// One kernel applies primitive `op` element-wise to operand arrays a, b, c and writes up to 8 result words per
// element; tests/test_gpu_zq_probe.py builds this file into a shared library and compares every word with Python
// integers.
#include <cstdio>
#include <cuda_runtime.h>

#include "../../fhe_rs_b200/csrc/zq.cuh"

using namespace fhe_b200;

enum Op {
  MUL_SHOUP_LAZY = 0, MUL_SHOUP, MUL_SOLINAS_LAZY, MUL_SOLINAS_LAZY_V1, FOLD63_SOLINAS, ADDBACK2P, SHOUP_OF,
  BARRETT128_LAZY, BARRETT128, BARRETT64, MULMOD, MUL128_62, FOLD192_SOLINAS, ACC192, ACC_THETA, MULMOD_LIMB_LAZY,
  MULMOD_LIMB, REDUCE128_LIMB, REDUCE94_LIMB, N_OPS
};

__global__ void probe_kernel(int op, LimbDev m, const u64* a, const u64* b, const u64* c, const u64* d, u64 n,
                             u64* out) {
  const u64 i = blockIdx.x * (u64)blockDim.x + threadIdx.x;
  if (i >= n) return;
  const u64 x = a[i], y = b[i], z = c[i], k = d[i];
  u64* o = out + i * 8;
  switch (op) {
    case MUL_SHOUP_LAZY: o[0] = mul_shoup_lazy(x, y, z, m.p); break;
    case MUL_SHOUP: o[0] = mul_shoup(x, y, z, m.p); break;
    case MUL_SOLINAS_LAZY: o[0] = mul_solinas_lazy(x, y, z, (u32)m.sol_c); break;
    case MUL_SOLINAS_LAZY_V1: o[0] = mul_solinas_lazy_v1(x, y, z, (u32)m.sol_c); break;
    case FOLD63_SOLINAS: o[0] = fold63_solinas(x, (u32)(2 * m.sol_c)); break;
    case ADDBACK2P: o[0] = addback2p(x, m.p2); break;
    case SHOUP_OF: o[0] = shoup_of(x, m.p, m.bhi, m.blo); break;
    case BARRETT128_LAZY: o[0] = barrett128_lazy(x, y, m.p, m.bhi, m.blo); break;
    case BARRETT128: o[0] = barrett128(x, y, m.p, m.bhi, m.blo); break;
    case BARRETT64: o[0] = barrett64(x, m.p, m.bhi, m.blo); break;
    case MULMOD: o[0] = mulmod(x, y, m.p, m.bhi, m.blo); break;
    case MUL128_62: mul128_62(x, y, o[0], o[1]); break;
    case FOLD192_SOLINAS: o[0] = fold192_solinas(x, y, z, (u32)m.sol_c); break;
    case ACC192: {
      // k terms x * y, then one add64(z): the merged words, reduce and reduce_lazy
      Acc192 acc;
      acc.clear();
      for (u64 t = 0; t < k; t++) acc.mac(x, y);
      acc.add64(z);
      u32 hi;
      acc.merged(o[0], o[1], hi);
      o[2] = hi;
      o[3] = acc.reduce(m);
      o[4] = acc.reduce_lazy(m);
      break;
    }
    case ACC_THETA: {
      // k terms r = x times theta = z:y with AccTheta and with mac_theta: 7 words each, packed two per u64
      AccTheta at;
      at.clear();
      u32 ref[7] = {0, 0, 0, 0, 0, 0, 0};
      for (u64 t = 0; t < k; t++) {
        at.mac(x, y, z);
        mac_theta(ref, x, y, z);
      }
      u32 w[7];
      at.words(w);
      for (int j = 0; j < 4; j++) {
        o[j] = (u64)w[2 * j] | (j < 3 ? (u64)w[2 * j + 1] << 32 : 0);
        o[4 + j] = (u64)ref[2 * j] | (j < 3 ? (u64)ref[2 * j + 1] << 32 : 0);
      }
      break;
    }
    case MULMOD_LIMB_LAZY: o[0] = mulmod_limb_lazy(x, y, m); break;
    case MULMOD_LIMB: o[0] = mulmod_limb(x, y, m); break;
    case REDUCE128_LIMB: o[0] = reduce128_limb(x, y, m); break;
    case REDUCE94_LIMB: o[0] = reduce94_limb(x, y, m); break;
    default: break;
  }
}

// limb = {p, 2p, floor(2^128/p) >> 64, floor(2^128/p) mod 2^64, 2^128 mod p, c (Solinas) or 0}; a, b, c, d: n words
// each; out: 8n words.  Returns 0, or the CUDA error code.
extern "C" int zq_probe_run(int op, const u64* limb, const u64* a, const u64* b, const u64* c, const u64* d, u64 n,
                            u64* out) {
  if (op < 0 || op >= N_OPS) return -1;
  LimbDev m = {};
  m.p = limb[0]; m.p2 = limb[1]; m.bhi = limb[2]; m.blo = limb[3]; m.c128 = limb[4]; m.sol_c = limb[5];
  u64* dev = nullptr;
  const size_t in_bytes = n * sizeof(u64), out_bytes = 8 * n * sizeof(u64);
  cudaError_t e = cudaMalloc(&dev, 4 * in_bytes + out_bytes);
  if (e != cudaSuccess) return (int)e;
  u64 *da = dev, *db = dev + n, *dc = dev + 2 * n, *dd = dev + 3 * n, *dout = dev + 4 * n;
  if ((e = cudaMemcpy(da, a, in_bytes, cudaMemcpyHostToDevice)) == cudaSuccess &&
      (e = cudaMemcpy(db, b, in_bytes, cudaMemcpyHostToDevice)) == cudaSuccess &&
      (e = cudaMemcpy(dc, c, in_bytes, cudaMemcpyHostToDevice)) == cudaSuccess &&
      (e = cudaMemcpy(dd, d, in_bytes, cudaMemcpyHostToDevice)) == cudaSuccess &&
      (e = cudaMemset(dout, 0, out_bytes)) == cudaSuccess) {
    probe_kernel<<<(unsigned)((n + 127) / 128), 128>>>(op, m, da, db, dc, dd, n, dout);
    if ((e = cudaGetLastError()) == cudaSuccess && (e = cudaDeviceSynchronize()) == cudaSuccess)
      e = cudaMemcpy(out, dout, out_bytes, cudaMemcpyDeviceToHost);
  }
  cudaFree(dev);
  return (int)e;
}
