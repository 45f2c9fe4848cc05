// Test-only probe of the three-product accumulator AccKara of fhe_rs_b200/csrc/zq.cuh (never linked into
// libfhe_b200.so).  Case c sums the terms r[t] * w[t] for t in [off[c], off[c+1]) and then adds add[c] with add64;
// tests/test_gpu_acc_kara.py builds this file into a shared library and compares the words with Python integers.
#include <cuda_runtime.h>

#include "../../fhe_rs_b200/csrc/zq.cuh"

using namespace fhe_b200;

__global__ void acc_kara_kernel(LimbDev m, const u64* r, const u64* w, const u32* off, const u64* add, u32 n_cases,
                                u64* out) {
  const u32 c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= n_cases) return;
  AccKara acc;
  acc.clear();
  for (u32 t = off[c]; t < off[c + 1]; t++) acc.mac(split31(r[t]), split31(w[t]));
  acc.add64(add[c]);
  u64* o = out + (size_t)c * 4;
  u32 hi;
  acc.merged(o[0], o[1], hi);
  o[2] = hi;
  o[3] = acc.reduce(m);
}

// limb = {p, 2p, floor(2^128/p) >> 64, floor(2^128/p) mod 2^64, 2^128 mod p, c (Solinas) or 0}; r, w: off[n_cases]
// terms; off: n_cases + 1 offsets; add: n_cases addends; out: 4 words per case (merged lo, mid, hi, reduce).
// Returns 0, or the CUDA error code.
extern "C" int acc_kara_probe_run(const u64* limb, const u64* r, const u64* w, const u32* off, const u64* add,
                                  u32 n_cases, u64* out) {
  LimbDev m = {};
  m.p = limb[0]; m.p2 = limb[1]; m.bhi = limb[2]; m.blo = limb[3]; m.c128 = limb[4]; m.sol_c = limb[5];
  const size_t n_terms = off[n_cases];
  const size_t term_bytes = (n_terms ? n_terms : 1) * sizeof(u64), off_bytes = (n_cases + 1) * sizeof(u32);
  const size_t add_bytes = n_cases * sizeof(u64), out_bytes = 4 * n_cases * sizeof(u64);
  char* dev = nullptr;
  cudaError_t e = cudaMalloc(&dev, 2 * term_bytes + add_bytes + out_bytes + off_bytes);
  if (e != cudaSuccess) return (int)e;
  u64* dr = reinterpret_cast<u64*>(dev);
  u64* dw = reinterpret_cast<u64*>(dev + term_bytes);
  u64* dadd = reinterpret_cast<u64*>(dev + 2 * term_bytes);
  u64* dout = reinterpret_cast<u64*>(dev + 2 * term_bytes + add_bytes);
  u32* doff = reinterpret_cast<u32*>(dev + 2 * term_bytes + add_bytes + out_bytes);
  if ((e = cudaMemcpy(dr, r, n_terms * sizeof(u64), cudaMemcpyHostToDevice)) == cudaSuccess &&
      (e = cudaMemcpy(dw, w, n_terms * sizeof(u64), cudaMemcpyHostToDevice)) == cudaSuccess &&
      (e = cudaMemcpy(dadd, add, add_bytes, cudaMemcpyHostToDevice)) == cudaSuccess &&
      (e = cudaMemcpy(doff, off, off_bytes, cudaMemcpyHostToDevice)) == cudaSuccess &&
      (e = cudaMemset(dout, 0, out_bytes)) == cudaSuccess) {
    acc_kara_kernel<<<(n_cases + 127) / 128, 128>>>(m, dr, dw, doff, dadd, n_cases, dout);
    if ((e = cudaGetLastError()) == cudaSuccess && (e = cudaDeviceSynchronize()) == cudaSuccess)
      e = cudaMemcpy(out, dout, out_bytes, cudaMemcpyDeviceToHost);
  }
  cudaFree(dev);
  return (int)e;
}
