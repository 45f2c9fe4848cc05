// NTT launcher: picks the (N1, N2) split and tile shapes for a given N and instantiates
// the tile kernels of ntt.cuh.
#include <algorithm>
#include <climits>
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <map>
#include <mutex>
#include <utility>

#include "engine.hpp"
#include "ntt_fast.cuh"
#include "ntt_tma.cuh"

namespace fhe_b200 {

std::atomic<unsigned long long> g_launches{0};
std::atomic<unsigned long long> g_ntt_rows[2] = {{0}, {0}};

const Switches& switches() {
  static const Switches s = [] {
    auto set = [](const char* name) { return getenv(name) != nullptr; };
    auto is = [](const char* name, const char* value) {
      const char* e = getenv(name);
      return e && !strcmp(e, value);
    };
    auto number = [](const char* name, int dflt) {
      const char* e = getenv(name);
      return e ? atoi(e) : dflt;
    };
    auto clamped = [&](const char* name, int dflt, int lo, int hi) {
      const int v = number(name, dflt);
      return (u32)(v < lo ? lo : v > hi ? hi : v);
    };
    Switches w;
    // ~28 GB of scratch per in-flight chunk at set C (108 MB per ciphertext); larger chunks mean fewer kernel
    // boundaries per ciphertext
    w.chunk = clamped("FHE_B200_CHUNK", 256, 1, INT_MAX);
    w.streams = clamped("FHE_B200_STREAMS", 2, 1, 4);
    w.ntt = is("FHE_B200_NTT", "fast") ? Switches::NTT_FAST : is("FHE_B200_NTT", "tma") ? Switches::NTT_TMA
                                                                                         : Switches::NTT_AUTO;
    w.generic_ntt = set("FHE_B200_GENERIC_NTT");
    w.solinas_ntt = set("FHE_B200_SOLINAS_NTT");
    w.no_solinas = set("FHE_B200_NO_SOLINAS");
    w.no_tensor_fusion = set("FHE_B200_NO_TENSOR_FUSION");
    w.classic_scaler = is("FHE_B200_SCALER", "classic");
    w.ksmac = is("FHE_B200_KSMAC", "tma")       ? Switches::KSMAC_TMA
              : is("FHE_B200_KSMAC", "classic") ? Switches::KSMAC_CLASSIC
                                                : Switches::KSMAC_FUSED;
    w.tma_cols = number("FHE_B200_TMA_COLS", 3);
    w.scale_unroll = number("FHE_B200_SCALE_UNROLL", 2);
    w.ks_stages = clamped("FHE_B200_KS_STAGES", 2, 2, 4);
    return w;
  }();
  return s;
}

EncodeTiledFn tensor_map_encoder() {
  static EncodeTiledFn fn = [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q = cudaDriverEntryPointSymbolNotFound;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess ||
        q != cudaDriverEntryPointSuccess)
      p = nullptr;
    cudaGetLastError();
    return (EncodeTiledFn)p;
  }();
  return fn;
}

bool box_map(CUtensorMap* m, const u64* base, u64 rows, u32 logn, u32 box_cols, u32 box_rows) {
  const cuuint64_t gdim[2] = {(cuuint64_t)1 << logn, rows};
  const cuuint64_t gstride[1] = {(cuuint64_t)8 << logn};
  const cuuint32_t box[2] = {box_cols, box_rows};
  const cuuint32_t es[2] = {1, 1};
  return tensor_map_encoder() &&
         tensor_map_encoder()(m, CU_TENSOR_MAP_DATA_TYPE_UINT64, 2, (void*)base, gdim, gstride, box, es,
                              CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
                              CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

int sm_count() {
  static std::mutex mu;
  static std::map<int, int> cache;
  int dev = 0;
  FHE_CUDA(cudaGetDevice(&dev));
  std::lock_guard<std::mutex> g(mu);
  auto it = cache.find(dev);
  if (it != cache.end()) return it->second;
  int n = 0;
  FHE_CUDA(cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev));
  return cache[dev] = n;
}

void ensure_dynamic_smem(const void* kernel, size_t bytes) {
  if (bytes <= 48 * 1024) return;   // the default limit needs no opt-in
  static std::mutex mu;
  static std::map<std::pair<int, const void*>, size_t> granted;
  int dev = 0;
  FHE_CUDA(cudaGetDevice(&dev));
  std::lock_guard<std::mutex> g(mu);
  size_t& have = granted[std::make_pair(dev, kernel)];
  if (have >= bytes) return;
  FHE_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
  have = bytes;
}

namespace {

constexpr int kTileLog = 12;  // 4096 words (32 KiB + padding) of shared memory per CTA

template <int LOGP, int LOGB, bool INV>
void run_rows(const NttArgs& a, cudaStream_t st) {
  constexpr u32 T = 1u << (LOGP + LOGB);
  const u32 tiles = (1u << a.logn1) >> LOGB;
  const u32 threads = T / 8 >= 256 ? 256 : (T / 8 < 32 ? 32 : T / 8);
  const size_t smem = (T + (T >> 5) + 1) * sizeof(u64);
  ntt_rows_kernel<LOGP, LOGB, INV><<<a.n_rows * tiles, threads, smem, st>>>(a);
  g_launches++;
}
template <int LOGP, int LOGB, bool INV>
void run_cols(const NttArgs& a, cudaStream_t st) {
  constexpr u32 T = 1u << (LOGP + LOGB);
  const u32 tiles = (1u << (a.logn - LOGP)) >> LOGB;
  const size_t smem = (T + (T >> 5) + 1) * sizeof(u64);
  ntt_cols_kernel<LOGP, LOGB, INV><<<a.n_rows * tiles, 256, smem, st>>>(a);
  g_launches++;
}

template <int LOGP, bool COLS, bool INV, int TLOG>
void run_fast(const NttArgs& a, cudaStream_t st) {
  constexpr size_t smem = 2 * FastTile<LOGP, COLS, INV, TLOG>::TW * sizeof(u64);
  ensure_dynamic_smem((const void*)ntt_fast_kernel<LOGP, COLS, INV, TLOG>, smem);
  constexpr int LOGB = TLOG - LOGP;
  const u32 tiles = COLS ? ((1u << (a.logn - LOGP)) >> LOGB) : ((1u << a.logn1) >> LOGB);
  ntt_fast_kernel<LOGP, COLS, INV, TLOG><<<a.n_rows * tiles, 1 << (TLOG - 3), smem, st>>>(a);
  g_launches++;
}
// 2048-word cols tiles; N = 2^16 keeps 4096 words (a 2048-word tile would be two columns wide there)
template <bool INV>
void run_fast_cols_for(const NttArgs& a, cudaStream_t st) {
  switch (a.logn1) {
    case 7: run_fast<7, true, INV, 11>(a, st); break;
    case 8: run_fast<8, true, INV, 11>(a, st); break;
    case 9: run_fast<9, true, INV, 11>(a, st); break;
    case 10: run_fast<10, true, INV, 12>(a, st); break;
    default: break;
  }
}

template <bool INV>
void run_single(const NttArgs& a, cudaStream_t st) {
  switch (a.logn) {
    case 3: run_rows<3, 0, INV>(a, st); break;
    case 4: run_rows<4, 0, INV>(a, st); break;
    case 5: run_rows<5, 0, INV>(a, st); break;
    case 6: run_rows<6, 0, INV>(a, st); break;
    case 7: run_rows<7, 0, INV>(a, st); break;
    case 8: run_rows<8, 0, INV>(a, st); break;
    case 9: run_rows<9, 0, INV>(a, st); break;
    case 10: run_rows<10, 0, INV>(a, st); break;
    case 11: run_rows<11, 0, INV>(a, st); break;
    case 12: run_rows<12, 0, INV>(a, st); break;
    default: break;
  }
}
template <bool INV>
void run_cols_for(const NttArgs& a, cudaStream_t st) {
  switch (a.logn1) {
    case 7: run_cols<7, kTileLog - 7, INV>(a, st); break;
    case 8: run_cols<8, kTileLog - 8, INV>(a, st); break;
    case 9: run_cols<9, kTileLog - 9, INV>(a, st); break;
    case 10: run_cols<10, kTileLog - 10, INV>(a, st); break;
    default: break;
  }
}

// ---- TMA-fed persistent kernels (ntt_tma.cuh)
struct TmaFail {};
// the buffer [rows][N] u64 as 128-byte box rows: dims {16, rows*N/16}, box {16, box_rows}, 128-byte swizzle
CUtensorMap rows_map(const u64* base, u64 rows, u32 logn, u32 box_rows) {
  CUtensorMap m;
  const cuuint64_t gdim[2] = {16, (rows << logn) >> 4};
  const cuuint64_t gstride[1] = {128};
  const cuuint32_t box[2] = {16, box_rows};
  const cuuint32_t es[2] = {1, 1};
  if (gdim[1] >= (1ull << 31) ||
      tensor_map_encoder()(&m, CU_TENSOR_MAP_DATA_TYPE_UINT64, 2, (void*)base, gdim, gstride, box, es,
                           CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                           CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
    throw TmaFail{};
  return m;
}
// the buffer as [rows][N1][64] u64: box {16 columns, box_rows points, 1 row}, no swizzle
CUtensorMap cols_map(const u64* base, u64 rows, u32 logn, u32 box_rows) {
  CUtensorMap m;
  const cuuint64_t gdim[3] = {64, (cuuint64_t)1 << (logn - 6), rows};
  const cuuint64_t gstride[2] = {512, (cuuint64_t)8 << logn};
  const cuuint32_t box[3] = {16, box_rows, 1};
  const cuuint32_t es[3] = {1, 1, 1};
  if (tensor_map_encoder()(&m, CU_TENSOR_MAP_DATA_TYPE_UINT64, 3, (void*)base, gdim, gstride, box, es,
                           CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                           CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
    throw TmaFail{};
  return m;
}

constexpr int kRowsRlog = 4;

// one tile per CTA iteration
template <bool INV, int STAGES, int MINB>
void run_tma_rows_one(const u64* in, u64 in_rows, u64* out, u64 out_rows, NttTmaArgs A, cudaStream_t st) {
  using Cfg = RowsCfg<kRowsRlog, STAGES>;
  const CUtensorMap mi = rows_map(in, in_rows, A.logn, 4 * Cfg::R), mo = rows_map(out, out_rows, A.logn, 4 * Cfg::R);
  A.tiles_per_row = (1u << (A.logn - 6)) / Cfg::R;
  A.tiles_total = A.lpp * A.tiles_per_row * A.n_polys;
  const u32 grid = std::min<u64>(A.tiles_total, (u64)sm_count() * MINB);
  if (!INV && A.lazy_out) {
    auto k = ntt_tma_rows_kernel<INV, kRowsRlog, STAGES, MINB, !INV>;
    ensure_dynamic_smem((const void*)k, Cfg::SMEM);
    k<<<grid, Cfg::NT + 32, Cfg::SMEM, st>>>(mi, mo, A);
  } else {
    auto k = ntt_tma_rows_kernel<INV, kRowsRlog, STAGES, MINB, false>;
    ensure_dynamic_smem((const void*)k, Cfg::SMEM);
    k<<<grid, Cfg::NT + 32, Cfg::SMEM, st>>>(mi, mo, A);
  }
  g_launches++;
}
// two polynomials per CTA iteration (ntt_tma_rows_pair_kernel); needs an even number of polynomials
template <bool INV, int STAGES, int MINB>
void run_tma_rows_pair(const u64* in, u64 in_rows, u64* out, u64 out_rows, NttTmaArgs A, cudaStream_t st) {
  using Cfg = RowsCfg<kRowsRlog, STAGES>;
  constexpr size_t smem = (size_t)STAGES * 2 * Cfg::TILE_BYTES + Cfg::TW_PAIRS * 16 + 2 * STAGES * 8 + 1024;
  const CUtensorMap mi = rows_map(in, in_rows, A.logn, 4 * Cfg::R), mo = rows_map(out, out_rows, A.logn, 4 * Cfg::R);
  A.tiles_per_row = (1u << (A.logn - 6)) / Cfg::R;
  A.n_polys /= 2;   // pairs
  A.tiles_total = A.lpp * A.tiles_per_row * A.n_polys;
  const u32 grid = std::min<u64>(A.tiles_total, (u64)sm_count() * MINB);
  if (!INV && A.lazy_out) {
    auto k = ntt_tma_rows_pair_kernel<INV, kRowsRlog, STAGES, MINB, !INV>;
    ensure_dynamic_smem((const void*)k, smem);
    k<<<grid, Cfg::NT + 32, smem, st>>>(mi, mo, A);
  } else {
    auto k = ntt_tma_rows_pair_kernel<INV, kRowsRlog, STAGES, MINB, false>;
    ensure_dynamic_smem((const void*)k, smem);
    k<<<grid, Cfg::NT + 32, smem, st>>>(mi, mo, A);
  }
  g_launches++;
}

template <bool INV>
void run_tma_rows(const u64* in, u64 in_rows, u64* out, u64 out_rows, const NttTmaArgs& A, cudaStream_t st) {
  // two polynomials per CTA iteration (ring depth 3 x 3 CTAs per SM) wherever the polynomials pair up; the one-tile
  // kernel (4 x 4) serves an odd polynomial count, or a digit-adjacent launch with an odd digit count
  if (A.n_polys % 2 == 0 && !(A.digit_adjacent && A.n_dig % 2))
    run_tma_rows_pair<INV, 3, 3>(in, in_rows, out, out_rows, A, st);
  else
    run_tma_rows_one<INV, 4, 4>(in, in_rows, out, out_rows, A, st);
}
template <int LOGP, bool INV, int STAGES, int MINB>
void run_tma_cols(const u64* in, u64 in_rows, u64* out, u64 out_rows, NttTmaArgs A, cudaStream_t st) {
  using Cfg = ColsCfg<LOGP, STAGES>;
  const CUtensorMap mi = cols_map(in, in_rows, A.logn, Cfg::BOX_ROWS), mo = cols_map(out, out_rows, A.logn, Cfg::BOX_ROWS);
  A.tiles_per_row = 4;
  A.tiles_total = A.lpp * 4 * A.n_polys;
  const u32 grid = std::min<u64>(A.tiles_total, (u64)sm_count() * MINB);
  if (!INV && A.reduce_on_load) {
    auto k = ntt_tma_cols_kernel<LOGP, INV, STAGES, MINB, !INV>;
    ensure_dynamic_smem((const void*)k, Cfg::SMEM);
    k<<<grid, Cfg::NT + 32, Cfg::SMEM, st>>>(mi, mo, A);
  } else {
    auto k = ntt_tma_cols_kernel<LOGP, INV, STAGES, MINB, false>;
    ensure_dynamic_smem((const void*)k, Cfg::SMEM);
    k<<<grid, Cfg::NT + 32, Cfg::SMEM, st>>>(mi, mo, A);
  }
  g_launches++;
}
// ring depth 3 (FHE_B200_TMA_COLS=2: 2); resident CTAs per SM by tile height
template <bool INV>
void run_tma_cols_for(const u64* in, u64 in_rows, u64* out, u64 out_rows, const NttTmaArgs& A, cudaStream_t st) {
  const bool d2 = switches().tma_cols == 2;
  switch (A.logn - 6) {
    case 7:
      if (d2) run_tma_cols<7, INV, 2, 6>(in, in_rows, out, out_rows, A, st);
      else run_tma_cols<7, INV, 3, 4>(in, in_rows, out, out_rows, A, st);
      break;
    case 8:
      if (d2) run_tma_cols<8, INV, 2, 3>(in, in_rows, out, out_rows, A, st);
      else run_tma_cols<8, INV, 3, 2>(in, in_rows, out, out_rows, A, st);
      break;
    case 9:
      if (d2) run_tma_cols<9, INV, 2, 1>(in, in_rows, out, out_rows, A, st);
      else run_tma_cols<9, INV, 3, 1>(in, in_rows, out, out_rows, A, st);
      break;
    default: throw TmaFail{};
  }
}

// Both passes through the TMA kernels.  Returns false when the shape is outside their domain (the caller then uses
// the register-resident kernels).
bool launch_ntt_tma(const u64* in, u64* out, u32 n_rows, const RowIds& ids, const LimbDev* limbs, u32 logn, bool inverse,
                    u32 in_div, bool reduce_on_load, cudaStream_t st, bool lazy_out, bool digit_adjacent, u32 n_dig) {
  const u32 lpp = ids.limbs_per_poly;
  if (logn < 13 || logn > 15 || !tensor_map_encoder()) return false;
  if (n_rows % lpp != 0 || (in_div != 1 && in_div != lpp)) return false;
  if (digit_adjacent && ((n_rows / lpp) % n_dig != 0 || n_dig == 0)) return false;
  if ((reinterpret_cast<uintptr_t>(in) | reinterpret_cast<uintptr_t>(out)) & 127) return false;
  NttTmaArgs A;
  std::memset(&A, 0, sizeof(A));
  A.limbs = limbs;
  A.n_polys = n_rows / lpp;
  A.lpp = lpp;
  A.logn = logn;
  A.digit_adjacent = digit_adjacent ? 1 : 0;
  A.n_dig = digit_adjacent ? n_dig : 1;
  for (int i = 0; i < kMaxPos; i++) A.ids[i] = ids.ids[i];
  const u64 in_rows = in_div == 1 ? n_rows : n_rows / lpp;
  try {
    NttTmaArgs first = A, second = A;
    first.in_bcast = first.limb_inner = in_div != 1;
    if (!inverse) {
      first.reduce_on_load = reduce_on_load;
      second.lazy_out = lazy_out;
      run_tma_cols_for<false>(in, in_rows, out, n_rows, first, st);
      run_tma_rows<false>(out, n_rows, out, n_rows, second, st);
    } else {
      if (reduce_on_load || in_div != 1) return false;
      run_tma_rows<true>(in, in_rows, out, n_rows, first, st);
      run_tma_cols_for<true>(out, n_rows, out, n_rows, second, st);
    }
  } catch (const TmaFail&) {
    return false;
  }
  return true;
}

// tensor product + first inverse pass fused (ntt_tma_tensor_rows_kernel), then the inverse cols pass in place on T
template <int STAGES, int MINB>
void run_tensor_rows(const CUtensorMap& ma, const CUtensorMap& mb, const CUtensorMap& mxa, const CUtensorMap& mxb,
                     const CUtensorMap& mo, TensorRowsArgs A, cudaStream_t st) {
  using Cfg = TensorRowsCfg<kRowsRlog, STAGES>;
  auto k = ntt_tma_tensor_rows_kernel<kRowsRlog, STAGES, MINB>;
  ensure_dynamic_smem((const void*)k, Cfg::SMEM);
  const u32 grid = std::min<u64>(A.items_total, (u64)sm_count() * MINB);
  k<<<grid, Cfg::NT + 32, Cfg::SMEM, st>>>(ma, mb, mxa, mxb, mo, A);
  g_launches++;
}

// tensor product + first inverse pass fused (ntt_tma_tensor_rows_kernel), then the inverse cols pass in place on T
bool launch_tensor_intt_tma(const u64* a, const u64* b, const u64* xa, const u64* xb, u64* T, u32 cts, u32 L, u32 K,
                            const RowIds& mul_ids, const LimbDev* limbs, u32 logn, cudaStream_t st) {
  constexpr u32 R = 1u << kRowsRlog;
  const u32 E = K - L;
  try {
    const CUtensorMap ma = rows_map(a, (u64)cts * 2 * L, logn, 4 * R), mb = rows_map(b, (u64)cts * 2 * L, logn, 4 * R);
    const CUtensorMap mxa = rows_map(xa, (u64)cts * 2 * E, logn, 4 * R), mxb = rows_map(xb, (u64)cts * 2 * E, logn, 4 * R);
    const CUtensorMap mo = rows_map(T, (u64)cts * 3 * K, logn, 4 * R);
    TensorRowsArgs A;
    std::memset(&A, 0, sizeof(A));
    A.limbs = limbs; A.cts = cts; A.L = L; A.K = K; A.logn = logn;
    A.tiles_per_row = (1u << (logn - 6)) / R;
    A.items_total = K * A.tiles_per_row * cts;
    for (int i = 0; i < kMaxPos; i++) A.ids[i] = mul_ids.ids[i];
    run_tensor_rows<2, 2>(ma, mb, mxa, mxb, mo, A, st);   // ring depth 2 x 2 CTAs per SM
    // second pass of the inverse transform of the 3K product rows, in place
    NttTmaArgs C;
    std::memset(&C, 0, sizeof(C));
    C.limbs = limbs; C.n_polys = cts * 3; C.lpp = K; C.logn = logn; C.n_dig = 1;
    for (int i = 0; i < kMaxPos; i++) C.ids[i] = mul_ids.ids[i];
    run_tma_cols_for<true>(T, (u64)cts * 3 * K, T, (u64)cts * 3 * K, C, st);
  } catch (const TmaFail&) {
    return false;
  }
  return true;
}

template <int STAGES, class Kern, class Keys>
void run_ks_rows_mac_with(Kern k, const CUtensorMap& mi, const CUtensorMap& m0, const CUtensorMap& m1,
                          const KsRowsArgs& A, const Keys& keys, cudaStream_t st) {
  using Cfg = KsRowsCfg<STAGES>;
  const size_t smem = Cfg::smem(A.n_dig);
  ensure_dynamic_smem((const void*)k, smem);
  int per_sm = 0;
  FHE_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, (const void*)k, Cfg::NT + 32, smem));
  const u32 grid = (u32)std::min<u64>(A.items_total, (u64)sm_count() * std::max(per_sm, 1));
  k<<<grid, Cfg::NT + 32, smem, st>>>(mi, m0, m1, A, keys);
  g_launches++;
}

template <int STAGES>
void run_ks_rows_mac(const CUtensorMap& mi, const CUtensorMap& m0, const CUtensorMap& m1, const KsRowsArgs& A,
                     const KeyTable& keys, cudaStream_t st) {
  if (keys.n == 1) {   // one key: its tensor maps, and no key table in the launch parameters
    run_ks_rows_mac_with<STAGES>(ks_rows_mac_tma_kernel<STAGES, 3, OneKey>, mi, m0, m1, A, OneKey{}, st);
    return;
  }
  run_ks_rows_mac_with<STAGES>(ks_rows_mac_tma_kernel<STAGES, 3, KeyTable>, mi, mi, mi, A, keys, st);
}

}  // namespace

// TMA-fed persistent kernels: the default whenever a launch carries enough polynomials per limb to amortise the
// per-(limb, tile position) twiddle staging; FHE_B200_NTT=fast keeps the register-resident kernels, =tma forces the
// TMA ones for any batch size (tests)
bool ntt_uses_tma(u32 n_rows, const RowIds& ids, u32 logn, u32 in_div, const u64* in, const u64* out) {
  const Switches& sw = switches();
  const u32 lpp = ids.limbs_per_poly;
  if (!sw.tma_allowed() || logn < 13 || logn > 15 || !tensor_map_encoder()) return false;
  if (n_rows % lpp != 0 || (in_div != 1 && in_div != lpp)) return false;
  if ((reinterpret_cast<uintptr_t>(in) | reinterpret_cast<uintptr_t>(out)) & 127) return false;
  return sw.ntt == Switches::NTT_TMA || n_rows / lpp >= 8;
}

bool launch_tensor_inverse_ntt(const u64* a, const u64* b, const u64* xa, const u64* xb, u64* T, u32 cts, u32 L, u32 K,
                               const RowIds& mul_ids, const LimbDev* limbs, u32 logn, cudaStream_t st) {
  if (switches().no_tensor_fusion || K <= L || !ntt_uses_tma(cts * 3 * K, mul_ids, logn, 1, T, T)) return false;
  if ((reinterpret_cast<uintptr_t>(a) | reinterpret_cast<uintptr_t>(b) | reinterpret_cast<uintptr_t>(xa) |
       reinterpret_cast<uintptr_t>(xb)) & 127)
    return false;
  return launch_tensor_intt_tma(a, b, xa, xb, T, cts, L, K, mul_ids, limbs, logn, st);
}

bool launch_key_switch_tma(const u64* c2, u64* inter, const std::vector<KeyRange>& ranges, const u64* base0,
                           const u64* base1, u64* out0, u64* out1, u32 cts, u32 n_dig, u32 Lk, u32 out_ct_rows,
                           const RowIds& ids, const LimbDev* limbs, u32 logn, bool reduce, cudaStream_t st) {
  // ring depth of the digit tiles: 2 (default) or 3 (FHE_B200_KS_STAGES >= 3); both keep 3 CTAs per SM at n_dig = 14
  const int stages = switches().ks_stages >= 3 ? 3 : 2;
  using Cfg = KsRowsCfg<2>;
  const u32 n_rows = cts * n_dig * Lk;
  if (logn < 13 || logn > 15 || !tensor_map_encoder() || ids.limbs_per_poly != Lk || n_dig == 0 || n_dig > 256)
    return false;
  if ((reinterpret_cast<uintptr_t>(c2) | reinterpret_cast<uintptr_t>(inter)) & 127) return false;
  // the key tiles travel as 1 KiB row segments (cp.async.bulk: 16-byte aligned)
  for (const KeyRange& r : ranges)
    for (u32 s = 0; s < r.keys.n; s++)
      if ((reinterpret_cast<uintptr_t>(r.keys.k0[s]) | reinterpret_cast<uintptr_t>(r.keys.k1[s])) & 127) return false;
  if ((stages == 3 ? KsRowsCfg<3>::smem(n_dig) : Cfg::smem(n_dig)) > 227 * 1024) return false;
  try {
    // every tensor map first: a shape the TMA cannot describe launches nothing.  A one-key range reads its key
    // [Lk][n_dig][N] as {128-coefficient, n_dig-row} boxes; a range of several keys copies 1 KiB row segments.
    std::vector<CUtensorMap> mi(ranges.size()), m0(ranges.size()), m1(ranges.size());
    for (size_t r = 0; r < ranges.size(); r++) {
      mi[r] = rows_map(inter + (((size_t)ranges[r].ct0 * n_dig * Lk) << logn), (u64)ranges[r].cts * n_dig * Lk, logn,
                       4 * Cfg::R);
      const KeyTable& K = ranges[r].keys;
      if (K.n == 1 && (!box_map(&m0[r], K.k0[0], (u64)Lk * n_dig, logn, Cfg::TC, n_dig) ||
                       !box_map(&m1[r], K.k1[0], (u64)Lk * n_dig, logn, Cfg::TC, n_dig)))
        return false;
    }
    // digit broadcast + large-stride stages: inter [ct][j][d][N] (in_bcast: the source row of polynomial (ct, d) is
    // row ct*n_dig + d of c2 for every limb j)
    NttTmaArgs C;
    std::memset(&C, 0, sizeof(C));
    C.limbs = limbs;
    C.n_polys = cts * n_dig;
    C.lpp = Lk;
    C.in_bcast = C.limb_inner = 1;
    C.digit_adjacent = 1;
    C.n_dig = n_dig;
    C.reduce_on_load = reduce ? 1 : 0;
    C.logn = logn;
    for (int i = 0; i < kMaxPos; i++) C.ids[i] = ids.ids[i];
    run_tma_cols_for<false>(c2, (u64)cts * n_dig, inter, n_rows, C, st);
    // the rows pass fused with the inner product, one launch per key range over the same transformed digits
    KsRowsArgs A;
    std::memset(&A, 0, sizeof(A));
    A.limbs = limbs;
    A.n_dig = n_dig; A.Lk = Lk; A.out_ct_rows = out_ct_rows; A.logn = logn;
    A.tiles_per_row = (1u << logn) / Cfg::TC;
    for (int i = 0; i < kMaxPos; i++) A.ids[i] = ids.ids[i];
    for (size_t r = 0; r < ranges.size(); r++) {
      const size_t o = ((size_t)ranges[r].ct0 * out_ct_rows) << logn;
      A.base0 = base0 ? base0 + o : nullptr; A.base1 = base1 ? base1 + o : nullptr;
      A.out0 = out0 + o; A.out1 = out1 + o;
      A.cts = ranges[r].cts;
      A.items_total = Lk * A.tiles_per_row * A.cts;
      if (stages == 3) run_ks_rows_mac<3>(mi[r], m0[r], m1[r], A, ranges[r].keys, st);
      else run_ks_rows_mac<2>(mi[r], m0[r], m1[r], A, ranges[r].keys, st);
    }
  } catch (const TmaFail&) {
    return false;
  }
  return true;
}

void launch_ntt(const u64* in, u64* out, u32 n_rows, const RowIds& ids, const LimbDev* limbs, u32 logn,
                bool inverse, u32 in_div, bool reduce_on_load, cudaStream_t st, bool lazy_out, bool digit_adjacent,
                u32 n_dig) {
  if (n_rows == 0) return;
  g_ntt_rows[inverse ? 1 : 0].fetch_add(n_rows, std::memory_order_relaxed);
  NttArgs a;
  a.in = in;
  a.out = out;
  a.limbs = limbs;
  a.n_rows = n_rows;
  a.limbs_per_poly = ids.limbs_per_poly;
  a.in_div = in_div;
  a.reduce_on_load = reduce_on_load ? 1 : 0;
  a.lazy_out = (lazy_out && !inverse) ? 1 : 0;
  a.logn = logn;
  for (int i = 0; i < kMaxPos; i++) a.ids[i] = ids.ids[i];
  if (logn <= 12) {
    a.logn1 = 0;
    if (inverse) run_single<true>(a, st); else run_single<false>(a, st);
    return;
  }
  // two passes: N2 = 64 contiguous points (rows kernel), N1 = N / 64 (cols kernel)
  a.logn1 = logn - 6;
  NttArgs second = a;  // second pass runs in place on `out`
  second.in = out;
  second.in_div = 1;
  second.reduce_on_load = 0;
  if (ntt_uses_tma(n_rows, ids, logn, in_div, in, out) &&
      launch_ntt_tma(in, out, n_rows, ids, limbs, logn, inverse, in_div, reduce_on_load, st, lazy_out, digit_adjacent,
                     n_dig))
    return;
  if (digit_adjacent) throw CudaFail{cudaErrorNotSupported, "digit-adjacent NTT output needs the TMA kernels"};
  // the register-resident kernels carry the Shoup butterflies only (the Solinas form measured no faster and doubled
  // their code size); FHE_B200_SOLINAS_NTT therefore selects the generic tile kernels, which keep both
  if (switches().generic_tiles()) {
    if (!inverse) {
      run_cols_for<false>(a, st);
      run_rows<6, 6, false>(second, st);
    } else {
      run_rows<6, 6, true>(a, st);
      run_cols_for<true>(second, st);
    }
    return;
  }
  // Tile sizes: 1024-word rows tiles, 2048-word cols tiles.  Smaller CTAs (same 8 words and <= 64 registers per
  // thread, so the same number of resident warps) put more independent CTAs on an SM; their load / butterfly /
  // exchange phases interleave and the multiplier pipe idles less (1024-word cols tiles would mean 16-byte column
  // segments at N = 2^15).
  if (!inverse) {
    run_fast_cols_for<false>(a, st);
    run_fast<6, false, false, 10>(second, st);
  } else {
    run_fast<6, false, true, 10>(a, st);
    run_fast_cols_for<true>(second, st);
  }
}

}  // namespace fhe_b200
