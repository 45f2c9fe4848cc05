// C ABI of the engine (include/fhe_b200.h): parameter precompute + upload, device batches,
// key material, and the batched homomorphic operations built from the kernels of
// ntt.cu / kernels.cu.  No CPU fallback: compute entry points require a CUDA device.
#include <algorithm>
#include <atomic>
#include <cstring>
#include <functional>
#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <vector>

#include "../../include/fhe_b200.h"
#include "engine.hpp"
#include "host/precompute.hpp"

using namespace fhe_b200;

namespace {

thread_local std::string g_last_error;

struct ScalerData {
  ScalerTablesH h;
  ScalerDev dev;
};

struct LevelData {
  u32 level = 0, L = 0, E = 0, K = 0;
  RowIds ctx_ids, mul_ids;
  RowIds ext_ids;                       // the E extension limbs of the multiplication basis
  std::vector<u64> mul_moduli;
  u64 q_min = 0, q_max = 0;             // of the level's moduli
  // a lift of plaintext words (< t) onto the level's limbs needs the reduction on load of the forward transform,
  // whose butterflies take inputs below 4 q_j: t > 4 q_min - 1
  bool lift_reduce = false;
  ScalerData ext, down;
  bool has_sd = false;
  SwitchDownDev sd;
  // CipherPlainContext (parameters.rs:604-643): Q_level mod t (when t fits a Modulus), delta = (-t)^-1 mod q_i and
  // the scaler from the level's basis to the plaintext context by t / Q_level
  u64 q_mod_t = 0;
  std::vector<u64> delta;
  const u64 *d_delta = nullptr, *d_delta_s = nullptr;
  ScalerData plain;
  // noise measurement: garner [L][L] with (i, j < i) = q_j^-1 mod q_i, and Q_level as W little-endian 64-bit words
  const u64* garner = nullptr;
  const u64* q_words = nullptr;
  u32 W = 0;
};

// Selects a device for the lifetime of the guard and puts the caller's device back afterwards.  Create and compute
// paths check (`check`): a failed cudaSetDevice throws, and the guard of a parameter set refuses one made without a
// device with NO_DEVICE before it selects anything.  Release paths never throw and leave no error behind.
struct DeviceGuard {
  int prev = -1;
  const bool check;
  DeviceGuard(int device, bool check_) : check(check_) {
    if (device < 0) return;
    if (cudaGetDevice(&prev) != cudaSuccess) { cudaGetLastError(); prev = -1; }
    if (prev == device) prev = -1;
    else if (check) FHE_CUDA(cudaSetDevice(device));
    else cudaSetDevice(device);
    if (!check) cudaGetLastError();
  }
  explicit DeviceGuard(const fhe_b200_params* p);
  ~DeviceGuard() {
    if (prev >= 0) cudaSetDevice(prev);
    if (!check) cudaGetLastError();
  }
  DeviceGuard(const DeviceGuard&) = delete;
  DeviceGuard& operator=(const DeviceGuard&) = delete;
};

// The owner of a handle's immutable device tables: `put` uploads a vector on the owner's device and keeps the
// allocation until the owner goes.  Not thread-safe: the parameter set calls put only while it holds its mutex (the
// lazy tables of level() and expansion_monomial_dev()); the other owners fill theirs before their handle is
// handed out.
class DeviceTables {
 public:
  explicit DeviceTables(int device) : device_(device) {}
  DeviceTables(const DeviceTables&) = delete;
  DeviceTables& operator=(const DeviceTables&) = delete;
  ~DeviceTables() {
    if (allocs_.empty()) return;
    DeviceGuard g(device_, false);
    for (void* d : allocs_) cudaFree(d);
  }
  // nullptr for an empty vector or a host-only parameter set (device < 0)
  template <typename T>
  T* put(const std::vector<T>& v) {
    if (device_ < 0 || v.empty()) return nullptr;
    DeviceGuard g(device_, true);   // tables are built lazily, possibly from a thread on another device
    T* d = nullptr;
    FHE_CUDA(cudaMalloc(&d, v.size() * sizeof(T)));
    allocs_.push_back(d);
    FHE_CUDA(cudaMemcpy(d, v.data(), v.size() * sizeof(T), cudaMemcpyHostToDevice));
    return d;
  }

 private:
  const int device_;
  std::vector<void*> allocs_;
};

// the slot of prime q in a limb table, -1 when it has none
int prime_index(const std::vector<u64>& primes, u64 q) {
  for (size_t i = 0; i < primes.size(); i++)
    if (primes[i] == q) return (int)i;
  return -1;
}

// Device copy of one RnsScaler's tables (rns/scaler.rs:79-175), owned by `tables`.  `limb_primes` are the primes of the
// limb table the kernels will be given, in which every modulus of the `to` basis has its slot.
void upload_scaler_tables(ScalerData& s, const std::vector<u64>& to_moduli, const std::vector<u64>& limb_primes,
                          DeviceTables& tables) {
  ScalerDev& d = s.dev;
  std::memset(&d, 0, sizeof(d));
  d.n_from = s.h.n_from; d.n_to = s.h.n_to; d.is_one = s.h.is_one; d.shift = s.h.shift;
  d.tg_lo = s.h.theta_gamma_lo; d.tg_hi = s.h.theta_gamma_hi; d.tg_sign = s.h.theta_gamma_sign;
  for (size_t j = 0; j < to_moduli.size(); j++) d.to_ids[j] = (unsigned short)prime_index(limb_primes, to_moduli[j]);
  d.all_solinas = switches().no_solinas ? 0 : 1;
  for (u64 q : to_moduli)
    if ((q >> 61) != 1 || ((1ull << 62) - q) >= (1ull << 28)) d.all_solinas = 0;
  d.gamma = tables.put(s.h.gamma);
  d.omega = tables.put(s.h.omega);
  d.to_lo = tables.put(s.h.theta_omega_lo);
  d.to_hi = tables.put(s.h.theta_omega_hi);
  d.to_sign = tables.put(s.h.theta_omega_sign);
  // source indices of the theta_omega terms, positive sign first (the kernel makes one pass per sign).  Terms whose
  // fractional part is exactly zero add nothing (rns/scaler.rs:282-298 multiplies them by zero) and are left out:
  // in the down scaler of the multiplication basis that is every extension limb (garner_i * t / Q is an integer).
  std::vector<unsigned char> order;
  d.n_pos = 0;
  for (int sg = 0; sg < 2; sg++)
    for (size_t i = 0; i < s.h.theta_omega_sign.size(); i++)
      if ((int)s.h.theta_omega_sign[i] == sg && (s.h.theta_omega_lo[i] | s.h.theta_omega_hi[i]) != 0) {
        order.push_back((unsigned char)i);
        d.n_pos += sg == 0;
      }
  d.n_terms = (u32)order.size();
  if (order.empty()) order.push_back(0);   // keep the table non-empty (never read: n_terms == 0)
  d.to_order = tables.put(order);
  d.tgar_lo = tables.put(s.h.theta_garner_lo);
  d.tgar_hi = tables.put(s.h.theta_garner_hi);
}

// Per-prime device constants and twiddle tables (NttOperator::new, ntt/native.rs:35-73, as (value, companion) pairs).
LimbDev make_limb_dev(u64 q, const NttTablesH& t, DeviceTables& tables) {
  ModulusH m(q);
  LimbDev d;
  std::memset(&d, 0, sizeof(d));
  d.p = q; d.p2 = 2 * q; d.bhi = m.bhi; d.blo = m.blo; d.c128 = m.c128;
  d.ninv = t.ninv; d.zn = t.zn;
  // limb mode: p = 2^62 - c with c < 2^28 takes the Solinas constant-multiplication form
  const u64 cc = (1ull << 62) - q;
  const bool sol = (q >> 61) == 1 && cc < (1ull << 28) && !switches().no_solinas;
  // NTT butterflies: Shoup pairs by default (no Solinas instruction selection timed in bench_micro/bf_bench.cu beat
  // them); FHE_B200_SOLINAS_NTT=1 selects the (w, w*2^32 mod p) pairs instead
  const bool sol_ntt = switches().solinas_ntt;
  auto pairs = [&](const std::vector<u64>& v, const std::vector<u64>& shoup) {
    std::vector<ulonglong2> o(v.size());
    for (size_t k = 0; k < v.size(); k++) {
      o[k].x = v[k];
      o[k].y = (sol && sol_ntt) ? (u64)((((u128)v[k]) << 32) % q) : shoup[k];
    }
    return o;
  };
  d.sol_c = sol ? cc : 0;
  d.sol_ntt = (sol && sol_ntt) ? 1 : 0;
  d.ninv_s = (sol && sol_ntt) ? (u64)((((u128)t.ninv) << 32) % q) : t.ninv_s;
  d.zn_s = (sol && sol_ntt) ? (u64)((((u128)t.zn) << 32) % q) : t.zn_s;
  d.om = tables.put(pairs(t.om, t.om_s));
  d.zi = tables.put(pairs(t.zi, t.zi_s));
  return d;
}

}  // namespace

struct fhe_b200_params {
  // Arc-like lifetime (the reference shares Arc<BfvParameters>): batches and keys hold a
  // reference, so the tables outlive every handle that points at them regardless of the order
  // in which a garbage-collected host releases its objects.
  std::atomic<int> refs{1};
  const int device;
  u32 N = 0, logn = 0, Lmax = 0;
  std::vector<u64> moduli, ext, primes, psi;
  std::vector<u32> moduli_sizes;
  BigUint t;
  bool t_small = false;            // BfvParameters::plaintext.small(): t is a zq::Modulus (2 <= t < 2^62)
  PlainMod t_mod{0, 0, 0};
  std::vector<NttTablesH> tables;  // host copies (kept for inspection / host-only handles)
  std::vector<LimbDev> h_limbs;
  LimbDev* d_limbs = nullptr;
  mutable DeviceTables uploads;
  // scratch of the batched operations comes from a stream-ordered pool this parameter set owns (the device's default
  // pool, which a host application may be using for its own cudaMallocAsync calls, is left untouched)
  cudaMemPool_t pool = nullptr;
  // side streams over which ChunkRunner deals the chunks of one batched call (created on first use)
  mutable cudaStream_t side[4] = {nullptr, nullptr, nullptr, nullptr};
  mutable std::mutex mu;
  mutable std::map<u32, std::unique_ptr<LevelData>> levels;

  explicit fhe_b200_params(int dev) : device(dev), uploads(dev) {}

  // the plaintext context: the first moduli whose sizes add up to bits(t) + 60 (parameters.rs:579-595)
  u32 plaintext_moduli_count() const {
    const size_t t_bits = t.bits();
    u32 pc = 0, acc = 0;
    for (u32 sz : moduli_sizes) {
      acc += sz;
      pc++;
      if (acc >= t_bits + 60) break;
    }
    return std::min(std::max(pc, 1u), Lmax);
  }

  // ContextLevel + MultiplicationParameters of one level (bfv/parameters.rs:600-700, :793-813)
  const LevelData& level(u32 lv) const {
    std::lock_guard<std::mutex> g(mu);
    auto it = levels.find(lv);
    if (it != levels.end()) return *it->second;
    if (lv >= Lmax) throw FheError(FHE_B200_INVALID_LEVEL, "InvalidLevel: level " + std::to_string(lv));
    std::unique_ptr<LevelData> d(new LevelData());
    d->level = lv;
    d->L = Lmax - lv;
    u32 bits = 0;
    for (u32 i = 0; i < d->L; i++) bits += moduli_sizes[i];
    d->E = (bits + 60 + 61) / 62;  // (modulus_size + 60).div_ceil(62), parameters.rs:689
    d->K = d->L + d->E;
    if (d->K > (u32)kMaxPos) throw FheError(FHE_B200_UNSUPPORTED, "too many limbs");
    std::vector<u64> ctx(moduli.begin(), moduli.begin() + d->L);
    d->mul_moduli = ctx;
    d->mul_moduli.insert(d->mul_moduli.end(), ext.begin(), ext.begin() + d->E);
    std::memset(&d->ctx_ids, 0, sizeof(RowIds));
    std::memset(&d->mul_ids, 0, sizeof(RowIds));
    std::memset(&d->ext_ids, 0, sizeof(RowIds));
    d->ctx_ids.limbs_per_poly = d->L;
    d->mul_ids.limbs_per_poly = d->K;
    d->ext_ids.limbs_per_poly = d->E;
    for (u32 i = 0; i < d->L; i++) d->ctx_ids.ids[i] = d->mul_ids.ids[i] = (unsigned short)i;
    for (u32 j = 0; j < d->E; j++) d->mul_ids.ids[d->L + j] = d->ext_ids.ids[j] = (unsigned short)(Lmax + j);
    d->q_min = *std::min_element(ctx.begin(), ctx.end());
    d->q_max = *std::max_element(ctx.begin(), ctx.end());
    d->lift_reduce = t_mod.t > 4 * d->q_min - 1;
    RnsContextH from(ctx), to(d->mul_moduli);
    d->ext.h = make_scaler_tables(from, to, BigUint(1), BigUint(1));
    d->down.h = make_scaler_tables(to, from, t, from.product);
    upload_scaler_tables(d->ext, d->mul_moduli, primes, uploads);
    upload_scaler_tables(d->down, ctx, primes, uploads);
    if (d->L >= 2) {  // rq/context.rs:65-71 and rq/mod.rs:444-468
      d->has_sd = true;
      u64 ql = ctx.back();
      std::vector<u64> half_mod, inv, inv_s;
      for (u32 i = 0; i + 1 < d->L; i++) {
        u64 qi = ctx[i], iv;
        if (!invmod_h(ql % qi, qi, &iv)) throw FheError(FHE_B200_INVALID_MODULUS, "NonCoprimeModuli");
        half_mod.push_back(qi - (ql / 2) % qi);
        inv.push_back(iv);
        inv_s.push_back(ModulusH(qi).shoup(iv));
      }
      d->sd.q_last = ql;
      d->sd.q_last_half = ql / 2;
      d->sd.half_mod = uploads.put(half_mod);
      d->sd.inv = uploads.put(inv);
      d->sd.inv_s = uploads.put(inv_s);
    }
    if (t_small) d->q_mod_t = from.product.mod_u64(t_mod.t);
    std::vector<u64> delta_s;
    for (u64 qi : ctx) {
      u64 iv;
      if (!invmod_h(qi - t.mod_u64(qi), qi, &iv)) throw FheError(FHE_B200_INVALID_MODULUS, "PlaintextModulusNotCoprime");
      d->delta.push_back(iv);
      delta_s.push_back(ModulusH(qi).shoup(iv));
    }
    d->d_delta = uploads.put(d->delta);
    d->d_delta_s = uploads.put(delta_s);
    const std::vector<u64> plain(moduli.begin(), moduli.begin() + plaintext_moduli_count());
    d->plain.h = make_scaler_tables(from, RnsContextH(plain), t, from.product);   // parameters.rs:638-643
    upload_scaler_tables(d->plain, plain, primes, uploads);
    std::vector<u64> garner((size_t)d->L * d->L, 0);
    for (u32 i = 0; i < d->L; i++)
      for (u32 j = 0; j < i; j++)
        if (!invmod_h(ctx[j] % ctx[i], ctx[i], &garner[(size_t)i * d->L + j]))
          throw FheError(FHE_B200_INVALID_MODULUS, "NonCoprimeModuli");
    d->garner = uploads.put(garner);
    std::vector<u64> qw;
    const BigUint& Q = from.product;
    for (size_t k = 0; k < Q.w.size(); k += 2)
      qw.push_back((u64)Q.w[k] | (k + 1 < Q.w.size() ? (u64)Q.w[k + 1] << 32 : 0));
    d->W = (u32)qw.size();
    d->q_words = uploads.put(qw);
    auto* raw = d.get();
    levels[lv] = std::move(d);
    return *raw;
  }

  // The expansion monomial -x^(N - 2^l) of EvaluationKey (evaluation_key.rs:465-474) at level `lv`, NTT words [L][N].
  // The forward NTT evaluates at psi^(2 bitrev(i) + 1) and psi^N = -1, so -z^(N - 2^l) = z^(-2^l) at every point z:
  // word i of limb q is psi_q^(-(2^l) (2 bitrev(i) + 1) mod 2N).  l < log2 N.
  std::vector<u64> expansion_monomial(u32 lv, u32 l) const {
    const u32 L = level(lv).L;
    const u64 m = 2 * (u64)N;
    std::vector<u64> out((size_t)L * N), pw(m);
    for (u32 j = 0; j < L; j++) {
      const u64 q = moduli[j];
      pw[0] = 1;
      for (u64 k = 1; k < m; k++) pw[k] = mulmod_h(pw[k - 1], psi[j], q);
      for (u32 i = 0; i < N; i++) {
        u32 r = 0;
        for (u32 b = 0; b < logn; b++) r |= ((i >> b) & 1) << (logn - 1 - b);
        const u64 e = (((u64)(2 * r + 1)) << l) % m;
        out[(size_t)j * N + i] = pw[(m - e) % m];
      }
    }
    return out;
  }
  // the same as (value, Shoup companion) pairs on the device, built on first use per (level, l)
  const ulonglong2* expansion_monomial_dev(u32 lv, u32 l) const {
    {
      std::lock_guard<std::mutex> g(mu);
      auto it = monos.find({lv, l});
      if (it != monos.end()) return it->second;
    }
    const std::vector<u64> w = expansion_monomial(lv, l);   // level() takes the mutex itself
    std::lock_guard<std::mutex> g(mu);
    auto it = monos.find({lv, l});
    if (it != monos.end()) return it->second;
    std::vector<ulonglong2> pairs(w.size());
    for (size_t j = 0; j < w.size() / N; j++) {
      const ModulusH mq(moduli[j]);
      for (size_t k = j * N; k < (j + 1) * N; k++) {
        pairs[k].x = w[k];
        pairs[k].y = mq.shoup(w[k]);
      }
    }
    const ulonglong2* d = uploads.put(pairs);
    monos[{lv, l}] = d;
    return d;
  }
  mutable std::map<std::pair<u32, u32>, const ulonglong2*> monos;
};

namespace {

void params_release(const fhe_b200_params* cp) {
  fhe_b200_params* p = const_cast<fhe_b200_params*>(cp);
  if (!p || p->refs.fetch_sub(1) != 1) return;
  if (p->device >= 0) {
    DeviceGuard g(p->device, false);
    for (cudaStream_t ss : p->side)
      if (ss) cudaStreamDestroy(ss);
    if (p->pool) {
      cudaDeviceSynchronize();   // scratch freed with cudaFreeAsync must have retired before its pool goes away
      cudaMemPoolDestroy(p->pool);
    }
  }
  delete p;   // its device tables go with it
}
const fhe_b200_params* params_retain(const fhe_b200_params* p) {
  const_cast<fhe_b200_params*>(p)->refs.fetch_add(1);
  return p;
}

// A handle's reference on its parameter set (fhe_b200_params::refs): retained when the handle is made, released when
// it goes.  Every handle declares it first, so that its other members, device memory included, are released while the
// set and its device are still there.
class ParamsRef {
 public:
  explicit ParamsRef(const fhe_b200_params* p) : p_(params_retain(p)) {}
  ~ParamsRef() { params_release(p_); }
  ParamsRef(const ParamsRef&) = delete;
  ParamsRef& operator=(const ParamsRef&) = delete;
  operator const fhe_b200_params*() const { return p_; }
  const fhe_b200_params* operator->() const { return p_; }

 private:
  const fhe_b200_params* const p_;
};

// Device words derived from a secret (SecretKey's s, the relinearization-key generator's u), erased before they are
// freed as SecretKey's Zeroize erases s (secret_key.rs:28-40).  Work that reads the words may still be queued on
// streams that do not order against the legacy stream the memset runs on (the chunk runner's side streams, a caller's
// non-blocking stream): the release waits for the device first, as cudaFree would, so that releasing the handle right
// after an enqueue-only call is as safe as releasing any other handle.
struct SecretBuffer {
  const int device;
  const size_t bytes;
  u64* d = nullptr;
  SecretBuffer(int dev, size_t words) : device(dev), bytes(words * sizeof(u64)) { FHE_CUDA(cudaMalloc(&d, bytes)); }
  ~SecretBuffer() {
    DeviceGuard g(device, false);
    cudaDeviceSynchronize();
    cudaMemset(d, 0, bytes);
    cudaDeviceSynchronize();
    cudaFree(d);
  }
  SecretBuffer(const SecretBuffer&) = delete;
  SecretBuffer& operator=(const SecretBuffer&) = delete;
};

}  // namespace

DeviceGuard::DeviceGuard(const fhe_b200_params* p) : DeviceGuard(p->device, true) {
  if (p->device < 0) throw FheError(FHE_B200_NO_DEVICE, "parameter set was created without a CUDA device");
}

struct fhe_b200_batch {
  ParamsRef par;
  u32 count = 0, parts = 0, level = 0, limbs = 0;
  int repr = 0;
  bool mul_basis = false;
  u64* d = nullptr;
  explicit fhe_b200_batch(const fhe_b200_params* p) : par(p) {}
  ~fhe_b200_batch() {
    DeviceGuard g(par->device, false);
    cudaFree(d);
  }
  size_t words_per_ct() const { return ((size_t)parts * limbs) << par->logn; }
};

struct fhe_b200_ksk {
  ParamsRef par;
  u32 ct_level = 0, ksk_level = 0, n_dig = 0, Lk = 0;
  u32 log_base = 0;   // 0: RNS-digit variant; else base-2^log_base decomposition (single-modulus key level)
  u64 *k0 = nullptr, *k1 = nullptr;
  explicit fhe_b200_ksk(const fhe_b200_params* p) : par(p) {}
  ~fhe_b200_ksk() {
    DeviceGuard g(par->device, false);
    cudaFree(k0);
    cudaFree(k1);
  }
};

// Multiplicator::new / new_leveled (bfv/ops/mul.rs:37-98): custom scaling factors and extended basis.
struct fhe_b200_multiplicator {
  ParamsRef par;
  u32 level = 0, L = 0, K = 0;
  u32 nc_l = 0, nc_r = 0, nc_d = 0;     // Scaler::number_common_moduli of the two extenders and the down scaler
  std::vector<u64> mul_moduli, plan_primes;
  RowIds mul_ids;
  std::vector<LimbDev> h_limbs;          // the parameter set's limbs followed by the primes only this basis has
  LimbDev* d_limbs = nullptr;
  ScalerData ext_l, ext_r, down;
  DeviceTables uploads;
  explicit fhe_b200_multiplicator(const fhe_b200_params* p) : par(p), uploads(p->device) {}
};

// The plaintext side of BfvParameters: the NTT operator of t (parameters.rs:71-75, :598) and the SIMD slot map
// (matrix_reps_index_map, :713-726).  Its limb table is the parameter set's followed by t, so the level RowIds of
// the parameter set index it unchanged.
struct fhe_b200_encoder {
  ParamsRef par;
  bool has_ntt = false;                 // NttOperator::new(t) is Some (ntt/native.rs:35-73)
  u64 psi_t = 0;
  NttTablesH tables;                    // of t, when has_ntt
  std::vector<u32> index_map;           // slot i -> coefficient index
  std::vector<LimbDev> h_limbs;
  LimbDev* d_limbs = nullptr;
  u32* d_inv_map = nullptr;             // coefficient index -> slot
  int* d_index_map = nullptr;           // index_map on the device (the decoders' gather)
  RowIds t_ids;                         // one row per plaintext, all modulo t
  DeviceTables uploads;
  explicit fhe_b200_encoder(const fhe_b200_params* p) : par(p), uploads(p->device) {}
};

// SecretKey (keys/secret_key.rs:25-53) on the device: s as NTT words modulo every modulus of the parameter set (the
// context of level l is the prefix moduli[..L-l], so every level reads a prefix of the same rows).  The tables that
// decryption and noise measurement read are the level's (LevelData).
struct fhe_b200_secret_key {
  ParamsRef par;
  SecretBuffer s;                       // [n_moduli][N]
  explicit fhe_b200_secret_key(const fhe_b200_params* p) : par(p), s(p->device, (size_t)p->Lmax * p->N) {}
};

namespace {

// stream-ordered scratch memory from the parameter set's own pool
struct Workspace {
  cudaStream_t st;
  cudaMemPool_t pool;
  std::vector<void*> ptrs;
  std::vector<std::pair<void*, size_t>> secret;
  Workspace(const fhe_b200_params* par, cudaStream_t s) : st(s), pool(par->pool) {}
  u64* words(size_t n) {
    void* p = nullptr;
    FHE_CUDA(cudaMallocFromPoolAsync(&p, n * sizeof(u64), pool, st));
    ptrs.push_back(p);
    return (u64*)p;
  }
  // scratch that will hold values derived from a secret key: zeroed on the stream before it goes back to the pool
  u64* secret_words(size_t n) {
    u64* p = words(n);
    secret.emplace_back(p, n * sizeof(u64));
    return p;
  }
  ~Workspace() {
    for (auto& s : secret) cudaMemsetAsync(s.first, 0, s.second, st);
    for (void* p : ptrs) cudaFreeAsync(p, st);
  }
};

u32 chunk_size() { return switches().chunk; }

// A batched call works through its ciphertexts chunk by chunk.  On ONE stream every kernel boundary costs the tail of
// one persistent grid plus the ring fill and table staging of the next, 18 boundaries per chunk.
// When a call has more than one chunk the runner therefore deals the chunks over side streams of the parameter set
// (two by default, FHE_B200_STREAMS=1..4): the kernels of one chunk fill the SMs that the kernels of another leave at
// their boundaries, and kernels bound by different resources (integer pipe, HBM) share an SM.  The caller's stream is the
// only one it ever sees: the side streams start behind an event recorded on it and it waits for all of them before the
// call returns.  Each side stream works on chunks of chunk_size() / streams ciphertexts, so the scratch in flight is what
// one full chunk takes.  FHE_B200_STREAMS=1 keeps everything on the caller's stream.
struct ChunkRunner {
  const fhe_b200_params* par;
  cudaStream_t user;
  u32 count, chunk, ns;
  cudaEvent_t ev[5] = {nullptr, nullptr, nullptr, nullptr, nullptr};
  static u32 streams() { return switches().streams; }
  // items_per_chunk: 0 for chunk_size() ciphertexts; a call whose items are larger than a ciphertext passes its own
  ChunkRunner(const fhe_b200_params* p, u32 n, cudaStream_t st, u32 items_per_chunk = 0)
      : par(p), user(st), count(n), chunk(items_per_chunk ? items_per_chunk : chunk_size()), ns(1) {
    if (streams() < 2 || count <= chunk || chunk < streams()) return;
    ns = streams();
    chunk = (chunk + ns - 1) / ns;
    {
      std::lock_guard<std::mutex> g(par->mu);
      for (u32 i = 0; i < ns; i++)
        if (!par->side[i]) FHE_CUDA(cudaStreamCreateWithFlags(&par->side[i], cudaStreamNonBlocking));
    }
    for (u32 i = 0; i <= ns; i++) FHE_CUDA(cudaEventCreateWithFlags(&ev[i], cudaEventDisableTiming));
    FHE_CUDA(cudaEventRecord(ev[ns], user));
    for (u32 i = 0; i < ns; i++) FHE_CUDA(cudaStreamWaitEvent(par->side[i], ev[ns], 0));
  }
  // body(first ciphertext, number of ciphertexts, stream)
  template <class F>
  void run(F&& body) {
    u32 k = 0;
    for (u32 c0 = 0; c0 < count; c0 += chunk, k++) body(c0, std::min(chunk, count - c0), ns > 1 ? par->side[k % ns] : user);
    join();
  }
  void join() {
    if (ns < 2 || joined) return;
    joined = true;
    for (u32 i = 0; i < ns; i++)
      if (cudaEventRecord(ev[i], par->side[i]) == cudaSuccess) cudaStreamWaitEvent(user, ev[i], 0);
  }
  ~ChunkRunner() {
    join();                         // also when a chunk failed half way: the caller's stream still has to wait
    for (cudaEvent_t e : ev)
      if (e) cudaEventDestroy(e);   // released once the recorded work has completed
  }
  bool joined = false;
};

void check_same(const fhe_b200_batch* a, const fhe_b200_batch* b) {
  if (a->par != b->par) throw FheError(FHE_B200_CONTEXT_MISMATCH, "ParameterMismatch: batches use different parameters");
  if (a->level != b->level) throw FheError(FHE_B200_INVALID_LEVEL, "InvalidLevel: operands are at different levels");
  if (a->mul_basis != b->mul_basis || a->limbs != b->limbs)
    throw FheError(FHE_B200_CONTEXT_MISMATCH, "PolynomialContextMismatch");
}
void need_repr(const fhe_b200_batch* b, int repr) {
  if (b->repr != repr) throw FheError(FHE_B200_INVALID_REPRESENTATION, "IncorrectRepresentation");
}
const RowIds& ids_of(const fhe_b200_batch* b) {
  const LevelData& lv = b->par->level(b->level);
  return b->mul_basis ? lv.mul_ids : lv.ctx_ids;
}

// Ciphertext::switch_down of `polys` NTT polynomials at `level` (L >= 2), in place: d [polys][L][N] becomes
// [polys][L-1][N], compacted at the start of the same buffer
void switch_down_polys(const fhe_b200_params* par, u32 level, u64* d, u32 polys, Workspace& ws, cudaStream_t st) {
  const LevelData& lv = par->level(level);
  const LevelData& nl = par->level(level + 1);
  u64* tmp = ws.words((size_t)polys * nl.L << par->logn);
  launch_ntt(d, d, polys * lv.L, lv.ctx_ids, par->d_limbs, par->logn, true, 1, false, st);
  launch_switch_down(lv.sd, d, tmp, polys, lv.L, lv.ctx_ids, par->d_limbs, par->logn, st);
  launch_ntt(tmp, d, polys * nl.L, nl.ctx_ids, par->d_limbs, par->logn, false, 1, false, st);
}

// The keys of a key switch: ciphertext c of the call uses keys[index[c]], or keys[0] when index is null (the
// single-key entry points).  Every key has the levels, digit count and base of keys[0] (check_keys).  A Galois call
// also gives each key's exponent (reduced mod 2N) and may name each output's source ciphertext.
struct KeySet {
  const fhe_b200_ksk* const* keys;
  u32 n;
  const u32* index;            // host memory, one entry per ciphertext; nullable
  const u32* exps = nullptr;   // Galois calls: exps[k] is the exponent of keys[k]
  const u32* source = nullptr; // Galois calls, host memory, one entry per output; nullable (output c reads input c)
  // the same keys for the ciphertexts from c0 on
  KeySet from(u32 c0) const { return {keys, n, index ? index + c0 : nullptr, exps, source ? source + c0 : nullptr}; }
  u32 key_of(u32 c) const { return index ? index[c] : 0; }
};

// The inner-product launches of `cts` ciphertexts: consecutive ranges of at most kKeyPairs distinct keys (a handle
// listed twice is one key) and, once a range holds two keys, at most kKeySlots ciphertexts.  One key: one range.
std::vector<KeyRange> key_ranges(const KeySet& K, u32 cts) {
  std::vector<KeyRange> out;
  KeyRange* r = nullptr;
  for (u32 c = 0; c < cts; c++) {
    const fhe_b200_ksk* k = K.keys[K.index ? K.index[c] : 0];
    u32 s = 0;
    if (r) {
      while (s < r->keys.n && r->keys.k0[s] != k->k0) s++;
      const u32 n_after = r->keys.n + (s == r->keys.n);
      if (n_after > kKeyPairs || (n_after > 1 && r->cts >= kKeySlots)) r = nullptr;
    }
    if (!r) {
      out.emplace_back();
      r = &out.back();
      std::memset(r, 0, sizeof(KeyRange));
      r->ct0 = c;
      s = 0;
    }
    if (s == r->keys.n) {
      r->keys.k0[s] = k->k0;
      r->keys.k1[s] = k->k1;
      r->keys.n++;
    }
    if (r->cts < kKeySlots) r->keys.slot[r->cts] = (unsigned char)s;
    r->cts++;
  }
  return out;
}

// Whether the digit transforms reduce their input on load.  The reference lazily reduces the digit modulo q_j before
// its lazy transform; the forward butterflies accept any input below 4*q_j, so the reduction on load is only needed
// when a digit (< max q_i) can reach 4 * min q_j (mixed modulus sizes).  The digits are those of the ciphertext level
// (n_dig = its L), the rows those of the key level.
bool digit_reduce(const fhe_b200_params* par, const fhe_b200_ksk* k) {
  const u64 qmax = par->level(k->ct_level).q_max, qmin = par->level(k->ksk_level).q_min;
  // The lifts of plaintext words (LevelData::lift_reduce) test only t > 4 * q_min - 1: the butterflies take [0, 4p)
  // for any modulus, down to q_min = 193 < 2^8 (tests/test_gpu_client_edges.py).  The extra clause here changes the
  // choice only when every modulus of the key level is below 2^10, which needs N <= 64.
  return qmax > 4 * qmin - 1 || qmin < (1ull << 8);
}

// KeySwitchingKey::key_switch core on a contiguous power-basis buffer c2 [cts][L][N]
// (key_switching_key.rs:241-270): out0/out1 (+ optional bases), rows (ct, j) at (ct*out_ct_rows + j).  The digit
// transforms do not depend on the key; the inner product runs once per key range (key_ranges).
void key_switch_core(const fhe_b200_params* par, const KeySet& K, const u64* c2, u32 cts, const u64* base0,
                     const u64* base1, u64* out0, u64* out1, u32 out_ct_rows, Workspace& ws, cudaStream_t st) {
  const fhe_b200_ksk* k = K.keys[0];
  const std::vector<KeyRange> ranges = key_ranges(K, cts);
  const LevelData& kl = par->level(k->ksk_level);
  const u32 L = k->n_dig, Lk = k->Lk;
  u64* inter = ws.words(((size_t)cts * L * Lk) << par->logn);
  bool adjacent = false;
  if (k->log_base) {
    // key_switch_decomposition (key_switching_key.rs:323-362): the digits of the single residue, each below
    // 2^log_base < q, transformed lazily like the RNS digits
    u64* dig = ws.words(((size_t)cts * L) << par->logn);
    launch_decompose(c2, dig, cts, L, k->log_base, par->logn, st);
    launch_ntt(dig, inter, cts * L, kl.ctx_ids, par->d_limbs, par->logn, false, 1, false, st, true);
  } else {
  // digit broadcast (rq/mod.rs:563-586), then NTT of every (digit, limb) row
  const bool reduce = digit_reduce(par, k);
  // forward_vt_lazy (rq/mod.rs:580): the digits stay in [0,4q_j); the lazy accumulator of the inner product takes
  // any 64-bit operand and reduces once
  // with the TMA kernels the transform deposits the digits of one (ciphertext, limb) in adjacent rows, which the
  // inner product streams fastest (bench_micro/stride_read.cu)
  adjacent = Lk > 1 && ntt_uses_tma(cts * L * Lk, kl.ctx_ids, par->logn, Lk, c2, inter);
  // default: the rows pass of the digit transforms and the inner product run as one kernel, so the transformed digits
  // never go through HBM.  FHE_B200_KSMAC=tma keeps the unfused TMA chain (rows pass, then ksmac_tma_kernel),
  // =classic the per-thread inner product.
  if (adjacent && switches().ksmac == Switches::KSMAC_FUSED &&
      launch_key_switch_tma(c2, inter, ranges, base0, base1, out0, out1, cts, L, Lk, out_ct_rows, kl.ctx_ids,
                            par->d_limbs, par->logn, reduce, st))
    return;
  launch_ntt(c2, inter, cts * L * Lk, kl.ctx_ids, par->d_limbs, par->logn, false, Lk, reduce, st, true, adjacent, L);
  }
  launch_ksmac(inter, ranges, base0, base1, out0, out1, L, Lk, out_ct_rows, kl.ctx_ids, par->d_limbs, par->logn, st,
               adjacent);
}

void key_switch_leveled_tail(const fhe_b200_params* par, const fhe_b200_ksk* k, u64* cur, u32 cts, u64* out,
                             int base_mode, u64* base, Workspace& ws, cudaStream_t st);

// key switch + the reference's post-processing (relinearization_key.rs:88-95, galois_key.rs:69-76):
// when the key lives at a lower level number than the ciphertext (more moduli), the (c0, c1) pair is
// taken to power basis, switched down to the ciphertext context and transformed back before it is added.
// c2: [cts][L][N] power basis at the ciphertext level; out: [cts][2][L][N]; base (nullable) is added:
// base_mode 0: none, 1: out += result (in place), 2: out = result + (base part 0 only; base is [cts][2][L][N])
void key_switch_apply(const fhe_b200_params* par, const KeySet& K, const u64* c2, u32 cts, u64* out,
                      int base_mode, u64* base, Workspace& ws, cudaStream_t st) {
  const fhe_b200_ksk* k = K.keys[0];
  const LevelData& cl = par->level(k->ct_level);
  const u32 L = cl.L, Lk = k->Lk, logn = par->logn;
  const size_t row = (size_t)1 << logn;
  if (Lk == L) {
    const u64* b0 = base_mode == 1 ? out : base_mode == 2 ? base : nullptr;
    const u64* b1 = base_mode == 1 ? out + L * row : nullptr;
    key_switch_core(par, K, c2, cts, b0, b1, out, out + L * row, 2 * L, ws, st);
    return;
  }
  u64* cur = ws.words((size_t)cts * 2 * Lk * row);
  key_switch_core(par, K, c2, cts, nullptr, nullptr, cur, cur + Lk * row, 2 * Lk, ws, st);
  key_switch_leveled_tail(par, k, cur, cts, out, base_mode, base, ws, st);
}

// The tail of key_switch_apply for a leveled key: cur [cts][2][Lk][N] (NTT, the key level) is taken to power basis,
// switched down to the ciphertext level, transformed back and written to or added into out as base_mode says.
void key_switch_leveled_tail(const fhe_b200_params* par, const fhe_b200_ksk* k, u64* cur, u32 cts, u64* out,
                             int base_mode, u64* base, Workspace& ws, cudaStream_t st) {
  const LevelData& cl = par->level(k->ct_level);
  const u32 L = cl.L, Lk = k->Lk, logn = par->logn;
  const size_t row = (size_t)1 << logn;
  const LevelData& kl = par->level(k->ksk_level);
  launch_ntt(cur, cur, cts * 2 * Lk, kl.ctx_ids, par->d_limbs, logn, true, 1, false, st);
  for (u32 lv = k->ksk_level; lv < k->ct_level; lv++) {  // Poly::switch_down_to, rq/mod.rs:498-507
    const LevelData& from = par->level(lv);
    u64* nxt = ws.words((size_t)cts * 2 * (from.L - 1) * row);
    launch_switch_down(from.sd, cur, nxt, cts * 2, from.L, from.ctx_ids, par->d_limbs, logn, st);
    cur = nxt;
  }
  launch_ntt(cur, cur, cts * 2 * L, cl.ctx_ids, par->d_limbs, logn, false, 1, false, st);
  if (base_mode == 1) {
    launch_ew(EW_ADD, out, cur, (size_t)cts * 2 * L, cl.ctx_ids, par->d_limbs, logn, st);
  } else {
    FHE_CUDA(cudaMemcpyAsync(out, cur, (size_t)cts * 2 * L * row * sizeof(u64), cudaMemcpyDeviceToDevice, st));
    if (base_mode == 2) {
      // only part 0 of `base` takes part: clear its part 1 (a scratch buffer of the caller) and add everything
      FHE_CUDA(cudaMemset2DAsync(base + L * row, 2 * L * row * sizeof(u64), 0, L * row * sizeof(u64), cts, st));
      launch_ew(EW_ADD, out, base, (size_t)cts * 2 * L, cl.ctx_ids, par->d_limbs, logn, st);
    }
  }
}

// GaloisKey::relinearize (galois_key.rs:63-86) of n 2-part NTT ciphertexts into `dst` ([n][2][L][N]), on one stream:
// the chunk body of every Galois call.  Output c reads ciphertext gk.source[c] of `src` (src0 + c without a source
// list) and uses the exponent of its key.  sum: one inner-sum step, dst = src + galois(src) (dst must not alias src):
// the substitution kernel writes (sigma(c0) + c0, c1) to dst and the key switch's in-place add finishes the step.
void galois_range(const fhe_b200_params* par, const LevelData& lv, const KeySet& gk, const u64* src, u32 src0, u64* dst,
                  u32 n, bool sum, cudaStream_t st) {
  const size_t row = (size_t)1 << par->logn, L = lv.L;
  std::vector<u32> exps(n), source(n);
  for (u32 c = 0; c < n; c++) {
    exps[c] = gk.exps[gk.key_of(c)];
    source[c] = gk.source ? gk.source[c] : src0 + c;
  }
  Workspace ws(par, st);
  u64* s = sum ? nullptr : ws.words((size_t)n * 2 * L * row);
  u64* c2 = ws.words((size_t)n * L * row);
  // galois_key.rs:66: substitute both parts; part 1 becomes the key-switch input
  launch_substitute_ntt(src, 2 * L * row, sum ? dst : s, 2 * L * row, c2, L * row, exps.data(), source.data(), n,
                        (u32)L, sum, lv.ctx_ids, par->d_limbs, par->logn, st);
  launch_ntt(c2, c2, n * (u32)L, lv.ctx_ids, par->d_limbs, par->logn, true, 1, false, st);
  // galois_key.rs:67 + :78: out0 = key_switch0 + substitute(ct[0]); out1 = key_switch1 (sum: both added in place)
  key_switch_apply(par, gk, c2, n, dst, sum ? 1 : 2, s, ws, st);
}

// extend -> tensor -> scale down of bfv/ops/mul.rs:192-206 for `cts` ciphertext pairs.
// a, b: [cts][2][L][N] NTT.  split == 0: out0 = [cts][3][L][N] power basis (all three parts);
// split == 1: out0 = [cts][2][L][N] (c0, c1), out1 = [cts][L][N] (c2), all power basis.
void mul_core(const fhe_b200_params* par, const LevelData& lv, const u64* a, const u64* b, u32 cts, u64* out0,
              u64* out1, int split, Workspace& ws, cudaStream_t st) {
  const u32 L = lv.L, E = lv.E, K = lv.K, logn = par->logn;
  const size_t row = (size_t)1 << logn;
  u64* A_l = ws.words((size_t)cts * 2 * L * row);
  u64* A_r = ws.words((size_t)cts * 2 * L * row);
  u64* X_l = ws.words((size_t)cts * 2 * E * row);
  u64* X_r = ws.words((size_t)cts * 2 * E * row);
  u64* T = ws.words((size_t)cts * 3 * K * row);
  // rq/scaler.rs:69-79: backward NTT of the source rows
  launch_ntt(a, A_l, cts * 2 * L, lv.ctx_ids, par->d_limbs, logn, true, 1, false, st);
  launch_ntt(b, A_r, cts * 2 * L, lv.ctx_ids, par->d_limbs, logn, true, 1, false, st);
  // rq/scaler.rs:85-94: exact base extension to the E new limbs (common prefix is kept as is, :61-65)
  launch_scale(lv.ext.dev, par->d_limbs, A_l, X_l, nullptr, cts * 2, E, L, E, 0, logn, st);
  launch_scale(lv.ext.dev, par->d_limbs, A_r, X_r, nullptr, cts * 2, E, L, E, 0, logn, st);
  // rq/scaler.rs:97-115: forward NTT of the new rows
  launch_ntt(X_l, X_l, cts * 2 * E, lv.ext_ids, par->d_limbs, logn, false, 1, false, st);
  launch_ntt(X_r, X_r, cts * 2 * E, lv.ext_ids, par->d_limbs, logn, false, 1, false, st);
  // mul.rs:198-201 tensor product, then mul.rs:204-206 scale down by t/Q (backward NTT of the 3K rows, exact scaling
  // K -> L); product and first inverse pass run as one kernel where the TMA kernels serve the shape
  if (!launch_tensor_inverse_ntt(a, b, X_l, X_r, T, cts, L, K, lv.mul_ids, par->d_limbs, logn, st)) {
    launch_tensor(a, b, X_l, X_r, T, cts, L, L, L, K, lv.mul_ids, par->d_limbs, logn, st);
    launch_ntt(T, T, cts * 3 * K, lv.mul_ids, par->d_limbs, logn, true, 1, false, st);
  }
  launch_scale(lv.down.dev, par->d_limbs, T, out0, out1, cts * 3, L, 0, L, split, logn, st);
}

// &ct * &ct for any part counts (ops/mod.rs:259-358): out [cts][na+nb-1][L][N] power basis
void mul_core_parts(const fhe_b200_params* par, const LevelData& lv, const u64* a, u32 na, const u64* b, u32 nb, u32 cts,
                    u64* out, Workspace& ws, cudaStream_t st) {
  const u32 L = lv.L, E = lv.E, K = lv.K, logn = par->logn, nc = na + nb - 1;
  const size_t row = (size_t)1 << logn;
  const u64* src[2] = {a, b};
  const u32 np[2] = {na, nb};
  u64* X[2];
  for (int s = 0; s < 2; s++) {
    u64* pb = ws.words((size_t)cts * np[s] * L * row);
    X[s] = ws.words((size_t)cts * np[s] * E * row);
    launch_ntt(src[s], pb, cts * np[s] * L, lv.ctx_ids, par->d_limbs, logn, true, 1, false, st);
    launch_scale(lv.ext.dev, par->d_limbs, pb, X[s], nullptr, cts * np[s], E, L, E, 0, logn, st);
    launch_ntt(X[s], X[s], cts * np[s] * E, lv.ext_ids, par->d_limbs, logn, false, 1, false, st);
  }
  u64* T = ws.words((size_t)cts * nc * K * row);
  launch_tensor_nm(a, b, X[0], X[1], T, cts, L, E, na, nb, lv.mul_ids, par->d_limbs, logn, st);
  launch_ntt(T, T, cts * nc * K, lv.mul_ids, par->d_limbs, logn, true, 1, false, st);
  launch_scale(lv.down.dev, par->d_limbs, T, out, nullptr, cts * nc, L, 0, L, 0, logn, st);
}

// The same pipeline for a custom strategy (mul.rs:192-206 with the Scalers of Multiplicator::new): every extender
// keeps its common prefix only when its factor is one (rq/scaler.rs:35-43), so a side with a non-unit factor gets all
// K limbs from the exact scaler.  out: [cts][3][L][N] power basis.
void mul_core_general(const fhe_b200_multiplicator* m, const u64* a, const u64* b, u32 cts, u64* out, Workspace& ws,
                      cudaStream_t st) {
  const fhe_b200_params* par = m->par;
  const LevelData& lv = par->level(m->level);
  const u32 L = m->L, K = m->K, logn = par->logn;
  const size_t row = (size_t)1 << logn;
  const u64* src[2] = {a, b};
  const ScalerData* ext[2] = {&m->ext_l, &m->ext_r};
  const u32 nc[2] = {m->nc_l, m->nc_r};
  u64* X[2] = {nullptr, nullptr};
  for (int s = 0; s < 2; s++) {
    const u32 E = K - nc[s];
    if (!E) continue;
    u64* pb = ws.words((size_t)cts * 2 * L * row);
    X[s] = ws.words((size_t)cts * 2 * E * row);
    launch_ntt(src[s], pb, cts * 2 * L, lv.ctx_ids, par->d_limbs, logn, true, 1, false, st);
    launch_scale(ext[s]->dev, m->d_limbs, pb, X[s], nullptr, cts * 2, E, nc[s], E, 0, logn, st);
    RowIds ids;
    std::memset(&ids, 0, sizeof(ids));
    ids.limbs_per_poly = E;
    for (u32 j = 0; j < E; j++) ids.ids[j] = m->mul_ids.ids[nc[s] + j];
    launch_ntt(X[s], X[s], cts * 2 * E, ids, m->d_limbs, logn, false, 1, false, st);
  }
  u64* T = ws.words((size_t)cts * 3 * K * row);
  launch_tensor(a, b, X[0], X[1], T, cts, L, nc[0], nc[1], K, m->mul_ids, m->d_limbs, logn, st);
  launch_ntt(T, T, cts * 3 * K, m->mul_ids, m->d_limbs, logn, true, 1, false, st);
  if (m->nc_d)  // common prefix of a factor-one down scaler: kept as is (power basis here, transformed by the caller)
    FHE_CUDA(cudaMemcpy2DAsync(out, L * row * 8, T, K * row * 8, m->nc_d * row * 8, (size_t)cts * 3,
                               cudaMemcpyDeviceToDevice, st));
  launch_scale(m->down.dev, m->d_limbs, T, out + m->nc_d * row, nullptr, cts * 3, L, m->nc_d, L - m->nc_d, 0, logn, st);
}

}  // namespace

extern "C" {

#define API_BEGIN try {
#define API_END                                                                   \
  }                                                                               \
  catch (const FheError& e) { g_last_error = e.what(); return e.code; }           \
  catch (const CudaFail& f) {                                                     \
    g_last_error = std::string(f.what) + ": " + cudaGetErrorString(f.err);        \
    cudaGetLastError();                                                           \
    return f.err == cudaErrorMemoryAllocation ? FHE_B200_OUT_OF_MEMORY : FHE_B200_CUDA_ERROR; \
  }                                                                               \
  catch (const std::bad_alloc&) { g_last_error = "host out of memory"; return FHE_B200_OUT_OF_MEMORY; } \
  catch (const std::exception& e) { g_last_error = e.what(); return FHE_B200_INVALID_ARGUMENT; } \
  return FHE_B200_OK;
#define REQUIRE(c, code, msg) \
  do { if (!(c)) throw FheError(code, msg); } while (0)

const char* fhe_b200_version(void) { return "fhe_b200 0.1 (sm_90a)"; }
const char* fhe_b200_last_error(void) { return g_last_error.c_str(); }
uint64_t fhe_b200_launch_count(void) { return g_launches.load(); }
uint64_t fhe_b200_ntt_row_count(int inverse) { return g_ntt_rows[inverse ? 1 : 0].load(); }

static int params_build(int device, uint32_t degree, const std::vector<u64>& moduli, const uint8_t* pt,
                        uint32_t pt_len, const uint64_t* psi, fhe_b200_params** out) {
  API_BEGIN
  REQUIRE(out && pt && pt_len, FHE_B200_INVALID_ARGUMENT, "null argument");
  // BfvParametersBuilder::validate_configuration (parameters.rs:440-468)
  REQUIRE(degree >= 8 && degree <= 65536 && (degree & (degree - 1)) == 0, FHE_B200_INVALID_DEGREE,
          "InvalidPolynomialDegree: " + std::to_string(degree));
  REQUIRE(!moduli.empty() && moduli.size() < 32, FHE_B200_INVALID_ARGUMENT, "MissingCiphertextModulusSpecification");
  // released through params_release on every exit path (frees the device tables and the pool of a half-built set)
  std::unique_ptr<fhe_b200_params, void (*)(const fhe_b200_params*)> p(new fhe_b200_params(device), params_release);
  p->N = degree;
  p->logn = (u32)__builtin_ctz(degree);
  p->Lmax = (u32)moduli.size();
  p->moduli = moduli;
  p->t = BigUint::from_le_bytes(pt, pt_len);
  REQUIRE(!p->t.is_zero(), FHE_B200_INVALID_ARGUMENT, "plaintext modulus is zero");
  if (p->t.bits() <= 62 && p->t.to_u64() >= 2) {
    const ModulusH tm(p->t.to_u64());
    p->t_small = true;
    p->t_mod = PlainMod{tm.p, tm.bhi, tm.blo};
  }
  // validate_moduli (parameters.rs:471-552)
  BigUint Q(1);
  for (size_t i = 0; i < moduli.size(); i++) {
    ModulusH m(moduli[i]);
    for (size_t j = 0; j < i; j++) REQUIRE(moduli[j] != moduli[i], FHE_B200_INVALID_MODULUS, "DuplicateModuli");
    REQUIRE(moduli[i] % (2 * (u64)degree) == 1 && is_prime_u64(moduli[i]), FHE_B200_NTT_UNAVAILABLE,
            "CiphertextModulusNotNttFriendly: " + std::to_string(moduli[i]));
    u64 tm = p->t.mod_u64(moduli[i]), dummy;
    REQUIRE(tm != 0 && invmod_h(tm, moduli[i], &dummy), FHE_B200_INVALID_MODULUS, "PlaintextModulusNotCoprime");
    p->moduli_sizes.push_back(64 - (u32)clz64(moduli[i]));
    Q = Q * BigUint(moduli[i]);
  }
  REQUIRE(p->t < Q, FHE_B200_INVALID_ARGUMENT, "PlaintextModulusExceedsCiphertextModulus");
  // extended basis (parameters.rs:660-676)
  u64 ub = 1ull << 62;
  while (p->ext.size() != moduli.size() + 1) {
    REQUIRE(generate_prime(62, 2 * (u64)degree, ub, &ub), FHE_B200_INVALID_MODULUS, "NotEnoughPrimes");
    bool dup = false;
    for (u64 q : p->ext) dup |= q == ub;
    for (u64 q : moduli) dup |= q == ub;
    if (!dup) p->ext.push_back(ub);
  }
  p->primes = moduli;
  p->primes.insert(p->primes.end(), p->ext.begin(), p->ext.end());
  if (device >= 0) {
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || device >= ndev) {
      cudaGetLastError();
      throw FheError(FHE_B200_NO_DEVICE, "CUDA device " + std::to_string(device) + " not available");
    }
  }
  DeviceGuard g(device, true);   // selects nothing for a host-only set
  if (device >= 0) {
    cudaMemPoolProps props;
    std::memset(&props, 0, sizeof(props));
    props.allocType = cudaMemAllocationTypePinned;
    props.handleTypes = cudaMemHandleTypeNone;
    props.location.type = cudaMemLocationTypeDevice;
    props.location.id = device;
    FHE_CUDA(cudaMemPoolCreate(&p->pool, &props));
    unsigned long long thr = ~0ull;   // keep freed scratch for the next chunk instead of returning it to the OS
    FHE_CUDA(cudaMemPoolSetAttribute(p->pool, cudaMemPoolAttrReleaseThreshold, &thr));
    // scratch freed on one stream must not be handed to another stream through an inserted dependency: that
    // serialises callers that pipeline chunks over several streams (bench.py e2e); let each stream keep its own
    int off = 0;
    FHE_CUDA(cudaMemPoolSetAttribute(p->pool, cudaMemPoolReuseAllowInternalDependencies, &off));
  }
  for (size_t i = 0; i < p->primes.size(); i++) {
    u64 q = p->primes[i];
    u64 r = psi ? psi[i] : default_psi(q, degree);
    p->psi.push_back(r);
    p->tables.push_back(make_ntt_tables(q, degree, r));
    p->h_limbs.push_back(make_limb_dev(q, p->tables.back(), p->uploads));
  }
  p->d_limbs = p->uploads.put(p->h_limbs);
  *out = p.release();
  API_END
}

int fhe_b200_params_create(int device, uint32_t degree, const uint64_t* moduli, uint32_t n_moduli,
                           const uint8_t* plaintext_le, uint32_t plaintext_len, const uint64_t* psi,
                           fhe_b200_params** out) {
  if (!moduli || !n_moduli) { g_last_error = "null moduli"; return FHE_B200_INVALID_ARGUMENT; }
  std::vector<u64> m(moduli, moduli + n_moduli);
  return params_build(device, degree, m, plaintext_le, plaintext_len, psi, out);
}

int fhe_b200_params_create_from_sizes(int device, uint32_t degree, const uint32_t* sizes, uint32_t n_moduli,
                                      const uint8_t* plaintext_le, uint32_t plaintext_len, fhe_b200_params** out) {
  if (!sizes || !n_moduli) { g_last_error = "null sizes"; return FHE_B200_INVALID_ARGUMENT; }
  if (degree < 8 || (degree & (degree - 1))) { g_last_error = "InvalidPolynomialDegree"; return FHE_B200_INVALID_DEGREE; }
  // BfvParametersBuilder::generate_moduli (parameters.rs:391-431)
  std::vector<u64> m;
  for (uint32_t i = 0; i < n_moduli; i++) {
    if (sizes[i] > 62 || sizes[i] < 10) { g_last_error = "InvalidModulusSize"; return FHE_B200_INVALID_MODULUS; }
    u64 ub = 1ull << sizes[i];
    for (;;) {
      u64 q;
      if (!generate_prime((int)sizes[i], 2 * (u64)degree, ub, &q)) { g_last_error = "NotEnoughPrimes"; return FHE_B200_INVALID_MODULUS; }
      bool dup = false;
      for (u64 x : m) dup |= x == q;
      if (!dup) { m.push_back(q); break; }
      ub = q;
    }
  }
  return params_build(device, degree, m, plaintext_le, plaintext_len, nullptr, out);
}

int fhe_b200_params_destroy(fhe_b200_params* p) {
  params_release(p);
  return FHE_B200_OK;
}
uint32_t fhe_b200_params_degree(const fhe_b200_params* p) { return p ? p->N : 0; }
uint32_t fhe_b200_params_n_moduli(const fhe_b200_params* p) { return p ? p->Lmax : 0; }
int fhe_b200_params_moduli(const fhe_b200_params* p, uint64_t* out) {
  if (!p || !out) return FHE_B200_INVALID_ARGUMENT;
  for (u32 i = 0; i < p->Lmax; i++) out[i] = p->moduli[i];
  return FHE_B200_OK;
}
int fhe_b200_params_mul_basis(const fhe_b200_params* p, uint32_t level, uint64_t* out, uint32_t* n) {
  API_BEGIN
  REQUIRE(p && n, FHE_B200_INVALID_ARGUMENT, "null argument");
  const LevelData& lv = p->level(level);
  *n = lv.K;
  if (out) for (u32 i = 0; i < lv.K; i++) out[i] = lv.mul_moduli[i];
  API_END
}
int fhe_b200_params_psi(const fhe_b200_params* p, uint64_t q, uint64_t* psi) {
  if (!p || !psi) return FHE_B200_INVALID_ARGUMENT;
  int i = prime_index(p->primes, q);
  if (i < 0) { g_last_error = "prime not in parameter set"; return FHE_B200_INVALID_MODULUS; }
  *psi = p->psi[i];
  return FHE_B200_OK;
}

// ------------------------------------------------------------------------------ batches
static int batch_alloc(const fhe_b200_params* p, uint32_t count, uint32_t parts, uint32_t level, int repr,
                       bool mul_basis, fhe_b200_batch** out) {
  API_BEGIN
  REQUIRE(p && out, FHE_B200_INVALID_ARGUMENT, "null argument");
  REQUIRE(count > 0 && parts > 0, FHE_B200_INVALID_ARGUMENT, "empty batch");
  REQUIRE(repr == FHE_B200_POWER_BASIS || repr == FHE_B200_NTT, FHE_B200_INVALID_REPRESENTATION, "bad representation");
  DeviceGuard g(p);
  const LevelData& lv = p->level(level);
  std::unique_ptr<fhe_b200_batch> b(new fhe_b200_batch(p));
  b->count = count; b->parts = parts; b->level = level; b->repr = repr;
  b->mul_basis = mul_basis;
  b->limbs = mul_basis ? lv.K : lv.L;
  FHE_CUDA(cudaMalloc(&b->d, b->words_per_ct() * count * sizeof(u64)));
  *out = b.release();
  API_END
}
int fhe_b200_batch_alloc(const fhe_b200_params* p, uint32_t count, uint32_t parts, uint32_t level, int repr,
                         fhe_b200_batch** out) {
  return batch_alloc(p, count, parts, level, repr, false, out);
}
int fhe_b200_batch_alloc_mul_basis(const fhe_b200_params* p, uint32_t count, uint32_t parts, uint32_t level,
                                   int repr, fhe_b200_batch** out) {
  return batch_alloc(p, count, parts, level, repr, true, out);
}
int fhe_b200_batch_free(fhe_b200_batch* b) {
  delete b;
  return FHE_B200_OK;
}
int fhe_b200_batch_info(const fhe_b200_batch* b, uint32_t* count, uint32_t* parts, uint32_t* level, uint32_t* limbs,
                        int* repr) {
  if (!b) return FHE_B200_INVALID_ARGUMENT;
  if (count) *count = b->count;
  if (parts) *parts = b->parts;
  if (level) *level = b->level;
  if (limbs) *limbs = b->limbs;
  if (repr) *repr = b->repr;
  return FHE_B200_OK;
}
int fhe_b200_batch_upload(fhe_b200_batch* b, uint32_t first, uint32_t n, const uint64_t* host, void* stream) {
  API_BEGIN
  REQUIRE(b && host, FHE_B200_INVALID_ARGUMENT, "null argument");
  REQUIRE((uint64_t)first + n <= b->count, FHE_B200_INVALID_ARGUMENT, "range exceeds batch");
  DeviceGuard g(b->par);
  size_t w = b->words_per_ct();
  FHE_CUDA(cudaMemcpyAsync(b->d + w * first, host, w * n * sizeof(u64), cudaMemcpyHostToDevice, (cudaStream_t)stream));
  API_END
}
int fhe_b200_batch_download(const fhe_b200_batch* b, uint32_t first, uint32_t n, uint64_t* host, void* stream) {
  API_BEGIN
  REQUIRE(b && host, FHE_B200_INVALID_ARGUMENT, "null argument");
  REQUIRE((uint64_t)first + n <= b->count, FHE_B200_INVALID_ARGUMENT, "range exceeds batch");
  DeviceGuard g(b->par);
  size_t w = b->words_per_ct();
  FHE_CUDA(cudaMemcpyAsync(host, b->d + w * first, w * n * sizeof(u64), cudaMemcpyDeviceToHost, (cudaStream_t)stream));
  FHE_CUDA(cudaStreamSynchronize((cudaStream_t)stream));
  API_END
}
int fhe_b200_batch_download_async(const fhe_b200_batch* b, uint32_t first, uint32_t n, uint64_t* host, void* stream) {
  API_BEGIN
  REQUIRE(b && host, FHE_B200_INVALID_ARGUMENT, "null argument");
  REQUIRE((uint64_t)first + n <= b->count, FHE_B200_INVALID_ARGUMENT, "range exceeds batch");
  DeviceGuard g(b->par);
  size_t w = b->words_per_ct();
  FHE_CUDA(cudaMemcpyAsync(host, b->d + w * first, w * n * sizeof(u64), cudaMemcpyDeviceToHost, (cudaStream_t)stream));
  API_END
}
int fhe_b200_batch_copy(fhe_b200_batch* dst, const fhe_b200_batch* src, void* stream) {
  API_BEGIN
  REQUIRE(dst && src, FHE_B200_INVALID_ARGUMENT, "null argument");
  check_same(dst, src);
  REQUIRE(dst->parts == src->parts && dst->count == src->count, FHE_B200_BAD_POLY_COUNT, "shapes differ");
  DeviceGuard g(src->par);
  FHE_CUDA(cudaMemcpyAsync(dst->d, src->d, src->words_per_ct() * src->count * sizeof(u64), cudaMemcpyDeviceToDevice,
                           (cudaStream_t)stream));
  dst->repr = src->repr;
  API_END
}
int fhe_b200_batch_copy_range(fhe_b200_batch* dst, uint32_t dst_first, const fhe_b200_batch* src, uint32_t src_first,
                              uint32_t src_stride, uint32_t n, void* stream) {
  API_BEGIN
  REQUIRE(dst && src && dst != src, FHE_B200_INVALID_ARGUMENT, "null or aliased argument");
  check_same(dst, src);
  REQUIRE(dst->parts == src->parts, FHE_B200_BAD_POLY_COUNT, "shapes differ");
  REQUIRE(dst->repr == src->repr, FHE_B200_INVALID_REPRESENTATION, "IncorrectRepresentation");
  REQUIRE(n > 0 && src_stride > 0, FHE_B200_INVALID_ARGUMENT, "empty range or zero stride");
  REQUIRE((uint64_t)dst_first + n <= dst->count &&
              (uint64_t)src_first + (uint64_t)(n - 1) * src_stride < src->count,
          FHE_B200_INVALID_ARGUMENT, "range exceeds batch");
  DeviceGuard g(src->par);
  const size_t w = src->words_per_ct() * sizeof(u64);
  FHE_CUDA(cudaMemcpy2DAsync(dst->d + src->words_per_ct() * dst_first, w, src->d + src->words_per_ct() * src_first,
                             w * src_stride, w, n, cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
  API_END
}
int fhe_b200_host_alloc(size_t bytes, int write_combined, void** out) {
  API_BEGIN
  REQUIRE(out && bytes, FHE_B200_INVALID_ARGUMENT, "null argument");
  void* p = nullptr;
  FHE_CUDA(cudaHostAlloc(&p, bytes, cudaHostAllocPortable | (write_combined ? cudaHostAllocWriteCombined : 0)));
  *out = p;
  API_END
}
int fhe_b200_host_free(void* p) {
  API_BEGIN
  if (p) FHE_CUDA(cudaFreeHost(p));
  API_END
}
int fhe_b200_batch_device_ptr(const fhe_b200_batch* b, uint64_t** dptr, size_t* n_words) {
  if (!b || !dptr) return FHE_B200_INVALID_ARGUMENT;
  *dptr = (uint64_t*)b->d;
  if (n_words) *n_words = b->words_per_ct() * b->count;
  return FHE_B200_OK;
}

// ------------------------------------------------------------------------------ keys
// The digit count of a key from its two levels (key_switching_key.rs:92-126).  log_base receives 0 for RNS digits (one
// per ciphertext limb) or, for a single-modulus key level, the base-2^(log_modulus/2) decomposition of the residue.
static u32 ksk_digits(const fhe_b200_params* p, const LevelData& cl, const LevelData& kl, u32& log_base) {
  log_base = 0;
  if (kl.L > 1) return cl.L;
  REQUIRE(cl.L == 1, FHE_B200_CONTEXT_MISMATCH, "ParameterMismatch: a single-modulus key serves the last level only");
  const u64 q = p->moduli[0];
  const u32 log_modulus = 64 - (u32)clz64(q - 1);   // next_power_of_two().ilog2()
  log_base = log_modulus / 2;
  REQUIRE(log_base >= 1, FHE_B200_UNSUPPORTED, "modulus too small for the decomposition");
  return (log_modulus + log_base - 1) / log_base;
}

// A key handle with room for its words: both parts in the device layout [limb][digit][N] of n_dig digits over the Lk
// limbs of the key level
static std::unique_ptr<fhe_b200_ksk> make_ksk(const fhe_b200_params* p, u32 ct_level, u32 ksk_level, u32 n_dig, u32 Lk,
                                              u32 log_base) {
  std::unique_ptr<fhe_b200_ksk> k(new fhe_b200_ksk(p));
  k->ct_level = ct_level; k->ksk_level = ksk_level; k->n_dig = n_dig; k->Lk = Lk; k->log_base = log_base;
  const size_t bytes = ((size_t)n_dig * Lk << p->logn) * sizeof(u64);
  FHE_CUDA(cudaMalloc(&k->k0, bytes));
  FHE_CUDA(cudaMalloc(&k->k1, bytes));
  return k;
}

int fhe_b200_ksk_upload(const fhe_b200_params* p, uint32_t ciphertext_level, uint32_t ksk_level, const uint64_t* c0,
                        const uint64_t* c1, uint32_t n_digits, fhe_b200_ksk** out) {
  API_BEGIN
  REQUIRE(p && c0 && c1 && out, FHE_B200_INVALID_ARGUMENT, "null argument");
  DeviceGuard g(p);
  const LevelData& cl = p->level(ciphertext_level);
  const LevelData& kl = p->level(ksk_level);
  REQUIRE(ksk_level <= ciphertext_level, FHE_B200_INVALID_LEVEL, "key level must not exceed the ciphertext level");
  u32 log_base = 0;
  const u32 want = ksk_digits(p, cl, kl, log_base);
  REQUIRE(n_digits == want, FHE_B200_CONTEXT_MISMATCH,
          log_base ? "n_digits must be ceil(log_modulus / log_base) for a single-modulus key"
                   : "n_digits must equal the ciphertext level's limb count");
  std::unique_ptr<fhe_b200_ksk> k = make_ksk(p, ciphertext_level, ksk_level, n_digits, kl.L, log_base);
  // host layout [digit][limb][N] -> device layout [limb][digit][N]: the inner product walks the digits of one limb
  const size_t rowb = sizeof(u64) << p->logn;
  for (u32 i = 0; i < n_digits; i++) {
    FHE_CUDA(cudaMemcpy2D((char*)k->k0 + i * rowb, n_digits * rowb, (const char*)c0 + (size_t)i * kl.L * rowb, rowb,
                          rowb, kl.L, cudaMemcpyHostToDevice));
    FHE_CUDA(cudaMemcpy2D((char*)k->k1 + i * rowb, n_digits * rowb, (const char*)c1 + (size_t)i * kl.L * rowb, rowb,
                          rowb, kl.L, cudaMemcpyHostToDevice));
  }
  *out = k.release();
  API_END
}
int fhe_b200_ksk_download(const fhe_b200_ksk* k, uint64_t* c0, uint64_t* c1, void* stream) {
  API_BEGIN
  REQUIRE(k && c0 && c1, FHE_B200_INVALID_ARGUMENT, "null argument");
  DeviceGuard g(k->par);
  cudaStream_t st = (cudaStream_t)stream;
  // device layout [limb][digit][N] -> host layout [digit][limb][N], the reverse of fhe_b200_ksk_upload
  const size_t rowb = sizeof(u64) << k->par->logn, row = (size_t)1 << k->par->logn;
  for (u32 i = 0; i < k->n_dig; i++) {
    FHE_CUDA(cudaMemcpy2DAsync(c0 + (size_t)i * k->Lk * row, rowb, k->k0 + i * row, k->n_dig * rowb, rowb, k->Lk,
                               cudaMemcpyDeviceToHost, st));
    FHE_CUDA(cudaMemcpy2DAsync(c1 + (size_t)i * k->Lk * row, rowb, k->k1 + i * row, k->n_dig * rowb, rowb, k->Lk,
                               cudaMemcpyDeviceToHost, st));
  }
  FHE_CUDA(cudaStreamSynchronize(st));
  API_END
}
int fhe_b200_ksk_free(fhe_b200_ksk* k) {
  delete k;
  return FHE_B200_OK;
}

// ------------------------------------------------------------------------------ primitives
static int ntt_batch(fhe_b200_batch* b, bool inverse, void* stream) {
  API_BEGIN
  REQUIRE(b, FHE_B200_INVALID_ARGUMENT, "null argument");
  need_repr(b, inverse ? FHE_B200_NTT : FHE_B200_POWER_BASIS);
  DeviceGuard g(b->par);
  launch_ntt(b->d, b->d, b->count * b->parts * b->limbs, ids_of(b), b->par->d_limbs, b->par->logn, inverse, 1, false,
             (cudaStream_t)stream);
  FHE_CUDA(cudaGetLastError());
  b->repr = inverse ? FHE_B200_POWER_BASIS : FHE_B200_NTT;
  API_END
}
int fhe_b200_ntt_forward(fhe_b200_batch* b, void* stream) { return ntt_batch(b, false, stream); }
int fhe_b200_ntt_backward(fhe_b200_batch* b, void* stream) { return ntt_batch(b, true, stream); }

static int ew(EwOp op, fhe_b200_batch* a, const fhe_b200_batch* b, void* stream) {
  API_BEGIN
  REQUIRE(a && (b || op == EW_NEG), FHE_B200_INVALID_ARGUMENT, "null argument");
  if (b) {
    check_same(a, b);
    REQUIRE(a->parts == b->parts && a->count == b->count, FHE_B200_BAD_POLY_COUNT, "operand shapes differ");
    REQUIRE(a->repr == b->repr, FHE_B200_INVALID_REPRESENTATION, "IncorrectRepresentation");
  }
  DeviceGuard g(a->par);
  launch_ew(op, a->d, b ? b->d : nullptr, (size_t)a->count * a->parts * a->limbs, ids_of(a), a->par->d_limbs,
            a->par->logn, (cudaStream_t)stream);
  FHE_CUDA(cudaGetLastError());
  API_END
}
int fhe_b200_add(fhe_b200_batch* a, const fhe_b200_batch* b, void* stream) { return ew(EW_ADD, a, b, stream); }
int fhe_b200_sub(fhe_b200_batch* a, const fhe_b200_batch* b, void* stream) { return ew(EW_SUB, a, b, stream); }
int fhe_b200_neg(fhe_b200_batch* a, void* stream) { return ew(EW_NEG, a, nullptr, stream); }

static int plain_op(fhe_b200_batch* a, const uint64_t* host_polys, uint32_t n_polys, u32 op, void* stream) {
  API_BEGIN
  REQUIRE(a && host_polys, FHE_B200_INVALID_ARGUMENT, "null argument");
  REQUIRE(n_polys == 1 || n_polys == a->count, FHE_B200_INVALID_ARGUMENT, "n_polys must be 1 or the batch size");
  REQUIRE(a->parts >= 1, FHE_B200_BAD_POLY_COUNT, "empty ciphertext");
  need_repr(a, FHE_B200_NTT);
  const fhe_b200_params* par = a->par;
  DeviceGuard g(par);
  cudaStream_t st = (cudaStream_t)stream;
  Workspace ws(par, st);
  const size_t words = ((size_t)n_polys * a->limbs) << par->logn;
  u64* pt = ws.words(words);
  FHE_CUDA(cudaMemcpyAsync(pt, host_polys, words * sizeof(u64), cudaMemcpyHostToDevice, st));
  launch_mul_plain(a->d, pt, a->count, a->parts, n_polys, ids_of(a), par->d_limbs, par->logn, st, op);
  FHE_CUDA(cudaGetLastError());
  // No synchronisation: a pageable host_polys has been staged by the runtime when cudaMemcpyAsync returns; a pinned
  // one must stay valid until the stream reaches this point -- the same contract as fhe_b200_batch_upload.
  API_END
}
int fhe_b200_mul_plain(fhe_b200_batch* a, const uint64_t* host_polys, uint32_t n_polys, void* stream) {
  return plain_op(a, host_polys, n_polys, 0, stream);
}
int fhe_b200_add_plain(fhe_b200_batch* a, const uint64_t* host_polys, uint32_t n_polys, int subtract, void* stream) {
  return plain_op(a, host_polys, n_polys, subtract ? 2 : 1, stream);
}

int fhe_b200_dot_product_scalar(const fhe_b200_batch* cts, const fhe_b200_batch* pts, uint32_t n_terms,
                                fhe_b200_batch* out, void* stream) {
  API_BEGIN
  REQUIRE(cts && pts && out, FHE_B200_INVALID_ARGUMENT, "null argument");
  REQUIRE(n_terms > 0 && cts->count > 0 && pts->count > 0, FHE_B200_INVALID_ARGUMENT, "DotProductError::EmptyInput");
  check_same(cts, pts);
  check_same(cts, out);
  REQUIRE(pts->parts == 1, FHE_B200_BAD_POLY_COUNT, "plaintext batch must hold one polynomial per entry");
  REQUIRE(out->parts == cts->parts, FHE_B200_BAD_POLY_COUNT, "DotProductError::CiphertextPolynomialCountMismatch");
  const size_t total = (size_t)out->count * n_terms;
  REQUIRE((cts->count == total || cts->count == n_terms) && (pts->count == total || pts->count == n_terms),
          FHE_B200_INVALID_ARGUMENT, "DotProductError::OperandCountMismatch");
  need_repr(cts, FHE_B200_NTT);
  need_repr(pts, FHE_B200_NTT);
  DeviceGuard g(cts->par);
  launch_dot(cts->d, pts->d, out->d, out->count, n_terms, cts->parts, cts->count, pts->count, ids_of(cts),
             cts->par->d_limbs, cts->par->logn, (cudaStream_t)stream);
  FHE_CUDA(cudaGetLastError());
  out->repr = FHE_B200_NTT;
  API_END
}

// AddAssign<&Ciphertext> (ops/mod.rs:54-69) folded over each run of n_terms entries, from out[g] or from
// Ciphertext::zero: one segment_sum launch for the whole batch.  It holds no scratch, so it needs no chunks.
int fhe_b200_batch_sum(const fhe_b200_batch* in, uint32_t n_terms, int accumulate, fhe_b200_batch* out,
                       void* stream) {
  API_BEGIN
  REQUIRE(in && out && in != out, FHE_B200_INVALID_ARGUMENT, "null or aliased argument");
  REQUIRE(n_terms > 0, FHE_B200_INVALID_ARGUMENT, "a sum takes at least one term");
  REQUIRE(in->count == (size_t)out->count * n_terms, FHE_B200_INVALID_ARGUMENT,
          "the input must hold n_terms entries per output entry");
  REQUIRE(in->par == out->par, FHE_B200_CONTEXT_MISMATCH, "ParameterMismatch: batches use different parameters");
  REQUIRE(in->parts == out->parts, FHE_B200_BAD_POLY_COUNT, "input and output part counts differ");
  check_same(in, out);
  if (accumulate) need_repr(out, in->repr);
  DeviceGuard g(in->par);
  const size_t W = in->words_per_ct();
  launch_segment_sum(in->d, W, n_terms, out->d, W, nullptr, 0, in->parts * in->limbs, out->count, W, accumulate != 0,
                     ids_of(in), in->par->d_limbs, in->par->logn, (cudaStream_t)stream);
  FHE_CUDA(cudaGetLastError());
  out->repr = in->repr;
  API_END
}

// ---- plaintext encoding
int fhe_b200_encoder_create(const fhe_b200_params* p, const uint64_t* psi_t, fhe_b200_encoder** out) {
  API_BEGIN
  REQUIRE(p && out, FHE_B200_INVALID_ARGUMENT, "null argument");
  std::unique_ptr<fhe_b200_encoder> e(new fhe_b200_encoder(p));
  const u32 N = p->N;
  // parameters.rs:713-726
  e->index_map.resize(N);
  auto brev = [&](u64 x) {
    u32 r = 0;
    for (u32 b = 0; b < p->logn; b++) r |= (u32)((x >> b) & 1) << (p->logn - 1 - b);
    return r;
  };
  const u64 m = 2 * (u64)N;
  u64 pos = 1;
  for (u32 i = 0; i < N / 2; i++) {
    e->index_map[i] = brev((pos - 1) >> 1);
    e->index_map[N / 2 + i] = brev((m - pos - 1) >> 1);
    pos = (pos * 3) & (m - 1);
  }
  std::vector<u32> inv(N);
  for (u32 i = 0; i < N; i++) inv[e->index_map[i]] = i;
  e->h_limbs = p->h_limbs;
  std::memset(&e->t_ids, 0, sizeof(RowIds));
  e->t_ids.limbs_per_poly = 1;
  e->t_ids.ids[0] = (unsigned short)p->h_limbs.size();
  // NttOperator::new (ntt/native.rs:35-73): t is a Modulus, prime, and 1 mod 2N
  const u64 t = p->t_mod.t;
  e->has_ntt = p->t_small && t % m == 1 && is_prime_u64(t);
  if (e->has_ntt) {
    e->psi_t = psi_t ? *psi_t : default_psi(t, N);
    e->tables = make_ntt_tables(t, N, e->psi_t);
    e->h_limbs.push_back(make_limb_dev(t, e->tables, e->uploads));
  }
  e->d_limbs = e->uploads.put(e->h_limbs);
  e->d_inv_map = e->uploads.put(inv);
  e->d_index_map = e->uploads.put(std::vector<int>(e->index_map.begin(), e->index_map.end()));
  *out = e.release();
  API_END
}

int fhe_b200_encoder_free(fhe_b200_encoder* e) {
  delete e;
  return FHE_B200_OK;
}

int fhe_b200_encode(const fhe_b200_encoder* e, int encoding, int is_signed, const void* values, size_t n_values,
                    fhe_b200_batch* out, void* stream) {
  API_BEGIN
  REQUIRE(e, FHE_B200_INVALID_ARGUMENT, "null encoder");
  const fhe_b200_params* par = e->par;
  DeviceGuard g(par);
  REQUIRE(out, FHE_B200_INVALID_ARGUMENT, "null argument");
  REQUIRE(encoding == FHE_B200_ENCODING_POLY || encoding == FHE_B200_ENCODING_SIMD, FHE_B200_INVALID_ARGUMENT,
          "unknown encoding");
  REQUIRE(par->t_small, FHE_B200_UNSUPPORTED, "the plaintext modulus does not fit a u64 Modulus");
  const bool simd = encoding == FHE_B200_ENCODING_SIMD;
  REQUIRE(!simd || e->has_ntt, FHE_B200_NTT_UNAVAILABLE, "EncodingError::SimdUnavailable");   // plaintext_vec.rs:47
  REQUIRE(out->par == par, FHE_B200_CONTEXT_MISMATCH, "ParameterMismatch");
  REQUIRE(!out->mul_basis, FHE_B200_CONTEXT_MISMATCH, "PolynomialContextMismatch");
  const LevelData& lv = par->level(out->level);
  REQUIRE(out->parts == 1, FHE_B200_BAD_POLY_COUNT, "a plaintext batch has one polynomial per entry");
  const size_t N = par->N;
  const size_t count = std::max<size_t>(1, (n_values + N - 1) / N);
  REQUIRE(out->count == count, FHE_B200_INVALID_ARGUMENT, "batch must hold max(1, ceil(n_values / N)) plaintexts");
  REQUIRE(values || !n_values, FHE_B200_INVALID_ARGUMENT, "null values");
  const u32 L = lv.L, logn = par->logn;
  const bool poly_u64 = !simd && !is_signed;
  // forward butterflies take inputs below 4 q_j: Poly u64 words are arbitrary, the other words are below t
  const bool reduce = poly_u64 || lv.lift_reduce;
  const char* src = (const char*)values;
  ChunkRunner chunks(par, (u32)count, (cudaStream_t)stream);
  chunks.run([&](u32 c0, u32 n, cudaStream_t st) {
    Workspace ws(par, st);
    const size_t v0 = (size_t)c0 * N, vn = n_values > v0 ? std::min(n_values - v0, (size_t)n * N) : 0;
    u64* staged = ws.words(std::max<size_t>(vn, 1));
    if (vn) FHE_CUDA(cudaMemcpyAsync(staged, src + v0 * sizeof(u64), vn * sizeof(u64), cudaMemcpyDefault, st));
    const u64* coeffs = staged;
    if (!(poly_u64 && vn == (size_t)n * N)) {
      u64* c = ws.words((size_t)n * N);
      launch_encode_load(staged, c, n, vn, simd ? e->d_inv_map : nullptr, is_signed != 0, par->t_mod, logn, st);
      if (simd) launch_ntt(c, c, n, e->t_ids, e->d_limbs, logn, true, 1, false, st);   // NttOperator::backward mod t
      coeffs = c;
    }
    // try_convert_from + into_ntt: every limb of plaintext k transforms row k of `coeffs`
    launch_ntt(coeffs, out->d + (size_t)c0 * L * N, n * L, lv.ctx_ids, e->d_limbs, logn, false, L, reduce, st);
  });
  FHE_CUDA(cudaGetLastError());
  out->repr = FHE_B200_NTT;
  API_END
}

// pts: 1-part NTT batch at a's level with 1 or a->count entries (the checks of plain_op plus the batch's shape)
static void check_plain_batch(const fhe_b200_batch* a, const fhe_b200_batch* pts) {
  REQUIRE(a && pts, FHE_B200_INVALID_ARGUMENT, "null argument");
  check_same(a, pts);
  REQUIRE(pts->count == 1 || pts->count == a->count, FHE_B200_INVALID_ARGUMENT, "plaintext count must be 1 or the batch size");
  REQUIRE(a->parts >= 1 && pts->parts == 1, FHE_B200_BAD_POLY_COUNT, "plaintext batch must hold one polynomial per entry");
  need_repr(a, FHE_B200_NTT);
  need_repr(pts, FHE_B200_NTT);
}

int fhe_b200_mul_plain_batch(fhe_b200_batch* a, const fhe_b200_batch* pts, void* stream) {
  API_BEGIN
  check_plain_batch(a, pts);
  DeviceGuard g(a->par);
  launch_mul_plain(a->d, pts->d, a->count, a->parts, pts->count, ids_of(a), a->par->d_limbs, a->par->logn,
                   (cudaStream_t)stream, 0);
  FHE_CUDA(cudaGetLastError());
  API_END
}

// RowIds of a single row modulo q_0
static RowIds q0_row_ids() {
  RowIds ids;
  std::memset(&ids, 0, sizeof(RowIds));
  ids.limbs_per_poly = 1;
  return ids;
}

// Plaintext::to_poly (plaintext.rs:172-197) up to the delta product, from the plaintexts' coefficients (t < q_0):
// x [n][N] power-basis words, in place ((x mod t) * q_mod_t) mod t, then lifted to every limb of the level and
// transformed into m [n][L][N]
static void to_poly_from_coefficients(const fhe_b200_params* par, const LevelData& lv, u64* x, u32 n, u64* m,
                                      cudaStream_t st) {
  launch_to_poly_load(x, (size_t)n << par->logn, par->t_mod, lv.q_mod_t, st);
  launch_ntt(x, m, n * lv.L, lv.ctx_ids, par->d_limbs, par->logn, false, lv.L, lv.lift_reduce, st);
}

// Plaintext::to_poly (plaintext.rs:172-197) of plaintexts [p0, p0 + n) of the 1-part NTT batch pts into m [n][L][N],
// before the delta product (t < q_0); x: scratch of n * N words
static void plain_to_poly(const fhe_b200_params* par, const LevelData& lv, const fhe_b200_batch* pts, u32 p0, u32 n,
                          u64* m, u64* x, cudaStream_t st) {
  const size_t N = par->N;
  FHE_CUDA(cudaMemcpy2DAsync(x, N * 8, pts->d + (size_t)p0 * lv.L * N, lv.L * N * 8, N * 8, n, cudaMemcpyDeviceToDevice,
                             st));
  launch_ntt(x, x, n, q0_row_ids(), par->d_limbs, par->logn, true, 1, false, st);   // limb 0 of into_power_basis
  to_poly_from_coefficients(par, lv, x, n, m, st);
}

int fhe_b200_add_plain_batch(fhe_b200_batch* a, const fhe_b200_batch* pts, int subtract, void* stream) {
  API_BEGIN
  check_plain_batch(a, pts);
  const fhe_b200_params* par = a->par;
  REQUIRE(par->t_small && par->t_mod.t < par->moduli[0], FHE_B200_UNSUPPORTED,
          "to_poly needs t below the first ciphertext modulus");
  DeviceGuard g(par);
  const LevelData& lv = par->level(a->level);
  const u32 L = lv.L, logn = par->logn;
  const size_t N = par->N;
  cudaStream_t user = (cudaStream_t)stream;
  Workspace shared_ws(par, user);
  const bool shared = pts->count == 1;
  u64* m_shared = nullptr;
  if (shared) {   // built once, before the chunks' side streams fork from `user`
    m_shared = shared_ws.words((size_t)L * N);
    plain_to_poly(par, lv, pts, 0, 1, m_shared, shared_ws.words(N), user);
  }
  ChunkRunner chunks(par, a->count, user);
  chunks.run([&](u32 c0, u32 n, cudaStream_t st) {
    Workspace ws(par, st);
    const u64* m = m_shared;
    if (!shared) {
      u64* mc = ws.words((size_t)n * L * N);
      plain_to_poly(par, lv, pts, c0, n, mc, ws.words((size_t)n * N), st);
      m = mc;
    }
    launch_add_scaled(a->d + (size_t)c0 * a->parts * L * N, m, n, a->parts, shared ? 1 : n, lv.d_delta, lv.d_delta_s,
                      subtract != 0, lv.ctx_ids, par->d_limbs, logn, st);
  });
  FHE_CUDA(cudaGetLastError());
  API_END
}

// ---- decryption, decoding and noise measurement
int fhe_b200_secret_key_create(const fhe_b200_params* p, const int64_t* coeffs, fhe_b200_secret_key** out) {
  API_BEGIN
  REQUIRE(p && coeffs && out, FHE_B200_INVALID_ARGUMENT, "null argument");
  REQUIRE(p->t_small, FHE_B200_UNSUPPORTED, "the plaintext modulus does not fit a u64 Modulus");
  DeviceGuard g(p);
  std::unique_ptr<fhe_b200_secret_key> sk(new fhe_b200_secret_key(p));
  const u32 N = p->N, Lmax = p->Lmax;
  // Poly::try_convert_from(&[i64], ctx, false) (rq/convert.rs:194-230): the canonical residue of every signed word
  std::vector<u64> res((size_t)Lmax * N);
  for (u32 j = 0; j < Lmax; j++) {
    const u64 q = p->moduli[j];
    for (u32 i = 0; i < N; i++) {
      const u64 w = (u64)coeffs[i], mag = coeffs[i] < 0 ? 0 - w : w, r = mag % q;
      res[(size_t)j * N + i] = (coeffs[i] < 0 && r) ? q - r : r;
    }
  }
  FHE_CUDA(cudaMemcpy(sk->s.d, res.data(), res.size() * sizeof(u64), cudaMemcpyHostToDevice));
  volatile u64* wipe = res.data();   // erase the host copy (volatile: the stores are not elided)
  for (size_t i = 0; i < res.size(); i++) wipe[i] = 0;
  const LevelData& l0 = p->level(0);
  launch_ntt(sk->s.d, sk->s.d, Lmax, l0.ctx_ids, p->d_limbs, p->logn, false, 1, false, nullptr);   // into_ntt
  FHE_CUDA(cudaGetLastError());
  FHE_CUDA(cudaStreamSynchronize(nullptr));
  *out = sk.release();
  API_END
}

int fhe_b200_secret_key_free(fhe_b200_secret_key* sk) {
  delete sk;
  return FHE_B200_OK;
}

// the checks shared by decrypt and measure_noise
static void check_secret_input(const fhe_b200_secret_key* sk, const fhe_b200_batch* ct) {
  REQUIRE(sk && ct, FHE_B200_INVALID_ARGUMENT, "null argument");
  REQUIRE(ct->par == sk->par, FHE_B200_CONTEXT_MISMATCH, "ParameterMismatch");
  REQUIRE(!ct->mul_basis, FHE_B200_CONTEXT_MISMATCH, "PolynomialContextMismatch");
  need_repr(ct, FHE_B200_NTT);
}

// try_decrypt (secret_key.rs:198-260) of ciphertexts [c0, c0 + n) of ct up to the scaled phase: w [n][N] receives
// ((v + t) mod q_0) mod t, v = row 0 of phase.scale(cipher_plain_context.scaler).  When ph_ntt is not null it receives
// the NTT-domain phase [n][L][N] (which measure_noise reuses); otherwise the phase is transformed in place in scratch.
static void decrypt_range(const fhe_b200_secret_key* sk, const fhe_b200_batch* ct, u32 c0, u32 n, u64* w, u64* ph_ntt,
                          Workspace& ws, cudaStream_t st) {
  const fhe_b200_params* par = sk->par;
  const LevelData& lv = par->level(ct->level);
  const u32 L = lv.L, logn = par->logn;
  const size_t rows = (size_t)n * L;
  u64* ph = ph_ntt ? ph_ntt : ws.secret_words(rows << logn);
  launch_phase(ct->d + (((size_t)c0 * ct->parts * L) << logn), sk->s.d, ph, n, ct->parts, lv.ctx_ids, par->d_limbs,
               logn, st);
  u64* pb = ph_ntt ? ws.secret_words(rows << logn) : ph;
  launch_ntt(ph, pb, (u32)rows, lv.ctx_ids, par->d_limbs, logn, true, 1, false, st);
  // only output row 0 (q_0): the reference keeps v[..degree], and every output limb of the scaler is independent
  launch_scale(lv.plain.dev, par->d_limbs, pb, w, nullptr, n, 1, 0, 1, 0, logn, st);
  const LimbDev& q0 = par->h_limbs[0];
  launch_decrypt_epilogue(w, (size_t)n << logn, PlainMod{q0.p, q0.bhi, q0.blo}, par->t_mod, st);
}

int fhe_b200_decrypt(const fhe_b200_secret_key* sk, const fhe_b200_batch* ct, fhe_b200_batch* out, void* stream) {
  API_BEGIN
  check_secret_input(sk, ct);
  REQUIRE(out, FHE_B200_INVALID_ARGUMENT, "null argument");
  REQUIRE(out->par == sk->par, FHE_B200_CONTEXT_MISMATCH, "ParameterMismatch");
  REQUIRE(!out->mul_basis, FHE_B200_CONTEXT_MISMATCH, "PolynomialContextMismatch");
  REQUIRE(out->parts == 1 && out->count == ct->count && out->level == ct->level, FHE_B200_INVALID_ARGUMENT,
          "out must be a 1-part batch of ct.count plaintexts at ct's level");
  const fhe_b200_params* par = sk->par;
  DeviceGuard g(par);
  const LevelData& lv = par->level(ct->level);
  const u32 L = lv.L, logn = par->logn;
  ChunkRunner chunks(par, ct->count, (cudaStream_t)stream);
  chunks.run([&](u32 c0, u32 n, cudaStream_t st) {
    Workspace ws(par, st);
    u64* w = ws.secret_words((size_t)n << logn);
    decrypt_range(sk, ct, c0, n, w, nullptr, ws, st);
    // Poly::try_convert_from(w, ctx).into_ntt(): every limb of plaintext k transforms row k of w
    launch_ntt(w, out->d + ((size_t)c0 * L << logn), n * L, lv.ctx_ids, par->d_limbs, logn, false, L, lv.lift_reduce,
               st);
  });
  FHE_CUDA(cudaGetLastError());
  out->repr = FHE_B200_NTT;
  API_END
}

int fhe_b200_measure_noise(const fhe_b200_secret_key* sk, const fhe_b200_batch* ct, uint32_t* noise_bits,
                           void* stream) {
  API_BEGIN
  check_secret_input(sk, ct);
  REQUIRE(noise_bits, FHE_B200_INVALID_ARGUMENT, "null argument");
  const fhe_b200_params* par = sk->par;
  REQUIRE(par->t_small && par->t_mod.t < par->moduli[0], FHE_B200_UNSUPPORTED,
          "to_poly needs t below the first ciphertext modulus");
  DeviceGuard g(par);
  const LevelData& lv = par->level(ct->level);
  const u32 L = lv.L, logn = par->logn;
  cudaStream_t user = (cudaStream_t)stream;
  Workspace out_ws(par, user);   // the per-ciphertext maxima, filled by the chunks' atomics
  u32* noise = (u32*)out_ws.words((ct->count + 1) / 2);
  FHE_CUDA(cudaMemsetAsync(noise, 0, ct->count * sizeof(u32), user));
  {
    ChunkRunner chunks(par, ct->count, user);
    chunks.run([&](u32 c0, u32 n, cudaStream_t st) {
      Workspace ws(par, st);
      const size_t words = ((size_t)n * L) << logn;
      u64* ph = ws.secret_words(words);
      u64* w = ws.secret_words((size_t)n << logn);
      decrypt_range(sk, ct, c0, n, w, ph, ws, st);
      // phase - to_poly(decrypt(ct)), back to the power basis (secret_key.rs:61-84)
      u64* m = ws.secret_words(words);
      to_poly_from_coefficients(par, lv, w, n, m, st);
      launch_add_scaled(ph, m, n, 1, n, lv.d_delta, lv.d_delta_s, true, lv.ctx_ids, par->d_limbs, logn, st);
      launch_ntt(ph, ph, n * L, lv.ctx_ids, par->d_limbs, logn, true, 1, false, st);
      launch_noise(ph, noise + c0, n, L, lv.garner, lv.q_words, lv.W, par->d_limbs, logn, st);
    });
  }
  FHE_CUDA(cudaMemcpyAsync(noise_bits, noise, ct->count * sizeof(u32), cudaMemcpyDefault, user));
  FHE_CUDA(cudaGetLastError());
  API_END
}

int fhe_b200_decode(const fhe_b200_encoder* e, int encoding, int is_signed, const fhe_b200_batch* pts, void* values,
                    size_t n_values, void* stream) {
  API_BEGIN
  REQUIRE(e, FHE_B200_INVALID_ARGUMENT, "null encoder");
  const fhe_b200_params* par = e->par;
  REQUIRE(encoding == FHE_B200_ENCODING_POLY || encoding == FHE_B200_ENCODING_SIMD, FHE_B200_INVALID_ARGUMENT,
          "unknown encoding");
  // Plaintext::coefficients (plaintext.rs:103-135): with t >= q_0 the reference lifts every limb
  REQUIRE(par->t_small && par->t_mod.t < par->moduli[0], FHE_B200_UNSUPPORTED,
          "decoding needs t below the first ciphertext modulus");
  DeviceGuard g(par);
  const bool simd = encoding == FHE_B200_ENCODING_SIMD;
  REQUIRE(!simd || e->has_ntt, FHE_B200_NTT_UNAVAILABLE, "EncodingError::SimdUnavailable");   // plaintext.rs:155-160
  REQUIRE(pts, FHE_B200_INVALID_ARGUMENT, "null argument");
  REQUIRE(pts->par == par, FHE_B200_CONTEXT_MISMATCH, "ParameterMismatch");
  REQUIRE(!pts->mul_basis, FHE_B200_CONTEXT_MISMATCH, "PolynomialContextMismatch");
  REQUIRE(pts->parts == 1, FHE_B200_BAD_POLY_COUNT, "a plaintext batch has one polynomial per entry");
  need_repr(pts, FHE_B200_NTT);
  const size_t N = par->N;
  REQUIRE(values && n_values == (size_t)pts->count * N, FHE_B200_INVALID_ARGUMENT,
          "values must hold pts.count * N words");
  const u32 L = pts->limbs, logn = par->logn;
  const RowIds q0_ids = q0_row_ids();
  char* dst = (char*)values;
  ChunkRunner chunks(par, pts->count, (cudaStream_t)stream);
  chunks.run([&](u32 c0, u32 n, cudaStream_t st) {
    Workspace ws(par, st);
    u64* x = ws.words((size_t)n * N);
    FHE_CUDA(cudaMemcpy2DAsync(x, N * 8, pts->d + (size_t)c0 * L * N, L * N * 8, N * 8, n, cudaMemcpyDeviceToDevice, st));
    launch_ntt(x, x, n, q0_ids, par->d_limbs, logn, true, 1, false, st);      // limb 0 of into_power_basis
    launch_to_poly_load(x, (size_t)n * N, par->t_mod, 1, st);                 // reduce_vec mod t
    if (simd) {   // decode_simd_u64 (plaintext.rs:155-170): NttOperator::forward mod t, then the slot gather
      launch_ntt(x, x, n, e->t_ids, e->d_limbs, logn, false, 1, false, st);
      u64* y = ws.words((size_t)n * N);
      launch_gather(x, y, n, e->d_index_map, logn, st);
      x = y;
    }
    if (is_signed) launch_center(x, (size_t)n * N, par->t_mod.t, st);       // center_vec (plaintext.rs:440-446)
    FHE_CUDA(cudaMemcpyAsync(dst + (size_t)c0 * N * 8, x, (size_t)n * N * 8, cudaMemcpyDefault, st));
  });
  FHE_CUDA(cudaGetLastError());
  API_END
}

// ---- encryption (keys/secret_key.rs:100-136, :181-193; keys/public_key.rs:45-92)
// the 32-byte seed as the key words of the ChaCha20 state
static EncSeed seed_words(const uint8_t* seed) {
  EncSeed K;
  for (int i = 0; i < 8; i++)
    K.w[i] = (u32)seed[4 * i] | (u32)seed[4 * i + 1] << 8 | (u32)seed[4 * i + 2] << 16 | (u32)seed[4 * i + 3] << 24;
  return K;
}

// the checks shared by both entry points; returns the seed as the key words of the ChaCha20 state
static EncSeed check_encrypt(const fhe_b200_params* par, const fhe_b200_batch* pts, const uint8_t* seed,
                             const fhe_b200_batch* out) {
  REQUIRE(seed && out, FHE_B200_INVALID_ARGUMENT, "null argument");
  REQUIRE(out->par == par, FHE_B200_CONTEXT_MISMATCH, "ParameterMismatch");
  REQUIRE(!out->mul_basis, FHE_B200_CONTEXT_MISMATCH, "PolynomialContextMismatch");
  REQUIRE(out->parts == 2, FHE_B200_INVALID_ARGUMENT, "out must be a batch of 2-part ciphertexts");
  if (pts) {
    REQUIRE(pts->par == par, FHE_B200_CONTEXT_MISMATCH, "ParameterMismatch");
    REQUIRE(!pts->mul_basis, FHE_B200_CONTEXT_MISMATCH, "PolynomialContextMismatch");
    REQUIRE(pts->parts == 1 && pts->count == out->count, FHE_B200_INVALID_ARGUMENT,
            "pts must be a 1-part batch with one plaintext per output ciphertext");
    REQUIRE(pts->level == out->level, FHE_B200_INVALID_LEVEL, "InvalidLevel: pts and out are at different levels");
    need_repr(pts, FHE_B200_NTT);
  }
  REQUIRE(par->t_small && par->t_mod.t < par->moduli[0], FHE_B200_UNSUPPORTED,
          "to_poly needs t below the first ciphertext modulus");
  return seed_words(seed);
}

static void check_variance(uint32_t variance) {   // BfvParametersBuilder::build (parameters.rs:449-454)
  REQUIRE(variance >= 1 && variance <= 32, FHE_B200_INVALID_ARGUMENT,
          "InvalidVariance: " + std::to_string(variance) + " is outside 1..32");
}

// part 0 of the ciphertexts dst [n][2][L][N] += Plaintext::to_poly of plaintexts [c0, c0 + n) of pts
static void add_to_poly(const fhe_b200_params* par, const LevelData& lv, const fhe_b200_batch* pts, u32 c0, u32 n,
                        u64* dst, Workspace& ws, cudaStream_t st) {
  u64* m = ws.secret_words(((size_t)n * lv.L) << par->logn);
  plain_to_poly(par, lv, pts, c0, n, m, ws.secret_words((size_t)n << par->logn), st);
  launch_add_scaled(dst, m, n, 2, n, lv.d_delta, lv.d_delta_s, false, lv.ctx_ids, par->d_limbs, par->logn, st);
}

int fhe_b200_encrypt_sk(const fhe_b200_secret_key* sk, const fhe_b200_batch* pts, uint32_t variance,
                        const uint8_t* seed, fhe_b200_batch* out, void* stream) {
  API_BEGIN
  check_variance(variance);
  REQUIRE(sk, FHE_B200_INVALID_ARGUMENT, "null argument");
  const fhe_b200_params* par = sk->par;
  const EncSeed K = check_encrypt(par, pts, seed, out);
  DeviceGuard g(par);
  const LevelData& lv = par->level(out->level);
  const u32 L = lv.L, logn = par->logn;
  ChunkRunner chunks(par, out->count, (cudaStream_t)stream);
  chunks.run([&](u32 c0, u32 n, cudaStream_t st) {
    Workspace ws(par, st);
    u64* e = ws.secret_words(((size_t)n * L) << logn);
    launch_cbd(e, n, c0, 1, 1, variance, K, lv.ctx_ids, par->d_limbs, logn, st);
    launch_ntt(e, e, n * L, lv.ctx_ids, par->d_limbs, logn, false, 1, false, st);
    u64* dst = out->d + (((size_t)c0 * 2 * L) << logn);
    launch_encrypt_sk(sk->s.d, e, dst, n, c0, K, lv.ctx_ids, par->d_limbs, logn, st);
    if (pts) add_to_poly(par, lv, pts, c0, n, dst, ws, st);
  });
  FHE_CUDA(cudaGetLastError());
  out->repr = FHE_B200_NTT;
  API_END
}

// the checks of a public key operand: one 2-part level-0 NTT ciphertext
static void check_public_key(const fhe_b200_batch* pk) {
  REQUIRE(pk, FHE_B200_INVALID_ARGUMENT, "null argument");
  REQUIRE(!pk->mul_basis, FHE_B200_CONTEXT_MISMATCH, "PolynomialContextMismatch");
  REQUIRE(pk->count == 1 && pk->parts == 2, FHE_B200_INVALID_ARGUMENT, "a public key is one 2-part ciphertext");
  REQUIRE(pk->level == 0, FHE_B200_INVALID_LEVEL, "InvalidPublicKeyLevel: " + std::to_string(pk->level));
  need_repr(pk, FHE_B200_NTT);
}

// the public key's c at `level`: the key itself at level 0, else a copy in ws switched down to the level
// (public_key.rs:60-70), enqueued on st
static const u64* public_key_at_level(const fhe_b200_batch* pk, u32 level, Workspace& ws, cudaStream_t st) {
  if (level == 0) return pk->d;
  const fhe_b200_params* par = pk->par;
  u64* sw = ws.words(((size_t)2 * par->Lmax) << par->logn);
  FHE_CUDA(cudaMemcpyAsync(sw, pk->d, pk->words_per_ct() * sizeof(u64), cudaMemcpyDeviceToDevice, st));
  for (u32 l = 0; l < level; l++) switch_down_polys(par, l, sw, 2, ws, st);
  return sw;
}

int fhe_b200_encrypt_pk(const fhe_b200_batch* pk, const fhe_b200_batch* pts, uint32_t variance, const uint8_t* seed,
                        fhe_b200_batch* out, void* stream) {
  API_BEGIN
  check_variance(variance);
  check_public_key(pk);
  const fhe_b200_params* par = pk->par;
  const EncSeed K = check_encrypt(par, pts, seed, out);
  DeviceGuard g(par);
  const LevelData& lv = par->level(out->level);
  const u32 L = lv.L, logn = par->logn;
  cudaStream_t user = (cudaStream_t)stream;
  Workspace key_ws(par, user);
  const u64* c = public_key_at_level(pk, out->level, key_ws, user);
  ChunkRunner chunks(par, out->count, user);
  chunks.run([&](u32 c0, u32 n, cudaStream_t st) {
    Workspace ws(par, st);
    u64* uee = ws.secret_words(((size_t)n * 3 * L) << logn);   // u, e1, e2
    launch_cbd(uee, n, c0, 2, 3, variance, K, lv.ctx_ids, par->d_limbs, logn, st);
    launch_ntt(uee, uee, n * 3 * L, lv.ctx_ids, par->d_limbs, logn, false, 1, false, st);
    u64* dst = out->d + (((size_t)c0 * 2 * L) << logn);
    launch_encrypt_pk(uee, c, dst, n, lv.ctx_ids, par->d_limbs, logn, st);
    if (pts) add_to_poly(par, lv, pts, c0, n, dst, ws, st);
  });
  FHE_CUDA(cudaGetLastError());
  out->repr = FHE_B200_NTT;
  API_END
}

// ---- SecretKey::random (secret_key.rs:42-45) for n_keys keys in one call.  Key k is sample_vec_cbd(N, variance) of
// the role-18 row (k, limb 0), written as its canonical residue into every limb (Poly::try_convert_from(&[i64])) and
// transformed: the words fhe_b200_secret_key_create makes from the same coefficients, which never reach the host.  The
// keys go through the chunk runner, per chunk at most chunk_size() rows of scratch (chunk_size() / Lmax keys): one
// launch draws the chunk's keys, one transform takes them to the NTT domain, then each key's rows are copied into its
// own SecretBuffer.  On failure the keys made so far are freed and out is left untouched.
int fhe_b200_secret_keys_random(const fhe_b200_params* p, uint32_t n_keys, uint32_t variance, const uint8_t* seed,
                                fhe_b200_secret_key** out, void* stream) {
  API_BEGIN
  REQUIRE(p && seed && out, FHE_B200_INVALID_ARGUMENT, "null argument");
  REQUIRE(n_keys, FHE_B200_INVALID_ARGUMENT, "n_keys is 0");
  check_variance(variance);
  REQUIRE(p->t_small, FHE_B200_UNSUPPORTED, "the plaintext modulus does not fit a u64 Modulus");
  DeviceGuard g(p);
  const EncSeed K = seed_words(seed);
  const LevelData& l0 = p->level(0);
  const u32 Lmax = p->Lmax, logn = p->logn;
  const size_t words = (size_t)Lmax << logn;
  std::vector<std::unique_ptr<fhe_b200_secret_key>> made;   // freed again unless the call succeeds
  for (u32 k = 0; k < n_keys; k++) made.emplace_back(new fhe_b200_secret_key(p));
  cudaStream_t user = (cudaStream_t)stream;
  {
    ChunkRunner chunks(p, n_keys, user, std::max(1u, chunk_size() / Lmax));
    chunks.run([&](u32 c0, u32 n, cudaStream_t st) {
      Workspace ws(p, st);
      u64* s = ws.secret_words(n * words);
      launch_cbd(s, n, c0, 18, 1, variance, K, l0.ctx_ids, p->d_limbs, logn, st);
      launch_ntt(s, s, n * Lmax, l0.ctx_ids, p->d_limbs, logn, false, 1, false, st);   // into_ntt
      for (u32 k = 0; k < n; k++)
        FHE_CUDA(cudaMemcpyAsync(made[c0 + k]->s.d, s + k * words, words * sizeof(u64), cudaMemcpyDeviceToDevice, st));
    });
  }
  FHE_CUDA(cudaGetLastError());
  FHE_CUDA(cudaStreamSynchronize(user));   // the keys are ready on every stream, as after fhe_b200_secret_key_create
  for (u32 k = 0; k < n_keys; k++) out[k] = made[k].release();
  API_END
}

// SecretKey.coeffs (secret_key.rs:25-30, read by to_bytes :142-148): limb 0 of s back to the power basis, each word
// centred modulo q_0 on the host (v - q_0 when v > q_0 / 2, by a mask)
int fhe_b200_secret_key_coeffs(const fhe_b200_secret_key* sk, int64_t* out, void* stream) {
  API_BEGIN
  REQUIRE(sk && out, FHE_B200_INVALID_ARGUMENT, "null argument");
  const fhe_b200_params* par = sk->par;
  DeviceGuard g(par);
  const u32 N = par->N;
  cudaStream_t st = (cudaStream_t)stream;
  {
    Workspace ws(par, st);
    u64* w = ws.secret_words(N);
    launch_ntt(sk->s.d, w, 1, par->level(0).ctx_ids, par->d_limbs, par->logn, true, 1, false, st);
    FHE_CUDA(cudaMemcpyAsync(out, w, (size_t)N * sizeof(u64), cudaMemcpyDefault, st));
  }
  FHE_CUDA(cudaGetLastError());
  FHE_CUDA(cudaStreamSynchronize(st));
  const u64 q0 = par->moduli[0];
  for (u32 i = 0; i < N; i++) {
    const u64 v = (u64)out[i];
    out[i] = (int64_t)(v - (q0 & (0 - (u64)(v > (q0 >> 1)))));
  }
  API_END
}

// ---- key generation (key_switching_key.rs:71-238, relinearization_key.rs:43-65, galois_key.rs:26-60,
// rgsw_ciphertext.rs:94-120).  Every value is a canonical residue and the NTT is linear, so the key is built in the NTT
// domain: c0_i = NTT(e_i) - c1_i s + G[i] x, with x the key's polynomial at the ciphertext level.  The switch-up of x
// to the key level (Switcher) is x (Q_key / Q_ct) on the ciphertext limbs and 0 on the others, and the Garner
// coefficient g_i of the ciphertext basis is δ_ij modulo its limbs, so G[i][j] = δ_ij (Q_key / Q_ct mod q_j).
static void check_key_levels(const fhe_b200_params* par, uint32_t ciphertext_level, uint32_t key_level) {
  REQUIRE(ciphertext_level < par->Lmax, FHE_B200_INVALID_LEVEL,
          "InvalidLevel: ciphertext level " + std::to_string(ciphertext_level));
  REQUIRE(key_level <= ciphertext_level, FHE_B200_INVALID_LEVEL,
          "InvalidLevel: key level " + std::to_string(key_level) + " above the ciphertext level");
}

// Makes n_keys keys at (ct_level, key_level) into out[0 .. n_keys).  x_of(k, x, st) writes key k's x [L_ct][N] (NTT)
// into scratch.  The (key, digit) items go through the chunk runner, per chunk at most chunk_size() error rows
// (chunk_size() / Lk items of Lk rows each; at set C 18 items, 64 MiB of errors) whatever the number of keys: per chunk
// the errors (role 6) are drawn and transformed at once, then the generator runs once per key the chunk touches.  On
// failure the keys made so far are freed and out is left untouched.
static void generate_keys(const fhe_b200_secret_key* sk, u32 n_keys, u32 ct_level, u32 key_level, u32 variance,
                          const EncSeed& K, const std::function<void(u32, u64*, cudaStream_t)>& x_of,
                          fhe_b200_ksk** out, cudaStream_t user) {
  const fhe_b200_params* par = sk->par;
  const LevelData& cl = par->level(ct_level);
  const LevelData& kl = par->level(key_level);
  u32 log_base = 0;
  const u32 n_dig = ksk_digits(par, cl, kl, log_base);
  const u32 Lk = kl.L, logn = par->logn;
  const size_t row = (size_t)1 << logn;
  KskG G;
  std::memset(&G, 0, sizeof(G));
  G.decomp = log_base ? 1 : 0;
  for (u32 j = 0; j < (log_base ? n_dig : cl.L); j++) {
    const u64 q = log_base ? par->moduli[0] : par->moduli[j];
    u64 v = log_base ? ((1ull << (j * log_base)) % q) : 1;   // i log_base < 64 (at most 3 digits of <= 31 bits)
    for (u32 l = cl.L; l < Lk; l++) v = mulmod_h(v, par->moduli[l] % q, q);
    G.g[j] = v;
    G.g_s[j] = ModulusH(q).shoup(v);
  }
  std::vector<std::unique_ptr<fhe_b200_ksk>> made;   // freed again unless the call succeeds
  for (u32 k = 0; k < n_keys; k++) made.push_back(make_ksk(par, ct_level, key_level, n_dig, Lk, log_base));
  ChunkRunner chunks(par, n_keys * n_dig, user, std::max(1u, chunk_size() / Lk));
  chunks.run([&](u32 c0, u32 n, cudaStream_t st) {
    Workspace ws(par, st);
    u64* e = ws.secret_words((size_t)n * Lk * row);
    launch_cbd(e, n, c0, 6, 1, variance, K, kl.ctx_ids, par->d_limbs, logn, st, n_dig);
    launch_ntt(e, e, n * Lk, kl.ctx_ids, par->d_limbs, logn, false, 1, false, st);
    u64* x = ws.secret_words((size_t)cl.L * row);
    for (u32 it = c0; it < c0 + n;) {
      const u32 key = it / n_dig, d0 = it % n_dig, nd = std::min(n_dig - d0, c0 + n - it);
      x_of(key, x, st);
      const fhe_b200_ksk* h = made[key].get();
      launch_ksk_gen(sk->s.d, e + (size_t)(it - c0) * Lk * row, x, h->k0, h->k1, key, d0, nd, n_dig, G, K, kl.ctx_ids,
                     par->d_limbs, logn, st);
      it += nd;
    }
  });
  FHE_CUDA(cudaGetLastError());
  for (u32 k = 0; k < n_keys; k++) out[k] = made[k].release();
}

// x = a * s on the limbs of the level (a: [L][N] NTT words, s the secret key's rows)
static void times_s(const fhe_b200_secret_key* sk, const LevelData& lv, const u64* a, u64* x, cudaStream_t st) {
  const fhe_b200_params* par = sk->par;
  const size_t words = (size_t)lv.L << par->logn;
  FHE_CUDA(cudaMemcpyAsync(x, a, words * sizeof(u64), cudaMemcpyDeviceToDevice, st));
  launch_mul_plain(x, sk->s.d, 1, 1, 1, lv.ctx_ids, par->d_limbs, par->logn, st, 0);
}

int fhe_b200_relin_key_generate(const fhe_b200_secret_key* sk, uint32_t ciphertext_level, uint32_t key_level,
                                uint32_t variance, const uint8_t* seed, fhe_b200_ksk** out, void* stream) {
  API_BEGIN
  check_variance(variance);
  REQUIRE(sk && seed && out, FHE_B200_INVALID_ARGUMENT, "null argument");
  const fhe_b200_params* par = sk->par;
  check_key_levels(par, ciphertext_level, key_level);
  REQUIRE(par->Lmax - key_level > 1, FHE_B200_UNSUPPORTED,
          "EvaluationKeyError::KeySwitchingNotSupported: a relinearization key needs two or more key moduli");
  DeviceGuard g(par);
  const LevelData& cl = par->level(ciphertext_level);
  // x = s * s (relinearization_key.rs:56-60)
  generate_keys(sk, 1, ciphertext_level, key_level, variance, seed_words(seed),
                [&](u32, u64* x, cudaStream_t st) { times_s(sk, cl, sk->s.d, x, st); }, out, (cudaStream_t)stream);
  API_END
}

int fhe_b200_galois_keys_generate(const fhe_b200_secret_key* sk, const uint32_t* exponents, uint32_t n_keys,
                                  uint32_t ciphertext_level, uint32_t key_level, uint32_t variance,
                                  const uint8_t* seed, fhe_b200_ksk** out, void* stream) {
  API_BEGIN
  check_variance(variance);
  REQUIRE(sk && seed && out && (exponents || !n_keys), FHE_B200_INVALID_ARGUMENT, "null argument");
  const fhe_b200_params* par = sk->par;
  check_key_levels(par, ciphertext_level, key_level);
  std::vector<u32> exps(n_keys);
  for (u32 k = 0; k < n_keys; k++) {   // SubstitutionExponent::new (rq/mod.rs:99-121)
    exps[k] = (u32)(exponents[k] % (2 * par->N));
    REQUIRE(exps[k] & 1, FHE_B200_INVALID_EXPONENT, "InvalidSubstitutionExponent: " + std::to_string(exponents[k]));
  }
  DeviceGuard g(par);
  const LevelData& cl = par->level(ciphertext_level);
  // x = s substituted by the exponent (galois_key.rs:40-46), a permutation of the NTT words
  generate_keys(sk, n_keys, ciphertext_level, key_level, variance, seed_words(seed),
                [&](u32 k, u64* x, cudaStream_t st) {
                  launch_substitute_ntt(sk->s.d, 0, x, 0, nullptr, 0, &exps[k], nullptr, 1, cl.L, false, cl.ctx_ids,
                                        par->d_limbs, par->logn, st);
                }, out, (cudaStream_t)stream);
  API_END
}

int fhe_b200_rgsw_encrypt(const fhe_b200_secret_key* sk, const fhe_b200_batch* pts, uint32_t variance,
                          const uint8_t* seed, fhe_b200_ksk** out, void* stream) {
  API_BEGIN
  check_variance(variance);
  REQUIRE(sk && pts && seed && out, FHE_B200_INVALID_ARGUMENT, "null argument");
  const fhe_b200_params* par = sk->par;
  REQUIRE(pts->par == par, FHE_B200_CONTEXT_MISMATCH, "ParameterMismatch");
  REQUIRE(!pts->mul_basis, FHE_B200_CONTEXT_MISMATCH, "PolynomialContextMismatch");
  REQUIRE(pts->parts == 1, FHE_B200_INVALID_ARGUMENT, "pts must be a 1-part batch");
  need_repr(pts, FHE_B200_NTT);
  DeviceGuard g(par);
  const LevelData& lv = par->level(pts->level);
  const size_t words = (size_t)lv.L << par->logn;
  // ksk0 of plaintext p has x = m, ksk1 has x = m s (rgsw_ciphertext.rs:106-116); m = pt.poly_ntt
  generate_keys(sk, 2 * pts->count, pts->level, pts->level, variance, seed_words(seed),
                [&](u32 k, u64* x, cudaStream_t st) {
                  const u64* m = pts->d + (k / 2) * words;
                  if (k & 1) times_s(sk, lv, m, x, st);
                  else FHE_CUDA(cudaMemcpyAsync(x, m, words * sizeof(u64), cudaMemcpyDeviceToDevice, st));
                },
                out, (cudaStream_t)stream);
  API_END
}

// ---- multiparty BFV (fhe::mbfv, crates/fhe/src/mbfv).  Experimental, incomplete, not audited, as the reference's
// module: the share errors are the ordinary variance errors, not smudging noise.
// a batch argument of this parameter set, over the level's own basis, NTT
static void check_operand(const fhe_b200_params* par, const fhe_b200_batch* b) {
  REQUIRE(b, FHE_B200_INVALID_ARGUMENT, "null argument");
  REQUIRE(b->par == par, FHE_B200_CONTEXT_MISMATCH, "ParameterMismatch");
  REQUIRE(!b->mul_basis, FHE_B200_CONTEXT_MISMATCH, "PolynomialContextMismatch");
  need_repr(b, FHE_B200_NTT);
}
// a 2-part ciphertext batch (InvalidPolynomialCount otherwise, secret_key_switch.rs:56-64)
static void check_ciphertexts(const fhe_b200_params* par, const fhe_b200_batch* ct) {
  check_operand(par, ct);
  REQUIRE(ct->parts == 2, FHE_B200_BAD_POLY_COUNT, "InvalidPolynomialCount: multiparty protocols take 2-part ciphertexts");
}
// an output batch: `parts` polynomials per entry, `count` entries at `level`
static void check_output(const fhe_b200_params* par, const fhe_b200_batch* out, u32 count, u32 parts, u32 level) {
  REQUIRE(out, FHE_B200_INVALID_ARGUMENT, "null argument");
  REQUIRE(out->par == par, FHE_B200_CONTEXT_MISMATCH, "ParameterMismatch");
  REQUIRE(!out->mul_basis, FHE_B200_CONTEXT_MISMATCH, "PolynomialContextMismatch");
  REQUIRE(out->count == count && out->parts == parts && out->level == level, FHE_B200_INVALID_ARGUMENT,
          "out must be a " + std::to_string(parts) + "-part batch of " + std::to_string(count) + " entries at level " +
              std::to_string(level));
}
// n shares, every one of the shape (count, parts, level) (MultipartyError::NoShares for n == 0)
static void check_shares(const fhe_b200_params* par, const fhe_b200_batch* const* shares, uint32_t n, u32 count,
                         u32 parts, u32 level) {
  REQUIRE(shares && n, FHE_B200_INVALID_ARGUMENT, "MultipartyError::NoShares");
  for (uint32_t i = 0; i < n; i++) {
    check_operand(par, shares[i]);
    REQUIRE(shares[i]->count == count && shares[i]->parts == parts && shares[i]->level == level,
            FHE_B200_INVALID_ARGUMENT, "share " + std::to_string(i) + " does not have the shape of the others");
  }
}

// entries [c0, c0 + n) of the shares: out item k = base item k + the sum of item c0 + k of every share.  An item is
// item_words words at word offset `part_off` of a share entry; base (nullable) and out point at the items of entry c0
// and have their own strides.
static void sum_shares(const fhe_b200_batch* const* shares, uint32_t n_sh, size_t part_off, size_t item_words,
                       const u64* base, size_t base_stride, u64* out, size_t out_stride, u32 c0, u32 n,
                       const LevelData& lv, cudaStream_t st) {
  const fhe_b200_params* par = shares[0]->par;
  const size_t src_stride = shares[0]->words_per_ct();
  std::vector<const u64*> src(n_sh);
  for (uint32_t i = 0; i < n_sh; i++) src[i] = shares[i]->d + (size_t)c0 * src_stride + part_off;
  launch_shares_sum(src.data(), n_sh, src_stride, base, base_stride, out, out_stride, n, item_words, lv.ctx_ids,
                    par->d_limbs, par->logn, st);
}

int fhe_b200_crp_generate(const fhe_b200_params* p, const uint8_t* seed, fhe_b200_batch* out, void* stream) {
  API_BEGIN
  REQUIRE(p && seed, FHE_B200_INVALID_ARGUMENT, "null argument");
  DeviceGuard g(p);
  REQUIRE(out, FHE_B200_INVALID_ARGUMENT, "null argument");
  check_output(p, out, out->count, 1, out->level);
  const EncSeed K = seed_words(seed);
  const LevelData& lv = p->level(out->level);
  ChunkRunner chunks(p, out->count, (cudaStream_t)stream);
  chunks.run([&](u32 c0, u32 n, cudaStream_t st) {
    launch_crp(out->d + (((size_t)c0 * lv.L) << p->logn), n, c0, K, lv.ctx_ids, p->d_limbs, p->logn, st);
  });
  FHE_CUDA(cudaGetLastError());
  out->repr = FHE_B200_NTT;
  API_END
}

int fhe_b200_pk_share(const fhe_b200_secret_key* sk, const fhe_b200_batch* crp, uint32_t variance, const uint8_t* seed,
                      fhe_b200_batch* out, void* stream) {
  API_BEGIN
  check_variance(variance);
  REQUIRE(sk && seed, FHE_B200_INVALID_ARGUMENT, "null argument");
  const fhe_b200_params* par = sk->par;
  check_operand(par, crp);
  REQUIRE(crp->parts == 1, FHE_B200_INVALID_ARGUMENT, "a crp batch holds one polynomial per entry");
  REQUIRE(crp->level == 0, FHE_B200_INVALID_LEVEL, "InvalidLevel: a public key share is made at level 0");
  check_output(par, out, crp->count, 1, 0);
  const EncSeed K = seed_words(seed);
  DeviceGuard g(par);
  const LevelData& lv = par->level(0);
  const u32 L = lv.L, logn = par->logn;
  ChunkRunner chunks(par, out->count, (cudaStream_t)stream);
  chunks.run([&](u32 c0, u32 n, cudaStream_t st) {
    Workspace ws(par, st);
    u64* e = ws.secret_words(((size_t)n * L) << logn);
    launch_cbd(e, n, c0, 8, 1, variance, K, lv.ctx_ids, par->d_limbs, logn, st);
    launch_ntt(e, e, n * L, lv.ctx_ids, par->d_limbs, logn, false, 1, false, st);
    const size_t off = ((size_t)c0 * L) << logn;
    launch_mbfv_share(SHARE_PK, sk->s.d, nullptr, crp->d + off, nullptr, e, out->d + off, n, lv.ctx_ids, par->d_limbs,
                      logn, st);
  });
  FHE_CUDA(cudaGetLastError());
  out->repr = FHE_B200_NTT;
  API_END
}

int fhe_b200_pk_aggregate(const fhe_b200_batch* const* shares, uint32_t n, const fhe_b200_batch* crp,
                          fhe_b200_batch* pk, void* stream) {
  API_BEGIN
  REQUIRE(crp, FHE_B200_INVALID_ARGUMENT, "null argument");
  const fhe_b200_params* par = crp->par;
  check_operand(par, crp);
  REQUIRE(crp->parts == 1, FHE_B200_INVALID_ARGUMENT, "a crp batch holds one polynomial per entry");
  REQUIRE(crp->level == 0, FHE_B200_INVALID_LEVEL, "InvalidLevel: a public key is made at level 0");
  check_shares(par, shares, n, crp->count, 1, 0);
  check_output(par, pk, crp->count, 2, 0);
  DeviceGuard g(par);
  const LevelData& lv = par->level(0);
  const size_t words = (size_t)lv.L << par->logn;
  ChunkRunner chunks(par, pk->count, (cudaStream_t)stream);
  chunks.run([&](u32 c0, u32 m, cudaStream_t st) {
    // PublicKey { c: (sum p0_i, crp) } (public_key_gen.rs:60-77)
    sum_shares(shares, n, 0, words, nullptr, 0, pk->d + 2 * (size_t)c0 * words, 2 * words, c0, m, lv, st);
    FHE_CUDA(cudaMemcpy2DAsync(pk->d + (2 * (size_t)c0 + 1) * words, 2 * words * 8, crp->d + (size_t)c0 * words,
                               words * 8, words * 8, m, cudaMemcpyDeviceToDevice, st));
  });
  FHE_CUDA(cudaGetLastError());
  pk->repr = FHE_B200_NTT;
  API_END
}

int fhe_b200_shares_sum(const fhe_b200_batch* const* shares, uint32_t n, fhe_b200_batch* out, void* stream) {
  API_BEGIN
  REQUIRE(out, FHE_B200_INVALID_ARGUMENT, "null argument");
  const fhe_b200_params* par = out->par;
  check_operand(par, out);
  check_shares(par, shares, n, out->count, out->parts, out->level);
  DeviceGuard g(par);
  const LevelData& lv = par->level(out->level);
  const size_t words = out->words_per_ct();
  ChunkRunner chunks(par, out->count, (cudaStream_t)stream);
  chunks.run([&](u32 c0, u32 m, cudaStream_t st) {
    sum_shares(shares, n, 0, words, nullptr, 0, out->d + (size_t)c0 * words, words, c0, m, lv, st);
  });
  FHE_CUDA(cudaGetLastError());
  API_END
}

int fhe_b200_sks_share(const fhe_b200_secret_key* sk_in, const fhe_b200_secret_key* sk_out, const fhe_b200_batch* ct,
                       uint32_t variance, const uint8_t* seed, fhe_b200_batch* out, void* stream) {
  API_BEGIN
  check_variance(variance);
  REQUIRE(sk_in && seed, FHE_B200_INVALID_ARGUMENT, "null argument");
  const fhe_b200_params* par = sk_in->par;
  REQUIRE(!sk_out || sk_out->par == par, FHE_B200_CONTEXT_MISMATCH, "ParameterMismatch: input and output keys");
  check_ciphertexts(par, ct);
  check_output(par, out, ct->count, 1, ct->level);
  const EncSeed K = seed_words(seed);
  DeviceGuard g(par);
  const LevelData& lv = par->level(ct->level);
  const u32 L = lv.L, logn = par->logn;
  ChunkRunner chunks(par, ct->count, (cudaStream_t)stream);
  chunks.run([&](u32 c0, u32 n, cudaStream_t st) {
    Workspace ws(par, st);
    u64* e = ws.secret_words(((size_t)n * L) << logn);
    launch_cbd(e, n, c0, 14, 1, variance, K, lv.ctx_ids, par->d_limbs, logn, st);
    launch_ntt(e, e, n * L, lv.ctx_ids, par->d_limbs, logn, false, 1, false, st);
    launch_mbfv_share(SHARE_SKS, sk_in->s.d, sk_out ? sk_out->s.d : nullptr, ct->d + ((2 * (size_t)c0 * L) << logn),
                      nullptr, e, out->d + (((size_t)c0 * L) << logn), n, lv.ctx_ids, par->d_limbs, logn, st);
  });
  FHE_CUDA(cudaGetLastError());
  out->repr = FHE_B200_NTT;
  API_END
}

int fhe_b200_sks_aggregate(const fhe_b200_batch* ct, const fhe_b200_batch* const* shares, uint32_t n,
                           fhe_b200_batch* out, void* stream) {
  API_BEGIN
  REQUIRE(ct, FHE_B200_INVALID_ARGUMENT, "null argument");
  const fhe_b200_params* par = ct->par;
  check_ciphertexts(par, ct);
  check_shares(par, shares, n, ct->count, 1, ct->level);
  check_output(par, out, ct->count, 2, ct->level);
  DeviceGuard g(par);
  const LevelData& lv = par->level(ct->level);
  const size_t words = (size_t)lv.L << par->logn;
  ChunkRunner chunks(par, ct->count, (cudaStream_t)stream);
  chunks.run([&](u32 c0, u32 m, cudaStream_t st) {
    // (c0 + sum h_i, c1) (secret_key_switch.rs:98-115)
    const size_t off = 2 * (size_t)c0 * words;
    sum_shares(shares, n, 0, words, ct->d + off, 2 * words, out->d + off, 2 * words, c0, m, lv, st);
    if (out != ct)
      FHE_CUDA(cudaMemcpy2DAsync(out->d + (2 * (size_t)c0 + 1) * words, 2 * words * 8,
                                 ct->d + (2 * (size_t)c0 + 1) * words, 2 * words * 8, words * 8, m,
                                 cudaMemcpyDeviceToDevice, st));
  });
  FHE_CUDA(cudaGetLastError());
  out->repr = FHE_B200_NTT;
  API_END
}

int fhe_b200_pks_share(const fhe_b200_secret_key* sk, const fhe_b200_batch* pk, const fhe_b200_batch* ct,
                       uint32_t variance, const uint8_t* seed, fhe_b200_batch* out, void* stream) {
  API_BEGIN
  check_variance(variance);
  REQUIRE(sk && seed, FHE_B200_INVALID_ARGUMENT, "null argument");
  const fhe_b200_params* par = sk->par;
  check_public_key(pk);
  REQUIRE(pk->par == par, FHE_B200_CONTEXT_MISMATCH, "ParameterMismatch: secret key and public key");
  check_ciphertexts(par, ct);
  check_output(par, out, ct->count, 2, ct->level);
  const EncSeed K = seed_words(seed);
  DeviceGuard g(par);
  const LevelData& lv = par->level(ct->level);
  const u32 L = lv.L, logn = par->logn;
  cudaStream_t user = (cudaStream_t)stream;
  Workspace key_ws(par, user);
  const u64* c = public_key_at_level(pk, ct->level, key_ws, user);
  ChunkRunner chunks(par, ct->count, user);
  chunks.run([&](u32 c0, u32 n, cudaStream_t st) {
    Workspace ws(par, st);
    u64* uee = ws.secret_words(((size_t)n * 3 * L) << logn);   // u, e0, e1
    launch_cbd(uee, n, c0, 15, 3, variance, K, lv.ctx_ids, par->d_limbs, logn, st);
    launch_ntt(uee, uee, n * 3 * L, lv.ctx_ids, par->d_limbs, logn, false, 1, false, st);
    const size_t off = ((2 * (size_t)c0 * L) << logn);
    launch_mbfv_share(SHARE_PKS, sk->s.d, nullptr, ct->d + off, c, uee, out->d + off, n, lv.ctx_ids, par->d_limbs, logn,
                      st);
  });
  FHE_CUDA(cudaGetLastError());
  out->repr = FHE_B200_NTT;
  API_END
}

int fhe_b200_pks_aggregate(const fhe_b200_batch* ct, const fhe_b200_batch* const* shares, uint32_t n,
                           fhe_b200_batch* out, void* stream) {
  API_BEGIN
  REQUIRE(ct, FHE_B200_INVALID_ARGUMENT, "null argument");
  const fhe_b200_params* par = ct->par;
  check_ciphertexts(par, ct);
  check_shares(par, shares, n, ct->count, 2, ct->level);
  check_output(par, out, ct->count, 2, ct->level);
  DeviceGuard g(par);
  const LevelData& lv = par->level(ct->level);
  const size_t words = (size_t)lv.L << par->logn;
  ChunkRunner chunks(par, ct->count, (cudaStream_t)stream);
  chunks.run([&](u32 c0, u32 m, cudaStream_t st) {
    // (c0 + sum h0_i, sum h1_i) (public_key_switch.rs:95-112)
    const size_t off = 2 * (size_t)c0 * words;
    sum_shares(shares, n, 0, words, ct->d + off, 2 * words, out->d + off, 2 * words, c0, m, lv, st);
    sum_shares(shares, n, words, words, nullptr, 0, out->d + off + words, 2 * words, c0, m, lv, st);
  });
  FHE_CUDA(cudaGetLastError());
  out->repr = FHE_B200_NTT;
  API_END
}

// RelinKeyGenerator (relin_key_gen.rs:36-96): the party's secret key, the level-0 CRPs a_i (one per level-0 limb,
// borrowed as in the reference) and u on the device, erased when the generator is freed.
struct fhe_b200_rkg {
  ParamsRef par;   // a reference of its own: freeing the generator never reads sk
  const fhe_b200_secret_key* sk;
  const fhe_b200_batch* crp;
  u32 variance;
  SecretBuffer u;   // [Lmax][N] NTT
  fhe_b200_rkg(const fhe_b200_secret_key* k, const fhe_b200_batch* c, u32 v)
      : par(static_cast<const fhe_b200_params*>(k->par)), sk(k), crp(c), variance(v),
        u(par->device, (size_t)par->Lmax << par->logn) {}
};

int fhe_b200_rkg_create(const fhe_b200_secret_key* sk, const fhe_b200_batch* crp, uint32_t variance,
                        const uint8_t* seed, fhe_b200_rkg** out, void* stream) {
  API_BEGIN
  check_variance(variance);
  REQUIRE(sk && seed && out, FHE_B200_INVALID_ARGUMENT, "null argument");
  const fhe_b200_params* par = sk->par;
  REQUIRE(par->Lmax > 1, FHE_B200_UNSUPPORTED, "EvaluationKeyError::KeySwitchingNotSupported: a single modulus");
  check_operand(par, crp);
  REQUIRE(crp->parts == 1, FHE_B200_INVALID_ARGUMENT, "a crp batch holds one polynomial per entry");
  REQUIRE(crp->level == 0, FHE_B200_INVALID_LEVEL, "InvalidLevel: the relinearization key protocol runs at level 0");
  REQUIRE(crp->count == par->Lmax, FHE_B200_INVALID_ARGUMENT,
          "MultipartyError::InvalidCommonRandomPolynomialCount: " + std::to_string(crp->count) + ", expected " +
              std::to_string(par->Lmax));
  const EncSeed K = seed_words(seed);
  DeviceGuard g(par);
  const LevelData& lv = par->level(0);
  std::unique_ptr<fhe_b200_rkg> r(new fhe_b200_rkg(sk, crp, variance));
  cudaStream_t st = (cudaStream_t)stream;
  launch_cbd(r->u.d, 1, 0, 9, 1, variance, K, lv.ctx_ids, par->d_limbs, par->logn, st);   // u: role 9
  launch_ntt(r->u.d, r->u.d, lv.L, lv.ctx_ids, par->d_limbs, par->logn, false, 1, false, st);
  FHE_CUDA(cudaGetLastError());
  *out = r.release();
  API_END
}

int fhe_b200_rkg_free(fhe_b200_rkg* r) {
  delete r;
  return FHE_B200_OK;
}

// one round of the generator: entries i of h0, h1 (1-part level-0 batches of Lmax entries) from the errors of roles
// role0, role0 + 1 (state word 15 = i)
static void rkg_round(const fhe_b200_rkg* r, MbfvShare kind, const fhe_b200_batch* x, const fhe_b200_batch* y,
                      const uint8_t* seed, fhe_b200_batch* h0, fhe_b200_batch* h1, u32 role0, cudaStream_t user) {
  const fhe_b200_params* par = r->par;
  const u32 L = par->Lmax, logn = par->logn;
  check_output(par, h0, L, 1, 0);
  check_output(par, h1, L, 1, 0);
  REQUIRE(h0 != h1, FHE_B200_INVALID_ARGUMENT, "h0 and h1 must be different batches");
  const EncSeed K = seed_words(seed);
  DeviceGuard g(par);
  const LevelData& lv = par->level(0);
  ChunkRunner chunks(par, L, user, std::max(1u, chunk_size() / (2 * L)));
  chunks.run([&](u32 c0, u32 n, cudaStream_t st) {
    Workspace ws(par, st);
    u64* e = ws.secret_words(((size_t)n * 2 * L) << logn);
    launch_cbd(e, n, c0, role0, 2, r->variance, K, lv.ctx_ids, par->d_limbs, logn, st, L);
    launch_ntt(e, e, n * 2 * L, lv.ctx_ids, par->d_limbs, logn, false, 1, false, st);
    const size_t off = ((size_t)c0 * L) << logn;
    launch_mbfv_share(kind, r->sk->s.d, nullptr, x->d + off, y ? y->d + off : nullptr, e, h0->d + off, n, lv.ctx_ids,
                      par->d_limbs, logn, st, r->u.d, h1->d + off, c0);
  });
  FHE_CUDA(cudaGetLastError());
  h0->repr = h1->repr = FHE_B200_NTT;
}

int fhe_b200_rkg_round1(const fhe_b200_rkg* r, const uint8_t* seed, fhe_b200_batch* h0, fhe_b200_batch* h1,
                        void* stream) {
  API_BEGIN
  REQUIRE(r && seed, FHE_B200_INVALID_ARGUMENT, "null argument");
  rkg_round(r, SHARE_RKG1, r->crp, nullptr, seed, h0, h1, 10, (cudaStream_t)stream);
  API_END
}

int fhe_b200_rkg_round2(const fhe_b200_rkg* r, const fhe_b200_batch* r1_h0, const fhe_b200_batch* r1_h1,
                        const uint8_t* seed, fhe_b200_batch* h0, fhe_b200_batch* h1, void* stream) {
  API_BEGIN
  REQUIRE(r && seed, FHE_B200_INVALID_ARGUMENT, "null argument");
  const fhe_b200_params* par = r->par;
  for (const fhe_b200_batch* b : {r1_h0, r1_h1}) {
    check_operand(par, b);
    REQUIRE(b->parts == 1 && b->count == par->Lmax, FHE_B200_INVALID_ARGUMENT,
            "a round-1 aggregate holds one polynomial per level-0 limb");
    REQUIRE(b->level == 0, FHE_B200_INVALID_LEVEL, "InvalidLevel: the round-1 aggregate is at level 0");
  }
  rkg_round(r, SHARE_RKG2, r1_h0, r1_h1, seed, h0, h1, 12, (cudaStream_t)stream);
  API_END
}

int fhe_b200_rkg_aggregate(const fhe_b200_batch* const* h0s, const fhe_b200_batch* const* h1s, uint32_t n,
                           const fhe_b200_batch* r1_h1, fhe_b200_ksk** out, void* stream) {
  API_BEGIN
  REQUIRE(r1_h1 && out, FHE_B200_INVALID_ARGUMENT, "null argument");
  const fhe_b200_params* par = r1_h1->par;
  const u32 L = par->Lmax, logn = par->logn;
  REQUIRE(L > 1, FHE_B200_UNSUPPORTED, "EvaluationKeyError::KeySwitchingNotSupported: a single modulus");
  check_operand(par, r1_h1);
  REQUIRE(r1_h1->parts == 1 && r1_h1->count == L, FHE_B200_INVALID_ARGUMENT,
          "a round-1 aggregate holds one polynomial per level-0 limb");
  REQUIRE(r1_h1->level == 0, FHE_B200_INVALID_LEVEL, "InvalidLevel: the round-1 aggregate is at level 0");
  check_shares(par, h0s, n, L, 1, 0);
  check_shares(par, h1s, n, L, 1, 0);
  DeviceGuard g(par);
  const LevelData& lv = par->level(0);
  const size_t words = (size_t)L << logn, row = (size_t)1 << logn;
  std::unique_ptr<fhe_b200_ksk> k = make_ksk(par, 0, 0, L, L, 0);
  std::vector<const fhe_b200_batch*> all(h0s, h0s + n);
  all.insert(all.end(), h1s, h1s + n);
  const fhe_b200_batch* r1[] = {r1_h1};
  u64 *k0 = k->k0, *k1 = k->k1;
  // digit i of the key: c0_i = sum h0'_i + sum h1'_i, c1_i = r1_h1_i, written straight into the key's device layout
  // [limb j][digit i][N] (relin_key_gen.rs:299-350): item i of the sum starts at digit i's row, rows L * N apart
  ChunkRunner chunks(par, L, (cudaStream_t)stream, std::max(1u, chunk_size() / L));
  chunks.run([&](u32 c0, u32 m, cudaStream_t st) {
    std::vector<const u64*> src(all.size());
    for (size_t i = 0; i < all.size(); i++) src[i] = all[i]->d + (size_t)c0 * words;
    launch_shares_sum(src.data(), (u32)src.size(), words, nullptr, 0, k0 + c0 * row, row, m, words, lv.ctx_ids,
                      par->d_limbs, logn, st, L * row);
    const u64* s1 = r1[0]->d + (size_t)c0 * words;
    launch_shares_sum(&s1, 1, words, nullptr, 0, k1 + c0 * row, row, m, words, lv.ctx_ids, par->d_limbs, logn, st,
                      L * row);
  });
  FHE_CUDA(cudaGetLastError());
  *out = k.release();
  API_END
}

int fhe_b200_decryption_aggregate(const fhe_b200_encoder* e, const fhe_b200_batch* ct,
                                  const fhe_b200_batch* const* shares, uint32_t n, fhe_b200_batch* pts_out,
                                  void* stream) {
  API_BEGIN
  REQUIRE(e, FHE_B200_INVALID_ARGUMENT, "null argument");
  const fhe_b200_params* par = e->par;
  DeviceGuard g(par);   // NO_DEVICE first: an encoder, unlike a batch, exists on a host-only parameter set
  check_ciphertexts(par, ct);
  check_shares(par, shares, n, ct->count, 1, ct->level);
  check_output(par, pts_out, ct->count, 1, ct->level);
  REQUIRE(par->t_small && par->t_mod.t < par->moduli[0], FHE_B200_UNSUPPORTED,
          "Plaintext::from_shares needs t below the first ciphertext modulus");
  const LevelData& lv = par->level(ct->level);
  const u32 L = lv.L, logn = par->logn;
  const size_t words = (size_t)L << logn;
  const bool q0_context = par->plaintext_moduli_count() == 1;
  ChunkRunner chunks(par, ct->count, (cudaStream_t)stream);
  chunks.run([&](u32 c0, u32 m, cudaStream_t st) {
    Workspace ws(par, st);
    // c = c0 + sum h_i (secret_key_switch.rs:150-154), taken to the power basis and scaled by t / Q into limb 0 of the
    // plaintext context; only that row is needed because the scaled value v has |v| <= t / 2 < q_0 / 2
    u64* c = ws.secret_words(m * words);
    sum_shares(shares, n, 0, words, ct->d + 2 * (size_t)c0 * words, 2 * words, c, words, c0, m, lv, st);
    launch_ntt(c, c, m * L, lv.ctx_ids, par->d_limbs, logn, true, 1, false, st);
    u64* w = ws.secret_words((size_t)m << logn);
    launch_scale(lv.plain.dev, par->d_limbs, c, w, nullptr, m, 1, 0, 1, 0, logn, st);
    // w = ((v + t) mod Q_p) mod t over the plaintext context Q_p (:164-173).  With one plaintext modulus Q_p = q_0 and
    // this is try_decrypt's lift; with more, (v + t) mod Q_p = v + t and w = v mod t.
    const LimbDev& q0 = par->h_limbs[0];
    if (q0_context) launch_decrypt_epilogue(w, (size_t)m << logn, PlainMod{q0.p, q0.bhi, q0.blo}, par->t_mod, st);
    else launch_from_shares_epilogue(w, (size_t)m << logn, q0.p, par->t_mod, st);
    launch_ntt(w, pts_out->d + (size_t)c0 * words, m * L, lv.ctx_ids, par->d_limbs, logn, false, L, lv.lift_reduce,
               st);
  });
  FHE_CUDA(cudaGetLastError());
  pts_out->repr = FHE_B200_NTT;
  API_END
}

int fhe_b200_mul(const fhe_b200_batch* a, const fhe_b200_batch* b, fhe_b200_batch* out3, void* stream) {
  API_BEGIN
  REQUIRE(a && b && out3, FHE_B200_INVALID_ARGUMENT, "null argument");
  check_same(a, b);
  check_same(a, out3);
  REQUIRE(!a->mul_basis, FHE_B200_CONTEXT_MISMATCH, "PolynomialContextMismatch");
  REQUIRE(a->parts >= 1 && b->parts >= 1 && out3->parts == a->parts + b->parts - 1, FHE_B200_BAD_POLY_COUNT,
          "MultiplicationPolynomialCount: expected n x m -> n + m - 1 parts");
  REQUIRE(a->count == b->count && a->count == out3->count, FHE_B200_INVALID_ARGUMENT, "batch sizes differ");
  need_repr(a, FHE_B200_NTT);
  need_repr(b, FHE_B200_NTT);
  DeviceGuard g(a->par);
  cudaStream_t st_user = (cudaStream_t)stream;
  const fhe_b200_params* par = a->par;
  const LevelData& lv = par->level(a->level);
  const size_t row = (size_t)1 << par->logn;
  const u32 na = a->parts, nb = b->parts, nc = na + nb - 1;
  ChunkRunner chunks(par, a->count, st_user);
  chunks.run([&](u32 c0, u32 n, cudaStream_t st) {
    Workspace ws(par, st);
    u64* o = out3->d + (size_t)c0 * nc * lv.L * row;
    const u64* pa = a->d + (size_t)c0 * na * lv.L * row;
    const u64* pb = b->d + (size_t)c0 * nb * lv.L * row;
    if (na == 2 && nb == 2) mul_core(par, lv, pa, pb, n, o, nullptr, 0, ws, st);
    else mul_core_parts(par, lv, pa, na, pb, nb, n, o, ws, st);
    // rq/scaler.rs:97-115 forward NTT of the scaled result
    launch_ntt(o, o, n * nc * lv.L, lv.ctx_ids, par->d_limbs, par->logn, false, 1, false, st);
  });
  FHE_CUDA(cudaGetLastError());
  out3->repr = FHE_B200_NTT;
  API_END
}

static void check_ksk(const fhe_b200_ksk* k, const fhe_b200_params* par, u32 level) {
  REQUIRE(k->par == par, FHE_B200_CONTEXT_MISMATCH, "ParameterMismatch: key belongs to other parameters");
  REQUIRE(k->ct_level == level, FHE_B200_INVALID_LEVEL, "InvalidLevel: key is for another ciphertext level");
}

// a keyed call's key list and index: present, non-empty, no NULL key
static KeySet key_list(const fhe_b200_ksk* const* keys, u32 n_keys, const u32* index) {
  REQUIRE(keys && n_keys && index, FHE_B200_INVALID_ARGUMENT, "null key list or index, or no keys");
  for (u32 i = 0; i < n_keys; i++) REQUIRE(keys[i], FHE_B200_INVALID_ARGUMENT, "null key");
  return {keys, n_keys, index};
}

// what a key switch over several keys needs beyond each key's own checks: one key level, digit count and base for
// every key, and every index of the `count` ciphertexts naming a key
static void check_key_set(const KeySet& K, u32 count) {
  const fhe_b200_ksk* k0 = K.keys[0];
  for (u32 i = 1; i < K.n; i++)
    REQUIRE(K.keys[i]->ksk_level == k0->ksk_level && K.keys[i]->n_dig == k0->n_dig &&
                K.keys[i]->log_base == k0->log_base,
            FHE_B200_INVALID_ARGUMENT, "keys of one call differ in key level, digit count or base");
  if (K.index)
    for (u32 c = 0; c < count; c++)
      REQUIRE(K.index[c] < K.n, FHE_B200_INVALID_ARGUMENT, "key index " + std::to_string(K.index[c]) + " of ciphertext " +
                                                               std::to_string(c) + " beyond the key list");
}

static void check_ksks(const KeySet& K, const fhe_b200_params* par, u32 level, u32 count) {
  for (u32 i = 0; i < K.n; i++) check_ksk(K.keys[i], par, level);
  check_key_set(K, count);
}

static void relinearize_run(const fhe_b200_batch* ct3, const KeySet& rk, fhe_b200_batch* out2, void* stream) {
  REQUIRE(ct3 && rk.keys[0] && out2, FHE_B200_INVALID_ARGUMENT, "null argument");
  check_same(ct3, out2);
  REQUIRE(!ct3->mul_basis, FHE_B200_CONTEXT_MISMATCH, "PolynomialContextMismatch");
  REQUIRE(ct3->parts == 3 && out2->parts == 2, FHE_B200_BAD_POLY_COUNT, "InvalidPolynomialCount: expected 3 -> 2");
  REQUIRE(ct3->count == out2->count, FHE_B200_INVALID_ARGUMENT, "batch sizes differ");
  need_repr(ct3, FHE_B200_NTT);
  check_ksks(rk, ct3->par, ct3->level, ct3->count);
  DeviceGuard g(ct3->par);
  cudaStream_t st_user = (cudaStream_t)stream;
  const fhe_b200_params* par = ct3->par;
  const LevelData& lv = par->level(ct3->level);
  const size_t row = (size_t)1 << par->logn, L = lv.L;
  ChunkRunner chunks(par, ct3->count, st_user);
  chunks.run([&](u32 c0, u32 n, cudaStream_t st) {
    Workspace ws(par, st);
    const u64* src = ct3->d + (size_t)c0 * 3 * L * row;
    u64* dst = out2->d + (size_t)c0 * 2 * L * row;
    u64* c2 = ws.words((size_t)n * L * row);
    FHE_CUDA(cudaMemcpy2DAsync(dst, 2 * L * row * 8, src, 3 * L * row * 8, 2 * L * row * 8, n, cudaMemcpyDeviceToDevice, st));
    FHE_CUDA(cudaMemcpy2DAsync(c2, L * row * 8, src + 2 * L * row, 3 * L * row * 8, L * row * 8, n, cudaMemcpyDeviceToDevice, st));
    // relinearization_key.rs:85: c2 -> power basis
    launch_ntt(c2, c2, n * (u32)L, lv.ctx_ids, par->d_limbs, par->logn, true, 1, false, st);
    key_switch_apply(par, rk.from(c0), c2, n, dst, 1, nullptr, ws, st);
  });
  FHE_CUDA(cudaGetLastError());
  out2->repr = FHE_B200_NTT;
}

int fhe_b200_relinearize(const fhe_b200_batch* ct3, const fhe_b200_ksk* rk, fhe_b200_batch* out2, void* stream) {
  API_BEGIN
  relinearize_run(ct3, {&rk, 1, nullptr}, out2, stream);
  API_END
}

int fhe_b200_relinearize_keyed(const fhe_b200_batch* ct3, const fhe_b200_ksk* const* rks, uint32_t n_keys,
                               const uint32_t* key_index, fhe_b200_batch* out2, void* stream) {
  API_BEGIN
  relinearize_run(ct3, key_list(rks, n_keys, key_index), out2, stream);
  API_END
}

static void mul_relin_run(const fhe_b200_batch* a, const fhe_b200_batch* b, const KeySet& rk, int mod_switch,
                          fhe_b200_batch* out2, void* stream) {
  REQUIRE(a && b && rk.keys[0] && out2, FHE_B200_INVALID_ARGUMENT, "null argument");
  check_same(a, b);
  REQUIRE(a->par == out2->par, FHE_B200_CONTEXT_MISMATCH, "ParameterMismatch");
  REQUIRE(!a->mul_basis && !out2->mul_basis, FHE_B200_CONTEXT_MISMATCH, "PolynomialContextMismatch");
  REQUIRE(a->parts == 2 && b->parts == 2 && out2->parts == 2, FHE_B200_BAD_POLY_COUNT,
          "MultiplicationPolynomialCount: expected 2 x 2 -> 2");
  REQUIRE(a->count == b->count && a->count == out2->count, FHE_B200_INVALID_ARGUMENT, "batch sizes differ");
  need_repr(a, FHE_B200_NTT);
  need_repr(b, FHE_B200_NTT);
  check_ksks(rk, a->par, a->level, a->count);
  const fhe_b200_params* par = a->par;
  const LevelData& lv = par->level(a->level);
  if (mod_switch) {
    REQUIRE(lv.L >= 2, FHE_B200_NO_MORE_CONTEXT, "NoMoreContext");  // mul.rs:155-162
    REQUIRE(out2->level == a->level + 1, FHE_B200_INVALID_LEVEL, "output batch must be one level down");
  } else {
    REQUIRE(out2->level == a->level, FHE_B200_INVALID_LEVEL, "output batch must be at the operand level");
  }
  DeviceGuard g(par);
  const size_t row = (size_t)1 << par->logn, L = lv.L;
  ChunkRunner chunks(par, a->count, (cudaStream_t)stream);
  chunks.run([&](u32 c0, u32 n, cudaStream_t st) {
    Workspace ws(par, st);
    u64* o = mod_switch ? ws.words((size_t)n * 2 * L * row) : out2->d + (size_t)c0 * 2 * L * row;
    u64* c2 = ws.words((size_t)n * L * row);
    mul_core(par, lv, a->d + (size_t)c0 * 2 * L * row, b->d + (size_t)c0 * 2 * L * row, n, o, c2, 1, ws, st);
    // c0, c1 back to NTT.  c2 stays in power basis: mul.rs:206 + :212 forward- then inverse-transform it,
    // and backward(forward(x)) == x for reduced x (ntt/mod.rs:73-74), so skipping both is bit-exact.
    launch_ntt(o, o, n * 2 * (u32)L, lv.ctx_ids, par->d_limbs, par->logn, false, 1, false, st);
    key_switch_apply(par, rk.from(c0), c2, n, o, 1, nullptr, ws, st);
    if (mod_switch) {  // Ciphertext::switch_down, ciphertext.rs:148-161
      launch_ntt(o, o, n * 2 * (u32)L, lv.ctx_ids, par->d_limbs, par->logn, true, 1, false, st);
      u64* dst = out2->d + (size_t)c0 * 2 * (L - 1) * row;
      launch_switch_down(lv.sd, o, dst, n * 2, (u32)L, lv.ctx_ids, par->d_limbs, par->logn, st);
      const LevelData& nl = par->level(a->level + 1);
      launch_ntt(dst, dst, n * 2 * (u32)(L - 1), nl.ctx_ids, par->d_limbs, par->logn, false, 1, false, st);
    }
  });
  FHE_CUDA(cudaGetLastError());
  out2->repr = FHE_B200_NTT;
}

int fhe_b200_mul_relin(const fhe_b200_batch* a, const fhe_b200_batch* b, const fhe_b200_ksk* rk, int mod_switch,
                       fhe_b200_batch* out2, void* stream) {
  API_BEGIN
  mul_relin_run(a, b, {&rk, 1, nullptr}, mod_switch, out2, stream);
  API_END
}

int fhe_b200_mul_relin_keyed(const fhe_b200_batch* a, const fhe_b200_batch* b, const fhe_b200_ksk* const* rks,
                             uint32_t n_keys, const uint32_t* key_index, int mod_switch, fhe_b200_batch* out2,
                             void* stream) {
  API_BEGIN
  mul_relin_run(a, b, key_list(rks, n_keys, key_index), mod_switch, out2, stream);
  API_END
}

// out[g] = switch_to_level(out.level, relinearizes(sum_i a[g*n + i] * b[g*n + i])) (examples/mulpir.rs:176-183; rk
// null: the 3-part sum).  An operand of n_terms entries is shared by every group.  The chunks run over groups, so the
// terms of one group stay on one stream; inside a chunk, slices of at most chunk_size() products go through mul_core
// (power basis, no forward NTT) and segment_sum adds them into the group accumulator.  The NTT is linear on canonical
// residues, so transforming the sum once gives the words of the reference's sum of transformed products; c2 stays in
// power basis for the key switch, as in mul_relin.
static void dot_product_run(const fhe_b200_batch* a, const fhe_b200_batch* b, uint32_t n_terms, const KeySet* rk,
                            fhe_b200_batch* out, void* stream) {
  REQUIRE(a && b && out && a != out && b != out, FHE_B200_INVALID_ARGUMENT, "null or aliased argument");
  REQUIRE(!rk || rk->keys[0], FHE_B200_INVALID_ARGUMENT, "null key");
  REQUIRE(a->par == b->par && a->par == out->par, FHE_B200_CONTEXT_MISMATCH,
          "ParameterMismatch: batches use different parameters");
  REQUIRE(!a->mul_basis && !b->mul_basis && !out->mul_basis, FHE_B200_CONTEXT_MISMATCH, "PolynomialContextMismatch");
  const u32 P = rk ? 2 : 3;
  REQUIRE(a->parts == 2 && b->parts == 2 && out->parts == P, FHE_B200_BAD_POLY_COUNT,
          rk ? "MultiplicationPolynomialCount: expected 2 x 2 -> 2" : "MultiplicationPolynomialCount: expected 2 x 2 -> 3");
  const size_t total = (size_t)out->count * n_terms;
  REQUIRE(n_terms > 0 && (a->count == total || a->count == n_terms) && (b->count == total || b->count == n_terms),
          FHE_B200_INVALID_ARGUMENT, "DotProductError::OperandCountMismatch");
  REQUIRE(a->level == b->level, FHE_B200_INVALID_LEVEL, "InvalidLevel: operands are at different levels");
  REQUIRE(out->level >= a->level, FHE_B200_INVALID_LEVEL, "InvalidLevel: output below the operand level");
  need_repr(a, FHE_B200_NTT);
  need_repr(b, FHE_B200_NTT);
  if (rk) check_ksks(*rk, a->par, a->level, out->count);
  const fhe_b200_params* par = a->par;
  DeviceGuard g(par);
  const LevelData& lv = par->level(a->level);
  const LevelData& ol = par->level(out->level);
  const u32 L = lv.L, logn = par->logn, S = chunk_size();
  const size_t row = (size_t)1 << logn, W = 2 * L * row, Wo = P * ol.L * row;
  ChunkRunner chunks(par, out->count, (cudaStream_t)stream, std::max(1u, S / n_terms));
  chunks.run([&](u32 g0, u32 ng, cudaStream_t st) {
    Workspace ws(par, st);
    // terms of one group per slice: a chunk of several groups holds at most S products and takes one slice
    const u32 tps = ng > 1 ? n_terms : std::min(S, n_terms);
    // the products of the chunk's terms [i0, i0 + m) of each group: a shared operand is repeated ng times
    auto operand = [&](const fhe_b200_batch* x, u32 i0) -> const u64* {
      if (x->count == total) return x->d + ((size_t)g0 * n_terms + i0) * W;
      if (ng == 1) return x->d + (size_t)i0 * W;
      const size_t run = (size_t)n_terms * W;
      u64* rep = ws.words(ng * run);
      FHE_CUDA(cudaMemcpyAsync(rep, x->d, run * 8, cudaMemcpyDeviceToDevice, st));
      for (u32 k = 1; k < ng; k *= 2)
        FHE_CUDA(cudaMemcpyAsync(rep + k * run, rep, std::min(k, ng - k) * run * 8, cudaMemcpyDeviceToDevice, st));
      return rep;
    };
    const bool direct = out->level == a->level;
    u64* o = direct ? out->d + (size_t)g0 * Wo : ws.words(ng * P * L * row);
    u64* c2 = rk ? ws.words(ng * L * row) : nullptr;
    u64* prod = ws.words((size_t)ng * tps * 3 * L * row);
    for (u32 i0 = 0; i0 < n_terms; i0 += tps) {
      const u32 m = std::min(tps, n_terms - i0);
      {
        Workspace slice(par, st);
        mul_core(par, lv, operand(a, i0), operand(b, i0), ng * m, prod, nullptr, 0, slice, st);
      }
      // (c0, c1[, c2]) into o, c2 into its own buffer when it is relinearized
      launch_segment_sum(prod, 3 * L * row, m, o, P * L * row, c2, L * row, P * L, ng, 3 * L * row, i0 > 0,
                         lv.ctx_ids, par->d_limbs, logn, st);
    }
    if (rk) {
      // relinearization_key.rs:70-103 on the sum: (c0, c1) to NTT, c2 switched from the power basis
      launch_ntt(o, o, ng * 2 * L, lv.ctx_ids, par->d_limbs, logn, false, 1, false, st);
      key_switch_apply(par, rk->from(g0), c2, ng, o, 1, nullptr, ws, st);
      if (!direct) launch_ntt(o, o, ng * 2 * L, lv.ctx_ids, par->d_limbs, logn, true, 1, false, st);
    }
    // Ciphertext::switch_to_level (ciphertext.rs:164-186): each switch_down goes through the power basis; the
    // transforms between two of them cancel (backward(forward(x)) == x for reduced x), so only the last one runs
    u64* cur = o;
    for (u32 l = a->level; l < out->level; l++) {
      const LevelData& from = par->level(l);
      u64* nxt = l + 1 == out->level ? out->d + (size_t)g0 * Wo : ws.words(ng * P * (from.L - 1) * row);
      launch_switch_down(from.sd, cur, nxt, ng * P, from.L, from.ctx_ids, par->d_limbs, logn, st);
      cur = nxt;
    }
    if (!rk || !direct) launch_ntt(cur, cur, ng * P * ol.L, ol.ctx_ids, par->d_limbs, logn, false, 1, false, st);
  });
  FHE_CUDA(cudaGetLastError());
  out->repr = FHE_B200_NTT;
}

int fhe_b200_dot_product(const fhe_b200_batch* a, const fhe_b200_batch* b, uint32_t n_terms, const fhe_b200_ksk* rk,
                         fhe_b200_batch* out, void* stream) {
  API_BEGIN
  const KeySet K{&rk, 1, nullptr};
  dot_product_run(a, b, n_terms, rk ? &K : nullptr, out, stream);
  API_END
}

int fhe_b200_dot_product_keyed(const fhe_b200_batch* a, const fhe_b200_batch* b, uint32_t n_terms,
                               const fhe_b200_ksk* const* rks, uint32_t n_keys, const uint32_t* key_index,
                               fhe_b200_batch* out, void* stream) {
  API_BEGIN
  const KeySet K = key_list(rks, n_keys, key_index);
  dot_product_run(a, b, n_terms, &K, out, stream);
  API_END
}

// ---- custom multiplication strategies
int fhe_b200_multiplicator_create(const fhe_b200_params* p, uint32_t level, const uint8_t* lhs_num, uint32_t lhs_num_len,
                                  const uint8_t* lhs_den, uint32_t lhs_den_len, const uint8_t* rhs_num,
                                  uint32_t rhs_num_len, const uint8_t* rhs_den, uint32_t rhs_den_len,
                                  const uint64_t* extended_basis, uint32_t n_basis, const uint64_t* psi,
                                  const uint8_t* post_num, uint32_t post_num_len, const uint8_t* post_den,
                                  uint32_t post_den_len, fhe_b200_multiplicator** out) {
  API_BEGIN
  REQUIRE(p && out && extended_basis && n_basis && lhs_num && lhs_den && rhs_num && rhs_den && post_num && post_den,
          FHE_B200_INVALID_ARGUMENT, "null argument");
  REQUIRE(n_basis <= (u32)kMaxPos, FHE_B200_UNSUPPORTED, "too many limbs");
  const LevelData& lv = p->level(level);   // context_at_level: InvalidLevel when out of range
  DeviceGuard g(p);
  std::unique_ptr<fhe_b200_multiplicator> m(new fhe_b200_multiplicator(p));
  m->level = level;
  m->L = lv.L;
  m->K = n_basis;
  m->mul_moduli.assign(extended_basis, extended_basis + n_basis);
  // Context::new(extended_basis) (rq/context.rs:42-92): distinct NTT-friendly primes
  for (u32 i = 0; i < n_basis; i++) {
    const u64 q = extended_basis[i];
    for (u32 j = 0; j < i; j++) REQUIRE(extended_basis[j] != q, FHE_B200_INVALID_MODULUS, "DuplicateModuli");
    REQUIRE(q >= 2 && (q >> 62) == 0, FHE_B200_INVALID_MODULUS, "InvalidModulus: " + std::to_string(q));
    REQUIRE(q % (2 * (u64)p->N) == 1 && is_prime_u64(q), FHE_B200_NTT_UNAVAILABLE,
            "modulus does not support the NTT: " + std::to_string(q));
  }
  m->plan_primes = p->primes;
  m->h_limbs = p->h_limbs;
  std::memset(&m->mul_ids, 0, sizeof(RowIds));
  m->mul_ids.limbs_per_poly = n_basis;
  for (u32 i = 0; i < n_basis; i++) {
    const u64 q = extended_basis[i];
    int idx = prime_index(m->plan_primes, q);
    if (idx >= 0 && psi && psi[i] != p->psi[(size_t)idx] && (size_t)idx < p->primes.size())
      throw FheError(FHE_B200_INVALID_ARGUMENT, "psi differs from the parameter set's root for " + std::to_string(q));
    if (idx < 0) {
      const u64 r = psi ? psi[i] : default_psi(q, p->N);
      NttTablesH t = make_ntt_tables(q, p->N, r);
      idx = (int)m->plan_primes.size();
      m->plan_primes.push_back(q);
      m->h_limbs.push_back(make_limb_dev(q, t, m->uploads));
    }
    m->mul_ids.ids[i] = (unsigned short)idx;
  }
  m->d_limbs = m->uploads.put(m->h_limbs);
  std::vector<u64> base(p->moduli.begin(), p->moduli.begin() + lv.L);
  RnsContextH from(base), to(m->mul_moduli);
  auto factor = [](const uint8_t* b, uint32_t n) { return BigUint::from_le_bytes(b, n); };
  const BigUint ln = factor(lhs_num, lhs_num_len), ld = factor(lhs_den, lhs_den_len);
  const BigUint rn = factor(rhs_num, rhs_num_len), rd = factor(rhs_den, rhs_den_len);
  const BigUint pn = factor(post_num, post_num_len), pd = factor(post_den, post_den_len);
  REQUIRE(!ld.is_zero() && !rd.is_zero() && !pd.is_zero(), FHE_B200_INVALID_ARGUMENT, "zero denominator");
  m->ext_l.h = make_scaler_tables(from, to, ln, ld);
  m->ext_r.h = make_scaler_tables(from, to, rn, rd);
  m->down.h = make_scaler_tables(to, from, pn, pd);
  auto common = [&](const ScalerData& sd, const std::vector<u64>& x, const std::vector<u64>& y) {
    u32 n = 0;
    if (sd.h.is_one)
      while (n < x.size() && n < y.size() && x[n] == y[n]) n++;
    return n;
  };
  m->nc_l = common(m->ext_l, base, m->mul_moduli);
  m->nc_r = common(m->ext_r, base, m->mul_moduli);
  m->nc_d = common(m->down, m->mul_moduli, base);
  upload_scaler_tables(m->ext_l, m->mul_moduli, m->plan_primes, m->uploads);
  upload_scaler_tables(m->ext_r, m->mul_moduli, m->plan_primes, m->uploads);
  upload_scaler_tables(m->down, base, m->plan_primes, m->uploads);
  *out = m.release();
  API_END
}

int fhe_b200_multiplicator_free(fhe_b200_multiplicator* m) {
  delete m;
  return FHE_B200_OK;
}

int fhe_b200_multiplicator_multiply(const fhe_b200_multiplicator* m, const fhe_b200_batch* a, const fhe_b200_batch* b,
                                    const fhe_b200_ksk* rk, int mod_switch, fhe_b200_batch* out, void* stream) {
  API_BEGIN
  REQUIRE(m && a && b && out, FHE_B200_INVALID_ARGUMENT, "null argument");
  const fhe_b200_params* par = m->par;
  REQUIRE(a->par == par && b->par == par && out->par == par, FHE_B200_CONTEXT_MISMATCH, "ParameterMismatch");
  REQUIRE(a->level == m->level && b->level == m->level, FHE_B200_INVALID_LEVEL, "InvalidLevel");  // mul.rs:168-181
  REQUIRE(!a->mul_basis && !b->mul_basis && !out->mul_basis, FHE_B200_CONTEXT_MISMATCH, "PolynomialContextMismatch");
  const u32 out_parts = rk ? 2 : 3;
  REQUIRE(a->parts == 2 && b->parts == 2 && out->parts == out_parts, FHE_B200_BAD_POLY_COUNT,
          "MultiplicationPolynomialCount");
  REQUIRE(a->count == b->count && a->count == out->count, FHE_B200_INVALID_ARGUMENT, "batch sizes differ");
  need_repr(a, FHE_B200_NTT);
  need_repr(b, FHE_B200_NTT);
  if (rk) {   // enable_relinearization (mul.rs:141-151): the key must live at the multiplicator's context
    REQUIRE(rk->par == par && rk->ct_level == m->level, FHE_B200_CONTEXT_MISMATCH,
            "ParameterMismatch: relinearization key and multiplicator contexts differ");
  }
  const LevelData& lv = par->level(m->level);
  if (mod_switch) {
    REQUIRE(lv.L >= 2, FHE_B200_NO_MORE_CONTEXT, "NoMoreContext");  // mul.rs:155-162
    REQUIRE(out->level == m->level + 1, FHE_B200_INVALID_LEVEL, "output batch must be one level down");
  } else {
    REQUIRE(out->level == m->level, FHE_B200_INVALID_LEVEL, "output batch must be at the operand level");
  }
  DeviceGuard g(par);
  const size_t row = (size_t)1 << par->logn, L = lv.L;
  ChunkRunner chunks(par, a->count, (cudaStream_t)stream);
  chunks.run([&](u32 c0, u32 n, cudaStream_t st) {
    Workspace ws(par, st);
    const bool direct = !rk && !mod_switch;
    u64* W = direct ? out->d + (size_t)c0 * 3 * L * row : ws.words((size_t)n * 3 * L * row);
    mul_core_general(m, a->d + (size_t)c0 * 2 * L * row, b->d + (size_t)c0 * 2 * L * row, n, W, ws, st);
    u64* o = W;   // [n][out_parts][L][N]
    if (rk) {
      o = mod_switch ? ws.words((size_t)n * 2 * L * row) : out->d + (size_t)c0 * 2 * L * row;
      u64* c2 = ws.words((size_t)n * L * row);
      FHE_CUDA(cudaMemcpy2DAsync(o, 2 * L * row * 8, W, 3 * L * row * 8, 2 * L * row * 8, n, cudaMemcpyDeviceToDevice, st));
      FHE_CUDA(cudaMemcpy2DAsync(c2, L * row * 8, W + 2 * L * row, 3 * L * row * 8, L * row * 8, n,
                                 cudaMemcpyDeviceToDevice, st));
      launch_ntt(o, o, n * 2 * (u32)L, lv.ctx_ids, par->d_limbs, par->logn, false, 1, false, st);
      key_switch_apply(par, {&rk, 1, nullptr}, c2, n, o, 1, nullptr, ws, st);   // mul.rs:210-228
    } else {
      launch_ntt(o, o, n * 3 * (u32)L, lv.ctx_ids, par->d_limbs, par->logn, false, 1, false, st);
    }
    if (mod_switch) {  // Ciphertext::switch_down, ciphertext.rs:148-161
      launch_ntt(o, o, n * out_parts * (u32)L, lv.ctx_ids, par->d_limbs, par->logn, true, 1, false, st);
      u64* dst = out->d + (size_t)c0 * out_parts * (L - 1) * row;
      launch_switch_down(lv.sd, o, dst, n * out_parts, (u32)L, lv.ctx_ids, par->d_limbs, par->logn, st);
      const LevelData& nl = par->level(m->level + 1);
      launch_ntt(dst, dst, n * out_parts * (u32)(L - 1), nl.ctx_ids, par->d_limbs, par->logn, false, 1, false, st);
    }
  });
  FHE_CUDA(cudaGetLastError());
  out->repr = FHE_B200_NTT;
  API_END
}

int fhe_b200_substitute(const fhe_b200_batch* in, uint32_t exponent, fhe_b200_batch* out, void* stream) {
  API_BEGIN
  REQUIRE(in && out && in != out, FHE_B200_INVALID_ARGUMENT, "null or aliased argument");
  check_same(in, out);
  REQUIRE(in->parts == out->parts && in->count == out->count, FHE_B200_BAD_POLY_COUNT, "shapes differ");
  const fhe_b200_params* par = in->par;
  exponent %= 2 * par->N;
  REQUIRE(exponent & 1, FHE_B200_INVALID_EXPONENT, "InvalidSubstitutionExponent");
  DeviceGuard g(par);
  const size_t rows = (size_t)in->count * in->parts * in->limbs;
  if (in->repr == FHE_B200_NTT)   // rq/mod.rs:360-389: a permutation of the bit-reversed evaluation points
    launch_substitute_ntt(in->d, 0, out->d, 0, nullptr, 0, &exponent, nullptr, 1, (u32)rows, false, ids_of(in),
                          par->d_limbs, par->logn, (cudaStream_t)stream);
  else                            // rq/mod.rs:390-408: a signed permutation of the coefficients
    launch_substitute_power(in->d, out->d, rows, exponent, ids_of(in), par->d_limbs, par->logn, (cudaStream_t)stream);
  FHE_CUDA(cudaGetLastError());
  out->repr = in->repr;
  API_END
}

// SubstitutionExponent::new (rq/mod.rs:99-121) of each key's exponent
static std::vector<u32> galois_exponents(const fhe_b200_params* par, const u32* exponents, u32 n_keys) {
  std::vector<u32> e(n_keys);
  for (u32 k = 0; k < n_keys; k++) {
    e[k] = exponents[k] % (2 * par->N);
    REQUIRE(e[k] & 1, FHE_B200_INVALID_EXPONENT, "InvalidSubstitutionExponent: " + std::to_string(exponents[k]));
  }
  return e;
}

// the argument checks of every Galois call; returns the exponents of gk.exps reduced mod 2N
static std::vector<u32> galois_check(const fhe_b200_batch* ct, const KeySet& gk, const fhe_b200_batch* out) {
  REQUIRE(ct && gk.keys[0] && out && ct != out, FHE_B200_INVALID_ARGUMENT, "null or aliased argument");
  check_same(ct, out);
  REQUIRE(!ct->mul_basis, FHE_B200_CONTEXT_MISMATCH, "PolynomialContextMismatch");
  REQUIRE(ct->parts == 2 && out->parts == 2, FHE_B200_BAD_POLY_COUNT, "InvalidPolynomialCount: expected 2");
  if (gk.source)
    for (u32 j = 0; j < out->count; j++)
      REQUIRE(gk.source[j] < ct->count, FHE_B200_INVALID_ARGUMENT, "source " + std::to_string(gk.source[j]) +
                                                                       " of output " + std::to_string(j) +
                                                                       " beyond the batch");
  else
    REQUIRE(ct->count == out->count, FHE_B200_INVALID_ARGUMENT, "batch sizes differ");
  need_repr(ct, FHE_B200_NTT);
  check_ksks(gk, ct->par, ct->level, out->count);
  return galois_exponents(ct->par, gk.exps, gk.n);
}

// output j = GaloisKey::relinearize of ciphertext gk.source[j] (j without a source list) with key gk.key_of(j) for
// its exponent gk.exps[key] (reduced), after galois_check
static void galois_chunks(const fhe_b200_batch* ct, const KeySet& gk, fhe_b200_batch* out, cudaStream_t stream) {
  const fhe_b200_params* par = ct->par;
  const LevelData& lv = par->level(ct->level);
  const size_t W = ct->words_per_ct();
  ChunkRunner chunks(par, out->count, stream);
  chunks.run([&](u32 c0, u32 n, cudaStream_t st) {
    galois_range(par, lv, gk.from(c0), ct->d, c0, out->d + c0 * W, n, false, st);
  });
}

static void galois_run(const fhe_b200_batch* ct, KeySet gk, fhe_b200_batch* out, void* stream) {
  const std::vector<u32> exps = galois_check(ct, gk, out);
  gk.exps = exps.data();
  DeviceGuard g(ct->par);
  galois_chunks(ct, gk, out, (cudaStream_t)stream);
  FHE_CUDA(cudaGetLastError());
  out->repr = FHE_B200_NTT;
}

int fhe_b200_galois(const fhe_b200_batch* ct, uint32_t exponent, const fhe_b200_ksk* gk, fhe_b200_batch* out,
                    void* stream) {
  API_BEGIN
  galois_run(ct, {&gk, 1, nullptr, &exponent}, out, stream);
  API_END
}

int fhe_b200_galois_keyed(const fhe_b200_batch* ct, uint32_t exponent, const fhe_b200_ksk* const* gks, uint32_t n_keys,
                          const uint32_t* key_index, fhe_b200_batch* out, void* stream) {
  API_BEGIN
  KeySet K = key_list(gks, n_keys, key_index);
  const std::vector<u32> exps(n_keys, exponent);
  K.exps = exps.data();
  galois_run(ct, K, out, stream);
  API_END
}

int fhe_b200_galois_many(const fhe_b200_batch* ct, const uint32_t* source, const fhe_b200_ksk* const* gks,
                         const uint32_t* exponents, uint32_t n_keys, const uint32_t* key_index, fhe_b200_batch* out,
                         void* stream) {
  API_BEGIN
  KeySet K = key_list(gks, n_keys, key_index);
  REQUIRE(exponents, FHE_B200_INVALID_ARGUMENT, "null exponent list");
  REQUIRE(ct && out && ct != out && out->d != ct->d, FHE_B200_INVALID_ARGUMENT, "null or aliased argument");
  K.exps = exponents;
  K.source = source;
  galois_run(ct, K, out, stream);
  API_END
}

// Item i of `in` ([n][words]) to item dst[i] of `out`: one copy per run of consecutive destinations.
static void scatter_items(const u64* in, u64* out, size_t words, const u32* dst, u32 n, cudaStream_t st) {
  for (u32 i = 0, e; i < n; i = e) {
    for (e = i + 1; e < n && dst[e] == dst[e - 1] + 1; e++) {}
    FHE_CUDA(cudaMemcpyAsync(out + dst[i] * words, in + i * words, (e - i) * words * sizeof(u64),
                             cudaMemcpyDeviceToDevice, st));
  }
}

// The hoisted outputs [c0, c0 + n) of `outs` (output indices, ordered by source) as kernel entries: each distinct
// source gets a digit slot and each distinct exponent a correction row, in order of first use.
struct HoistPlan {
  std::vector<HoistOut> h;
  std::vector<u32> sources, exps;
  HoistPlan(const KeySet& gk, const std::vector<u32>& outs, u32 c0, u32 n) {
    for (u32 i = 0; i < n; i++) {
      const u32 j = outs[c0 + i], s = gk.source ? gk.source[j] : j;
      const fhe_b200_ksk* k = gk.keys[gk.key_of(j)];
      const u32 e = gk.exps[gk.key_of(j)];
      u32 slot = (u32)sources.size(), m = 0;
      if (slot && sources.back() == s) slot--;
      else sources.push_back(s);
      while (m < exps.size() && exps[m] != e) m++;
      if (m == exps.size()) exps.push_back(e);
      h.push_back({k->k0, k->k1, e, slot, s, m, j});
    }
  }
};

// The power-basis c1 of the plan's sources: x [slot][L][N], canonical (the reference's c2 before its substitution)
static u64* hoist_c1(const fhe_b200_params* par, const LevelData& lv, const fhe_b200_batch* ct,
                     const std::vector<u32>& sources, Workspace& ws, cudaStream_t st) {
  const size_t rowb = ((size_t)lv.L << par->logn) * sizeof(u64), W = ct->words_per_ct();
  const u32 n = (u32)sources.size();
  u64* x = ws.words(((size_t)n * lv.L) << par->logn);
  for (u32 i = 0, e; i < n; i = e) {   // one 2-D copy per run of consecutive sources
    for (e = i + 1; e < n && sources[e] == sources[e - 1] + 1; e++) {}
    FHE_CUDA(cudaMemcpy2DAsync((char*)x + i * rowb, rowb, ct->d + sources[i] * W + ((size_t)lv.L << par->logn),
                               W * sizeof(u64), rowb, e - i, cudaMemcpyDeviceToDevice, st));
  }
  launch_ntt(x, x, n * lv.L, lv.ctx_ids, par->d_limbs, par->logn, true, 1, false, st);
  return x;
}

// fhe_b200_galois_many_hoisted after galois_check; returns how many outputs the hoisted kernels computed
static u32 galois_hoisted(const fhe_b200_batch* ct, const KeySet& gk, fhe_b200_batch* out, cudaStream_t user) {
  const fhe_b200_params* par = ct->par;
  const fhe_b200_ksk* k = gk.keys[0];
  const LevelData& lv = par->level(ct->level);
  const LevelData& kl = par->level(k->ksk_level);
  const u32 L = lv.L, Lk = k->Lk, logn = par->logn, count = out->count;
  const size_t row = (size_t)1 << logn, W = ct->words_per_ct();
  auto src_of = [&](u32 j) { return gk.source ? gk.source[j] : j; };
  // candidates: the outputs of sources with two or more outputs, by (source, key) so that outputs sharing either
  // are neighbours in the kernels' order.  Base-2^b digits of q - x are not a function of those of x: no candidates.
  std::vector<u32> uses(ct->count), cand;
  for (u32 j = 0; j < count; j++) uses[src_of(j)]++;
  for (u32 j = 0; j < count && !k->log_base; j++)
    if (uses[src_of(j)] >= 2) cand.push_back(j);
  if (cand.empty()) {
    galois_chunks(ct, gk, out, user);
    return 0;
  }
  std::stable_sort(cand.begin(), cand.end(), [&](u32 a, u32 b) {
    return src_of(a) != src_of(b) ? src_of(a) < src_of(b) : gk.key_of(a) < gk.key_of(b);
  });
  const u32 nc = (u32)cand.size();
  // the zero check: an output whose exponent negates a position where c1 has a zero residue takes galois_range
  std::vector<u32> zero(nc);
  {
    Workspace ws(par, user);
    u32* flags = (u32*)ws.words((nc + 1) / 2);
    FHE_CUDA(cudaMemsetAsync(flags, 0, nc * sizeof(u32), user));
    {
      ChunkRunner chunks(par, nc, user);
      chunks.run([&](u32 c0, u32 n, cudaStream_t st) {
        Workspace cws(par, st);
        const HoistPlan P(gk, cand, c0, n);
        const u64* x = hoist_c1(par, lv, ct, P.sources, cws, st);
        launch_hoist_zero(P.h.data(), n, x, flags + c0, L, logn, st);
      });
    }
    FHE_CUDA(cudaMemcpyAsync(zero.data(), flags, nc * sizeof(u32), cudaMemcpyDeviceToHost, user));
    FHE_CUDA(cudaStreamSynchronize(user));   // the one synchronisation of the call
  }
  std::vector<u32> hoisted, rest, rest_key, rest_src;
  std::vector<bool> is_hoisted(count);
  for (u32 i = 0; i < nc; i++)
    if (!zero[i]) {
      hoisted.push_back(cand[i]);
      is_hoisted[cand[i]] = true;
    }
  for (u32 j = 0; j < count; j++)
    if (!is_hoisted[j]) {
      rest.push_back(j);
      rest_key.push_back(gk.key_of(j));
      rest_src.push_back(src_of(j));
    }
  const u32 nh = (u32)hoisted.size(), nr = (u32)rest.size();
  const bool reduce = digit_reduce(par, k);
  ChunkRunner(par, nh, user).run([&](u32 c0, u32 n, cudaStream_t st) {
    Workspace ws(par, st);
    const HoistPlan P(gk, hoisted, c0, n);
    const u32 ns = (u32)P.sources.size(), ne = (u32)P.exps.size();
    const u64* x = hoist_c1(par, lv, ct, P.sources, ws, st);
    // D_k[j] = NTT_j(lazy(x_k)): key_switch_core's unfused digit transform, in the layout it would choose
    u64* D = ws.words(((size_t)ns * L * Lk) << logn);
    const bool adjacent = Lk > 1 && ntt_uses_tma(ns * L * Lk, kl.ctx_ids, logn, Lk, x, D);
    launch_ntt(x, D, ns * L * Lk, kl.ctx_ids, par->d_limbs, logn, false, Lk, reduce, st, true, adjacent, L);
    // M_e[j] = NTT_j(N_e) of every exponent of the chunk
    u64* Mrows = ws.words(((size_t)ne * Lk) << logn);
    launch_negation_rows(Mrows, P.exps.data(), ne, Lk, logn, st);
    launch_ntt(Mrows, Mrows, ne * Lk, kl.ctx_ids, par->d_limbs, logn, false, 1, false, st);
    if (Lk == L) {   // galois_key.rs:78: sigma(c0) is added in the kernel, which writes every output in place
      launch_hoist_mac(P.h.data(), n, D, adjacent, Mrows, ct->d, W, out->d, W, L, Lk, kl.ctx_ids, par->d_limbs,
                       logn, st);
      return;
    }
    // leveled key (galois_key.rs:69-76): the Lk-limb pairs take key_switch_apply's tail with sigma(c0) as its base
    std::vector<HoistOut> h = P.h;
    std::vector<u32> exps(n), srcs(n), dst(n);
    for (u32 i = 0; i < n; i++) {
      exps[i] = h[i].exponent;
      srcs[i] = h[i].src_ct;
      dst[i] = h[i].dst;
      h[i].dst = i;
    }
    u64* cur = ws.words(((size_t)n * 2 * Lk) << logn);
    launch_hoist_mac(h.data(), n, D, adjacent, Mrows, nullptr, 0, cur, 2 * Lk * row, L, Lk, kl.ctx_ids, par->d_limbs,
                     logn, st);
    u64* s = ws.words(n * W);
    u64* res = ws.words(n * W);
    launch_substitute_ntt(ct->d, W, s, W, nullptr, 0, exps.data(), srcs.data(), n, L, false, lv.ctx_ids,
                          par->d_limbs, logn, st);
    key_switch_leveled_tail(par, k, cur, n, res, 2, s, ws, st);
    scatter_items(res, out->d, W, dst.data(), n, st);
  });
  // every other output: galois_many's path, into place when the chunk's outputs are consecutive
  const KeySet R{gk.keys, gk.n, rest_key.data(), gk.exps, rest_src.data()};
  ChunkRunner(par, nr, user).run([&](u32 c0, u32 n, cudaStream_t st) {
    if (rest[c0 + n - 1] - rest[c0] == n - 1) {
      galois_range(par, lv, R.from(c0), ct->d, 0, out->d + rest[c0] * W, n, false, st);
      return;
    }
    Workspace ws(par, st);
    u64* tmp = ws.words(n * W);
    galois_range(par, lv, R.from(c0), ct->d, 0, tmp, n, false, st);
    scatter_items(tmp, out->d, W, rest.data() + c0, n, st);
  });
  return nh;
}

int fhe_b200_galois_many_hoisted(const fhe_b200_batch* ct, const uint32_t* source, const fhe_b200_ksk* const* gks,
                                 const uint32_t* exponents, uint32_t n_keys, const uint32_t* key_index,
                                 fhe_b200_batch* out, uint32_t* n_hoisted, void* stream) {
  API_BEGIN
  KeySet K = key_list(gks, n_keys, key_index);
  REQUIRE(exponents, FHE_B200_INVALID_ARGUMENT, "null exponent list");
  REQUIRE(ct && out && ct != out && out->d != ct->d, FHE_B200_INVALID_ARGUMENT, "null or aliased argument");
  K.exps = exponents;
  K.source = source;
  const std::vector<u32> exps = galois_check(ct, K, out);
  K.exps = exps.data();
  DeviceGuard g(ct->par);
  const u32 h = galois_hoisted(ct, K, out, (cudaStream_t)stream);
  FHE_CUDA(cudaGetLastError());
  out->repr = FHE_B200_NTT;
  if (n_hoisted) *n_hoisted = h;
  API_END
}

// ---- linear transforms (DESIGN §3.4): out[c] = sum_g rot_{g b}(sum_i D[g b + i] (.) B_i(ct[c])), B_0 the identity
struct LinearTransform {
  const fhe_b200_batch *ct, *diags;
  u32 n, b, G;
  bool per_ct;
  const fhe_b200_ksk* const* keys;
  u32 n_keys;
  const u32* exps;            // reduced, one per key
  std::vector<u32> baby_key;  // [b]: the key of baby step i >= 1 (entry 0 unused)
  std::vector<u32> giant_key; // [G]: the key of giant step g >= 1 (entry 0 unused)
  size_t W() const { return ct->words_per_ct(); }
  // GaloisKey::relinearize of items src[r] of `in` with keys key[r] into dst [m][W], at most chunk_size() at a time
  void rotate(const u64* in, const std::vector<u32>& src, const std::vector<u32>& key, u64* dst, cudaStream_t st) const {
    const fhe_b200_params* par = ct->par;
    const u32 m = (u32)src.size(), step = chunk_size();
    for (u32 r0 = 0; r0 < m; r0 += step)
      galois_range(par, par->level(ct->level), KeySet{keys, n_keys, key.data() + r0, exps, src.data() + r0}, in, 0,
                   dst + r0 * W(), std::min(step, m - r0), false, st);
  }
  // the giant steps of groups [g0, g0 + ng) of ciphertexts [c0, c0 + cts): P [cts][ng] holds their partial sums;
  // out[c] = (g0 == 0 ? P[c][0] : out[c]) + sum over the other groups of rot_{g b}(P[c][g - g0]), through R [cts][ng]
  void finish(u64* P, u64* R, u32 c0, u32 cts, u32 g0, u32 ng, u64* out, cudaStream_t st) const {
    const fhe_b200_params* par = ct->par;
    const u32 L = par->level(ct->level).L;
    std::vector<u32> src, key;
    for (u32 c = 0; c < cts; c++)
      for (u32 gi = g0 ? 0 : 1; gi < ng; gi++) {
        src.push_back(c * ng + gi);
        key.push_back(giant_key[g0 + gi]);
      }
    u64* o = out + (size_t)c0 * W();
    if (g0 == 0)
      launch_segment_sum(P, ng * W(), 1, o, W(), nullptr, 0, 2 * L, cts, W(), false, ids_of(ct), par->d_limbs,
                         par->logn, st);
    if (src.empty()) return;
    rotate(P, src, key, R, st);
    launch_segment_sum(R, W(), (u32)src.size() / cts, o, W(), nullptr, 0, 2 * L, cts, W(), true, ids_of(ct),
                       par->d_limbs, par->logn, st);
  }
  // groups per tile for a chunk of `cts` ciphertexts: a tile's giant rotations are at most chunk_size() outputs
  u32 group_tile(u32 cts) const { return std::min(G, std::max(1u, chunk_size() / cts)); }
  const u64* diag(u32 c, u32 k) const {
    return diags->d + ((per_ct ? (size_t)c * n : 0) + k) * diags->words_per_ct();
  }
};

// Keys at the ciphertext level without base-2^b digits: one hoisted decomposition per ciphertext and hoist_dot_kernel;
// returns the (ciphertext, baby step) terms that took galois_range because of the zero check
static u32 linear_transform_fused(const LinearTransform& T, fhe_b200_batch* out, cudaStream_t user) {
  const fhe_b200_batch* ct = T.ct;
  const fhe_b200_params* par = ct->par;
  const LevelData& lv = par->level(ct->level);
  const u32 L = lv.L, logn = par->logn, b = T.b, count = ct->count;
  const size_t W = T.W();
  std::vector<LtStep> steps(b);
  std::vector<u32> exps(b, 1);
  for (u32 i = 1; i < b; i++) {
    const fhe_b200_ksk* k = T.keys[T.baby_key[i]];
    exps[i] = T.exps[T.baby_key[i]];
    steps[i] = {k->k0, k->k1, exps[i], 0};
  }
  auto c1_of = [&](u32 c0, u32 n, Workspace& ws, cudaStream_t st) {
    std::vector<u32> src(n);
    for (u32 c = 0; c < n; c++) src[c] = c0 + c;
    return hoist_c1(par, lv, ct, src, ws, st);
  };
  // the zero check (DESIGN §8): term (c, i) falls back when exponent i negates a position where c1 has a zero residue
  std::vector<u32> zero((size_t)count * (b - 1));
  Workspace ws(par, user);
  if (b > 1) {
    u32* flags = (u32*)ws.words((zero.size() + 1) / 2);
    FHE_CUDA(cudaMemsetAsync(flags, 0, zero.size() * sizeof(u32), user));
    ChunkRunner(par, count, user).run([&](u32 c0, u32 n, cudaStream_t st) {
      Workspace cws(par, st);
      std::vector<HoistOut> h;
      for (u32 c = 0; c < n; c++)
        for (u32 i = 1; i < b; i++) h.push_back({steps[i].k0, steps[i].k1, exps[i], c, c0 + c, i, 0});
      launch_hoist_zero(h.data(), (u32)h.size(), c1_of(c0, n, cws, st), flags + (size_t)c0 * (b - 1), L, logn, st);
    });
    FHE_CUDA(cudaMemcpyAsync(zero.data(), flags, zero.size() * sizeof(u32), cudaMemcpyDeviceToHost, user));
    FHE_CUDA(cudaStreamSynchronize(user));   // the one synchronisation of the call
  }
  // the baby steps' keys and exponents, and M_e of each (DESIGN §8), for every chunk
  LtStep* d_steps = (LtStep*)ws.words((b * sizeof(LtStep) + 7) / 8);
  FHE_CUDA(cudaMemcpyAsync(d_steps, steps.data(), b * sizeof(LtStep), cudaMemcpyHostToDevice, user));
  u64* mrows = ws.words(((size_t)b * L) << logn);
  launch_negation_rows(mrows, exps.data(), b, L, logn, user);
  launch_ntt(mrows, mrows, b * L, lv.ctx_ids, par->d_limbs, logn, false, 1, false, user);
  const bool reduce = b > 1 && digit_reduce(par, T.keys[0]);
  u32 n_fallback = 0;
  for (u32 z : zero) n_fallback += z;
  ChunkRunner(par, count, user, std::max(1u, chunk_size() / T.G)).run([&](u32 c0, u32 n, cudaStream_t st) {
    Workspace cws(par, st);
    u64 *D = nullptr, *fb = nullptr;
    int* d_fallback = nullptr;
    bool adjacent = false;
    if (b > 1) {
      const u64* x = c1_of(c0, n, cws, st);
      D = cws.words(((size_t)n * L * L) << logn);
      adjacent = L > 1 && ntt_uses_tma(n * L * L, lv.ctx_ids, logn, L, x, D);
      launch_ntt(x, D, n * L * L, lv.ctx_ids, par->d_limbs, logn, false, L, reduce, st, true, adjacent, L);
      std::vector<int> fallback((size_t)n * b, -1);
      std::vector<u32> src, key;
      for (u32 c = 0; c < n; c++)
        for (u32 i = 1; i < b; i++)
          if (zero[(size_t)(c0 + c) * (b - 1) + i - 1]) {
            fallback[(size_t)c * b + i] = (int)src.size();
            src.push_back(c0 + c);
            key.push_back(T.baby_key[i]);
          }
      if (!src.empty()) {
        fb = cws.words(src.size() * W);
        T.rotate(ct->d, src, key, fb, st);
        d_fallback = (int*)cws.words((fallback.size() + 1) / 2);
        FHE_CUDA(cudaMemcpyAsync(d_fallback, fallback.data(), fallback.size() * sizeof(int), cudaMemcpyHostToDevice, st));
      }
    }
    const u32 gt = T.group_tile(n);
    u64* P = cws.words((size_t)n * gt * W);
    u64* R = cws.words((size_t)n * gt * W);
    for (u32 g0 = 0; g0 < T.G; g0 += gt) {
      const u32 ng = std::min(gt, T.G - g0);
      launch_hoist_dot(d_steps, d_fallback, fb, D, adjacent, mrows, ct->d + (size_t)c0 * W, W, n, T.diags->d, c0,
                       T.per_ct, T.n, b, g0, ng, P, L, lv.ctx_ids, par->d_limbs, logn, st);
      T.finish(P, R, c0, n, g0, ng, out->d, st);
    }
  });
  return n_fallback;
}

// Leveled keys and base-2^b keys: the composition itself -- every baby-step rotation through galois_range, the
// products and sums of each group through launch_dot, then the giant steps and the sum
static u32 linear_transform_unfused(const LinearTransform& T, fhe_b200_batch* out, cudaStream_t user) {
  const fhe_b200_batch* ct = T.ct;
  const fhe_b200_params* par = ct->par;
  const u32 b = T.b;
  const size_t W = T.W();
  ChunkRunner(par, ct->count, user, std::max(1u, chunk_size() / std::max(b, T.G))).run([&](u32 c0, u32 n, cudaStream_t st) {
    Workspace cws(par, st);
    // B [n][b]: ciphertext c, then its rotations by 1 .. b - 1
    u64* B = cws.words((size_t)n * b * W);
    FHE_CUDA(cudaMemcpy2DAsync(B, b * W * sizeof(u64), ct->d + (size_t)c0 * W, W * sizeof(u64), W * sizeof(u64), n,
                               cudaMemcpyDeviceToDevice, st));
    if (b > 1) {
      std::vector<u32> src, key;
      for (u32 c = 0; c < n; c++)
        for (u32 i = 1; i < b; i++) {
          src.push_back(c0 + c);
          key.push_back(T.baby_key[i]);
        }
      u64* rot = cws.words(src.size() * W);
      T.rotate(ct->d, src, key, rot, st);
      FHE_CUDA(cudaMemcpy2DAsync(B + W, b * W * sizeof(u64), rot, (b - 1) * W * sizeof(u64), (b - 1) * W * sizeof(u64),
                                 n, cudaMemcpyDeviceToDevice, st));
    }
    const u32 gt = T.group_tile(n);
    u64* P = cws.words((size_t)n * gt * W);
    u64* R = cws.words((size_t)n * gt * W);
    for (u32 g0 = 0; g0 < T.G; g0 += gt) {
      const u32 ng = std::min(gt, T.G - g0);
      for (u32 c = 0; c < n; c++)
        for (u32 gi = 0; gi < ng; gi++) {
          const u32 first = (g0 + gi) * b, terms = std::min(b, T.n - first);
          launch_dot(B + (size_t)c * b * W, T.diag(c0 + c, first), P + ((size_t)c * ng + gi) * W, 1, terms, 2, terms,
                     terms, ids_of(ct), par->d_limbs, par->logn, st);
        }
      T.finish(P, R, c0, n, g0, ng, out->d, st);
    }
  });
  return ct->count * (b - 1);
}

int fhe_b200_linear_transform(const fhe_b200_batch* ct, const fhe_b200_batch* diags, uint32_t n_diags, uint32_t baby,
                              const fhe_b200_ksk* const* gks, const uint32_t* exponents, uint32_t n_keys,
                              fhe_b200_batch* out, uint32_t* n_fallback, void* stream) {
  API_BEGIN
  REQUIRE(!n_keys || (gks && exponents), FHE_B200_INVALID_ARGUMENT, "null key list or exponents");
  for (u32 i = 0; i < n_keys; i++) REQUIRE(gks[i], FHE_B200_INVALID_ARGUMENT, "null key");
  REQUIRE(ct && diags && out && ct != out && out->d != ct->d && diags != out && diags->d != out->d,
          FHE_B200_INVALID_ARGUMENT, "null or aliased argument");
  check_same(ct, diags);
  REQUIRE(ct->par == out->par, FHE_B200_CONTEXT_MISMATCH, "ParameterMismatch: batches use different parameters");
  REQUIRE(ct->level == out->level, FHE_B200_INVALID_LEVEL, "InvalidLevel: operands are at different levels");
  REQUIRE(!ct->mul_basis && !out->mul_basis, FHE_B200_CONTEXT_MISMATCH, "PolynomialContextMismatch");
  REQUIRE(ct->parts == 2, FHE_B200_BAD_POLY_COUNT, "InvalidPolynomialCount: expected 2");
  REQUIRE(out->parts == 2 && out->count == ct->count, FHE_B200_INVALID_ARGUMENT,
          "the output must hold one 2-part ciphertext per input ciphertext");
  REQUIRE(diags->parts == 1, FHE_B200_INVALID_ARGUMENT, "diagonals must hold one polynomial per entry");
  const fhe_b200_params* par = ct->par;
  REQUIRE(n_diags >= 1 && n_diags <= par->N / 2, FHE_B200_INVALID_ARGUMENT,
          "n_diags must be 1 .. N/2, got " + std::to_string(n_diags));
  REQUIRE(baby >= 1 && baby <= n_diags, FHE_B200_INVALID_ARGUMENT,
          "the baby step must be 1 .. n_diags, got " + std::to_string(baby));
  REQUIRE(diags->count == n_diags || diags->count == (size_t)ct->count * n_diags, FHE_B200_INVALID_ARGUMENT,
          "diags must hold n_diags entries or n_diags per ciphertext");
  need_repr(ct, FHE_B200_NTT);
  need_repr(diags, FHE_B200_NTT);
  const std::vector<u32> exps = galois_exponents(par, exponents, n_keys);
  if (n_keys) check_ksks(KeySet{gks, n_keys, nullptr}, par, ct->level, 0);
  LinearTransform T{ct, diags, n_diags, baby, (n_diags + baby - 1) / baby, diags->count != n_diags, gks, n_keys,
                    exps.data(), std::vector<u32>(baby), std::vector<u32>()};
  T.giant_key.resize(T.G);
  // EvaluationKey::rotates_columns_by's key of each step (evaluation_key.rs:145-170, :278-286)
  auto key_of_step = [&](u32 step) {
    const u32 e = (u32)powmod_h(3, step, 2 * (u64)par->N);
    for (u32 k = 0; k < n_keys; k++)
      if (exps[k] == e) return k;
    throw FheError(FHE_B200_INVALID_ARGUMENT,
                   "EvaluationKeyError: column rotation by " + std::to_string(step) + " not supported by the key list");
  };
  for (u32 i = 1; i < baby; i++) T.baby_key[i] = key_of_step(i);
  for (u32 g = 1; g < T.G; g++) T.giant_key[g] = key_of_step(g * baby);
  DeviceGuard g(par);
  // the one routing decision, from the keys: a transform that needs no key is the plaintext products alone
  const fhe_b200_ksk* k = baby > 1 || T.G > 1 ? gks[0] : nullptr;
  const bool fused = !k || (k->log_base == 0 && k->Lk == par->level(ct->level).L);
  const u32 f = fused ? linear_transform_fused(T, out, (cudaStream_t)stream)
                      : linear_transform_unfused(T, out, (cudaStream_t)stream);
  FHE_CUDA(cudaGetLastError());
  out->repr = FHE_B200_NTT;
  if (n_fallback) *n_fallback = f;
  API_END
}

// EvaluationKey::computes_inner_sum (evaluation_key.rs:56-100) of every ciphertext: gks[s * n_gks + l] is the key of
// step l of key set s (column rotations by 1, 2, 4, ..., N/4, then the row rotation), set_index[c] (nullable: set 0)
// the key set of ciphertext c.  Step l of a chunk is one Galois call in sum mode, from the previous step's output; the
// steps alternate between `out` and one scratch buffer so that the last lands in `out`.
static void inner_sum_run(const fhe_b200_batch* ct, const fhe_b200_ksk* const* gks, uint32_t n_gks, uint32_t n_sets,
                          const uint32_t* set_index, fhe_b200_batch* out, void* stream) {
  REQUIRE(ct && out && gks, FHE_B200_INVALID_ARGUMENT, "null argument");
  REQUIRE(ct != out && out->d != ct->d, FHE_B200_INVALID_ARGUMENT, "out must not alias ct");
  const fhe_b200_params* par = ct->par;
  REQUIRE(n_gks == par->logn, FHE_B200_INVALID_ARGUMENT,
          "EvaluationKeyError: an inner sum takes log2 N = " + std::to_string(par->logn) + " keys per set, got " +
              std::to_string(n_gks));
  check_same(ct, out);
  REQUIRE(!ct->mul_basis, FHE_B200_CONTEXT_MISMATCH, "PolynomialContextMismatch");
  REQUIRE(ct->parts == 2 && out->parts == 2, FHE_B200_BAD_POLY_COUNT, "InvalidPolynomialCount: expected 2");
  REQUIRE(ct->count == out->count, FHE_B200_INVALID_ARGUMENT, "batch sizes differ");
  need_repr(ct, FHE_B200_NTT);
  const u32 Q = ct->count, steps = n_gks, m = 2 * par->N;
  // the exponent of step l: 3^(2^l) mod 2N (evaluation_key.rs:278-286), then 2N - 1 (:118)
  std::vector<u32> step_exp(steps);
  u64 e = 3;
  for (u32 l = 0; l + 1 < steps; l++) {
    step_exp[l] = (u32)e;
    e = e * e % m;
  }
  step_exp[steps - 1] = m - 1;
  std::vector<std::vector<const fhe_b200_ksk*>> keys(steps, std::vector<const fhe_b200_ksk*>(n_sets));
  std::vector<std::vector<u32>> exps(steps);
  for (u32 l = 0; l < steps; l++) {
    for (u32 k = 0; k < n_sets; k++) {
      keys[l][k] = gks[(size_t)k * n_gks + l];
      REQUIRE(keys[l][k], FHE_B200_INVALID_ARGUMENT,
              "EvaluationKeyError: Missing GaloisKey { element: " + std::to_string(step_exp[l]) + " }");
    }
    exps[l].assign(n_sets, step_exp[l]);
    check_ksks({keys[l].data(), n_sets, set_index}, par, ct->level, Q);
  }
  DeviceGuard g(par);
  const LevelData& lv = par->level(ct->level);
  const size_t W = ct->words_per_ct();
  ChunkRunner chunks(par, Q, (cudaStream_t)stream);
  chunks.run([&](u32 c0, u32 n, cudaStream_t st) {
    Workspace ws(par, st);
    u64* buf[2] = {out->d + c0 * W, ws.words(n * W)};
    const u64* src = ct->d + c0 * W;
    for (u32 l = 0; l < steps; l++) {
      u64* dst = buf[(steps - 1 - l) & 1];
      const KeySet K{keys[l].data(), n_sets, set_index ? set_index + c0 : nullptr, exps[l].data()};
      galois_range(par, lv, K, src, 0, dst, n, true, st);
      src = dst;
    }
  });
  FHE_CUDA(cudaGetLastError());
  out->repr = FHE_B200_NTT;
}

int fhe_b200_inner_sum(const fhe_b200_batch* ct, const fhe_b200_ksk* const* gks, uint32_t n_gks, fhe_b200_batch* out,
                       void* stream) {
  API_BEGIN
  inner_sum_run(ct, gks, n_gks, 1, nullptr, out, stream);
  API_END
}

int fhe_b200_inner_sum_keyed(const fhe_b200_batch* ct, const fhe_b200_ksk* const* gks, uint32_t n_gks, uint32_t n_sets,
                             const uint32_t* set_index, fhe_b200_batch* out, void* stream) {
  API_BEGIN
  REQUIRE(n_sets && set_index, FHE_B200_INVALID_ARGUMENT, "null key set index, or no key sets");
  inner_sum_run(ct, gks, n_gks, n_sets, set_index, out, stream);
  API_END
}

// gks[s * n_gks + l]: the key of expansion level l of key set s; set_index[q] (nullable: set 0 for every query) the
// key set of query q
static void expand_run(const fhe_b200_batch* ct, uint32_t size, const fhe_b200_ksk* const* gks, uint32_t n_gks,
                       uint32_t n_sets, const uint32_t* set_index, fhe_b200_batch* out, void* stream) {
  REQUIRE(ct && out, FHE_B200_INVALID_ARGUMENT, "null argument");
  const fhe_b200_params* par = ct->par;
  REQUIRE(size > 0 && size <= par->N, FHE_B200_INVALID_ARGUMENT,
          "InvalidExpansionSize: " + std::to_string(size) + " for degree " + std::to_string(par->N));
  REQUIRE(ct->parts == 2, FHE_B200_BAD_POLY_COUNT, "InvalidPolynomialCount: expected 2");
  REQUIRE(!ct->mul_basis, FHE_B200_CONTEXT_MISMATCH, "PolynomialContextMismatch");
  need_repr(ct, FHE_B200_NTT);
  const u32 Q = ct->count;
  REQUIRE(out != ct && out->d != ct->d, FHE_B200_INVALID_ARGUMENT, "out must not alias ct");
  REQUIRE(out->par == par && !out->mul_basis && out->level == ct->level && out->parts == 2 &&
              (uint64_t)out->count == (uint64_t)size * Q,
          FHE_B200_INVALID_ARGUMENT, "out must hold size * ct.count 2-part ciphertexts at ct's level");
  // level = ceil(log2 size) (evaluation_key.rs:212); the key of level l is for element (N >> l) + 1 (:222-228)
  u32 level = 0;
  while ((1u << level) < size) level++;
  REQUIRE(n_gks >= level && (level == 0 || gks), FHE_B200_INVALID_ARGUMENT,
          "EvaluationKeyError: Missing GaloisKey: expansion level " + std::to_string(level) + " needs that many keys");
  if (set_index)
    for (u32 q = 0; q < Q; q++)
      REQUIRE(set_index[q] < n_sets, FHE_B200_INVALID_ARGUMENT, "key set index " + std::to_string(set_index[q]) +
                                                                    " of query " + std::to_string(q) + " beyond the sets");
  // the keys of level l, one per key set, and the key set of each of its step * Q inputs (entry i*Q + q: query q)
  std::vector<std::vector<const fhe_b200_ksk*>> keys(level, std::vector<const fhe_b200_ksk*>(n_sets));
  std::vector<std::vector<u32>> index(set_index ? level : 0);
  for (u32 l = 0; l < level; l++) {
    for (u32 k = 0; k < n_sets; k++) {
      keys[l][k] = gks[(size_t)k * n_gks + l];
      REQUIRE(keys[l][k], FHE_B200_INVALID_ARGUMENT,
              "EvaluationKeyError: Missing GaloisKey { element: " + std::to_string((par->N >> l) + 1) + " }");
      check_ksk(keys[l][k], par, ct->level);
    }
    check_key_set({keys[l].data(), n_sets, nullptr}, Q);
    if (set_index) {
      index[l].resize((size_t)Q << l);
      for (u32 c = 0; c < index[l].size(); c++) index[l][c] = set_index[c % Q];
    }
  }
  DeviceGuard g(par);
  cudaStream_t user = (cudaStream_t)stream;
  const LevelData& lv = par->level(ct->level);
  const size_t W = ct->words_per_ct();
  // monomials first: building one allocates and uploads synchronously, which must not happen between enqueued levels
  std::vector<const ulonglong2*> monos(level);
  std::vector<std::vector<u32>> exps(level);
  for (u32 l = 0; l < level; l++) {
    monos[l] = par->expansion_monomial_dev(ct->level, l);
    exps[l].assign(n_sets, (par->N >> l) + 1);
  }
  // index-major order: entry i*Q + q of `out` is output i of query q, so the outputs 0 .. step-1 of every query are
  // the contiguous region [0, step*Q) and the ones a level adds, step .. 2*step-1, the region right after it
  FHE_CUDA(cudaMemcpyAsync(out->d, ct->d, W * Q * sizeof(u64), cudaMemcpyDeviceToDevice, user));
  // at a partial last level the Galois images of outputs i >= size - step have no slot in `out`: they only feed lo
  Workspace spill_ws(par, user);
  const u32 last_step = level ? 1u << (level - 1) : 0;
  u64* spill = level && 2 * last_step > size ? spill_ws.words((size_t)(2 * last_step - size) * Q * W) : nullptr;
  for (u32 l = 0; l < level; l++) {
    const u32 step = 1u << l, pairs = step * Q, n_hi = (std::min(2 * step, size) - step) * Q;
    u64* hi = out->d + (size_t)pairs * W;
    ChunkRunner chunks(par, pairs, user);
    const KeySet K{keys[l].data(), n_sets, set_index ? index[l].data() : nullptr, exps[l].data()};
    chunks.run([&](u32 c0, u32 n, cudaStream_t st) {
      const u32 e = c0 + n, mid = std::min(std::max(c0, n_hi), e);
      if (mid > c0) galois_range(par, lv, K.from(c0), out->d, c0, hi + c0 * W, mid - c0, false, st);
      if (e > mid) galois_range(par, lv, K.from(mid), out->d, mid, spill + (mid - n_hi) * W, e - mid, false, st);
    });
    launch_expand_butterfly(out->d, hi, spill, pairs, n_hi, monos[l], lv.ctx_ids, par->d_limbs, par->logn, user);
  }
  FHE_CUDA(cudaGetLastError());
  out->repr = FHE_B200_NTT;
}

int fhe_b200_expand(const fhe_b200_batch* ct, uint32_t size, const fhe_b200_ksk* const* gks, uint32_t n_gks,
                    fhe_b200_batch* out, void* stream) {
  API_BEGIN
  expand_run(ct, size, gks, n_gks, 1, nullptr, out, stream);
  API_END
}

int fhe_b200_expand_keyed(const fhe_b200_batch* ct, uint32_t size, const fhe_b200_ksk* const* gks, uint32_t n_gks,
                          uint32_t n_sets, const uint32_t* set_index, fhe_b200_batch* out, void* stream) {
  API_BEGIN
  REQUIRE(n_sets && set_index, FHE_B200_INVALID_ARGUMENT, "null key set index, or no key sets");
  expand_run(ct, size, gks, n_gks, n_sets, set_index, out, stream);
  API_END
}

static void key_switch_run(const fhe_b200_batch* pb, uint32_t part, const KeySet& K, fhe_b200_batch* out2,
                           void* stream) {
  REQUIRE(pb && K.keys[0] && out2, FHE_B200_INVALID_ARGUMENT, "null argument");
  for (u32 i = 0; i < K.n; i++)
    REQUIRE(pb->par == out2->par && pb->par == K.keys[i]->par, FHE_B200_CONTEXT_MISMATCH, "ParameterMismatch");
  REQUIRE(!pb->mul_basis && !out2->mul_basis, FHE_B200_CONTEXT_MISMATCH, "PolynomialContextMismatch");
  REQUIRE(part < pb->parts && out2->parts == 2, FHE_B200_BAD_POLY_COUNT, "bad part index / output parts");
  for (u32 i = 0; i < K.n; i++)
    REQUIRE(pb->level == K.keys[i]->ct_level && out2->level == K.keys[i]->ksk_level, FHE_B200_INVALID_LEVEL,
            "InvalidLevel");
  REQUIRE(pb->count == out2->count, FHE_B200_INVALID_ARGUMENT, "batch sizes differ");
  need_repr(pb, FHE_B200_POWER_BASIS);
  check_key_set(K, pb->count);
  const fhe_b200_params* par = pb->par;
  DeviceGuard g(par);
  cudaStream_t st_user = (cudaStream_t)stream;
  const size_t row = (size_t)1 << par->logn, L = pb->limbs, Lk = K.keys[0]->Lk;
  ChunkRunner chunks(par, pb->count, st_user);
  chunks.run([&](u32 c0, u32 n, cudaStream_t st) {
    Workspace ws(par, st);
    u64* c2 = ws.words((size_t)n * L * row);
    FHE_CUDA(cudaMemcpy2DAsync(c2, L * row * 8, pb->d + ((size_t)c0 * pb->parts + part) * L * row,
                               pb->parts * L * row * 8, L * row * 8, n, cudaMemcpyDeviceToDevice, st));
    u64* dst = out2->d + (size_t)c0 * 2 * Lk * row;
    key_switch_core(par, K.from(c0), c2, n, nullptr, nullptr, dst, dst + Lk * row, 2 * (u32)Lk, ws, st);
  });
  FHE_CUDA(cudaGetLastError());
  out2->repr = FHE_B200_NTT;
}

int fhe_b200_key_switch(const fhe_b200_batch* pb, uint32_t part, const fhe_b200_ksk* k, fhe_b200_batch* out2,
                        void* stream) {
  API_BEGIN
  key_switch_run(pb, part, {&k, 1, nullptr}, out2, stream);
  API_END
}

int fhe_b200_key_switch_keyed(const fhe_b200_batch* pb, uint32_t part, const fhe_b200_ksk* const* keys,
                              uint32_t n_keys, const uint32_t* key_index, fhe_b200_batch* out2, void* stream) {
  API_BEGIN
  key_switch_run(pb, part, key_list(keys, n_keys, key_index), out2, stream);
  API_END
}

int fhe_b200_switch_down(fhe_b200_batch* b, void* stream) {
  API_BEGIN
  REQUIRE(b, FHE_B200_INVALID_ARGUMENT, "null argument");
  REQUIRE(!b->mul_basis, FHE_B200_CONTEXT_MISMATCH, "PolynomialContextMismatch");
  need_repr(b, FHE_B200_NTT);
  const fhe_b200_params* par = b->par;
  const LevelData& lv = par->level(b->level);
  REQUIRE(lv.L >= 2, FHE_B200_NO_MORE_CONTEXT, "NoMoreContext");
  DeviceGuard g(par);
  cudaStream_t st = (cudaStream_t)stream;
  const LevelData& nl = par->level(b->level + 1);
  const u32 polys = b->count * b->parts;
  // Stream-ordered and in place: the L-1 surviving rows of every polynomial go through scratch memory and the forward
  // transform writes them back, compacted, at the start of the batch's own allocation (which keeps its size: the
  // pointer handed out by fhe_b200_batch_device_ptr stays valid, nothing is allocated, freed or synchronised here).
  Workspace ws(par, st);
  switch_down_polys(par, b->level, b->d, polys, ws, st);
  FHE_CUDA(cudaGetLastError());
  b->level += 1;
  b->limbs = nl.L;
  API_END
}

int fhe_b200_scale(const fhe_b200_batch* in, int which, fhe_b200_batch* out, void* stream) {
  API_BEGIN
  REQUIRE(in && out && in != out, FHE_B200_INVALID_ARGUMENT, "null or aliased argument");
  REQUIRE(in->par == out->par, FHE_B200_CONTEXT_MISMATCH, "ParameterMismatch");
  REQUIRE(in->level == out->level, FHE_B200_INVALID_LEVEL, "InvalidLevel");
  REQUIRE(in->count == out->count && in->parts == out->parts, FHE_B200_BAD_POLY_COUNT, "shapes differ");
  REQUIRE(which == 0 || which == 1, FHE_B200_INVALID_ARGUMENT, "which must be 0 or 1");
  REQUIRE(in->mul_basis == (which == 1) && out->mul_basis == (which == 0), FHE_B200_CONTEXT_MISMATCH,
          "PolynomialContextMismatch");
  need_repr(in, FHE_B200_NTT);
  const fhe_b200_params* par = in->par;
  DeviceGuard g(par);
  cudaStream_t st = (cudaStream_t)stream;
  const LevelData& lv = par->level(in->level);
  const size_t row = (size_t)1 << par->logn;
  const u32 polys = in->count * in->parts;
  Workspace ws(par, st);
  u64* pb = ws.words((size_t)polys * in->limbs * row);
  launch_ntt(in->d, pb, polys * in->limbs, ids_of(in), par->d_limbs, par->logn, true, 1, false, st);
  if (which == 0) {  // extender: common prefix copied, E new rows computed (rq/scaler.rs:61-65, :85-115)
    FHE_CUDA(cudaMemcpy2DAsync(out->d, lv.K * row * 8, in->d, lv.L * row * 8, lv.L * row * 8, polys,
                               cudaMemcpyDeviceToDevice, st));
    u64* x = ws.words((size_t)polys * lv.E * row);
    launch_scale(lv.ext.dev, par->d_limbs, pb, x, nullptr, polys, lv.E, lv.L, lv.E, 0, par->logn, st);
    launch_ntt(x, x, polys * lv.E, lv.ext_ids, par->d_limbs, par->logn, false, 1, false, st);
    FHE_CUDA(cudaMemcpy2DAsync(out->d + lv.L * row, lv.K * row * 8, x, lv.E * row * 8, lv.E * row * 8, polys,
                               cudaMemcpyDeviceToDevice, st));
  } else {
    launch_scale(lv.down.dev, par->d_limbs, pb, out->d, nullptr, polys, lv.L, 0, lv.L, 0, par->logn, st);
    launch_ntt(out->d, out->d, polys * lv.L, lv.ctx_ids, par->d_limbs, par->logn, false, 1, false, st);
  }
  FHE_CUDA(cudaGetLastError());
  out->repr = FHE_B200_NTT;
  API_END
}

// ------------------------------------------------------------------------------ wire format
static PackDev pack_desc(const fhe_b200_batch* b) {
  const fhe_b200_params* par = b->par;
  const LevelData& lv = par->level(b->level);
  PackDev P;
  std::memset(&P, 0, sizeof(P));
  P.limbs = b->limbs;
  u32 off = 0;
  for (u32 i = 0; i < b->limbs; i++) {
    const u64 q = b->mul_basis ? lv.mul_moduli[i] : par->moduli[i];
    const u32 nb = 64 - (u32)clz64(q - 1);          // Modulus::serialize_vec, zq/mod.rs:784
    P.nbits[i] = (unsigned char)nb;
    P.offs[i] = off;
    off += nb * (par->N / 8);                        // serialization_length, zq/mod.rs:773-777
  }
  P.poly_bytes = off;
  return P;
}
int fhe_b200_poly_packed_bytes(const fhe_b200_params* p, uint32_t level, size_t* nbytes) {
  API_BEGIN
  REQUIRE(p && nbytes, FHE_B200_INVALID_ARGUMENT, "null argument");
  const LevelData& lv = p->level(level);
  size_t n = 0;
  for (u32 i = 0; i < lv.L; i++) n += (size_t)(64 - clz64(p->moduli[i] - 1)) * (p->N / 8);
  *nbytes = n;
  API_END
}
int fhe_b200_batch_packed_bytes(const fhe_b200_batch* b, size_t* nbytes) {
  API_BEGIN
  REQUIRE(b && nbytes, FHE_B200_INVALID_ARGUMENT, "null argument");
  *nbytes = pack_desc(b).poly_bytes;
  API_END
}
int fhe_b200_batch_pack(const fhe_b200_batch* b, uint32_t first, uint32_t n, uint8_t* host_out, void* stream) {
  API_BEGIN
  REQUIRE(b && host_out, FHE_B200_INVALID_ARGUMENT, "null argument");
  REQUIRE((uint64_t)first + n <= b->count, FHE_B200_INVALID_ARGUMENT, "range exceeds batch");
  const fhe_b200_params* par = b->par;
  DeviceGuard g(par);
  cudaStream_t st = (cudaStream_t)stream;
  const PackDev P = pack_desc(b);
  const size_t rows = (size_t)n * b->parts * b->limbs, row = (size_t)1 << par->logn;
  Workspace ws(par, st);
  const u64* src = b->d + b->words_per_ct() * first;
  if (b->repr == FHE_B200_NTT) {   // rq/convert.rs:20-24: serialization is always in power basis
    u64* pb = ws.words(rows * row);
    launch_ntt(src, pb, (u32)rows, ids_of(b), par->d_limbs, par->logn, true, 1, false, st);
    src = pb;
  }
  const size_t nbytes = (size_t)n * b->parts * P.poly_bytes;
  unsigned char* dbytes = (unsigned char*)ws.words((nbytes + 7) / 8);
  launch_pack(P, src, dbytes, rows, par->logn, st);
  FHE_CUDA(cudaGetLastError());
  FHE_CUDA(cudaMemcpyAsync(host_out, dbytes, nbytes, cudaMemcpyDeviceToHost, st));
  FHE_CUDA(cudaStreamSynchronize(st));
  API_END
}
int fhe_b200_batch_unpack(fhe_b200_batch* b, uint32_t first, uint32_t n, const uint8_t* host_in, void* stream) {
  API_BEGIN
  REQUIRE(b && host_in, FHE_B200_INVALID_ARGUMENT, "null argument");
  REQUIRE((uint64_t)first + n <= b->count, FHE_B200_INVALID_ARGUMENT, "range exceeds batch");
  const fhe_b200_params* par = b->par;
  DeviceGuard g(par);
  cudaStream_t st = (cudaStream_t)stream;
  const PackDev P = pack_desc(b);
  const size_t rows = (size_t)n * b->parts * b->limbs;
  Workspace ws(par, st);
  const size_t nbytes = (size_t)n * b->parts * P.poly_bytes;
  unsigned char* dbytes = (unsigned char*)ws.words((nbytes + 7) / 8);
  FHE_CUDA(cudaMemcpyAsync(dbytes, host_in, nbytes, cudaMemcpyHostToDevice, st));
  u64* dst = b->d + b->words_per_ct() * first;
  launch_unpack(P, dbytes, dst, rows, par->logn, st);
  if (b->repr == FHE_B200_NTT)     // rq/convert.rs:128-129: p.into_ntt()
    launch_ntt(dst, dst, (u32)rows, ids_of(b), par->d_limbs, par->logn, false, 1, false, st);
  FHE_CUDA(cudaGetLastError());
  API_END
}

// ---- bit transcoding and the SealPIR reply fold
static bool device_resident(const void* ptr, int device) {
  cudaPointerAttributes a;
  if (cudaPointerGetAttributes(&a, ptr) != cudaSuccess) {
    cudaGetLastError();
    return false;
  }
  return a.type == cudaMemoryTypeManaged || (a.type == cudaMemoryTypeDevice && a.device == device);
}

// rows [r0, r0 + n) of a strided host or device array, as one contiguous copy when the rows are adjacent
static void copy_rows(char* dst, size_t dst_pitch, const char* src, size_t src_pitch, size_t width, size_t n,
                      cudaStream_t st) {
  if (!width || !n) return;
  if (dst_pitch == width && src_pitch == width)
    FHE_CUDA(cudaMemcpyAsync(dst, src, width * n, cudaMemcpyDefault, st));
  else
    FHE_CUDA(cudaMemcpy2DAsync(dst, dst_pitch, src, src_pitch, width, n, cudaMemcpyDefault, st));
}

int fhe_b200_transcode(const fhe_b200_params* p, const void* in, uint32_t in_elem, size_t in_len, size_t in_stride,
                       uint32_t in_bits, void* out, uint32_t out_elem, size_t out_len, size_t out_stride,
                       uint32_t out_bits, uint32_t n_rows, void* stream) {
  API_BEGIN
  REQUIRE(p, FHE_B200_INVALID_ARGUMENT, "null argument");
  REQUIRE(in_bits >= 1 && in_bits <= 64 && out_bits >= 1 && out_bits <= 64, FHE_B200_INVALID_ARGUMENT,
          "bit widths must be in 1..64");
  REQUIRE((in_elem == 8 || (in_elem == 1 && in_bits == 8)) && (out_elem == 8 || (out_elem == 1 && out_bits == 8)),
          FHE_B200_INVALID_ARGUMENT, "elements are u64 words (8) or bytes (1, with 8 bits)");
  REQUIRE(n_rows > 0, FHE_B200_INVALID_ARGUMENT, "no rows");
  REQUIRE(in_stride >= in_len && out_stride >= out_len, FHE_B200_INVALID_ARGUMENT, "stride shorter than the row");
  REQUIRE((in || !in_len) && (out || !out_len), FHE_B200_INVALID_ARGUMENT, "null rows");
  const uintptr_t ib = (uintptr_t)in, ob = (uintptr_t)out;
  const uintptr_t ie = ib + ((size_t)(n_rows - 1) * in_stride + in_len) * in_elem;
  const uintptr_t oe = ob + ((size_t)(n_rows - 1) * out_stride + out_len) * out_elem;
  REQUIRE(!in_len || !out_len || ie <= ob || oe <= ib, FHE_B200_INVALID_ARGUMENT, "in and out overlap");
  DeviceGuard g(p);
  const bool in_dev = !in_len || device_resident(in, p->device), out_dev = !out_len || device_resident(out, p->device);
  // a chunk stages at most what one chunk of level-0 ciphertexts holds
  const size_t budget = ((size_t)chunk_size() * 2 * p->Lmax) << p->logn;
  const size_t row_words = std::max<size_t>({1, (in_len * in_elem + 7) / 8, (out_len * out_elem + 7) / 8});
  const u32 rows_per_chunk = (u32)std::max<size_t>(1, std::min<size_t>(budget / row_words, n_rows));
  ChunkRunner chunks(p, n_rows, (cudaStream_t)stream, rows_per_chunk);
  chunks.run([&](u32 r0, u32 n, cudaStream_t st) {
    Workspace ws(p, st);
    TranscodeRows T;
    T.in_len = in_len; T.in_elem = in_elem; T.in_bits = in_bits;
    T.out_len = out_len; T.out_elem = out_elem; T.out_bits = out_bits;
    const char* src = (const char*)in + (size_t)r0 * in_stride * in_elem;
    char* dst = (char*)out + (size_t)r0 * out_stride * out_elem;
    if (in_dev) {
      T.in = src;
      T.in_stride = in_stride;
    } else {
      char* staged = (char*)ws.words(((size_t)n * in_len * in_elem + 7) / 8);
      copy_rows(staged, in_len * in_elem, src, in_stride * in_elem, in_len * in_elem, n, st);
      T.in = staged;
      T.in_stride = in_len;
    }
    if (out_dev) {
      T.out = dst;
      T.out_stride = out_stride;
    } else {
      T.out = ws.words(((size_t)n * out_len * out_elem + 7) / 8);
      T.out_stride = out_len;
    }
    launch_transcode(T, n, st);
    if (!out_dev) copy_rows(dst, out_stride * out_elem, (const char*)T.out, out_len * out_elem, out_len * out_elem, n, st);
  });
  FHE_CUDA(cudaGetLastError());
  API_END
}

int fhe_b200_fold(const fhe_b200_batch* ct, uint32_t in_bits, uint32_t out_bits, fhe_b200_batch* out, void* stream) {
  API_BEGIN
  REQUIRE(ct && out, FHE_B200_INVALID_ARGUMENT, "null argument");
  REQUIRE(ct->par == out->par, FHE_B200_CONTEXT_MISMATCH, "ParameterMismatch");
  REQUIRE(!ct->mul_basis && !out->mul_basis, FHE_B200_CONTEXT_MISMATCH, "PolynomialContextMismatch");
  REQUIRE(out->parts == 1, FHE_B200_BAD_POLY_COUNT, "a plaintext batch has one polynomial per entry");
  REQUIRE(in_bits >= 1 && in_bits <= 64 && out_bits >= 1 && out_bits <= 64, FHE_B200_INVALID_ARGUMENT,
          "bit widths must be in 1..64");
  REQUIRE(out != ct, FHE_B200_INVALID_ARGUMENT, "out aliases ct");
  const fhe_b200_params* par = ct->par;
  const size_t N = par->N, row_words = (size_t)ct->limbs * N;
  const size_t E = (row_words * in_bits + out_bits - 1) / out_bits;
  const size_t P = (ct->parts * E + N - 1) / N;
  REQUIRE(out->count == P * ct->count, FHE_B200_INVALID_ARGUMENT,
          "out must hold ceil(parts * ceil(L * N * in_bits / out_bits) / N) plaintexts per ciphertext");
  DeviceGuard g(par);
  const LevelData& lv = par->level(out->level);
  const u32 L = lv.L, logn = par->logn, count = ct->count;
  // Poly u64 words are arbitrary: the forward butterflies reduce them on load, as fhe_b200_encode does
  ChunkRunner chunks(par, count, (cudaStream_t)stream, std::max<u32>(1, chunk_size() / (u32)P));
  chunks.run([&](u32 c0, u32 n, cudaStream_t st) {
    Workspace ws(par, st);
    u64* coeffs = ws.words((P * n) << logn);
    launch_fold_stage(ct->d + c0 * ct->words_per_ct(), n, ct->parts, row_words, in_bits, out_bits, (u32)P, coeffs, logn,
                      st);
    for (size_t i = 0; i < P; i++)
      launch_ntt(coeffs + ((i * n) << logn), out->d + ((i * count + c0) * L << logn), n * L, lv.ctx_ids, par->d_limbs,
                 logn, false, L, true, st);
  });
  FHE_CUDA(cudaGetLastError());
  out->repr = FHE_B200_NTT;
  API_END
}

int fhe_b200_sync(void* stream) {
  API_BEGIN
  FHE_CUDA(cudaStreamSynchronize((cudaStream_t)stream));
  API_END
}

// ------------------------------------------------------------------------------ inspection
int fhe_b200_debug_scaler_tables(const fhe_b200_params* p, uint32_t level, int which, uint32_t* n_from, uint32_t* n_to,
                                 uint32_t* shift, uint64_t* gamma, uint64_t* omega, uint64_t* theta_gamma,
                                 uint64_t* theta_omega_lo, uint64_t* theta_omega_hi, uint8_t* theta_omega_sign,
                                 uint64_t* theta_garner_lo, uint64_t* theta_garner_hi) {
  API_BEGIN
  REQUIRE(p, FHE_B200_INVALID_ARGUMENT, "null argument");
  const LevelData& lv = p->level(level);
  REQUIRE(which >= 0 && which <= 2, FHE_B200_INVALID_ARGUMENT, "which must be 0, 1 or 2");
  const ScalerTablesH& h = which == 0 ? lv.ext.h : which == 1 ? lv.down.h : lv.plain.h;
  if (n_from) *n_from = h.n_from;
  if (n_to) *n_to = h.n_to;
  if (shift) *shift = h.shift;
  auto cp = [](uint64_t* dst, const std::vector<u64>& v) {
    if (dst) for (size_t i = 0; i < v.size(); i++) dst[i] = v[i];
  };
  cp(gamma, h.gamma);
  cp(omega, h.omega);
  if (theta_gamma) { theta_gamma[0] = h.theta_gamma_lo; theta_gamma[1] = h.theta_gamma_hi; theta_gamma[2] = h.theta_gamma_sign; }
  cp(theta_omega_lo, h.theta_omega_lo);
  cp(theta_omega_hi, h.theta_omega_hi);
  if (theta_omega_sign) for (size_t i = 0; i < h.theta_omega_sign.size(); i++) theta_omega_sign[i] = h.theta_omega_sign[i];
  cp(theta_garner_lo, h.theta_garner_lo);
  cp(theta_garner_hi, h.theta_garner_hi);
  API_END
}

int fhe_b200_debug_ntt_tables(const fhe_b200_params* p, uint64_t q, uint64_t* omegas, uint64_t* omegas_shoup,
                              uint64_t* zetas_inv, uint64_t* zetas_inv_shoup, uint64_t* size_inv) {
  API_BEGIN
  REQUIRE(p, FHE_B200_INVALID_ARGUMENT, "null argument");
  int i = prime_index(p->primes, q);
  REQUIRE(i >= 0, FHE_B200_INVALID_MODULUS, "prime not in parameter set");
  const NttTablesH& t = p->tables[i];
  auto cp = [](uint64_t* dst, const std::vector<u64>& v) {
    if (dst) for (size_t k = 0; k < v.size(); k++) dst[k] = v[k];
  };
  cp(omegas, t.om);
  cp(omegas_shoup, t.om_s);
  cp(zetas_inv, t.zi);
  cp(zetas_inv_shoup, t.zi_s);
  if (size_inv) *size_inv = t.ninv;
  API_END
}

int fhe_b200_debug_expansion_monomial(const fhe_b200_params* p, uint32_t level, uint32_t l, uint64_t* out) {
  API_BEGIN
  REQUIRE(p && out, FHE_B200_INVALID_ARGUMENT, "null argument");
  REQUIRE(l < p->logn, FHE_B200_INVALID_ARGUMENT, "expansion level must be below log2 N");
  const std::vector<u64> w = p->expansion_monomial(level, l);
  std::copy(w.begin(), w.end(), out);
  API_END
}

int fhe_b200_debug_encoder_tables(const fhe_b200_encoder* e, uint32_t level, uint32_t* index_map, uint64_t* omegas,
                                  uint64_t* zetas_inv, uint64_t* q_mod_t, uint64_t* delta) {
  API_BEGIN
  REQUIRE(e, FHE_B200_INVALID_ARGUMENT, "null argument");
  const fhe_b200_params* p = e->par;
  const LevelData& lv = p->level(level);
  if (index_map) std::copy(e->index_map.begin(), e->index_map.end(), index_map);
  if (omegas || zetas_inv) {
    REQUIRE(e->has_ntt, FHE_B200_NTT_UNAVAILABLE, "NttOperatorUnavailable: plaintext modulus");
    if (omegas) std::copy(e->tables.om.begin(), e->tables.om.end(), omegas);
    if (zetas_inv) std::copy(e->tables.zi.begin(), e->tables.zi.end(), zetas_inv);
  }
  if (q_mod_t) {
    REQUIRE(p->t_small, FHE_B200_UNSUPPORTED, "the plaintext modulus does not fit a u64 Modulus");
    *q_mod_t = lv.q_mod_t;
  }
  if (delta) std::copy(lv.delta.begin(), lv.delta.end(), delta);
  API_END
}

}  // extern "C"
