// Linear transforms through include/fhe_b200.hpp: linear_transform (with n_fallback) and
// EvaluationKey::linear_transform on words prepared by tests/test_gpu_linear_transform.py, whose results it writes back
// for the test to compare with the Python mirror's; encode_diagonals and linear_transform_steps are checked here.
// usage: linear_transform_test <dir>   with <dir>/args.txt = "degree t n_moduli count n_diags baby n_keys" followed by
// the moduli and the n_keys exponents, <dir>/a.bin = [count][2][L][N] words, <dir>/d.bin = [count * n_diags][1][L][N]
// words (one matrix per ciphertext), <dir>/k<k>_c0.bin / _c1.bin = [L][L][N] words of the Galois key k.
#include <cstdio>
#include <fstream>
#include <iterator>

#include "fhe_b200.hpp"

using namespace fhe_b200::bfv;

static std::vector<uint64_t> read_words(const std::string& path) {
  std::ifstream in(path, std::ios::binary);
  std::string data((std::istreambuf_iterator<char>(in)), std::istreambuf_iterator<char>());
  std::vector<uint64_t> w(data.size() / 8);
  std::copy(data.begin(), data.begin() + w.size() * 8, (char*)w.data());
  return w;
}
static void write_words(const std::string& path, const std::vector<uint64_t>& w) {
  std::ofstream out(path, std::ios::binary);
  out.write((const char*)w.data(), (std::streamsize)(w.size() * 8));
}

int main(int argc, char** argv) {
  if (argc < 2) return 2;
  const std::string dir = argv[1];
  try {
    std::ifstream args(dir + "/args.txt");
    uint32_t degree, nmod, count, n_diags, baby, nkeys;
    uint64_t t;
    args >> degree >> t >> nmod >> count >> n_diags >> baby >> nkeys;
    std::vector<uint64_t> moduli(nmod);
    for (auto& q : moduli) args >> q;
    std::vector<uint32_t> exps(nkeys);
    for (auto& e : exps) args >> e;
    auto par = BfvParametersBuilder().set_degree(degree).set_plaintext_modulus(t).set_moduli(moduli).build_arc();
    std::vector<GaloisKey> gk;
    EvaluationKey ek(par);
    for (uint32_t k = 0; k < nkeys; k++) {
      const std::string stem = dir + "/k" + std::to_string(k);
      auto ksk = std::make_shared<KeySwitchingKey>(par, read_words(stem + "_c0.bin"), read_words(stem + "_c1.bin"), nmod);
      gk.emplace_back(exps[k], ksk);
      ek.add_galois_key(std::make_shared<GaloisKey>(exps[k], ksk));
    }
    std::vector<const GaloisKey*> pgk;
    for (const GaloisKey& g : gk) pgk.push_back(&g);
    const Ciphertext a = Ciphertext::from_host(par, read_words(dir + "/a.bin"), count);
    const Ciphertext d = Ciphertext::from_host(par, read_words(dir + "/d.bin"), count * n_diags, 1);
    uint32_t n_fallback = 99;
    write_words(dir + "/out_call.bin", linear_transform(a, d, n_diags, baby, pgk, &n_fallback).to_host());
    write_words(dir + "/out_ek.bin", ek.linear_transform(a, d, baby, n_diags).to_host());
    if (linear_transform_steps(10, 3) != std::vector<uint32_t>{1, 2, 3, 6, 9}) {
      printf("FAIL linear_transform_steps\n");
      return 1;
    }
    // the identity matrix has one diagonal: encoded, it is the all-ones slot vector
    const size_t half = degree / 2;
    std::vector<uint64_t> id(2 * half * half);
    for (size_t q = 0; q < 2; q++)
      for (size_t r = 0; r < half; r++) id[(q * half + r) * half + r] = 1;
    const PlaintextVec pv = encode_diagonals(par, id, 1, 1, 0, 1);
    const Encoding simd = Encoding::simd();
    const std::vector<uint64_t> ones = pv.try_decode<uint64_t>(&simd);
    for (uint64_t v : ones)
      if (v != 1) {
        printf("FAIL encode_diagonals of the identity\n");
        return 1;
      }
    try {
      linear_transform(a, d, n_diags, n_diags + 1, pgk);
      printf("FAIL a baby step beyond n_diags accepted\n");
      return 1;
    } catch (const fhe_b200::Error& e) {
      if (e.code != FHE_B200_INVALID_ARGUMENT) throw;
    }
    printf("OK n_fallback %u\n", n_fallback);
    return 0;
  } catch (const std::exception& e) {
    printf("FAIL %s\n", e.what());
    return 1;
  }
}
