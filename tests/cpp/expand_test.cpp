// Oblivious expansion and inner sum through include/fhe_b200.hpp: EvaluationKey::expands / expands_batch /
// computes_inner_sum and Ciphertext::take on words prepared by tests/test_gpu_expand.py, whose results it writes back
// for the test to compare with the Python mirror's.
// usage: expand_test <dir>   with <dir>/args.txt = "degree t n_moduli size count n_keys" followed by the moduli and the
// key exponents, <dir>/ct.bin = [count][2][L][N] words, <dir>/gk<k>_c0.bin / _c1.bin = [L][L][N] words of key k
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
    uint32_t degree, nmod, size, count, nkeys;
    uint64_t t;
    args >> degree >> t >> nmod >> size >> count >> nkeys;
    std::vector<uint64_t> moduli(nmod);
    for (auto& q : moduli) args >> q;
    auto par = BfvParametersBuilder().set_degree(degree).set_plaintext_modulus(t).set_moduli(moduli).build_arc();
    EvaluationKey ek(par);
    for (uint32_t k = 0; k < nkeys; k++) {
      uint32_t e;
      args >> e;
      const std::string stem = dir + "/gk" + std::to_string(k);
      auto ksk = std::make_shared<KeySwitchingKey>(par, read_words(stem + "_c0.bin"), read_words(stem + "_c1.bin"), nmod);
      ek.add_galois_key(std::make_shared<GaloisKey>(e, ksk));
    }
    const Ciphertext ct = Ciphertext::from_host(par, read_words(dir + "/ct.bin"), count);
    uint32_t level = 0;
    while ((1u << level) < size) level++;
    if (!ek.supports_expansion(level) || ek.supports_expansion(31)) {   // 2^31 > N: never supported
      printf("FAIL supports_expansion\n");
      return 1;
    }
    write_words(dir + "/out_batch.bin", ek.expands_batch(ct, size).to_host());
    std::vector<uint64_t> listed;
    for (const Ciphertext& c : ek.expands(ct, size)) {
      const auto w = c.to_host();
      listed.insert(listed.end(), w.begin(), w.end());
    }
    write_words(dir + "/out_list.bin", listed);
    if (!ek.supports_inner_sum()) {
      printf("FAIL supports_inner_sum\n");
      return 1;
    }
    write_words(dir + "/out_inner.bin", ek.computes_inner_sum(ct).to_host());
    try {
      ek.expands_batch(ct, 0);
      printf("FAIL size 0 accepted\n");
      return 1;
    } catch (const fhe_b200::Error& e) {
      if (e.code != FHE_B200_INVALID_ARGUMENT) throw;
    }
    printf("OK\n");
    return 0;
  } catch (const std::exception& e) {
    printf("FAIL %s\n", e.what());
    return 1;
  }
}
