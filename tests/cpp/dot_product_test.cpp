// Ciphertext dot products and batch sums through include/fhe_b200.hpp: batch_sum, dot_product (with and without a key,
// switched one level down) and dot_product_keyed on words prepared by tests/test_gpu_dot_product.py, whose results it
// writes back for the test to compare with the Python mirror's.
// usage: dot_product_test <dir>   with <dir>/args.txt = "degree t n_moduli groups n_terms" followed by the moduli and
// the groups key indices, <dir>/a.bin = [groups * n_terms][2][L][N] words, <dir>/b.bin = [n_terms][2][L][N] words (shared
// by every group), <dir>/k<k>_c0.bin / _c1.bin = [L][L][N] words of relinearization key k (k = 0, 1).
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
    uint32_t degree, nmod, groups, n_terms;
    uint64_t t;
    args >> degree >> t >> nmod >> groups >> n_terms;
    std::vector<uint64_t> moduli(nmod);
    for (auto& q : moduli) args >> q;
    std::vector<uint32_t> index(groups);
    for (auto& i : index) args >> i;
    auto par = BfvParametersBuilder().set_degree(degree).set_plaintext_modulus(t).set_moduli(moduli).build_arc();
    std::vector<RelinearizationKey> rks;
    for (uint32_t k = 0; k < 2; k++) {
      const std::string stem = dir + "/k" + std::to_string(k);
      rks.emplace_back(std::make_shared<KeySwitchingKey>(par, read_words(stem + "_c0.bin"), read_words(stem + "_c1.bin"),
                                                         nmod));
    }
    const Ciphertext a = Ciphertext::from_host(par, read_words(dir + "/a.bin"), groups * n_terms);
    const Ciphertext b = Ciphertext::from_host(par, read_words(dir + "/b.bin"), n_terms);
    write_words(dir + "/out_sum.bin", batch_sum(a, n_terms).to_host());
    write_words(dir + "/out_dot.bin", dot_product(a, b, n_terms, &rks[0], 1).to_host());
    write_words(dir + "/out_dot3.bin", dot_product(a, b, n_terms).to_host());
    write_words(dir + "/out_keyed.bin", dot_product_keyed(a, b, n_terms, {&rks[0], &rks[1]}, index).to_host());
    try {
      dot_product(a, b, n_terms + 1, &rks[0]);
      printf("FAIL a run length that does not divide the batch accepted\n");
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
