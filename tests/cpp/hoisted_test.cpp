// Hoisted rotations through include/fhe_b200.hpp: galois_many_hoisted (with n_hoisted) and
// EvaluationKey::rotates_columns_by_many_hoisted on words prepared by tests/test_gpu_hoisted.py, whose results it writes
// back for the test to compare with the Python mirror's.
// usage: hoisted_test <dir>   with <dir>/args.txt = "degree t n_moduli n_ct count n_keys" followed by the moduli, the
// n_keys exponents, the count key indices and the count source indices, <dir>/a.bin = [n_ct][2][L][N] words,
// <dir>/k<k>_c0.bin / _c1.bin = [L][L][N] words of the Galois key for exponent k.
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
    uint32_t degree, nmod, n_ct, count, nkeys;
    uint64_t t;
    args >> degree >> t >> nmod >> n_ct >> count >> nkeys;
    std::vector<uint64_t> moduli(nmod);
    for (auto& q : moduli) args >> q;
    std::vector<uint32_t> exps(nkeys), index(count), source(count);
    for (auto& e : exps) args >> e;
    for (auto& i : index) args >> i;
    for (auto& s : source) args >> s;
    auto par = BfvParametersBuilder().set_degree(degree).set_plaintext_modulus(t).set_moduli(moduli).build_arc();
    std::vector<std::shared_ptr<KeySwitchingKey>> ksk;
    std::vector<GaloisKey> gk;
    EvaluationKey ek(par);
    for (uint32_t k = 0; k < nkeys; k++) {
      const std::string stem = dir + "/k" + std::to_string(k);
      ksk.push_back(std::make_shared<KeySwitchingKey>(par, read_words(stem + "_c0.bin"), read_words(stem + "_c1.bin"), nmod));
      gk.emplace_back(exps[k], ksk.back());
      ek.add_galois_key(std::make_shared<GaloisKey>(exps[k], ksk[k]));
    }
    std::vector<const GaloisKey*> pgk;
    for (const GaloisKey& g : gk) pgk.push_back(&g);
    const Ciphertext a = Ciphertext::from_host(par, read_words(dir + "/a.bin"), n_ct);
    uint32_t n_hoisted = 0;
    const Ciphertext many = galois_many_hoisted(a, pgk, index, source, &n_hoisted);
    const std::vector<uint64_t> many_words = many.to_host();
    if (many_words != galois_many(a, pgk, index, source).to_host()) {
      printf("FAIL hoisted words differ from galois_many\n");
      return 1;
    }
    write_words(dir + "/out_many.bin", many_words);
    write_words(dir + "/out_rot.bin", ek.rotates_columns_by_many_hoisted(a, {1, 2, 4}).to_host());
    std::vector<uint32_t> bad(source);
    bad[0] = n_ct;
    try {
      galois_many_hoisted(a, pgk, index, bad);
      printf("FAIL source beyond the batch accepted\n");
      return 1;
    } catch (const fhe_b200::Error& e) {
      if (e.code != FHE_B200_INVALID_ARGUMENT) throw;
    }
    printf("OK n_hoisted %u\n", n_hoisted);
    return 0;
  } catch (const std::exception& e) {
    printf("FAIL %s\n", e.what());
    return 1;
  }
}
