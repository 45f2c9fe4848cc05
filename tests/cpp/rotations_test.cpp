// Per-ciphertext Galois exponents and the batched inner sum through include/fhe_b200.hpp: galois_many,
// EvaluationKey::rotates_columns_by_many, EvaluationKey::computes_inner_sum and computes_inner_sum_keyed on words
// prepared by tests/test_gpu_rotations.py, whose results it writes back for the test to compare with the Python
// mirror's.
// usage: rotations_test <dir>   with <dir>/args.txt = "degree t n_moduli n_ct count n_keys" followed by the moduli, the
// n_keys exponents, the count key indices, the count source indices and the n_ct key-set indices, <dir>/a.bin =
// [n_ct][2][L][N] words, <dir>/k<k>_c0.bin / _c1.bin = [L][L][N] words of the Galois key for exponent k.  Key set 0
// holds key k for exponent k, key set 1 key k + 1 (mod n_keys) for it.
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
    std::vector<uint32_t> exps(nkeys), index(count), source(count), sets(n_ct);
    for (auto& e : exps) args >> e;
    for (auto& i : index) args >> i;
    for (auto& s : source) args >> s;
    for (auto& s : sets) args >> s;
    auto par = BfvParametersBuilder().set_degree(degree).set_plaintext_modulus(t).set_moduli(moduli).build_arc();
    std::vector<std::shared_ptr<KeySwitchingKey>> ksk;
    std::vector<GaloisKey> gk;
    for (uint32_t k = 0; k < nkeys; k++) {
      const std::string stem = dir + "/k" + std::to_string(k);
      ksk.push_back(std::make_shared<KeySwitchingKey>(par, read_words(stem + "_c0.bin"), read_words(stem + "_c1.bin"), nmod));
      gk.emplace_back(exps[k], ksk.back());
    }
    EvaluationKey ek0(par), ek1(par);
    for (uint32_t k = 0; k < nkeys; k++) {
      ek0.add_galois_key(std::make_shared<GaloisKey>(exps[k], ksk[k]));
      ek1.add_galois_key(std::make_shared<GaloisKey>(exps[k], ksk[(k + 1) % nkeys]));
    }
    std::vector<const GaloisKey*> pgk;
    for (const GaloisKey& g : gk) pgk.push_back(&g);
    const Ciphertext a = Ciphertext::from_host(par, read_words(dir + "/a.bin"), n_ct);
    write_words(dir + "/out_many.bin", galois_many(a, pgk, index, source).to_host());
    write_words(dir + "/out_rot.bin", ek0.rotates_columns_by_many(a, {1, 2, 4}).to_host());
    write_words(dir + "/out_isum.bin", ek0.computes_inner_sum(a).to_host());
    write_words(dir + "/out_isum_keyed.bin", computes_inner_sum_keyed(a, {&ek0, &ek1}, sets).to_host());
    std::vector<uint32_t> bad(source);
    bad[0] = n_ct;
    try {
      galois_many(a, pgk, index, bad);
      printf("FAIL source beyond the batch accepted\n");
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
