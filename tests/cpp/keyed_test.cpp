// Per-ciphertext keys through include/fhe_b200.hpp: multiply_keyed, relinearizes_keyed, galois_keyed, key_switch_keyed,
// external_products_keyed and expands_keyed on words prepared by tests/test_gpu_keyed.py, whose results it writes back
// for the test to compare with the Python mirror's.
// usage: keyed_test <dir>   with <dir>/args.txt = "degree t n_moduli count n_keys" followed by the moduli and the
// count key indices, <dir>/a.bin, b.bin = [count][2][L][N] words, <dir>/k<k>_c0.bin / _c1.bin = [L][L][N] words of
// key k (used as relinearization key, Galois key for 3, N + 1 and N/2 + 1, and both halves of an RGSW ciphertext)
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
    uint32_t degree, nmod, count, nkeys;
    uint64_t t;
    args >> degree >> t >> nmod >> count >> nkeys;
    std::vector<uint64_t> moduli(nmod);
    for (auto& q : moduli) args >> q;
    std::vector<uint32_t> index(count);
    for (auto& i : index) args >> i;
    auto par = BfvParametersBuilder().set_degree(degree).set_plaintext_modulus(t).set_moduli(moduli).build_arc();
    std::vector<std::shared_ptr<KeySwitchingKey>> ksk;
    std::vector<RelinearizationKey> rk;
    std::vector<GaloisKey> gk;
    std::vector<RGSWCiphertext> rgsw;
    std::vector<EvaluationKey> ek;
    for (uint32_t k = 0; k < nkeys; k++) {
      const std::string stem = dir + "/k" + std::to_string(k);
      ksk.push_back(std::make_shared<KeySwitchingKey>(par, read_words(stem + "_c0.bin"), read_words(stem + "_c1.bin"), nmod));
      rk.emplace_back(ksk.back());
      gk.emplace_back(3, ksk.back());
      rgsw.emplace_back(ksk.back(), ksk.back());
      ek.emplace_back(par);
      ek.back().add_galois_key(std::make_shared<GaloisKey>(degree + 1, ksk.back()));
      ek.back().add_galois_key(std::make_shared<GaloisKey>(degree / 2 + 1, ksk.back()));
    }
    std::vector<const KeySwitchingKey*> pk;
    std::vector<const RelinearizationKey*> prk;
    std::vector<const GaloisKey*> pgk;
    std::vector<const RGSWCiphertext*> prg;
    std::vector<const EvaluationKey*> pek;
    for (uint32_t k = 0; k < nkeys; k++) {
      pk.push_back(ksk[k].get());
      prk.push_back(&rk[k]);
      pgk.push_back(&gk[k]);
      prg.push_back(&rgsw[k]);
      pek.push_back(&ek[k]);
    }
    const Ciphertext a = Ciphertext::from_host(par, read_words(dir + "/a.bin"), count);
    const Ciphertext b = Ciphertext::from_host(par, read_words(dir + "/b.bin"), count);
    write_words(dir + "/out_mul.bin", multiply_keyed(a, b, prk, index).to_host());
    write_words(dir + "/out_relin.bin", relinearizes_keyed(a * b, prk, index).to_host());
    write_words(dir + "/out_galois.bin", galois_keyed(a, pgk, index).to_host());
    Ciphertext pb = a.clone();
    pb.into_power_basis();
    write_words(dir + "/out_ks.bin", key_switch_keyed(pb, 1, pk, index).to_host());
    write_words(dir + "/out_ext.bin", external_products_keyed(a, prg, index).to_host());
    std::vector<uint64_t> listed;
    for (const Ciphertext& c : expands_keyed(a, pek, index, 4)) {
      const auto w = c.to_host();
      listed.insert(listed.end(), w.begin(), w.end());
    }
    write_words(dir + "/out_expand.bin", listed);
    std::vector<uint32_t> bad(index);
    bad[0] = nkeys;
    try {
      multiply_keyed(a, b, prk, bad);
      printf("FAIL index beyond the key list accepted\n");
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
