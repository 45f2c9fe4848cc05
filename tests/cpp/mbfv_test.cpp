// Multiparty BFV through the mbfv namespace of include/fhe_b200.hpp (driven by
// tests/test_gpu_mbfv.py::test_cpp_mbfv):
//   argv: degree t count dir; dir holds moduli.bin (u64), sk0.bin and sk1.bin (SecretKey messages), seeds.bin (32-byte
//   seeds, used in the order below) and ct.bin (count 2-part level-0 ciphertexts, [count][2][L][N] u64).
// Writes the words of every object, u64 [..][N]: crp.bin (new_vec), pk.bin (the aggregated public key),
// dec.bin (Plaintext::from_shares of both parties' decryption shares), sks.bin (key switch from sk0 + sk1 to sk1 + sk0),
// pks.bin (public key switch to pk), r1.bin (round-1 aggregate h0 then h1), rk.bin (the relinearization key's c0 then
// c1, [digit][limb][N]).
#include <cstdio>
#include <fstream>
#include <iostream>
#include <string>
#include <vector>

#include "fhe_b200_wire.hpp"

using namespace fhe_b200;
using namespace fhe_b200::bfv;
namespace M = fhe_b200::mbfv;

template <typename T>
static std::vector<T> read_file(const std::string& path) {
  std::ifstream f(path, std::ios::binary | std::ios::ate);
  const size_t n = (size_t)f.tellg() / sizeof(T);
  std::vector<T> v(n);
  f.seekg(0);
  f.read(reinterpret_cast<char*>(v.data()), n * sizeof(T));
  return v;
}
template <typename T>
static void write_file(const std::string& path, const std::vector<T>& v) {
  std::ofstream(path, std::ios::binary).write(reinterpret_cast<const char*>(v.data()), v.size() * sizeof(T));
}
static void append(std::vector<uint64_t>& a, const std::vector<uint64_t>& b) { a.insert(a.end(), b.begin(), b.end()); }

int main(int argc, char** argv) {
  if (argc != 5) return 2;
  const size_t degree = std::stoul(argv[1]);
  const uint64_t t = std::stoull(argv[2]);
  const uint32_t count = (uint32_t)std::stoul(argv[3]);
  const std::string dir = argv[4];
  try {
    auto par = BfvParametersBuilder().set_degree(degree).set_plaintext_modulus(t)
                   .set_moduli(read_file<uint64_t>(dir + "/moduli.bin")).build_arc();
    std::vector<std::shared_ptr<SecretKey>> sks;
    for (const char* f : {"/sk0.bin", "/sk1.bin"}) {
      const auto msg = read_file<char>(dir + f);
      sks.push_back(secret_key_from_bytes(par, std::string(msg.begin(), msg.end())));
    }
    const auto seeds = read_file<uint8_t>(dir + "/seeds.bin");
    const uint8_t* sd = seeds.data();
    auto next = [&]() { const uint8_t* s = sd; sd += 32; return s; };
    const Ciphertext ct = Ciphertext::from_host(par, read_file<uint64_t>(dir + "/ct.bin"), count, 2, 0);

    const auto crps = M::CommonRandomPoly::new_vec(par, next());
    std::vector<uint64_t> crp_words;
    for (const auto& c : crps) append(crp_words, c.batch->to_host());
    write_file(dir + "/crp.bin", crp_words);

    std::vector<M::PublicKeyShare> pk_shares;
    for (const auto& sk : sks) pk_shares.emplace_back(*sk, crps[0], next());
    const PublicKey pk = M::public_key_from_shares(pk_shares);
    write_file(dir + "/pk.bin", pk.c().to_host());

    std::vector<M::DecryptionShare> dec;
    for (const auto& sk : sks) dec.emplace_back(*sk, ct, next());
    write_file(dir + "/dec.bin", M::plaintext_from_shares(dec).batch().to_host());

    std::vector<M::SecretKeySwitchShare> sw;
    sw.emplace_back(*sks[0], sks[1].get(), ct, next());
    sw.emplace_back(*sks[1], sks[0].get(), ct, next());
    write_file(dir + "/sks.bin", M::ciphertext_from_shares(sw).to_host());

    std::vector<M::PublicKeySwitchShare> pw;
    for (const auto& sk : sks) pw.emplace_back(*sk, pk, ct, next());
    write_file(dir + "/pks.bin", M::ciphertext_from_shares(pw).to_host());

    std::vector<std::unique_ptr<M::RelinKeyGenerator>> gens;
    for (const auto& sk : sks) gens.emplace_back(new M::RelinKeyGenerator(*sk, crps, next()));
    std::vector<M::RelinKeyShare> r1s;
    for (const auto& g : gens) r1s.push_back(g->round_1(next()));
    const auto r1 = std::make_shared<const M::RelinKeyShare>(M::r1_from_shares(r1s));
    std::vector<uint64_t> r1_words = r1->h0->to_host();
    append(r1_words, r1->h1->to_host());
    write_file(dir + "/r1.bin", r1_words);
    std::vector<M::RelinKeyShare> r2s;
    for (const auto& g : gens) r2s.push_back(g->round_2(r1, next()));
    const RelinearizationKey rk = M::relin_key_from_shares(r2s);
    auto w = rk.ksk->arrays();
    append(w.first, w.second);
    write_file(dir + "/rk.bin", w.first);

    try {
      M::plaintext_from_shares({});
      std::cout << "FAIL no shares accepted\n";
      return 1;
    } catch (const Error& e) {
      if (e.code != FHE_B200_INVALID_ARGUMENT) throw;
    }
    std::cout << "OK\n";
  } catch (const Error& e) {
    std::cout << "FAIL " << e.code << " " << e.what() << "\n";
    return 1;
  }
  return 0;
}
