// Generates keys through include/fhe_b200.hpp and serializes them through include/fhe_b200_wire.hpp (driven by
// tests/test_gpu_keygen.py::test_cpp_keygen):
//   argv: degree t dir; dir holds moduli.bin (u64), sk.bin (a SecretKey message), seeds.bin (four 32-byte seeds) and
//   values.bin (N u64 values below t).
// Writes the messages rk.bin (RelinearizationKey::new_key, seed 0), gk3.bin and gk_row.bin (one GaloisKey::generate
// call for the exponents 3 and 2N - 1, seed 1), gk_last.bin (the decomposition variant at the last level, seed 2) and
// rgsw.bin (try_encrypt_rgsw of the values as a Poly plaintext, seed 3).  Checks on its own that an inner-sum
// EvaluationKeyBuilder key sums the slots and that a failed generation throws with the reference's error.
#include <cstdio>
#include <fstream>
#include <iostream>
#include <string>
#include <vector>

#include "fhe_b200_wire.hpp"

using namespace fhe_b200;
using namespace fhe_b200::bfv;

template <typename T>
static std::vector<T> read_file(const std::string& path) {
  std::ifstream f(path, std::ios::binary | std::ios::ate);
  const size_t n = (size_t)f.tellg() / sizeof(T);
  std::vector<T> v(n);
  f.seekg(0);
  f.read(reinterpret_cast<char*>(v.data()), n * sizeof(T));
  return v;
}
static void write_msg(const std::string& path, const std::string& m) {
  std::ofstream(path, std::ios::binary).write(m.data(), (std::streamsize)m.size());
}

int main(int argc, char** argv) {
  if (argc != 4) return 2;
  const size_t degree = std::stoul(argv[1]);
  const uint64_t t = std::stoull(argv[2]);
  const std::string dir = argv[3];
  try {
    auto par = BfvParametersBuilder().set_degree(degree).set_plaintext_modulus(t)
                   .set_moduli(read_file<uint64_t>(dir + "/moduli.bin")).build_arc();
    const uint32_t last = (uint32_t)par->max_level();
    const auto msg = read_file<char>(dir + "/sk.bin");
    auto sk = secret_key_from_bytes(par, std::string(msg.begin(), msg.end()));
    const auto seeds = read_file<uint8_t>(dir + "/seeds.bin");
    const auto values = read_file<uint64_t>(dir + "/values.bin");
    write_msg(dir + "/rk.bin", to_bytes(RelinearizationKey::new_key(*sk, seeds.data())));
    const std::vector<GaloisKey> gks = GaloisKey::generate(*sk, {3, 2 * degree - 1}, 0, 0, seeds.data() + 32);
    write_msg(dir + "/gk3.bin", to_bytes(gks[0]));
    write_msg(dir + "/gk_row.bin", to_bytes(gks[1]));
    const GaloisKey low = GaloisKey::new_key(*sk, 2 * degree - 1, last, last, seeds.data() + 64);
    if (low.ksk->log_base() == 0 || low.ksk->n_digits() < 2) {
      std::cout << "FAIL the last-level key is not the decomposition variant\n";
      return 1;
    }
    write_msg(dir + "/gk_last.bin", to_bytes(low));
    const auto pts = PlaintextVec::try_encode(values, Encoding::poly(), par);
    write_msg(dir + "/rgsw.bin", to_bytes(sk->try_encrypt_rgsw(pts, seeds.data() + 96).at(0)));
    // the inner sum with keys made by the builder (fresh seeds)
    const EvaluationKey ek = EvaluationKeyBuilder(*sk).enable_inner_sum().build();
    const Encoding simd = Encoding::simd();
    const auto sum = sk->try_decrypt(ek.computes_inner_sum(sk->try_encrypt(PlaintextVec::try_encode(values, simd, par))))
                         .try_decode<uint64_t>(&simd);
    uint64_t want = 0;
    for (uint64_t v : values) want = (want + v) % t;
    for (uint64_t v : sum)
      if (v != want) {
        std::cout << "FAIL inner sum\n";
        return 1;
      }
    try {
      RelinearizationKey::new_leveled(*sk, last, last);
      std::cout << "FAIL a single-modulus relinearization key was made\n";
      return 1;
    } catch (const Error& e) {
      if (e.code != FHE_B200_UNSUPPORTED) throw;
    }
    try {
      GaloisKey::new_key(*sk, 4);
      std::cout << "FAIL an even exponent was accepted\n";
      return 1;
    } catch (const Error& e) {
      if (e.code != FHE_B200_INVALID_EXPONENT) throw;
    }
    std::cout << "OK\n";
  } catch (const Error& e) {
    std::cout << "FAIL " << e.code << " " << e.what() << "\n";
    return 1;
  }
  return 0;
}
