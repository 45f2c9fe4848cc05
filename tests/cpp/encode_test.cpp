// Encodes through include/fhe_b200.hpp (driven by tests/test_gpu_encode.py::test_cpp_encode):
//   argv: degree t dir; dir holds moduli.bin (u64), u64.bin (N slot values below t), i64.bin (N + 3 signed words).
// Writes simd.bin: SIMD encoding of u64.bin at level 0 (from page-locked memory), poly_l1.bin: Poly encoding of
// i64.bin at level 1 (two plaintexts), and checks that ct x pt with the SIMD plaintext equals the word form.
#include <cstdio>
#include <fstream>
#include <iostream>
#include <string>
#include <vector>

#include "fhe_b200.hpp"

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
static void write_file(const std::string& path, const std::vector<uint64_t>& v) {
  std::ofstream(path, std::ios::binary).write(reinterpret_cast<const char*>(v.data()), v.size() * sizeof(uint64_t));
}

int main(int argc, char** argv) {
  if (argc != 4) return 2;
  const size_t degree = std::stoul(argv[1]);
  const uint64_t t = std::stoull(argv[2]);
  const std::string dir = argv[3];
  try {
    auto par = BfvParametersBuilder().set_degree(degree).set_plaintext_modulus(t)
                   .set_moduli(read_file<uint64_t>(dir + "/moduli.bin")).build_arc();
    const auto u = read_file<uint64_t>(dir + "/u64.bin");
    const auto s = read_file<int64_t>(dir + "/i64.bin");
    PinnedWords pinned(u.size());
    std::copy(u.begin(), u.end(), pinned.data());
    auto simd = PlaintextVec::try_encode(pinned.data(), pinned.size(), Encoding::simd(), par);
    auto poly = PlaintextVec::try_encode(s, Encoding::poly_at_level(1), par);
    auto one = Plaintext::try_encode(u, Encoding::simd(), par);
    if (simd.len() != 1 || poly.len() != 2 || one.poly_ntt() != simd.poly_ntt()) {
      std::cout << "FAIL shapes\n";
      return 1;
    }
    write_file(dir + "/simd.bin", simd.poly_ntt());
    write_file(dir + "/poly_l1.bin", poly.poly_ntt());
    // ct x pt: device plaintext against its own words
    const size_t L = par->moduli().size();
    std::vector<uint64_t> ct_words(2 * L * degree);
    for (size_t i = 0; i < ct_words.size(); i++) ct_words[i] = (i * 2654435761u) % par->moduli()[(i / degree) % L];
    auto a = Ciphertext::from_host(par, ct_words, 1);
    auto b = Ciphertext::from_host(par, ct_words, 1);
    a.mul_plain(simd);
    b.mul_plain(simd.poly_ntt());
    if (a.to_host() != b.to_host()) {
      std::cout << "FAIL mul_plain\n";
      return 1;
    }
    std::cout << "OK\n";
  } catch (const Error& e) {
    std::cout << "FAIL " << e.code << " " << e.what() << "\n";
    return 1;
  }
  return 0;
}
