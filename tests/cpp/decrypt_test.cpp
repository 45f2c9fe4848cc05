// Decrypts through include/fhe_b200.hpp and include/fhe_b200_wire.hpp (driven by
// tests/test_gpu_decrypt.py::test_cpp_decrypt):
//   argv: degree t count dir; dir holds moduli.bin (u64), sk.bin (a SecretKey message, SecretKey::to_bytes) and
//   ct.bin (count fresh ciphertexts at level 0, [count][2][L][N] u64).
// Writes simd.bin (SIMD u64 decoding of every decryption), poly_i64.bin (Poly i64 decoding) and noise.bin
// (measure_noise, u32 per ciphertext).
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
template <typename T>
static void write_file(const std::string& path, const std::vector<T>& v) {
  std::ofstream(path, std::ios::binary).write(reinterpret_cast<const char*>(v.data()), v.size() * sizeof(T));
}

int main(int argc, char** argv) {
  if (argc != 5) return 2;
  const size_t degree = std::stoul(argv[1]);
  const uint64_t t = std::stoull(argv[2]);
  const uint32_t count = (uint32_t)std::stoul(argv[3]);
  const std::string dir = argv[4];
  try {
    auto par = BfvParametersBuilder().set_degree(degree).set_plaintext_modulus(t)
                   .set_moduli(read_file<uint64_t>(dir + "/moduli.bin")).build_arc();
    const auto msg = read_file<char>(dir + "/sk.bin");
    auto sk = secret_key_from_bytes(par, std::string(msg.begin(), msg.end()));
    if (to_bytes(*sk) != std::string(msg.begin(), msg.end())) {
      std::cout << "FAIL to_bytes\n";
      return 1;
    }
    auto ct = Ciphertext::from_host(par, read_file<uint64_t>(dir + "/ct.bin"), count);
    auto pts = sk->try_decrypt(ct);
    if (pts.len() != count || pts.has_encoding()) {
      std::cout << "FAIL shape\n";
      return 1;
    }
    try {
      pts.try_decode<uint64_t>();
      std::cout << "FAIL decode without an encoding\n";
      return 1;
    } catch (const Error& e) {
      if (e.code != FHE_B200_INVALID_ARGUMENT) throw;
    }
    const Encoding simd = Encoding::simd(), poly = Encoding::poly();
    write_file(dir + "/simd.bin", pts.try_decode<uint64_t>(&simd));
    write_file(dir + "/poly_i64.bin", pts.try_decode<int64_t>(&poly));
    write_file(dir + "/noise.bin", sk->measure_noise(ct));
    std::cout << "OK\n";
  } catch (const Error& e) {
    std::cout << "FAIL " << e.code << " " << e.what() << "\n";
    return 1;
  }
  return 0;
}
