// Encrypts through include/fhe_b200.hpp and include/fhe_b200_wire.hpp (driven by
// tests/test_gpu_encrypt.py::test_cpp_encrypt):
//   argv: degree t count dir; dir holds moduli.bin (u64), sk.bin (a SecretKey message), seeds.bin (three 32-byte seeds:
//   public key, secret-key encryption, public-key encryption) and values.bin (count * N u64 SIMD values).
// Writes pk.bin (the PublicKey message of PublicKey::new), ct_sk.bin and ct_pk.bin ([count][2][L][N] u64 words of the
// secret-key and public-key encryptions of the values, through a public key decoded from pk.bin).
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
    if (par->variance() != 10) {
      std::cout << "FAIL default variance\n";
      return 1;
    }
    const auto msg = read_file<char>(dir + "/sk.bin");
    auto sk = secret_key_from_bytes(par, std::string(msg.begin(), msg.end()));
    const auto seeds = read_file<uint8_t>(dir + "/seeds.bin");
    const auto values = read_file<uint64_t>(dir + "/values.bin");
    const auto pts = PlaintextVec::try_encode(values, Encoding::simd(), par);
    const std::string pk_msg = to_bytes(PublicKey::new_key(*sk, seeds.data()));
    write_file(dir + "/pk.bin", std::vector<char>(pk_msg.begin(), pk_msg.end()));
    const PublicKey pk = public_key_from_bytes(par, pk_msg);
    write_file(dir + "/ct_sk.bin", sk->try_encrypt(pts, seeds.data() + 32).to_host());
    write_file(dir + "/ct_pk.bin", pk.try_encrypt(pts, seeds.data() + 64).to_host());
    // default seeds: fresh entropy on every call, and the result decrypts
    const Ciphertext a = pk.try_encrypt(pts), b = pk.try_encrypt(pts);
    if (a.to_host() == b.to_host()) {
      std::cout << "FAIL two encryptions with fresh seeds are equal\n";
      return 1;
    }
    const Encoding simd = Encoding::simd();
    if (sk->try_decrypt(a).try_decode<uint64_t>(&simd) != values ||
        sk->try_decrypt(sk->try_encrypt(pts)).try_decode<uint64_t>(&simd) != values) {
      std::cout << "FAIL decryption\n";
      return 1;
    }
    try {
      BfvParametersBuilder().set_degree(degree).set_plaintext_modulus(t).set_variance(33)
          .set_moduli(read_file<uint64_t>(dir + "/moduli.bin")).build_arc();
      std::cout << "FAIL variance 33 accepted\n";
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
