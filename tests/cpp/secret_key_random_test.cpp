// GPU test driver of SecretKey::random in include/fhe_b200.hpp (tests/test_gpu_secret_key.py):
//   secret_key_random_test <params.bin> <seed.bin> <n_keys> <out dir>
// reads the parameters from their message, makes n_keys keys in one random_vec call and writes
//   par.bin        parameters_to_bytes of the decoded parameters
//   sk<k>.bin      to_bytes of key k (downloaded through fhe_b200_secret_key_coeffs)
//   one.bin        to_bytes of SecretKey::random with the same seed (key 0 of the call)
//   ct.bin         the words of two encryptions of zero under key 0 with the same seed
//   rebuilt.bin    the words of the same encryptions under secret_key_from_bytes(sk0.bin)
#include <cstdio>
#include <fstream>
#include <iterator>
#include <string>

#include "fhe_b200_wire.hpp"

using namespace fhe_b200;

static std::string slurp(const std::string& path) {
  std::ifstream in(path, std::ios::binary);
  return std::string((std::istreambuf_iterator<char>(in)), std::istreambuf_iterator<char>());
}
static void spill(const std::string& path, const void* p, size_t n) {
  std::ofstream(path, std::ios::binary).write((const char*)p, (std::streamsize)n);
}

int main(int argc, char** argv) {
  if (argc < 5) return 2;
  try {
    const std::string dir = argv[4];
    auto par = bfv::parameters_from_bytes(slurp(argv[1]), 0);
    const std::string seed = slurp(argv[2]);
    const uint8_t* s = (const uint8_t*)seed.data();
    const std::string pb = bfv::parameters_to_bytes(*par);
    spill(dir + "/par.bin", pb.data(), pb.size());
    auto keys = bfv::SecretKey::random_vec(par, (uint32_t)std::atoi(argv[3]), s);
    for (size_t k = 0; k < keys.size(); k++) {
      if (!keys[k]->coeffs().empty()) return 5;
      const std::string m = bfv::to_bytes(*keys[k]);
      spill(dir + "/sk" + std::to_string(k) + ".bin", m.data(), m.size());
    }
    const std::string one = bfv::to_bytes(*bfv::SecretKey::random(par, s));
    spill(dir + "/one.bin", one.data(), one.size());
    const std::vector<uint64_t> w = keys[0]->try_encrypt_zero(2, 0, s).to_host();
    spill(dir + "/ct.bin", w.data(), w.size() * 8);
    auto rebuilt = bfv::secret_key_from_bytes(par, bfv::to_bytes(*keys[0]));
    const std::vector<uint64_t> r = rebuilt->try_encrypt_zero(2, 0, s).to_host();
    spill(dir + "/rebuilt.bin", r.data(), r.size() * 8);
  } catch (const Error& e) {
    std::printf("error %d %s\n", e.code, e.what());
    return 4;
  }
  std::printf("OK\n");
  return 0;
}
