// CPU test driver of the SecretKey codec of include/fhe_b200_wire.hpp (tests/test_decrypt_cpu.py):
//   secret_key_wire_test e <coeffs.i64> <out.bin>            SecretKey::to_bytes of the coefficients
//   secret_key_wire_test d <message.bin> <degree> <out.i64>  SecretKey::from_bytes; on a refusal prints the variant
//                                                            and exits with 3
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <iterator>
#include <string>

#include "fhe_b200_wire.hpp"

using namespace fhe_b200;

static std::string slurp(const char* path) {
  std::ifstream in(path, std::ios::binary);
  return std::string((std::istreambuf_iterator<char>(in)), std::istreambuf_iterator<char>());
}

int main(int argc, char** argv) {
  if (argc < 4) return 2;
  const std::string mode = argv[1];
  if (mode == "e") {
    const std::string raw = slurp(argv[2]);
    std::vector<int64_t> c(raw.size() / 8);
    if (!c.empty()) std::memcpy(c.data(), raw.data(), c.size() * 8);
    const std::string msg = wire::encode_secret_key(c.data(), c.size());
    std::ofstream(argv[3], std::ios::binary).write(msg.data(), (std::streamsize)msg.size());
    return 0;
  }
  if (mode == "d" && argc >= 5) {
    const std::string msg = slurp(argv[2]);
    try {
      const std::vector<int64_t> c = wire::decode_secret_key(msg.data(), msg.size(), (size_t)std::atoll(argv[3]));
      std::ofstream(argv[4], std::ios::binary).write((const char*)c.data(), (std::streamsize)(c.size() * 8));
    } catch (const WireError& e) {
      std::printf("%s\n", e.variant.c_str());
      return 3;
    }
    return 0;
  }
  return 2;
}
