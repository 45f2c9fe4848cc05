// CPU test driver of the Parameters codec of include/fhe_b200_wire.hpp (tests/test_params_wire_cpu.py):
//   params_wire_test e <degree> <variance> <plaintext, little-endian hex> <moduli, comma-separated> <out.bin>
//                                          wire::encode_parameters
//   params_wire_test d <message.bin>       wire::decode_parameters; prints "degree variance plaintext-hex moduli"
//   params_wire_test r <message.bin> <out.bin>
//                                          parameters_from_bytes on a host-only parameter set, then
//                                          parameters_to_bytes
// A WireError prints its variant and exits with 3; any other Error prints its code and exits with 4.
#include <cstdio>
#include <cstdlib>
#include <fstream>
#include <iterator>
#include <sstream>
#include <string>

#include "fhe_b200_wire.hpp"

using namespace fhe_b200;

static std::string slurp(const char* path) {
  std::ifstream in(path, std::ios::binary);
  return std::string((std::istreambuf_iterator<char>(in)), std::istreambuf_iterator<char>());
}
static void spill(const char* path, const std::string& s) {
  std::ofstream(path, std::ios::binary).write(s.data(), (std::streamsize)s.size());
}

int main(int argc, char** argv) {
  if (argc < 3) return 2;
  const std::string mode = argv[1];
  try {
    if (mode == "e" && argc >= 7) {
      std::vector<uint8_t> t;
      for (const char* h = argv[4]; h[0] && h[1]; h += 2) t.push_back((uint8_t)std::strtoul(std::string(h, 2).c_str(), nullptr, 16));
      std::vector<uint64_t> moduli;
      std::stringstream ss(argv[5]);
      for (std::string q; std::getline(ss, q, ',');)
        if (!q.empty()) moduli.push_back(std::strtoull(q.c_str(), nullptr, 10));
      spill(argv[6], wire::encode_parameters((uint32_t)std::atol(argv[2]), moduli, t, (uint32_t)std::atol(argv[3])));
      return 0;
    }
    if (mode == "d") {
      const std::string msg = slurp(argv[2]);
      const wire::ParametersMsg m = wire::decode_parameters(msg.data(), msg.size());
      std::printf("%u %u ", m.degree, m.variance);
      for (uint8_t b : m.plaintext_le) std::printf("%02x", b);
      std::printf(" ");
      for (size_t i = 0; i < m.moduli.size(); i++) std::printf(i ? ",%llu" : "%llu", (unsigned long long)m.moduli[i]);
      std::printf("\n");
      return 0;
    }
    if (mode == "r" && argc >= 4) {
      auto par = bfv::parameters_from_bytes(slurp(argv[2]), -1);
      spill(argv[3], bfv::parameters_to_bytes(*par));
      return 0;
    }
  } catch (const WireError& e) {
    std::printf("%s\n", e.variant.c_str());
    return 3;
  } catch (const Error& e) {
    std::printf("%d\n", e.code);
    return 4;
  }
  return 2;
}
