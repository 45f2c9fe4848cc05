// Reads KeySwitchingKey messages with include/fhe_b200_wire.hpp's key_switching_key_from_bytes and writes every key it
// accepts back with to_bytes (driven by tests/test_widths_cpu.py and tests/test_gpu_widths.py):
//   argv: degree t device moduli.bin in.bin out.bin; moduli.bin holds u64 moduli, in.bin records (u32 length, message).
//   Output record per input: tag 'k' + u32 length + the re-encoded message; 'w' + u32 length + the WireError variant;
//   or 'e' + u32 length + the decimal status of any other error (NO_DEVICE for host-only parameters, device = -1).
#include <cstdio>
#include <cstring>
#include <fstream>
#include <iterator>
#include <string>
#include <vector>

#include "fhe_b200_wire.hpp"

using namespace fhe_b200;
using namespace fhe_b200::bfv;

static std::string slurp(const char* path) {
  std::ifstream in(path, std::ios::binary);
  return std::string((std::istreambuf_iterator<char>(in)), std::istreambuf_iterator<char>());
}

static void put(std::ofstream& out, char tag, const std::string& s) {
  const uint32_t n = (uint32_t)s.size();
  out.write(&tag, 1);
  out.write((const char*)&n, 4);
  out.write(s.data(), n);
}

int main(int argc, char** argv) {
  if (argc != 7) return 2;
  const std::string raw = slurp(argv[4]);
  std::vector<uint64_t> moduli(raw.size() / 8);
  std::memcpy(moduli.data(), raw.data(), moduli.size() * 8);
  auto par = BfvParametersBuilder().set_degree(std::stoul(argv[1])).set_plaintext_modulus(std::stoull(argv[2]))
                 .set_moduli(moduli).set_device(std::stoi(argv[3])).build_arc();
  const std::string data = slurp(argv[5]);
  std::ofstream out(argv[6], std::ios::binary);
  size_t pos = 0;
  while (pos + 4 <= data.size()) {
    uint32_t n;
    std::memcpy(&n, &data[pos], 4);
    const char* p = data.data() + pos + 4;
    pos += 4 + n;
    try {
      put(out, 'k', to_bytes(*key_switching_key_from_bytes(par, p, n)));
    } catch (const WireError& e) {
      put(out, 'w', e.variant);
    } catch (const Error& e) {
      put(out, 'e', std::to_string(e.code));
    }
  }
  return 0;
}
