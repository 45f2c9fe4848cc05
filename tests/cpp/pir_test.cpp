// The SealPIR pieces of include/fhe_b200.hpp / fhe_b200_wire.hpp, driven by tests/test_pir_cpu.py and
// tests/test_gpu_pir.py:
//   argv: mode degree t device moduli.bin in.bin out.bin; moduli.bin holds u64 moduli; in.bin and out.bin are records
//   (tag byte, u32 length, payload).  A refused call writes 'w' + the WireError variant or 'e' + the decimal status.
//   mode "codec": in = 'h' (u32 ciphertext_level, u32 evaluation_key_level) then 'g' GaloisKey messages.  Writes 'k'
//     encode_evaluation_key(messages, levels), 'g' every message decode_evaluation_key returns from it, then the
//     outcome of evaluation_key_from_bytes on a message without keys at those levels ('l' + its two levels).
//   mode "device": in = 'h' (u32 count, parts, level, repr, in_bits, out_bits, out_level, rows, in_len, t_in_bits,
//     t_out_bits), 'c' ciphertext words, 'r' transcoder rows (rows * in_len u64), 'm' an EvaluationKey message.
//     Writes 'f' the fold's poly_ntt words, 't' transcode_bidirectional of every row, 'b' transcode_to_bytes and 'y'
//     transcode_from_bytes(to_bytes) of row 0, 'k' to_bytes(evaluation_key_from_bytes(message)).
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

static void put(std::ofstream& out, char tag, const void* p, size_t len) {
  const uint32_t n = (uint32_t)len;
  out.write(&tag, 1);
  out.write((const char*)&n, 4);
  out.write((const char*)p, n);
}
static void put(std::ofstream& out, char tag, const std::string& s) { put(out, tag, s.data(), s.size()); }
template <class T>
static void put(std::ofstream& out, char tag, const std::vector<T>& v) { put(out, tag, v.data(), v.size() * sizeof(T)); }

template <class F>
static void guarded(std::ofstream& out, F&& f) {
  try {
    f();
  } catch (const WireError& e) {
    put(out, 'w', e.variant);
  } catch (const Error& e) {
    put(out, 'e', std::to_string(e.code));
  }
}

int main(int argc, char** argv) {
  if (argc != 8) return 2;
  const std::string mode = argv[1];
  const std::string raw = slurp(argv[5]);
  std::vector<uint64_t> moduli(raw.size() / 8);
  std::memcpy(moduli.data(), raw.data(), moduli.size() * 8);
  auto par = BfvParametersBuilder().set_degree(std::stoul(argv[2])).set_plaintext_modulus(std::stoull(argv[3]))
                 .set_moduli(moduli).set_device(std::stoi(argv[4])).build_arc();
  const std::string data = slurp(argv[6]);
  std::vector<std::pair<char, std::string>> rec;
  for (size_t pos = 0; pos + 5 <= data.size();) {
    uint32_t n;
    std::memcpy(&n, &data[pos + 1], 4);
    rec.emplace_back(data[pos], data.substr(pos + 5, n));
    pos += 5 + n;
  }
  std::ofstream out(argv[7], std::ios::binary);
  auto u32s = [](const std::string& s) {
    std::vector<uint32_t> v(s.size() / 4);
    std::memcpy(v.data(), s.data(), v.size() * 4);
    return v;
  };
  auto u64s = [](const std::string& s) {
    std::vector<uint64_t> v(s.size() / 8);
    std::memcpy(v.data(), s.data(), v.size() * 8);
    return v;
  };
  if (mode == "codec") {
    const std::vector<uint32_t> h = u32s(rec[0].second);
    std::vector<std::string> gks;
    for (size_t i = 1; i < rec.size(); i++) gks.push_back(rec[i].second);
    const std::string msg = wire::encode_evaluation_key(gks, h[0], h[1]);
    put(out, 'k', msg);
    for (const wire::Span& g : wire::decode_evaluation_key(msg.data(), msg.size()).gk) put(out, 'g', g.p, g.n);
    guarded(out, [&] {
      const EvaluationKey ek = evaluation_key_from_bytes(par, wire::encode_evaluation_key({}, h[0], h[1]));
      put(out, 'l', std::vector<uint32_t>{ek.ciphertext_level(), ek.evaluation_key_level()});
    });
    return 0;
  }
  const std::vector<uint32_t> h = u32s(rec[0].second);
  guarded(out, [&] {
    const Ciphertext ct = Ciphertext::from_host(par, u64s(rec[1].second), h[0], h[1], h[2], (Representation)h[3]);
    put(out, 'f', ct.fold(h[4], h[5], h[6]).poly_ntt());
  });
  const std::vector<uint64_t> rows = u64s(rec[2].second);
  std::vector<uint64_t> all;
  for (uint32_t r = 0; r < h[7]; r++) {
    const std::vector<uint64_t> row(rows.begin() + (size_t)r * h[8], rows.begin() + (size_t)(r + 1) * h[8]);
    const std::vector<uint64_t> t = transcode_bidirectional(par, row, h[9], h[10]);
    all.insert(all.end(), t.begin(), t.end());
  }
  put(out, 't', all);
  const std::vector<uint64_t> row0(rows.begin(), rows.begin() + h[8]);
  const std::vector<uint8_t> bytes = transcode_to_bytes(par, row0, h[9]);
  put(out, 'b', bytes);
  put(out, 'y', transcode_from_bytes(par, bytes, h[9]));
  guarded(out, [&] { put(out, 'k', to_bytes(evaluation_key_from_bytes(par, rec[3].second))); });
  return 0;
}
