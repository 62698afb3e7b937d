// CRC-32C (Castagnoli, reflected polynomial 0x82f63b78) of host bytes, slicing by 8 (include/p2pvg_b200.h, p2pvg_crc32c).
// TensorBoard frames every event record with masked CRC-32Cs of its length and payload; the writer thread computes them
// on serialized host bytes, so this is host code.
#include "common.cuh"

#include <cstring>

namespace {

struct Tables {
  uint32_t t[8][256];
  Tables() {
    for (uint32_t i = 0; i < 256; ++i) {
      uint32_t c = i;
      for (int k = 0; k < 8; ++k) c = (c & 1u) ? (c >> 1) ^ 0x82f63b78u : c >> 1;
      t[0][i] = c;
    }
    for (uint32_t i = 0; i < 256; ++i)
      for (int s = 1; s < 8; ++s) t[s][i] = (t[s - 1][i] >> 8) ^ t[0][t[s - 1][i] & 255u];
  }
};

const Tables kTab;

}  // namespace

extern "C" uint32_t p2pvg_crc32c(const void* data, size_t n, uint32_t crc) {
  const uint8_t* p = static_cast<const uint8_t*>(data);
  const auto& t = kTab.t;
  uint32_t c = ~crc;
  for (; n && (reinterpret_cast<uintptr_t>(p) & 7); --n) c = t[0][(c ^ *p++) & 255u] ^ (c >> 8);
  for (; n >= 8; n -= 8, p += 8) {
    uint32_t lo, hi;
    std::memcpy(&lo, p, 4);
    std::memcpy(&hi, p + 4, 4);
    lo ^= c;   // little-endian host
    c = t[7][lo & 255u] ^ t[6][(lo >> 8) & 255u] ^ t[5][(lo >> 16) & 255u] ^ t[4][lo >> 24] ^ t[3][hi & 255u] ^
        t[2][(hi >> 8) & 255u] ^ t[1][(hi >> 16) & 255u] ^ t[0][hi >> 24];
  }
  for (; n; --n) c = t[0][(c ^ *p++) & 255u] ^ (c >> 8);
  return ~c;
}
