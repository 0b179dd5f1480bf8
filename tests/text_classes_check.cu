// Host check of the two-byte clean test (dev_common.cuh): for every (pw, w) whose governing bytes (w and pw's last
// three bytes) hold no lead of a 3- or 4-byte sequence, utf8_unclean2 must flag exactly the bits utf8_unclean4 flags.
// Exhaustive over an alphabet of the bytes the rule turns on, then `argv[1]` random pairs of bytes < 0xE0 (pw's
// first byte: any).  Also: the end-of-text check utf8_unclean4(tail, spaces) flags nothing when tail's last three bytes
// are ASCII.  Prints the counts; exits 1 on the first mismatch.   nvcc -std=c++17 -gencode arch=compute_90a,code=sm_90a
#include <cstdio>
#include <cstdlib>

#include "../distributed_crawler_b200/csrc/dev_common.cuh"

using namespace tgi;

static bool same(uint32_t pw, uint32_t w) {
  if (((utf8_lead3(w) | utf8_lead3(pw & 0xFFFFFF00u))) != 0) {
    std::printf("utf8_lead3 flags a byte < 0xE0: pw %08x w %08x\n", pw, w);
    return false;
  }
  const uint32_t a = utf8_unclean4(pw, w), b = utf8_unclean2(pw, w);
  if (a != b) std::printf("mismatch: pw %08x w %08x: utf8_unclean4 %08x utf8_unclean2 %08x\n", pw, w, a, b);
  return a == b;
}

int main(int argc, char** argv) {
  for (uint32_t b = 0; b < 256; b++) {  // utf8_lead3 is exact in every byte position
    for (int k = 0; k < 4; k++) {
      const uint32_t w = (b << (8 * k)) | (0x41414141u & ~(0xFFu << (8 * k)));
      if ((utf8_lead3(w) != 0) != (b >= 0xE0) || (utf8_lead3(w) & ~(0x80u << (8 * k)))) {
        std::printf("utf8_lead3 wrong for byte %02x in position %d\n", b, k);
        return 1;
      }
    }
  }
  const uint8_t A[] = {0x00, 0x0A, 0x20, 0x41, 0x7F, 0x80, 0x9F, 0xA0, 0xBF, 0xC0, 0xC1, 0xC2, 0xD0, 0xDF};
  const int NA = sizeof A;
  const uint8_t P0[] = {0x20, 0xC3, 0xE2, 0xF0, 0xFF};  // pw's first byte governs nothing in w
  uint64_t n = 0;
  for (int i = 0; i < NA * NA * NA; i++) {
    const uint32_t pw_hi = (uint32_t)A[i % NA] << 8 | (uint32_t)A[i / NA % NA] << 16 | (uint32_t)A[i / NA / NA] << 24;
    for (int j = 0; j < NA * NA * NA * NA; j++) {
      const uint32_t w = A[j % NA] | (uint32_t)A[j / NA % NA] << 8 | (uint32_t)A[j / NA / NA % NA] << 16 |
                         (uint32_t)A[j / NA / NA / NA] << 24;
      if (!same(pw_hi | P0[j % 5], w)) return 1;
      n++;
    }
  }
  // the end-of-text check of the last strip's last word is skipped when its last three bytes are ASCII: nothing is open
  for (uint32_t t = 0; t < (1u << 21); t++) {
    const uint32_t tail = (t & 0x7F) << 8 | (t >> 7 & 0x7F) << 16 | (t >> 14 & 0x7F) << 24 | P0[t % 5];
    if (utf8_unclean4(tail, 0x20202020u) != 0) {
      std::printf("utf8_unclean4(%08x, spaces) flags a byte\n", tail);
      return 1;
    }
  }
  const uint64_t R = argc > 1 ? std::strtoull(argv[1], nullptr, 10) : 100000000ull;
  uint64_t s = 0x9E3779B97F4A7C15ull;
  for (uint64_t r = 0; r < R; r++) {
    s ^= s << 13, s ^= s >> 7, s ^= s << 17;
    uint64_t x = s;
    uint32_t v[8];
    for (int k = 0; k < 8; k++, x >>= 8) {
      const uint32_t u = x & 0xFF;
      // half of the bytes from the two-byte alphabet's interesting end (0x80..0xDF), the others anything < 0xE0
      v[k] = (k & 1) ? 0x80 + u % 0x60 : u % 0xE0;
    }
    const uint32_t pw = (uint32_t)(s >> 56) | v[1] << 8 | v[2] << 16 | v[3] << 24;
    const uint32_t w = (r & 1) ? (v[4] | v[5] << 8 | v[6] << 16 | v[7] << 24) : (v[5] | v[4] << 8 | v[7] << 16 | v[6] << 24);
    if (!same(pw, w)) return 1;
    n++;
  }
  std::printf("ok: %llu pairs\n", (unsigned long long)n);
  return 0;
}
