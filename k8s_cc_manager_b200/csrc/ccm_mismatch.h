// ccm_mismatch.h — host-side classification of the windows a tagged check found not holding their tags
// (include/ccm.h: ccm_mismatch_kind).  Plain C++17, no CUDA: a CPU test compiles it on its own.
//
// The tag of the 4-byte word at address a (i = a >> 2) is  lo32(i) * K1  ^  hi32(i) * K2  ^  seed  with both
// constants odd (scrub_kernels.cuh: tag_word).  Within one 16 GiB window (hi32(i) fixed) that is a bijection of
// lo32(i), so a word that holds THIS call's tag of some address can be inverted back to it:
//     lo32(i) = (w ^ seed ^ hi32(i) * K2) * K1^-1  (mod 2^32)
// for every hi32(i) the mapping spans.  classify() decides, in this order:
//   ZERO     every byte of the window inside the region reads 0;
//   ALIAS    the bytes are exactly this call's tags of a DIFFERENT 16-aligned window inside the mapping
//            (a second view of one physical range);
//   PARTIAL  some byte still holds its own tag (flipped or overwritten bytes in an otherwise tagged window);
//   FOREIGN  anything else: data this call did not write.
#pragma once
#include <algorithm>
#include <cstddef>
#include <cstdint>
#include <vector>

namespace ccm_mismatch {

constexpr uint32_t kK1 = 0x9E3779B1u;
constexpr uint32_t kK2 = 0x85EBCA77u;

// Inverse of an odd k mod 2^32 (Newton: each step doubles the number of correct low bits).
constexpr uint32_t inverse32(uint32_t k) {
  uint32_t x = k;                       // correct to 3 bits for any odd k
  for (int i = 0; i < 5; ++i) x *= 2u - k * x;
  return x;
}
constexpr uint32_t kK1Inv = inverse32(kK1);
static_assert(kK1 * kK1Inv == 1u, "K1 must be odd");

inline uint32_t tag_word(uint32_t seed, uint64_t a) {
  const uint64_t i = a >> 2;
  return ((uint32_t)i * kK1) ^ ((uint32_t)(i >> 32) * kK2) ^ seed;
}

inline uint8_t tag_byte(uint32_t seed, uint64_t x) { return (uint8_t)(tag_word(seed, x & ~3ull) >> (8 * (x & 3))); }

// Values of include/ccm.h: ccm_mismatch_kind.
constexpr int kZero = 1, kAlias = 2, kPartial = 3, kForeign = 4;

struct Range { uint64_t lo, hi; };      // [lo, hi): addresses the call mapped (or the region checked)

struct Verdict {
  int kind;
  uint64_t source;                      // ALIAS: address of the window whose tags these are; otherwise 0
};

inline bool mapped(uint64_t a, const Range* r, size_t n) {
  for (size_t k = 0; k < n; ++k)
    if (a >= r[k].lo && a < r[k].hi) return true;
  return false;
}

// The window at the 16-aligned address w, as read (`bytes`), of which the bytes `present` (bit i: byte w + i)
// lie inside the region that was checked; `ranges` is what the call mapped.
inline Verdict classify(uint32_t seed, uint64_t w, const uint8_t bytes[16], uint32_t present, const Range* ranges,
                        size_t nranges) {
  bool zero = true, own = false;
  for (int i = 0; i < 16; ++i)
    if (present >> i & 1) {
      zero &= bytes[i] == 0;
      own |= bytes[i] == tag_byte(seed, w + i);
    }
  if (zero) return {kZero, 0};
  int k = 0;                            // the first whole word inside the region
  while (k < 4 && ((present >> (4 * k)) & 0xFu) != 0xFu) ++k;
  if (k < 4) {
    const uint32_t word = (uint32_t)bytes[4 * k] | (uint32_t)bytes[4 * k + 1] << 8 | (uint32_t)bytes[4 * k + 2] << 16 |
                          (uint32_t)bytes[4 * k + 3] << 24;
    std::vector<uint64_t> his;          // every hi32(a >> 2) the mapping spans, ascending
    for (size_t r = 0; r < nranges; ++r)
      if (ranges[r].hi > ranges[r].lo)
        for (uint64_t hi = ranges[r].lo >> 34; hi <= (ranges[r].hi - 1) >> 34; ++hi) his.push_back(hi);
    std::sort(his.begin(), his.end());
    his.erase(std::unique(his.begin(), his.end()), his.end());
    for (const uint64_t hi : his) {
      const uint32_t lo = (word ^ seed ^ (uint32_t)hi * kK2) * kK1Inv;
      const uint64_t src = 4 * (hi << 32 | lo) - 4 * (uint64_t)k;
      if (src % 16 != 0 || src == w) continue;
      bool ok = true;
      for (int i = 0; i < 16 && ok; ++i)
        if (present >> i & 1) ok = mapped(src + i, ranges, nranges) && bytes[i] == tag_byte(seed, src + i);
      if (ok) return {kAlias, src};
    }
  }
  return {own ? kPartial : kForeign, 0};
}

}  // namespace ccm_mismatch
