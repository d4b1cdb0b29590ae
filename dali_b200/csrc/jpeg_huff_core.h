// dali_b200/csrc/jpeg_huff_core.h -- the first-level Huffman tables of the baseline JPEG entropy passes (jpeg.cu: huff_sync_intra,
// huff_sync_walk, huff_write): their entry format, the host builder, and the rule that picks the step a decoder takes at an entry.
// Plain functions of values, so that tests/test_jpeg_huff_core_cpu.py runs them on the host (tools/emul/jpeg_huff_emul.cc).
//
// An entry may decode two AC symbols of one block in one lookup.  Every pass keeps the state sequence (pos, c, z, blocks) of a
// one-symbol-per-lookup decoder at every step it takes: a pair step is taken only where it equals two single steps, so the
// synchronisation records, the block counts and the behaviour on damaged streams do not depend on whether pairs were taken.
#ifndef DALI_B200_CSRC_JPEG_HUFF_CORE_H_
#define DALI_B200_CSRC_JPEG_HUFF_CORE_H_
#include <stdint.h>
#include <string.h>
#include "host_device.h"

namespace dalib200 {

constexpr int kDcLutBits = 9, kAcLutBits = 11;   // first-level Huffman lookup widths (std DC codes are <= 9 bits)
constexpr int kDcLutSize = 1 << kDcLutBits, kAcLutSize = 1 << kAcLutBits;
constexpr int kLutWords = 2 * kDcLutSize + 2 * kAcLutSize;          // DC0 DC1 AC0 AC1 back to back: 20 KB
DB_HD int LutOffset(int t) { return t < 2 ? t * kDcLutSize : 2 * kDcLutSize + (t - 2) * kAcLutSize; }

// The canonical tables for codes longer than the first level (T.81 F.2.2.3), which the passes search in slow_lookup (jpeg.cu).
constexpr int kLongLut = 512;
struct HuffSlow {
  int32_t maxcode[18];        // T.81 F.2.2.3: maxcode[l] left-aligned to 16 bits (+1)
  int32_t valoff[18];         // valptr[l] - mincode[l]
  uint8_t vals[256];
  // canonical codes grow with their length, so the codes longer than the first-level LUT occupy the top [long_base, 65536) of the
  // left-aligned 16-bit code space -- 192 values for the standard tables.  When that range fits, ONE lookup indexed by
  // (window - long_base) replaces the length search (which ran on a single lane while the warp waited).  Entry = code length | symbol << 8, 0 = not a code.  long_n == 0: use the search.
  int32_t long_base, long_n;
  uint16_t long_lut[kLongLut];
};

// A step: [4:0] bits consumed (codes + magnitudes, <= 31), [8:5] magnitude size s of its LAST symbol, [15:9] zig-zag advance (run + 1;
// 16 for ZRL; 64 for EOB; 1 for DC; the sum of both for a pair).
//
// An entry: [31:16] the single step (the first symbol alone), [15:0] the pair step (the first symbol and the next one), or the single
// step again where the entry has no pair.  0 = a code longer than the first-level width (slow_lookup).  The funnel shifts of the bit
// window take the selected word itself as the shift amount (bits [4:0]), so a pair costs the decode loop one select.
//
// A pair is stored when the first symbol is an AC symbol but not an EOB (a ZRL pairs) and the second code ends inside the index bits
// behind the first symbol's code and magnitude; the second may be any symbol, and its magnitude may reach past the index (a pair
// consumes <= 11 + 15 bits).  DC entries, long codes and invalid codes (17 bits, symbol 0) are single steps.
DB_HD uint32_t huff_single(uint32_t len, uint32_t sym, bool is_dc) {
  const uint32_t s = sym & 15u, r = sym >> 4;
  const uint32_t adv = is_dc ? 1u : (s == 0 ? (r == 15u ? 16u : 64u) : r + 1u);
  return (len + s) | (s << 5) | (adv << 9);
}
DB_HD uint32_t huff_entry(uint32_t len, uint32_t sym, bool is_dc) { const uint32_t h = huff_single(len, sym, is_dc); return h | (h << 16); }

// The step to take at entry `e` in state (z, pos): the pair only when the single-step decoder would decode the second symbol in the
// same block and table, that is when the block is still open after the first symbol (z + adv1 < 64: a block that fills coefficient
// 63 without an EOB is followed by a DC code) and the second symbol starts before `limit` (a symbol at or behind it belongs to the
// next decoder).  A pair's first symbol takes at most kAcLutBits - 1 bits, so the second test holds wherever limit - pos >=
// kAcLutBits; closer to the limit (once per span) no pair is taken.  Both tests then fold into one threshold on the entry, known
// before the lookup (pair_threshold): adv1 sits in the entry's top bits, so e < (64 - z) << 25 iff adv1 < 64 - z.
DB_HD uint32_t pair_threshold(int z, uint32_t pos, uint32_t limit) {
  return limit - pos >= (uint32_t)kAcLutBits ? (64u - (uint32_t)z) << 25 : 0u;
}
DB_HD uint32_t huff_step(uint32_t e, uint32_t threshold) { return e < threshold ? e : e >> 16; }
DB_HD uint32_t step_bits(uint32_t st) { return st & 31u; }
DB_HD uint32_t step_size(uint32_t st) { return (st >> 5) & 15u; }
DB_HD uint32_t step_adv(uint32_t st) { return (st >> 9) & 127u; }

// EXTEND (T.81 F.2.2.1) of the s magnitude bits that end `end` bits into the window `hi`: s == 0 gives 0.
DB_HD int huff_extend(uint32_t hi, uint32_t end, uint32_t s) {
  const uint32_t bits = (uint32_t)(((uint64_t)(hi << (end - s))) >> (32u - s));      // 64-bit shift: s == 0 -> 0
  // (measured: a funnel-shift + sign-mask formulation of EXTEND is 3 instructions shorter but made huff_write slower)
  return (int)bits - ((s == 0 || ((bits >> (s - 1u)) & 1u)) ? 0 : (int)((1u << s) - 1u));
}

// The first-level table (1 << kDcLutBits or 1 << kAcLutBits entries) and the long-code tables of one DHT table; bits[1..16] = the
// code counts per length, vals = the symbols.
inline void BuildDeviceTable(const uint8_t *bits, const uint8_t *vals, uint32_t *lut, HuffSlow &t, bool is_dc) {
  const int kLutBits = is_dc ? kDcLutBits : kAcLutBits, kLutSize = 1 << kLutBits;
  memset(&t, 0, sizeof(t));
  memset(lut, 0, sizeof(uint32_t) * kLutSize);
  int code = 0, k = 0;
  for (int l = 1; l <= 16; l++) {
    const int mincode = code;
    t.valoff[l] = k - mincode;
    for (int i = 0; i < bits[l]; i++, k++, code++) {
      if (l <= kLutBits) {
        const int lo = code << (kLutBits - l), cnt = 1 << (kLutBits - l);
        for (int e = 0; e < cnt && lo + e < kLutSize; e++) lut[lo + e] = huff_entry(l, vals[k & 255], is_dc);
      }
    }
    // a 16-bit window belongs to length l iff it is < maxcode[l] (exclusive bound, left-aligned) and matched
    // no shorter length; for an empty length the bound equals the previous one, so nothing matches
    t.maxcode[l] = code << (16 - l);
    code <<= 1;
  }
  t.maxcode[17] = 0x7fffffff;
  memcpy(t.vals, vals, 256);
  // pairs: the second code is read from the index bits behind the first symbol (the bits past the index read as 0, so the entry
  // there decodes the second code only when its length fits in what is left)
  if (!is_dc) {
    for (int i = 0; i < kLutSize; i++) {
      const uint32_t one = lut[i] >> 16, tb1 = step_bits(one), adv1 = step_adv(one);
      if (one == 0 || adv1 == 64 || tb1 >= (uint32_t)kLutBits) continue;
      const uint32_t two = lut[((uint32_t)i << tb1) & (uint32_t)(kLutSize - 1)] >> 16;
      const uint32_t len2 = step_bits(two) - step_size(two);
      if (two == 0 || tb1 + len2 > (uint32_t)kLutBits) continue;
      lut[i] = (one << 16) | (tb1 + step_bits(two)) | (step_size(two) << 5) | ((adv1 + step_adv(two)) << 9);
    }
  }
  // direct table for the codes behind the first level (see HuffSlow)
  t.long_base = t.maxcode[kLutBits];
  const int range = 65536 - t.long_base;
  t.long_n = 0;
  if (range > 0 && range <= kLongLut) {
    t.long_n = range;
    int c2 = 0, k2 = 0;
    for (int l = 1; l <= 16; l++) {
      for (int i = 0; i < bits[l]; i++, k2++, c2++) {
        if (l > kLutBits) {
          const int lo = (c2 << (16 - l)) - t.long_base, cnt = 1 << (16 - l);
          for (int e = 0; e < cnt; e++)
            if (lo + e >= 0 && lo + e < range) t.long_lut[lo + e] = (uint16_t)(l | (vals[k2 & 255] << 8));
        }
      }
      c2 <<= 1;
    }
  }
}

}  // namespace dalib200

#endif  // DALI_B200_CSRC_JPEG_HUFF_CORE_H_
