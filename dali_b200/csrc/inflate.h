// dali_b200/csrc/inflate.h -- zlib inflate (RFC 1950 / 1951) written once for device and host, shared by the PNG decoder (png_core.h:
// one zlib stream over the payloads of an image's IDAT chunks) and the TIFF decoder (tiff_core.h: one zlib stream per strip or tile).
//
// The two formats differ only in what happens at the end of the output, and that is the `kStopWhenFull` parameter of inflate_zlib:
//   * libpng (kStopWhenFull = false) decodes on past the image's last byte until a surplus byte would be produced, and from there only
//     drains the stream: malformed data or a bad Adler-32 there is a warning.  Running out of data is always an error.
//   * libtiff (kStopWhenFull = true) hands zlib an output buffer of exactly the segment's size.  zlib stops at the first step that would
//     write a byte into the full buffer (a literal, or the copy of a match); up to there it decodes on, so a malformed block header or a
//     bad Adler-32 met before it is an error.  Running out of data once the buffer is full is not; surplus input is ignored.
#ifndef DALI_B200_CSRC_INFLATE_H_
#define DALI_B200_CSRC_INFLATE_H_
#include <stdint.h>
#include "host_device.h"

namespace dalib200 {

// Bit reader over a list of byte ranges read as one stream (`R` has `off` and `len`, relative to `raw`).  Bytes past the last range read
// as zero; `used` counts the bits consumed, so running past the data is detected exactly.
template <class R>
struct InflateBits {
  const uint8_t *raw;
  const R *ranges;
  int k, kend;                 // current range, end of the ranges
  uint32_t pos;                // next byte inside range k
  uint64_t acc;                // LSB first
  int nbits;
  int64_t used, avail;         // bits consumed / bits of data in all ranges
};
template <class R>
DB_HD void ibits_init(InflateBits<R> &b, const uint8_t *raw, const R *ranges, int k, int kend) {
  b.raw = raw; b.ranges = ranges; b.k = k; b.kend = kend; b.pos = 0; b.acc = 0; b.nbits = 0; b.used = 0; b.avail = 0;
  for (int i = k; i < kend; i++) b.avail += 8 * (int64_t)ranges[i].len;
}
template <class R>
DB_HD void ibits_fill(InflateBits<R> &b) {
  while (b.nbits <= 56) {
    while (b.k < b.kend && b.pos >= b.ranges[b.k].len) { b.k++; b.pos = 0; }
    uint32_t v = 0;
    if (b.k < b.kend) v = b.raw[b.ranges[b.k].off + b.pos++];
    b.acc |= (uint64_t)v << b.nbits;
    b.nbits += 8;
  }
}
template <class R>
DB_HD uint32_t ibits_get(InflateBits<R> &b, int n) {        // n <= 32
  if (b.nbits < n) ibits_fill(b);
  const uint32_t v = n ? (uint32_t)(b.acc & ((1ull << n) - 1)) : 0u;
  b.acc >>= n; b.nbits -= n; b.used += n;
  return v;
}
template <class R>
DB_HD bool ibits_dry(const InflateBits<R> &b) { return b.used > b.avail; }

// zlib header (RFC 1950): deflate, window <= 32 KiB, check bits, no preset dictionary
DB_HD bool zlib_header_ok(uint32_t cmf, uint32_t flg) {
  return (cmf & 15) == 8 && (cmf >> 4) <= 7 && ((cmf << 8) | flg) % 31 == 0 && !(flg & 0x20);
}

// Canonical Huffman code (RFC 1951 3.2.2) as zlib's puff.c decodes it, with a 9-bit first-level table in front.
constexpr int kInflLutBits = 9;
struct InflateHuff {
  uint16_t lut[1 << kInflLutBits];   // (length << 9) | symbol for codes of at most 9 bits, 0 = longer code or no code
  uint16_t count[16];                // codes of each length
  uint16_t symbol[288];              // symbols in canonical order
};

// builds the code from `n` code lengths; returns false for an over-subscribed set, or an incomplete one that is not a single code
// of length 1 or that may not be incomplete at all (zlib inflate_table: a single length-1 code is accepted for the literal / length
// and distance codes, never for the code-length code; a code without any symbol is left empty)
DB_HD bool inflate_build(InflateHuff &h, const uint8_t *len, int n, bool allow_incomplete) {
  for (int l = 0; l < 16; l++) h.count[l] = 0;
  for (int s = 0; s < n; s++) h.count[len[s]]++;
  for (int i = 0; i < (1 << kInflLutBits); i++) h.lut[i] = 0;
  if (h.count[0] == n) return true;                       // no codes: any use of it is an undefined symbol
  int left = 1, maxlen = 0;
  for (int l = 1; l < 16; l++) {
    left <<= 1; left -= h.count[l];
    if (left < 0) return false;
    if (h.count[l]) maxlen = l;
  }
  if (left > 0 && !(allow_incomplete && maxlen == 1)) return false;
  uint16_t offs[16];
  offs[1] = 0;
  for (int l = 1; l < 15; l++) offs[l + 1] = offs[l] + h.count[l];
  // canonical codes: first code of length l = (first code of length l - 1 + count[l - 1]) << 1
  uint16_t next[16];
  int code = 0;
  for (int l = 1; l < 16; l++) { code = (code + (l > 1 ? h.count[l - 1] : 0)) << 1; next[l] = (uint16_t)code; }
  for (int s = 0; s < n; s++) {
    const int l = len[s];
    if (!l) continue;
    h.symbol[offs[l]++] = (uint16_t)s;
    const uint32_t c = next[l]++;
    if (l <= kInflLutBits) {
      uint32_t r = 0;                                       // the stream sends the code MSB first into an LSB-first bit order
      for (int i = 0; i < l; i++) r |= ((c >> i) & 1u) << (l - 1 - i);
      for (uint32_t e = r; e < (1u << kInflLutBits); e += 1u << l) h.lut[e] = (uint16_t)((l << 9) | s);
    }
  }
  return true;
}

// next symbol, -1 = no such code
template <class R>
DB_HD int inflate_decode(InflateBits<R> &b, const InflateHuff &h) {
  if (b.nbits < 16) ibits_fill(b);
  const uint16_t e = h.lut[b.acc & ((1u << kInflLutBits) - 1)];
  if (e) { const int l = e >> 9; b.acc >>= l; b.nbits -= l; b.used += l; return e & 511; }
  int code = 0, first = 0, index = 0;                    // puff.c decode(): one bit at a time
  for (int l = 1; l < 16; l++) {
    code |= (int)((b.acc >> (l - 1)) & 1u);
    const int cnt = h.count[l];
    if (code - cnt < first) { b.acc >>= l; b.nbits -= l; b.used += l; return h.symbol[index + (code - first)]; }
    index += cnt; first += cnt; first <<= 1; code <<= 1;
  }
  return -1;
}

struct InflateWork { InflateHuff lit, dist, cl; uint8_t lens[288 + 32]; };     // the decoder's working memory (per stream)

// Inflates the deflate blocks and the Adler-32 trailer behind the zlib header (already consumed from `b`) into `dst` (`total` bytes).
// Returns 0, or 1 for a malformed or short stream.  Reads stay inside the ranges; writes stay inside [dst, dst + total).  The end of
// the output follows libpng (kStopWhenFull = false) or libtiff (true), as the head of this file describes.
template <bool kStopWhenFull, class R>
DB_HD int inflate_zlib(InflateBits<R> &b, uint8_t *dst, int64_t total, InflateWork &w) {
  int64_t out = 0;                                        // bytes produced, surplus included
  bool drain = false;
  uint32_t s1 = 1, s2 = 0, nmod = 0;                      // Adler-32
  auto put = [&](uint8_t v) {
    if (out < total) {
      dst[out] = v;
      s1 += v; s2 += s1;
      if (++nmod == 5552) { s1 %= 65521u; s2 %= 65521u; nmod = 0; }
    } else {
      drain = true;
    }
    out++;
  };
  auto full = [&] { return kStopWhenFull && out >= total; };        // libtiff: the next write ends the decode
  auto bad = [&] { return drain ? 0 : 1; };               // malformed data: an error unless libpng is only draining
  auto dry = [&] { return full() ? 0 : 1; };              // the data ran out: an error unless libtiff's buffer is full
  bool last = false;
  while (!last) {
    last = ibits_get(b, 1) != 0;
    const uint32_t type = ibits_get(b, 2);
    if (ibits_dry(b)) return dry();
    if (type == 0) {                                      // stored
      const int drop = b.nbits & 7;                       // to the byte boundary
      ibits_get(b, drop);
      const uint32_t len = ibits_get(b, 16), nlen = ibits_get(b, 16);
      if (ibits_dry(b)) return dry();
      if ((len ^ 0xFFFFu) != nlen) return bad();
      for (uint32_t i = 0; i < len; i++) {
        if (full()) return 0;
        const uint8_t v = (uint8_t)ibits_get(b, 8);
        if (ibits_dry(b)) return 1;
        put(v);
      }
    } else if (type == 1 || type == 2) {
      if (type == 1) {                                    // fixed codes (RFC 1951 3.2.6)
        for (int s = 0; s < 288; s++) w.lens[s] = s < 144 ? 8 : s < 256 ? 9 : s < 280 ? 7 : 8;
        inflate_build(w.lit, w.lens, 288, true);
        for (int s = 0; s < 32; s++) w.lens[s] = 5;      // 30 and 31 complete the code; decoding one is an error
        inflate_build(w.dist, w.lens, 32, true);
      } else {                                            // dynamic codes (3.2.7)
        const int nlen = (int)ibits_get(b, 5) + 257, ndist = (int)ibits_get(b, 5) + 1, ncode = (int)ibits_get(b, 4) + 4;
        if (ibits_dry(b)) return dry();
        if (nlen > 286 || ndist > 30) return bad();
        const uint8_t order[19] = { 16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15 };
        uint8_t cl[19];
        for (int i = 0; i < 19; i++) cl[order[i]] = i < ncode ? (uint8_t)ibits_get(b, 3) : 0;
        if (ibits_dry(b)) return dry();
        if (!inflate_build(w.cl, cl, 19, false)) return bad();
        int i = 0;
        while (i < nlen + ndist) {
          const int sym = inflate_decode(b, w.cl);
          if (ibits_dry(b)) return dry();
          if (sym < 0) return bad();
          if (sym < 16) { w.lens[i++] = (uint8_t)sym; continue; }
          int rep, v = 0;
          if (sym == 16) { if (i == 0) return bad(); v = w.lens[i - 1]; rep = 3 + (int)ibits_get(b, 2); }
          else if (sym == 17) rep = 3 + (int)ibits_get(b, 3);
          else rep = 11 + (int)ibits_get(b, 7);
          if (ibits_dry(b)) return dry();
          if (i + rep > nlen + ndist) return bad();
          while (rep--) w.lens[i++] = (uint8_t)v;
        }
        if (w.lens[256] == 0) return bad();               // no end-of-block code
        if (!inflate_build(w.lit, w.lens, nlen, true)) return bad();
        if (!inflate_build(w.dist, w.lens + nlen, ndist, true)) return bad();
      }
      while (true) {
        const int sym = inflate_decode(b, w.lit);
        if (ibits_dry(b)) return dry();
        if (sym < 0) return bad();
        if (sym < 256) { if (full()) return 0; put((uint8_t)sym); continue; }
        if (sym == 256) break;
        const int li = sym - 257;
        if (li >= 29) return bad();                       // 286, 287
        int len;
        if (li < 8) len = 3 + li;
        else if (li == 28) len = 258;
        else { const int e = (li >> 2) - 1; len = ((4 + (li & 3)) << e) + 3 + (int)ibits_get(b, e); }
        const int ds = inflate_decode(b, w.dist);
        if (ibits_dry(b)) return dry();
        if (ds < 0 || ds >= 30) return bad();
        int dist;
        if (ds < 4) dist = ds + 1;
        else { const int e = (ds >> 1) - 1; dist = ((2 + (ds & 1)) << e) + 1 + (int)ibits_get(b, e); }
        if (ibits_dry(b)) return dry();
        if (full()) return 0;                             // zlib checks the distance only when it copies
        if (dist > out) return bad();                     // a distance behind the output start
        for (int k = 0; k < len; k++) {
          if (full()) return 0;
          put(out < total ? dst[out - dist] : 0);         // past the image only the count matters
        }
      }
    } else {
      return bad();                                       // block type 3
    }
  }
  if (out < total) return 1;                              // the stream ends before the output does
  ibits_get(b, b.nbits & 7);                              // the Adler-32 trailer
  uint32_t adler = 0;
  for (int i = 0; i < 4; i++) adler = (adler << 8) | ibits_get(b, 8);
  if (ibits_dry(b)) return dry();
  return adler != (((s2 % 65521u) << 16) | (s1 % 65521u)) ? bad() : 0;
}

}  // namespace dalib200
#endif  // DALI_B200_CSRC_INFLATE_H_
