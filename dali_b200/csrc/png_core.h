// dali_b200/csrc/png_core.h -- PNG decoding written once for device and host: inflate + unfilter of one image (png_inflate_unfilter)
// and the conversion of one output pixel (png_pixel).
//
// A PNG image is one zlib stream (RFC 1950 / 1951) spread over the payloads of consecutive IDAT chunks, inflating to the filtered
// scanlines of the image (of each Adam7 pass in turn), every row led by its filter byte.  Deflate is a serial chain -- a symbol's bit
// position depends on every symbol in front of it, and a back-reference on the bytes already produced -- so png_inflate runs one
// working thread per image, like the progressive-JPEG scans (jpeg_prog_core.h).  The same function compiled by a host compiler is what
// tools/emul/png_emul.cc runs to pin it against zlib + a numpy unfilter without a GPU (tests/test_png_cpu.py).
//
// Parity target: cv2.imdecode (OpenCV 4.13 / libpng).  How libpng treats the tail of the stream:
//   * the data ending before the image's last row is an error ("Not enough image data");
//   * the data running out before the end of the zlib stream is an error, even behind the image's last row;
//   * a malformed block or a bad Adler-32 trailer behind the last row is an error, unless the stream holds more data than the image
//     needs: libpng then only drains it and warns (png_inflate).
#ifndef DALI_B200_CSRC_PNG_CORE_H_
#define DALI_B200_CSRC_PNG_CORE_H_
#include <stdint.h>

#if defined(__CUDACC__)
#define PNG_HD __host__ __device__ __forceinline__
#else
#define PNG_HD inline
#endif

namespace dalib200 {

enum PngColorType : int32_t { kPngGray = 0, kPngRGB = 2, kPngPalette = 3, kPngGrayAlpha = 4, kPngRGBA = 6 };

struct PngChunk {              // payload of one IDAT chunk: type at off - 4, CRC-32 at off + len (big endian)
  uint32_t off, len;           // relative to the image's staged bytes
  int32_t image;               // index into the PngImage array
};

struct PngImage {
  int64_t raw_off;             // byte offset of the image's staged bytes (the first IDAT's type field .. the last IDAT's CRC)
  int64_t scan_off;            // byte offset of the image's filtered scanlines in the scratch buffer
  int64_t scan_bytes;          // size of the filtered scanlines of all passes (filter bytes included)
  int64_t pass_off[7];         // start of each Adam7 pass inside the scanlines (pass 0 only when not interlaced)
  int32_t pass_row[7];         // bytes per row of each pass, filter byte included (0: the pass is empty)
  int32_t chunk_begin, chunk_end;
  int32_t sample;              // batch index (status word)
  int32_t width, height, depth, ctype, interlace;
  int32_t spp;                 // samples per pixel (palette: 1)
  // output, filled at launch: the window [win_x0, win_x0 + win_w) x [win_y0, win_y0 + win_h) of the image goes to `out` as a tight
  // win_h x win_w x C buffer, C = 1 for GRAY (cv2 IMREAD_GRAYSCALE), 3 for RGB / BGR (IMREAD_COLOR)
  uint8_t *out;
  int32_t win_x0, win_y0, win_w, win_h, out_type;
  int64_t first_px;            // prefix of window pixels over the PNG images (png_color's sample search)
  uint8_t pal[256][3];         // PLTE, zero behind the last entry (libpng: an index past the palette reads black)
};

// Adam7: pass p starts at (x0, y0) and steps (dx, dy); a non-interlaced image is one pass (0, 0, 1, 1)
PNG_HD void png_pass_geom(int interlace, int p, int &x0, int &y0, int &dx, int &dy) {
  if (!interlace) { x0 = y0 = 0; dx = dy = 1; return; }
  switch (p) {
    case 0: x0 = 0; y0 = 0; dx = 8; dy = 8; break;
    case 1: x0 = 4; y0 = 0; dx = 8; dy = 8; break;
    case 2: x0 = 0; y0 = 4; dx = 4; dy = 8; break;
    case 3: x0 = 2; y0 = 0; dx = 4; dy = 4; break;
    case 4: x0 = 0; y0 = 2; dx = 2; dy = 4; break;
    case 5: x0 = 1; y0 = 0; dx = 2; dy = 2; break;
    default: x0 = 0; y0 = 1; dx = 1; dy = 2; break;
  }
}

// Adam7 pass of pixel (x, y): the 8 x 8 pattern of the PNG specification (8.2), decided on (y & 7, x & 7)
PNG_HD int png_adam7_pass(int x, int y) {
  const int xm = x & 7, ym = y & 7;
  if (ym & 1) return 6;
  if (xm & 1) return 5;
  if (ym & 2) return 4;                // rows 2, 6
  if (xm & 2) return 3;                // rows 0, 4, columns 2, 6
  if (ym & 4) return 2;                // row 4, columns 0, 4
  if (xm & 4) return 1;                // row 0, column 4
  return 0;
}

// CRC-32 (ISO 3309, as PNG uses it) over an IDAT chunk's type and data, against the value stored behind them.  `table`: the 256
// entries of the reflected polynomial 0xEDB88320, indexed by the low byte.
PNG_HD bool png_chunk_crc_ok(const uint8_t *type, uint32_t len, const uint32_t *table) {
  uint32_t c = 0xFFFFFFFFu;
  for (uint32_t i = 0; i < len + 4; i++) c = table[(c ^ type[i]) & 255] ^ (c >> 8);
  const uint8_t *e = type + 4 + len;
  return (c ^ 0xFFFFFFFFu) == (((uint32_t)e[0] << 24) | ((uint32_t)e[1] << 16) | ((uint32_t)e[2] << 8) | e[3]);
}
PNG_HD uint32_t png_crc_table_entry(uint32_t i) {
  uint32_t c = i;
  for (int k = 0; k < 8; k++) c = c & 1 ? 0xEDB88320u ^ (c >> 1) : c >> 1;
  return c;
}

// ---------------------------------------------------------------------------------------------------------------------------------
// Inflate.  Bit reader over the IDAT payloads as one stream, hopping the 12-byte gaps (CRC, length, type) between chunks.  Bytes past
// the last payload read as zero; `used` counts the bits consumed, so running past the data is detected exactly.
struct PngBits {
  const uint8_t *raw;          // the image's staged bytes
  const PngChunk *chunks;
  int k, kend;                 // current chunk, end of the image's chunks
  uint32_t pos;                // next byte inside chunk k
  uint64_t acc;                // LSB first
  int nbits;
  int64_t used, avail;         // bits consumed / bits of data in all payloads
};
PNG_HD void pbits_fill(PngBits &b) {
  while (b.nbits <= 56) {
    while (b.k < b.kend && b.pos >= b.chunks[b.k].len) { b.k++; b.pos = 0; }
    uint32_t v = 0;
    if (b.k < b.kend) v = b.raw[b.chunks[b.k].off + b.pos++];
    b.acc |= (uint64_t)v << b.nbits;
    b.nbits += 8;
  }
}
PNG_HD uint32_t pbits_get(PngBits &b, int n) {        // n <= 32
  if (b.nbits < n) pbits_fill(b);
  const uint32_t v = n ? (uint32_t)(b.acc & ((1ull << n) - 1)) : 0u;
  b.acc >>= n; b.nbits -= n; b.used += n;
  return v;
}
PNG_HD bool pbits_dry(const PngBits &b) { return b.used > b.avail; }

// Canonical Huffman code (RFC 1951 3.2.2) as zlib's puff.c decodes it, with a 9-bit first-level table in front.
constexpr int kPngLutBits = 9;
struct PngHuff {
  uint16_t lut[1 << kPngLutBits];    // (length << 9) | symbol for codes of at most 9 bits, 0 = longer code or no code
  uint16_t count[16];                // codes of each length
  uint16_t symbol[288];              // symbols in canonical order
};

// builds the code from `n` code lengths; returns false for an over-subscribed set, or an incomplete one that is not a single code
// of length 1 or that may not be incomplete at all (zlib inflate_table: a single length-1 code is accepted for the literal / length
// and distance codes, never for the code-length code; a code without any symbol is left empty)
PNG_HD bool png_build(PngHuff &h, const uint8_t *len, int n, bool allow_incomplete) {
  for (int l = 0; l < 16; l++) h.count[l] = 0;
  for (int s = 0; s < n; s++) h.count[len[s]]++;
  for (int i = 0; i < (1 << kPngLutBits); i++) h.lut[i] = 0;
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
    if (l <= kPngLutBits) {
      uint32_t r = 0;                                       // the stream sends the code MSB first into an LSB-first bit order
      for (int i = 0; i < l; i++) r |= ((c >> i) & 1u) << (l - 1 - i);
      for (uint32_t e = r; e < (1u << kPngLutBits); e += 1u << l) h.lut[e] = (uint16_t)((l << 9) | s);
    }
  }
  return true;
}

// next symbol, -1 = no such code
PNG_HD int png_decode(PngBits &b, const PngHuff &h) {
  if (b.nbits < 16) pbits_fill(b);
  const uint16_t e = h.lut[b.acc & ((1u << kPngLutBits) - 1)];
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

struct PngWork { PngHuff lit, dist, cl; uint8_t lens[288 + 32]; };     // the kernel's working memory (per image)

// Inflates the image's zlib stream into `scan` (im.scan_bytes bytes).  Returns 0, or 1 for a malformed stream.  Reads stay inside
// the chunks' payloads; writes stay inside [scan, scan + scan_bytes).
//
// The stream's tail follows libpng + zlib (pinned against cv2 by tests/test_png_cpu.py):
//   * the data running out before the end of the zlib stream is an error, before or after the image is complete ("Not enough image
//     data");
//   * the zlib call that produces the image's last byte decodes on until it would have to produce another one: a malformed block or a
//     bad Adler-32 trailer met before that is an error;
//   * once a byte beyond the image (a surplus) would be produced, libpng only drains the rest of the stream: malformed data or a bad
//     trailer there is a warning, so the rest is decoded without output ("draining") and only its end is required.
PNG_HD int png_inflate(const PngImage &im, const PngChunk *chunks, const uint8_t *raw, uint8_t *scan, PngWork &w) {
  PngBits b;
  b.raw = raw + im.raw_off; b.chunks = chunks; b.k = im.chunk_begin; b.kend = im.chunk_end; b.pos = 0; b.acc = 0; b.nbits = 0; b.used = 0;
  b.avail = 0;
  for (int k = im.chunk_begin; k < im.chunk_end; k++) b.avail += 8 * (int64_t)chunks[k].len;
  const int64_t total = im.scan_bytes;
  int64_t out = 0;                                        // bytes produced, surplus included
  bool drain = false;
  uint32_t s1 = 1, s2 = 0, nmod = 0;                      // Adler-32
  auto put = [&](uint8_t v) {
    if (out < total) {
      scan[out] = v;
      s1 += v; s2 += s1;
      if (++nmod == 5552) { s1 %= 65521u; s2 %= 65521u; nmod = 0; }
    } else {
      drain = true;
    }
    out++;
  };
  auto bad = [&] { return drain ? 0 : 1; };               // malformed data: an error unless libpng is only draining
  pbits_get(b, 16);                                       // CMF / FLG, checked by the planner
  bool last = false;
  while (!last) {
    last = pbits_get(b, 1) != 0;
    const uint32_t type = pbits_get(b, 2);
    if (pbits_dry(b)) return 1;
    if (type == 0) {                                      // stored
      const int drop = b.nbits & 7;                       // to the byte boundary
      pbits_get(b, drop);
      const uint32_t len = pbits_get(b, 16), nlen = pbits_get(b, 16);
      if (pbits_dry(b)) return 1;
      if ((len ^ 0xFFFFu) != nlen) return bad();
      for (uint32_t i = 0; i < len; i++) {
        const uint8_t v = (uint8_t)pbits_get(b, 8);
        if (pbits_dry(b)) return 1;
        put(v);
      }
    } else if (type == 1 || type == 2) {
      if (type == 1) {                                    // fixed codes (RFC 1951 3.2.6)
        for (int s = 0; s < 288; s++) w.lens[s] = s < 144 ? 8 : s < 256 ? 9 : s < 280 ? 7 : 8;
        png_build(w.lit, w.lens, 288, true);
        for (int s = 0; s < 32; s++) w.lens[s] = 5;      // 30 and 31 complete the code; decoding one is an error
        png_build(w.dist, w.lens, 32, true);
      } else {                                            // dynamic codes (3.2.7)
        const int nlen = (int)pbits_get(b, 5) + 257, ndist = (int)pbits_get(b, 5) + 1, ncode = (int)pbits_get(b, 4) + 4;
        if (pbits_dry(b)) return 1;
        if (nlen > 286 || ndist > 30) return bad();
        const uint8_t order[19] = { 16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15 };
        uint8_t cl[19];
        for (int i = 0; i < 19; i++) cl[order[i]] = i < ncode ? (uint8_t)pbits_get(b, 3) : 0;
        if (pbits_dry(b)) return 1;
        if (!png_build(w.cl, cl, 19, false)) return bad();
        int i = 0;
        while (i < nlen + ndist) {
          const int sym = png_decode(b, w.cl);
          if (pbits_dry(b)) return 1;
          if (sym < 0) return bad();
          if (sym < 16) { w.lens[i++] = (uint8_t)sym; continue; }
          int rep, v = 0;
          if (sym == 16) { if (i == 0) return bad(); v = w.lens[i - 1]; rep = 3 + (int)pbits_get(b, 2); }
          else if (sym == 17) rep = 3 + (int)pbits_get(b, 3);
          else rep = 11 + (int)pbits_get(b, 7);
          if (pbits_dry(b)) return 1;
          if (i + rep > nlen + ndist) return bad();
          while (rep--) w.lens[i++] = (uint8_t)v;
        }
        if (w.lens[256] == 0) return bad();               // no end-of-block code
        if (!png_build(w.lit, w.lens, nlen, true)) return bad();
        if (!png_build(w.dist, w.lens + nlen, ndist, true)) return bad();
      }
      while (true) {
        const int sym = png_decode(b, w.lit);
        if (pbits_dry(b)) return 1;
        if (sym < 0) return bad();
        if (sym < 256) { put((uint8_t)sym); continue; }
        if (sym == 256) break;
        const int li = sym - 257;
        if (li >= 29) return bad();                       // 286, 287
        int len;
        if (li < 8) len = 3 + li;
        else if (li == 28) len = 258;
        else { const int e = (li >> 2) - 1; len = ((4 + (li & 3)) << e) + 3 + (int)pbits_get(b, e); }
        const int ds = png_decode(b, w.dist);
        if (pbits_dry(b)) return 1;
        if (ds < 0 || ds >= 30) return bad();
        int dist;
        if (ds < 4) dist = ds + 1;
        else { const int e = (ds >> 1) - 1; dist = ((2 + (ds & 1)) << e) + 1 + (int)pbits_get(b, e); }
        if (pbits_dry(b)) return 1;
        if (dist > out) return bad();                     // a distance behind the output start
        for (int k = 0; k < len; k++) put(out < total ? scan[out - dist] : 0);     // past the image only the count matters
      }
    } else {
      return bad();                                       // block type 3
    }
  }
  if (out < total) return 1;                              // the stream ends before the image does
  pbits_get(b, b.nbits & 7);                              // the Adler-32 trailer
  uint32_t adler = 0;
  for (int i = 0; i < 4; i++) adler = (adler << 8) | pbits_get(b, 8);
  if (pbits_dry(b)) return 1;
  return adler != (((s2 % 65521u) << 16) | (s1 % 65521u)) ? bad() : 0;
}

// png_inflate, then the unfilter in place.  Returns 0, or 1 for a malformed stream or filter byte.
PNG_HD int png_inflate_unfilter(const PngImage &im, const PngChunk *chunks, const uint8_t *raw, uint8_t *scan, PngWork &w) {
  if (png_inflate(im, chunks, raw, scan, w)) return 1;
  // unfilter in place, pass by pass (filter types 0..4 of the PNG specification, 9.2); bpp = bytes of a whole pixel, at least 1
  const int bpp = (im.spp * im.depth + 7) >> 3;
  for (int p = 0; p < 7; p++) {
    const int rb = im.pass_row[p];
    if (rb == 0) continue;
    int x0, y0, dx, dy;
    png_pass_geom(im.interlace, p, x0, y0, dx, dy);
    const int rows = (im.height - y0 + dy - 1) / dy;
    uint8_t *prev = nullptr;
    for (int y = 0; y < rows; y++) {
      uint8_t *row = scan + im.pass_off[p] + (int64_t)y * rb;
      const int f = row[0];
      uint8_t *c = row + 1;
      const uint8_t *u = prev ? prev + 1 : nullptr;
      const int n = rb - 1;
      switch (f) {
        case 0: break;
        case 1: for (int i = bpp; i < n; i++) c[i] = (uint8_t)(c[i] + c[i - bpp]); break;
        case 2: if (u) for (int i = 0; i < n; i++) c[i] = (uint8_t)(c[i] + u[i]); break;
        case 3:
          for (int i = 0; i < n; i++) {
            const int a = i >= bpp ? c[i - bpp] : 0, up = u ? u[i] : 0;
            c[i] = (uint8_t)(c[i] + ((a + up) >> 1));
          }
          break;
        case 4:
          for (int i = 0; i < n; i++) {
            const int a = i >= bpp ? c[i - bpp] : 0, up = u ? u[i] : 0, ul = (u && i >= bpp) ? u[i - bpp] : 0;
            const int pp = a + up - ul;
            const int pa = pp > a ? pp - a : a - pp, pb = pp > up ? pp - up : up - pp, pc = pp > ul ? pp - ul : ul - pp;
            c[i] = (uint8_t)(c[i] + ((pa <= pb && pa <= pc) ? a : pb <= pc ? up : ul));
          }
          break;
        default: return 1;
      }
      prev = row;
    }
  }
  return 0;
}

// ---------------------------------------------------------------------------------------------------------------------------------
// One output pixel of the window (lx, ly): unpacks the sample(s) from the unfiltered scanlines and writes cv2's IMREAD_COLOR (RGB
// order; BGR swaps) or IMREAD_GRAYSCALE value.  Rules pinned against cv2 4.13 (tests/png_oracle.py):
//   * 1/2/4-bit gray scales to 8 bits (v * 255 / (2^depth - 1)); a palette index reads PLTE (black past its end);
//   * 16-bit samples keep their high byte; alpha is dropped;
//   * GRAY of a colour or palette pixel: (9797 R + 19234 G + 3737 B) >> 15 on 8-bit values, and on 16-bit samples
//     ((9797 R + 19234 G + 3737 B + 16384) >> 15) >> 8.
PNG_HD void png_pixel(const PngImage &im, const uint8_t *scan, int lx, int ly) {
  const int x = im.win_x0 + lx, y = im.win_y0 + ly;
  int p = 0, px = x, py = y;
  if (im.interlace) {
    int x0, y0, dx, dy;
    p = png_adam7_pass(x, y);
    png_pass_geom(1, p, x0, y0, dx, dy);
    px = (x - x0) / dx; py = (y - y0) / dy;
  }
  const uint8_t *row = scan + im.pass_off[p] + (int64_t)py * im.pass_row[p] + 1;
  uint32_t r, g, bl;                                       // 8-bit values
  uint32_t r16 = 0, g16 = 0, b16 = 0;
  bool colour = false, wide = false;
  if (im.depth < 8) {
    const int64_t bit = (int64_t)px * im.depth;
    const uint32_t v = (row[bit >> 3] >> (8 - im.depth - (bit & 7))) & ((1u << im.depth) - 1);
    if (im.ctype == kPngPalette) { r = im.pal[v][0]; g = im.pal[v][1]; bl = im.pal[v][2]; colour = true; }
    else r = g = bl = v * (255u / ((1u << im.depth) - 1));
  } else if (im.depth == 8) {
    const uint8_t *s = row + (int64_t)px * im.spp;
    if (im.ctype == kPngPalette) { r = im.pal[s[0]][0]; g = im.pal[s[0]][1]; bl = im.pal[s[0]][2]; colour = true; }
    else if (im.ctype == kPngRGB || im.ctype == kPngRGBA) { r = s[0]; g = s[1]; bl = s[2]; colour = true; }
    else r = g = bl = s[0];
  } else {
    const uint8_t *s = row + (int64_t)px * im.spp * 2;
    if (im.ctype == kPngRGB || im.ctype == kPngRGBA) {
      r = s[0]; g = s[2]; bl = s[4]; colour = wide = true;
      r16 = (s[0] << 8) | s[1]; g16 = (s[2] << 8) | s[3]; b16 = (s[4] << 8) | s[5];
    } else r = g = bl = s[0];
  }
  const int64_t o = (int64_t)ly * im.win_w + lx;
  if (im.out_type == 2 /* DALIB200_GRAY */) {
    uint32_t v = r;
    if (wide) v = ((9797u * r16 + 19234u * g16 + 3737u * b16 + 16384u) >> 15) >> 8;
    else if (colour) v = (9797u * r + 19234u * g + 3737u * bl) >> 15;
    im.out[o] = (uint8_t)v;
    return;
  }
  uint8_t *d = im.out + o * 3;
  if (im.out_type == 1 /* DALIB200_BGR */) { d[0] = (uint8_t)bl; d[1] = (uint8_t)g; d[2] = (uint8_t)r; }
  else { d[0] = (uint8_t)r; d[1] = (uint8_t)g; d[2] = (uint8_t)bl; }
}

}  // namespace dalib200
#endif  // DALI_B200_CSRC_PNG_CORE_H_
