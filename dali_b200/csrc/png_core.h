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
#include "inflate.h"
#include "host_device.h"

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
DB_HD void png_pass_geom(int interlace, int p, int &x0, int &y0, int &dx, int &dy) {
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
DB_HD int png_adam7_pass(int x, int y) {
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
DB_HD bool png_chunk_crc_ok(const uint8_t *type, uint32_t len, const uint32_t *table) {
  uint32_t c = 0xFFFFFFFFu;
  for (uint32_t i = 0; i < len + 4; i++) c = table[(c ^ type[i]) & 255] ^ (c >> 8);
  const uint8_t *e = type + 4 + len;
  return (c ^ 0xFFFFFFFFu) == (((uint32_t)e[0] << 24) | ((uint32_t)e[1] << 16) | ((uint32_t)e[2] << 8) | e[3]);
}
DB_HD uint32_t png_crc_table_entry(uint32_t i) {
  uint32_t c = i;
  for (int k = 0; k < 8; k++) c = c & 1 ? 0xEDB88320u ^ (c >> 1) : c >> 1;
  return c;
}

// ---------------------------------------------------------------------------------------------------------------------------------
// Inflates the image's zlib stream into `scan` (im.scan_bytes bytes): inflate.h over the IDAT payloads read as one stream, hopping the
// 12-byte gaps (CRC, length, type) between chunks.  Returns 0, or 1 for a malformed stream.  Reads stay inside the chunks' payloads;
// writes stay inside [scan, scan + scan_bytes).
//
// The stream's tail follows libpng + zlib (pinned against cv2 by tests/test_png_cpu.py):
//   * the data running out before the end of the zlib stream is an error, before or after the image is complete ("Not enough image
//     data");
//   * the zlib call that produces the image's last byte decodes on until it would have to produce another one: a malformed block or a
//     bad Adler-32 trailer met before that is an error;
//   * once a byte beyond the image (a surplus) would be produced, libpng only drains the rest of the stream: malformed data or a bad
//     trailer there is a warning, so the rest is decoded without output ("draining") and only its end is required.
DB_HD int png_inflate(const PngImage &im, const PngChunk *chunks, const uint8_t *raw, uint8_t *scan, InflateWork &w) {
  InflateBits<PngChunk> b;
  ibits_init(b, raw + im.raw_off, chunks, im.chunk_begin, im.chunk_end);
  ibits_get(b, 16);                                       // CMF / FLG, checked by the planner
  return inflate_zlib<false>(b, scan, im.scan_bytes, w);
}

// png_inflate, then the unfilter in place.  Returns 0, or 1 for a malformed stream or filter byte.
DB_HD int png_inflate_unfilter(const PngImage &im, const PngChunk *chunks, const uint8_t *raw, uint8_t *scan, InflateWork &w) {
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
DB_HD void png_pixel(const PngImage &im, const uint8_t *scan, int lx, int ly) {
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
