// dali_b200/csrc/tiff_core.h -- TIFF decoding written once for device and host: the decode of one segment (tiff_decode_segment) and
// the conversion of one output pixel (tiff_pixel).
//
// A TIFF image is cut into segments -- strips or tiles, one plane each when PlanarConfiguration is 2 -- compressed one by one.  Each is
// an independent serial chain, so tiff_segment runs one working lane per segment: a cv2-written 1080p RGB image is 1 080 one-row LZW
// strips.  The same functions compiled by a host compiler are what tools/emul/tiff_emul.cc runs to pin them against tests/tiff_oracle.py
// without a GPU (tests/test_tiff_cpu.py).
//
// Parity target: cv2.imdecode (OpenCV 4.13 / libtiff 4.7).  A segment decodes to exactly its size (a strip: its rows; a tile: the whole
// padded tile); surplus input is ignored and a segment that ends early is an error, for every codec (libtiff's "Not enough data").
#ifndef DALI_B200_CSRC_TIFF_CORE_H_
#define DALI_B200_CSRC_TIFF_CORE_H_
#include <stdint.h>
#include "inflate.h"
#include "host_device.h"

namespace dalib200 {

enum TiffCompression : int32_t { kTiffNone = 1, kTiffLzw = 5, kTiffDeflate = 8, kTiffPackBits = 32773 };
enum TiffPhotometric : int32_t { kTiffMinIsWhite = 0, kTiffMinIsBlack = 1, kTiffRGB = 2, kTiffPalette = 3 };

// working memory of one segment decode, a plan-owned global slot per working lane of tiff_segment: the LZW string starts, or the inflate
// tables (a per-thread stack frame of this size would make the driver reserve it for every resident thread of the GPU)
constexpr int kTiffLzwStarts = 4096 - 258 + 2;               // start of every code since the last Clear that a 12-bit code can name
constexpr uint32_t kTiffSlotBytes = 16384;
static_assert(sizeof(InflateWork) <= kTiffSlotBytes && kTiffLzwStarts * 4 <= kTiffSlotBytes, "TIFF slot too small");

struct TiffSeg {               // one strip or tile of one plane
  uint32_t off, len;           // compressed bytes, relative to the image's staged bytes (an inflate.h byte range)
  int32_t image;               // index into the TiffImage array
  uint32_t rows;               // decoded rows (a strip at the bottom edge has fewer; a tile is always whole)
  int64_t dec_off;             // offset of the decoded bytes in the scratch buffer (rows * TiffImage::row_bytes)
};

struct TiffImage {
  int64_t raw_off;             // byte offset of the image's staged bytes (the span of its segments)
  int32_t seg_begin, seg_end;
  int32_t sample;              // batch index (status word)
  int32_t width, height, bps, spp, photometric, planar, compression, predictor;
  int32_t big_endian;          // byte order of 16-bit samples (and of the predictor's differences)
  int32_t premultiply;         // ExtraSamples = unassociated alpha: libtiff's RGBA path premultiplies colour by alpha
  int32_t seg_w, seg_h;        // pixel size of a segment (a strip: width x RowsPerStrip)
  int32_t segs_across, segs_per_plane;
  uint32_t row_bytes;          // bytes of one decoded segment row
  // output, filled at launch: the window [win_x0, win_x0 + win_w) x [win_y0, win_y0 + win_h) of the image goes to `out` as a tight
  // win_h x win_w x C buffer, C = 1 for GRAY (cv2 IMREAD_GRAYSCALE), 3 for RGB / BGR (IMREAD_COLOR)
  uint8_t *out;
  int32_t win_x0, win_y0, win_w, win_h, out_type;
  int64_t first_px;            // prefix of window pixels over the TIFF images (tiff_color's sample search)
  uint8_t pal[256][3];         // ColorMap scaled to 8 bits
};

// ---------------------------------------------------------------------------------------------------------------------------------
// LZW (TIFF 6.0 section 13, the MSB-first variant with early change), as libtiff's LZWDecode runs it.  Every string of the code table
// is a copy of earlier output of the segment plus one byte: code 258 + j is the output of the j-th code since the last Clear followed by
// the first byte of the next one.  So the table is only the output offset where each code's string starts, `start` (kTiffLzwStarts
// entries), and strings are copied out of the segment's own output.  Errors, as libtiff's: a first code that is not Clear, a code past
// the next free one, a literal expected after Clear, a full table, EOI or the end of the data before the segment is complete.
DB_HD int tiff_lzw(const uint8_t *src, uint32_t n, uint8_t *dst, uint32_t total, uint32_t *start) {
  uint64_t acc = 0;
  int nb = 0;
  uint32_t pos = 0, out = 0;
  int width = 9, mask = 511;   // code width; libtiff widens when the next free entry reaches mask
  int k = -1;                  // codes since the last Clear, -1 = no Clear yet
  while (out < total) {
    if (nb < width) {
      if (pos + 2 <= n) { acc = (acc << 16) | ((uint32_t)src[pos] << 8) | src[pos + 1]; pos += 2; nb += 16; }
      else { while (nb < width && pos < n) { acc = (acc << 8) | src[pos++]; nb += 8; } if (nb < width) return 1; }
    }
    nb -= width;
    const int code = (int)((acc >> nb) & ((1u << width) - 1));
    if (code == 257) return 1;                               // EOI before the segment is complete
    if (code == 256) { k = 0; width = 9; mask = 511; continue; }
    if (k < 0) return 1;
    const int fr = 257 + k;                                   // the entry this code defines (k >= 1)
    if (k == 0) {
      if (code > 255) return 1;
    } else {
      if (fr >= 5119) return 1;                               // libtiff's table (CSIZE) is full
      if (code > 255 && code > fr) return 1;                  // an undefined code
      if (fr + 1 > mask - 1 && width < 12) { width++; mask = (1 << width) - 1; }
    }
    if (k < kTiffLzwStarts) start[k] = out;
    k++;
    if (code < 256) { dst[out++] = (uint8_t)code; continue; }
    const uint32_t j = (uint32_t)(code - 258);
    const uint32_t s = start[j], len = start[j + 1] - s + 1;  // start[j + 1] == out for the code being defined (KwKwK)
    for (uint32_t i = 0; i < len && out < total; i++, out++) dst[out] = dst[s + i];
  }
  return 0;
}

// PackBits (libtiff PackBitsDecode): a run longer than the rest of the segment is clipped, data ending early is an error
DB_HD int tiff_packbits(const uint8_t *src, uint32_t n, uint8_t *dst, uint32_t total) {
  uint32_t pos = 0, out = 0;
  while (pos < n && out < total) {
    int c = (int8_t)src[pos++];
    if (c == -128) continue;
    if (c < 0) {
      if (pos >= n) break;
      const uint8_t v = src[pos++];
      for (int i = 0; i < 1 - c && out < total; i++) dst[out++] = v;
    } else {
      uint32_t m = (uint32_t)c + 1;
      if (m > total - out) m = total - out;
      if (m > n - pos) break;
      for (uint32_t i = 0; i < m; i++) dst[out++] = src[pos++];
    }
  }
  return out < total ? 1 : 0;
}

// Decodes segment `s` into `dst` (s.rows * im.row_bytes bytes) and undoes the horizontal predictor row by row.  Returns 0, or 1 for a
// malformed or short segment.  Reads stay inside the segment's bytes; writes inside [dst, dst + size).  `slot`: kTiffSlotBytes of
// working memory (4-byte aligned).
DB_HD int tiff_decode_segment(const TiffImage &im, const TiffSeg &s, const uint8_t *raw, uint8_t *dst, void *slot) {
  const uint8_t *src = raw + im.raw_off + s.off;
  const uint32_t total = s.rows * im.row_bytes;
  int rc = 0;
  if (im.compression == kTiffLzw) {
    rc = tiff_lzw(src, s.len, dst, total, static_cast<uint32_t *>(slot));
  } else if (im.compression == kTiffPackBits) {
    rc = tiff_packbits(src, s.len, dst, total);
  } else if (im.compression == kTiffDeflate) {
    InflateBits<TiffSeg> b;
    ibits_init(b, raw + im.raw_off, &s, 0, 1);
    const uint32_t cmf = ibits_get(b, 8), flg = ibits_get(b, 8);
    rc = ibits_dry(b) || !zlib_header_ok(cmf, flg) ? 1 : inflate_zlib<true>(b, dst, total, *static_cast<InflateWork *>(slot));
  } else {
    if (s.len < total) return 1;
    for (uint32_t i = 0; i < total; i++) dst[i] = src[i];
  }
  if (rc || im.predictor != 2) return rc;
  // horizontal differencing: each sample adds the same sample of the pixel before it in the row (16-bit: in the file's byte order)
  const int stride = im.planar == 2 ? 1 : im.spp;
  for (uint32_t r = 0; r < s.rows; r++) {
    uint8_t *row = dst + (int64_t)r * im.row_bytes;
    if (im.bps == 8) {
      for (uint32_t i = stride; i < im.row_bytes; i++) row[i] = (uint8_t)(row[i] + row[i - stride]);
    } else {
      const int hi = im.big_endian ? 0 : 1, lo = 1 - hi;
      for (uint32_t i = 2 * stride; i + 1 < im.row_bytes; i += 2) {
        const uint32_t v = (((uint32_t)row[i + hi] << 8) | row[i + lo]) + (((uint32_t)row[i - 2 * stride + hi] << 8) | row[i - 2 * stride + lo]);
        row[i + hi] = (uint8_t)(v >> 8); row[i + lo] = (uint8_t)v;
      }
    }
  }
  return 0;
}

// sample c of pixel (x, y), as stored (1 to 16 bits)
DB_HD uint32_t tiff_sample(const TiffImage &im, const TiffSeg *segs, const uint8_t *dec, int x, int y, int c) {
  const int plane = im.planar == 2 ? c : 0, sx = x / im.seg_w, sy = y / im.seg_h;
  const TiffSeg &s = segs[im.seg_begin + plane * im.segs_per_plane + sy * im.segs_across + sx];
  const int64_t bit = (int64_t)(x - sx * im.seg_w) * (im.planar == 2 ? 1 : im.spp) * im.bps + (im.planar == 2 ? 0 : c * im.bps);
  const uint8_t *p = dec + s.dec_off + (int64_t)(y - sy * im.seg_h) * im.row_bytes + (bit >> 3);
  if (im.bps == 16) return im.big_endian ? ((uint32_t)p[0] << 8) | p[1] : ((uint32_t)p[1] << 8) | p[0];
  if (im.bps == 8) return p[0];
  return (p[0] >> (8 - im.bps - (bit & 7))) & ((1u << im.bps) - 1);
}

// One output pixel of the window (lx, ly): libtiff's TIFFReadRGBA* conversion, then cv2's RGBA -> BGR / GRAY.  Rules pinned against
// cv2 4.13 (tests/tiff_oracle.py):
//   * gray, contiguous: 1/2/4/8 bits -> v * 255 / (2^bps - 1) (MinIsWhite: (2^bps - 1 - v) * 255 / (2^bps - 1)); 16 bits -> high byte
//     (MinIsWhite: 255 - high byte); an extra sample is dropped;
//   * RGB, and gray + extra sample with PlanarConfiguration 2 (libtiff reads those as RGB with R = G = B): 16 bits -> (v + 128) / 257,
//     no MinIsWhite inversion; unassociated alpha premultiplies, (c * a + 127) / 255 on the 8-bit values;
//   * palette: the ColorMap scaled to 8 bits by the planner;
//   * GRAY of a colour pixel: (1868 B + 9617 G + 4899 R + 8192) >> 14 (OpenCV's BGRA -> gray, the CMYK JPEG path's rule).
DB_HD void tiff_pixel(const TiffImage &im, const TiffSeg *segs, const uint8_t *dec, int lx, int ly) {
  const int x = im.win_x0 + lx, y = im.win_y0 + ly;
  uint32_t r, g, b;
  if (im.photometric == kTiffPalette) {
    const uint32_t v = tiff_sample(im, segs, dec, x, y, 0);
    r = im.pal[v][0]; g = im.pal[v][1]; b = im.pal[v][2];
  } else if (im.photometric == kTiffRGB || im.planar == 2) {
    const bool gray = im.photometric != kTiffRGB;
    const int ac = gray ? 1 : 3;                             // the alpha sample
    auto to8 = [&](uint32_t v) { return im.bps == 16 ? (v + 128) / 257 : v; };
    r = to8(tiff_sample(im, segs, dec, x, y, 0));
    g = gray ? r : to8(tiff_sample(im, segs, dec, x, y, 1));
    b = gray ? r : to8(tiff_sample(im, segs, dec, x, y, 2));
    if (im.premultiply) {
      const uint32_t a = to8(tiff_sample(im, segs, dec, x, y, ac));
      r = (r * a + 127) / 255; g = (g * a + 127) / 255; b = (b * a + 127) / 255;
    }
  } else {
    const uint32_t v = tiff_sample(im, segs, dec, x, y, 0);
    const uint32_t range = im.bps == 16 ? 255u : (1u << im.bps) - 1, s = im.bps == 16 ? v >> 8 : v;
    r = g = b = ((im.photometric == kTiffMinIsWhite ? range - s : s) * 255u) / range;
  }
  const int64_t o = (int64_t)ly * im.win_w + lx;
  if (im.out_type == 2 /* DALIB200_GRAY */) { im.out[o] = (uint8_t)((b * 1868u + g * 9617u + r * 4899u + 8192u) >> 14); return; }
  uint8_t *d = im.out + o * 3;
  if (im.out_type == 1 /* DALIB200_BGR */) { d[0] = (uint8_t)b; d[1] = (uint8_t)g; d[2] = (uint8_t)r; }
  else { d[0] = (uint8_t)r; d[1] = (uint8_t)g; d[2] = (uint8_t)b; }
}

}  // namespace dalib200
#endif  // DALI_B200_CSRC_TIFF_CORE_H_
