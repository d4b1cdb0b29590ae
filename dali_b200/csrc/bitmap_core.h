// dali_b200/csrc/bitmap_core.h -- BMP and PNM (PBM / PGM / PPM) decoding written once for device and host: the serial unpack of one
// RLE-compressed BMP or ASCII PNM image into a plane of plan scratch (bitmap_unpack), and the conversion of a group of output pixels
// (bitmap_group).
//
// Most of these images are an uncompressed raster: bitmap_color reads the staged bytes directly, with no decode and no copy.  Only
// RLE4 / RLE8 BMP and ASCII P1-P3 are serial chains; bitmap_unpack expands them into an 8-bit plane (palette indices or final samples),
// which bitmap_color then reads like an uncompressed 8-bit raster.  The same functions compiled by a host compiler are what
// tools/emul/bitmap_emul.cc runs to pin them against cv2.imdecode without a GPU (tests/test_bitmap_cpu.py).
//
// Parity target: cv2.imdecode (OpenCV 4.13, grfmt_bmp.cpp / grfmt_pxm.cpp).  DESIGN section 2 lists the rules.
#ifndef DALI_B200_CSRC_BITMAP_CORE_H_
#define DALI_B200_CSRC_BITMAP_CORE_H_
#include <stdint.h>
#include <vector_types.h>
#include "host_device.h"

namespace dalib200 {

// how bitmap_color reads a pixel of the source (the staged raster, or the plane bitmap_unpack wrote)
enum BitmapLayout : int32_t {
  kBitmapIndexed = 0,          // 1-, 4- or 8-bit palette indices, most significant bits first (`bits`)
  kBitmap555 = 1,              // 16-bit little-endian x-R5-G5-B5
  kBitmap565 = 2,              // 16-bit little-endian R5-G6-B5
  kBitmapBytes = 3,            // `channels` samples of `sample_bytes` bytes each (2: big-endian, the high byte is read), `px_bytes` apart
};
// the serial pass an image needs before bitmap_color, or none
enum BitmapUnpack : int32_t { kBitmapDirect = 0, kBitmapRle8 = 1, kBitmapRle4 = 2, kBitmapAscii = 3 };

struct BitmapImage {
  int64_t raw_off;             // byte offset of the image's staged bytes (BMP: pixel array or RLE data; PNM: the raster)
  int64_t plane_off;           // unpack != kBitmapDirect: offset of the plane bitmap_unpack writes, in the scratch buffer
  uint32_t raw_len;            // staged bytes; bitmap_unpack reads no further
  int32_t sample;              // batch index (status word)
  int32_t width, height;
  int32_t unpack;              // BitmapUnpack
  int32_t layout;              // BitmapLayout of the source bitmap_color reads
  int32_t bits;                // kBitmapIndexed: 1, 4 or 8
  int32_t px_bytes, sample_bytes, channels, bgr;   // kBitmapBytes; bgr: the colour samples are in B, G, R order (BMP)
  int32_t bottom_up;           // the source's row 0 is the bottom row of the image (BMP with a positive height)
  uint32_t stride;             // bytes per source row
  int32_t ascii_channels;      // kBitmapAscii: 1 (P1 / P2) or 3 (P3) samples per pixel
  int32_t ascii_bits;          // kBitmapAscii: P1 (one digit per pixel, 1 = black)
  int32_t maxval;              // kBitmapAscii: PNM maxval
  int32_t gray_float;          // GRAY by cv2's float rule (32-bit BITFIELDS with R, G, B masks in a V3 - V5 header), else the integer rule
  // output, filled at launch: the window [win_x0, win_x0 + win_w) x [win_y0, win_y0 + win_h) of the image goes to `out` as a tight
  // win_h x win_w x C buffer, C = 1 for GRAY (cv2 IMREAD_GRAYSCALE), 3 for RGB / BGR (IMREAD_COLOR)
  uint8_t *out;
  int32_t win_x0, win_y0, win_w, win_h, out_type;
  int64_t first_px;            // prefix of window pixels over the bitmap images
  int64_t first_grp;           // prefix of pixel groups (kBitmapGroup pixels each) over the bitmap images: bitmap_color's search key
  uint8_t pal[256][3];         // R, G, B; entries past the stream's palette are 0
};

// ---------------------------------------------------------------------------------------------------------------------------------
// OpenCV's PxM ReadNumber: skips whitespace and '#' comments (up to '\n' or '\r'), reads decimal digits (at most `maxdigits`, 0 = no
// limit) and consumes the byte behind them.  Any other byte in front of the number, a value above INT_MAX or the end of the data is an
// error (returns false).
DB_HD bool pnm_read_number(const uint8_t *s, uint32_t n, uint32_t &pos, int maxdigits, int32_t &val) {
  auto space = [](int c) { return c == ' ' || (c >= '\t' && c <= '\r'); };
  auto digit = [](int c) { return c >= '0' && c <= '9'; };
  if (pos >= n) return false;
  int c = s[pos++];
  while (!digit(c)) {
    if (c == '#') {
      do { if (pos >= n) return false; c = s[pos++]; } while (c != '\n' && c != '\r');
      if (pos >= n) return false;
      c = s[pos++];
    } else if (space(c)) {
      while (space(c)) { if (pos >= n) return false; c = s[pos++]; }
    } else {
      return false;
    }
  }
  int64_t v = 0;
  int digits = 0;
  for (;;) {
    v = v * 10 + (c - '0');
    if (v > 0x7FFFFFFF) return false;
    if (maxdigits && ++digits >= maxdigits) break;
    if (pos >= n) return false;
    c = s[pos++];
    if (!digit(c)) break;
  }
  val = (int32_t)v;
  return true;
}

// cv2's FillUniColor: `count` pixels of palette index v from (x, y) on, wrapping at the end of each row, stopping behind the last row
DB_HD void bitmap_fill(uint8_t *plane, int64_t W, int64_t H, int64_t &x, int64_t &y, int64_t count, uint8_t v) {
  do {
    const int64_t end = x + count < W ? x + count : W;
    count -= end - x;
    for (uint8_t *row = plane + y * W; x < end; x++) row[x] = v;
    if (x >= W) { x = 0; if (++y >= H) break; }
  } while (count > 0);
}

// RLE8 / RLE4 as cv2's BmpDecoder reads them, into a W x H plane of palette indices in the file's row order.  Pixels that an
// end-of-line, delta or end-of-bitmap code skips take index 0; a delta (dx, dy) skips dx + dy * W pixels in RLE8 and dx in RLE4 (whose
// dy byte is read and ignored), and RLE4's end-of-bitmap ends the image only on its last row (elsewhere it acts as end-of-line).  A run
// past the end of its row, or data that ends before the last row is complete, is an error.
DB_HD int bitmap_rle(const BitmapImage &im, const uint8_t *s, uint8_t *plane) {
  const int64_t W = im.width, H = im.height;
  const uint32_t n = im.raw_len;
  const bool rle8 = im.unpack == kBitmapRle8;
  uint32_t pos = 0;
  int64_t x = 0, y = 0;
  bool wrapped = false;                                      // RLE8: the last run ended its row exactly (an end-of-line behind it is void)
  for (;;) {
    if (n - pos < 2) return 1;
    const int len = s[pos], code = s[pos + 1];
    pos += 2;
    if (len) {                                               // a run of `len` pixels
      if (x + len > W) return 1;
      if (rle8) {
        const int64_t y0 = y;
        bitmap_fill(plane, W, H, x, y, len, (uint8_t)code);
        wrapped = y != y0;
        if (y >= H) return 0;
      } else {
        uint8_t *row = plane + y * W;
        for (int i = 0; i < len; i++) row[x + i] = (uint8_t)(i & 1 ? code & 15 : code >> 4);
        x += len;
      }
    } else if (code > 2) {                                   // absolute mode: `code` literal pixels, padded to 16 bits
      if (x + code > W) return 1;
      const uint32_t sz = rle8 ? (code + 1) & ~1 : (((code + 1) >> 1) + 1) & ~1;
      if (n - pos < sz) return 1;
      uint8_t *row = plane + y * W;
      for (int i = 0; i < code; i++) row[x + i] = rle8 ? s[pos + i] : (uint8_t)((s[pos + (i >> 1)] >> (i & 1 ? 0 : 4)) & 15);
      x += code;
      pos += sz;
      wrapped = false;
    } else {                                                 // 0: end of line, 1: end of bitmap, 2: delta
      int64_t dx = W - x, dy = H - y;
      if (!rle8 || code || !wrapped || dx < W) {
        if (code == 2) {
          if (n - pos < 2) return 1;
          dx = s[pos]; dy = s[pos + 1];
          pos += 2;
        }
        bitmap_fill(plane, W, H, x, y, rle8 && code ? dx + dy * W : dx, 0);
        if (y >= H) return 0;
      }
      wrapped = false;
    }
  }
}

// ASCII P1 / P2 / P3 as cv2's PxMDecoder reads them, into a plane of `ascii_channels` bytes per pixel: P1 one digit per pixel (index 1
// for a non-zero digit: black), P2 / P3 samples clamped to maxval, then v * 255 / maxval for maxval < 256 or v >> 8 above.
DB_HD int bitmap_ascii(const BitmapImage &im, const uint8_t *s, uint8_t *plane) {
  const int64_t count = (int64_t)im.width * im.height * im.ascii_channels;
  uint32_t pos = 0;
  for (int64_t i = 0; i < count; i++) {
    int32_t v;
    if (!pnm_read_number(s, im.raw_len, pos, im.ascii_bits ? 1 : 0, v)) return 1;
    if (im.ascii_bits) { plane[i] = v != 0; continue; }
    if (v > im.maxval) v = im.maxval;
    plane[i] = (uint8_t)(im.maxval < 256 ? v * 255 / im.maxval : v >> 8);
  }
  return 0;
}

// bitmap_unpack_kernel's body: the plane of one RLE or ASCII image.  Returns 0, or 1 for data cv2 refuses.  Reads stay inside the
// image's raw_len staged bytes, writes inside its plane (width * height * ascii_channels bytes; RLE: width * height).
DB_HD int bitmap_unpack(const BitmapImage &im, const uint8_t *raw, uint8_t *plane) {
  return im.unpack == kBitmapAscii ? bitmap_ascii(im, raw, plane) : bitmap_rle(im, raw, plane);
}

// R, G, B of image pixel (x, y) from the source raster `src`
DB_HD void bitmap_rgb(const BitmapImage &im, const uint8_t *src, int x, int y, uint32_t &r, uint32_t &g, uint32_t &b) {
  const uint8_t *row = src + (int64_t)(im.bottom_up ? im.height - 1 - y : y) * im.stride;
  if (im.layout == kBitmapIndexed) {
    const uint32_t i = im.bits == 8 ? row[x] : im.bits == 4 ? (row[x >> 1] >> (x & 1 ? 0 : 4)) & 15 : (row[x >> 3] >> (7 - (x & 7))) & 1;
    r = im.pal[i][0]; g = im.pal[i][1]; b = im.pal[i][2];
  } else if (im.layout == kBitmapBytes) {
    const uint8_t *p = row + (int64_t)x * im.px_bytes;
    const uint32_t c0 = p[0];
    if (im.channels == 1) { r = g = b = c0; return; }
    const uint32_t c1 = p[im.sample_bytes], c2 = p[2 * im.sample_bytes];
    if (im.bgr) { b = c0; g = c1; r = c2; } else { r = c0; g = c1; b = c2; }
  } else {                                                   // 5-5-5 / 5-6-5: shifted up, no bit replication (cv2's rule)
    const uint32_t v = row[2 * x] | (uint32_t)row[2 * x + 1] << 8;
    b = (v << 3) & 0xF8;
    if (im.layout == kBitmap565) { g = (v >> 3) & 0xFC; r = (v >> 8) & 0xF8; }
    else { g = (v >> 2) & 0xF8; r = (v >> 7) & 0xF8; }
  }
}

// bitmap_color_kernel's work item: window pixels [16 g, 16 g + 16) of the image, in row-major window order.  A whole group whose output
// is 16-byte aligned is written with 16-byte stores (one for GRAY, three for RGB / BGR), any other with byte stores.  GRAY of a colour
// pixel: (1868 B + 9617 G + 4899 R + 8192) >> 14 (cv2's BGR -> gray in both decoders), except for gray_float images, which cv2 reads
// through its bitfield-mask path: the float32 sum (0.299 R + 0.587 G) + 0.114 B, each product and sum rounded once, truncated.
constexpr int kBitmapGroup = 16;
DB_HD uint32_t bitmap_gray(const BitmapImage &im, uint32_t r, uint32_t g, uint32_t b) {
  if (!im.gray_float) return (b * 1868u + g * 9617u + r * 4899u + 8192u) >> 14;
#if defined(__CUDA_ARCH__)
  return (uint32_t)__fadd_rn(__fadd_rn(__fmul_rn(0.299f, (float)r), __fmul_rn(0.587f, (float)g)), __fmul_rn(0.114f, (float)b));
#else
  return (uint32_t)((0.299f * (float)r + 0.587f * (float)g) + 0.114f * (float)b);   // built with -ffp-contract=off
#endif
}
DB_HD void bitmap_group(const BitmapImage &im, const uint8_t *src, int64_t g) {
  const int64_t p0 = g * kBitmapGroup, npx = (int64_t)im.win_w * im.win_h;
  const int cnt = npx - p0 < kBitmapGroup ? (int)(npx - p0) : kBitmapGroup;
  int ly = (int)(p0 / im.win_w), lx = (int)(p0 - (int64_t)ly * im.win_w);
  const bool gray = im.out_type == 2 /* DALIB200_GRAY */, bgr = im.out_type == 1 /* DALIB200_BGR */;
  uint32_t w[3 * kBitmapGroup / 4] = {0};
  auto put = [&](int i, uint32_t v) { w[i >> 2] |= v << (8 * (i & 3)); };
#if defined(__CUDACC__)
#pragma unroll
#endif
  for (int k = 0; k < kBitmapGroup; k++) {
    if (k < cnt) {
      uint32_t r, gg, b;
      bitmap_rgb(im, src, im.win_x0 + lx, im.win_y0 + ly, r, gg, b);
      if (gray) put(k, bitmap_gray(im, r, gg, b));
      else if (bgr) { put(3 * k, b); put(3 * k + 1, gg); put(3 * k + 2, r); }
      else { put(3 * k, r); put(3 * k + 1, gg); put(3 * k + 2, b); }
      if (++lx == im.win_w) { lx = 0; ly++; }
    }
  }
  const int C = gray ? 1 : 3;
  uint8_t *d = im.out + p0 * C;
  if (cnt == kBitmapGroup && ((uintptr_t)d & 15) == 0) {
    uint4 *q = reinterpret_cast<uint4 *>(d);
    auto quad = [](uint32_t a, uint32_t b, uint32_t c, uint32_t e) { uint4 v; v.x = a; v.y = b; v.z = c; v.w = e; return v; };
    q[0] = quad(w[0], w[1], w[2], w[3]);
    if (!gray) { q[1] = quad(w[4], w[5], w[6], w[7]); q[2] = quad(w[8], w[9], w[10], w[11]); }
  } else {
#if defined(__CUDACC__)
#pragma unroll
#endif
    for (int i = 0; i < 3 * kBitmapGroup; i++)             // unrolled, so that w stays in registers
      if (i < cnt * C) d[i] = (uint8_t)(w[i >> 2] >> (8 * (i & 3)));
  }
}

}  // namespace dalib200
#endif  // DALI_B200_CSRC_BITMAP_CORE_H_
