// dali_b200/csrc/bitmap_plan.h -- host-side planning of a BMP or PNM (PBM / PGM / PPM) stream inside the image decoder plan: format
// detection, the header walk (BMP file and info headers, palette, bitfield masks; PNM magic, size and maxval), the validation cv2 4.13
// applies, and the BitmapImage descriptor.  No per-byte work on the pixel data.  Plain C++ (no CUDA types): jpeg.cu calls it from
// JpegGetInfo / JpegPlanSetup, tools/emul/bitmap_emul.cc from the CPU tests.
//
// BMP: BITMAPINFOHEADER and larger (V2 - V5), or the 12-byte OS/2 core header; 1-, 4-, 8-bit palettes, RLE4, RLE8, 16-bit 5-5-5 (BI_RGB
// or BITFIELDS) and 5-6-5 (BITFIELDS), 24-bit, 32-bit BI_RGB or BITFIELDS (masks ignored, as in cv2: B, G, R, alpha bytes).  PNM: P1 - P6,
// ASCII or binary, maxval 1 - 65535.  What cv2 refuses is refused: DALIB200_ERROR_UNSUPPORTED for a valid stream of a kind cv2 does not
// decode (2-bit BMP, JPEG / PNG / RLE24 compression, other 16-bit masks, the size limits), DALIB200_ERROR_BAD_DATA for a malformed or
// truncated one.
#ifndef DALI_B200_CSRC_BITMAP_PLAN_H_
#define DALI_B200_CSRC_BITMAP_PLAN_H_
#include <algorithm>
#include <cstring>
#include <string>
#include "../../include/dali_b200.h"
#include "bitmap_core.h"
#include "stream_info.h"

namespace dalib200 {

inline bool IsBmpStream(const uint8_t *p, size_t n) { return n >= 2 && p[0] == 'B' && p[1] == 'M'; }
// cv2's PxM signature: 'P', '1' - '6', whitespace
inline bool IsPnmStream(const uint8_t *p, size_t n) {
  return n >= 3 && p[0] == 'P' && p[1] >= '1' && p[1] <= '6' && (p[2] == ' ' || (p[2] >= '\t' && p[2] <= '\r'));
}
inline bool IsBitmapStream(const uint8_t *p, size_t n) { return IsBmpStream(p, n) || IsPnmStream(p, n); }

// OpenCV's validateInputImageSize: at most 2^20 pixels on a side and 2^30 pixels in all
constexpr int64_t kBitmapMaxSide = 1 << 20;
constexpr int64_t kBitmapMaxPixels = 1ll << 30;

// Plans one BMP or PNM image.  Its plane (RLE and ASCII images only) goes to `plane_base` of the scratch buffer; *plane_bytes receives
// its size, 16-byte aligned (0 for an image bitmap_color reads straight from the staged bytes).  The staged bytes, info->stage_begin ..
// stage_end, are the BMP pixel array (RLE: the data from the pixel offset to the end of the stream) or the PNM raster behind the header.
// Returns a DALIB200 status.
inline int PlanBitmap(const uint8_t *p, size_t n, BitmapImage *im, int64_t plane_base, int64_t *plane_bytes, StreamInfo *info,
                      std::string *err) {
  const bool bmp = IsBmpStream(p, n);
  auto fail = [&](int rc, const std::string &m) { if (err) *err = (bmp ? "BMP: " : "PNM: ") + m; return rc; };
  auto bad = [&](const std::string &m) { return fail(DALIB200_ERROR_BAD_DATA, m); };
  auto unsupported = [&](const std::string &m) { return fail(DALIB200_ERROR_UNSUPPORTED, m); };
  memset(im, 0, sizeof(*im));
  *info = StreamInfo();
  *plane_bytes = 0;
  if (!bmp && !IsPnmStream(p, n)) return bad("missing signature");
  int64_t W = 0, H = 0;
  size_t begin = 0, end = n;
  if (bmp) {
    auto u16 = [&](size_t o) -> uint32_t { return p[o] | (uint32_t)p[o + 1] << 8; };
    auto i32 = [&](size_t o) -> int32_t { return (int32_t)(p[o] | (uint32_t)p[o + 1] << 8 | (uint32_t)p[o + 2] << 16 | (uint32_t)p[o + 3] << 24); };
    if (n < 18) return bad("truncated header");
    const int32_t offset = i32(10), size = i32(14);
    if (size <= 0) return bad("bad info header size");
    int bpp = 0, comp = 0;
    int64_t colours = 0;                                      // palette entries in the stream
    size_t pal_at = 0, entry = 4;
    bool colour = true;
    if (size >= 36) {
      if (n < 50) return bad("truncated header");
      W = i32(18); H = i32(22); bpp = (int)u16(28); comp = i32(30);
      const int32_t clrused = i32(46);
      if (comp < 0 || comp > 3) return unsupported("compression " + std::to_string(comp) + " is not supported (BI_RGB, RLE8, RLE4, BITFIELDS)");
      const bool ok = ((bpp == 1 || bpp == 4 || bpp == 8 || bpp == 24 || bpp == 32) && comp == 0) ||
                      ((bpp == 16 || bpp == 32) && (comp == 0 || comp == 3)) || (bpp == 4 && comp == 2) || (bpp == 8 && comp == 1);
      if (!ok) return unsupported(std::to_string(bpp) + "-bit pixels with compression " + std::to_string(comp) + " are not supported");
      pal_at = 14 + (size_t)size;
      if (bpp <= 8) {
        if (clrused < 0 || clrused > 256) return bad("more than 256 palette entries");
        colours = clrused ? clrused : 1 << bpp;
      } else if (bpp == 16 && comp == 3) {
        if (pal_at + 12 > n) return bad("truncated bitfield masks");
        const int32_t rm = i32(pal_at), gm = i32(pal_at + 4), bm = i32(pal_at + 8);
        if (bm == 0x1F && gm == 0x3E0 && rm == 0x7C00) bpp = 15;
        else if (!(bm == 0x1F && gm == 0x7E0 && rm == 0xF800)) return unsupported("16-bit masks other than 5-5-5 and 5-6-5 are not supported");
      } else if (bpp == 16) {
        bpp = 15;
      } else if (bpp == 32 && comp == 3 && size >= 56) {
        // a V3 - V5 header holds R, G, B, A masks.  With all three colour masks set, cv2 4.13 decodes through its mask path, whose GRAY
        // is a float rule; with any of them empty it reads B, G, R, alpha bytes as for a 40-byte header.  Of the mask path, the
        // standard masks (B, G, R, alpha bytes) are matched; cv2's extraction of other masks is not restated here
        if (n < 70) return bad("truncated header");
        const uint32_t rm = (uint32_t)i32(54), gm = (uint32_t)i32(58), bm = (uint32_t)i32(62);
        if (rm && gm && bm) {
          if (rm != 0xFF0000 || gm != 0xFF00 || bm != 0xFF) return unsupported("32-bit colour masks other than 0xFF0000 / 0xFF00 / 0xFF are not supported");
          im->gray_float = 1;
        }
      }
    } else if (size == 12) {
      if (n < 26) return bad("truncated header");
      W = u16(18); H = u16(20); bpp = (int)u16(24);
      if (!(bpp == 1 || bpp == 4 || bpp == 8 || bpp == 24 || bpp == 32)) return unsupported(std::to_string(bpp) + "-bit OS/2 bitmaps are not supported");
      pal_at = 26; entry = 3;
      if (bpp <= 8) colours = 1 << bpp;
    } else {
      return bad("info header size " + std::to_string(size) + " is not supported");
    }
    if (W <= 0 || H == 0) return bad("bad image size");
    im->bottom_up = H > 0;
    H = H < 0 ? -H : H;
    if (W > kBitmapMaxSide || H > kBitmapMaxSide || W * H > kBitmapMaxPixels)
      return unsupported("images wider or taller than 2^20 pixels or larger than 2^30 pixels are not supported (OpenCV's limit)");
    if (W * H * 3 >= (1ll << 30)) return unsupported("images of 2^30 / 3 pixels or more are not supported (OpenCV's BMP limit)");
    if (colours) {
      if (pal_at > n || (size_t)colours * entry > n - pal_at) return bad("truncated palette");
      for (int64_t i = 0; i < colours; i++) {
        const uint8_t *e = p + pal_at + i * entry;
        im->pal[i][0] = e[2]; im->pal[i][1] = e[1]; im->pal[i][2] = e[0];
      }
      colour = false;                                         // reported as 1 component when every entry is gray (cv2's IsColorPalette)
      for (int i = 0; i < (1 << bpp); i++) colour |= im->pal[i][0] != im->pal[i][1] || im->pal[i][1] != im->pal[i][2];
    }
    if (offset < 0 || (size_t)offset >= n) return bad("pixel data offset outside the stream");
    begin = (size_t)offset;
    im->width = (int)W; im->height = (int)H;
    if (comp == 1 || comp == 2) {
      im->unpack = comp == 1 ? kBitmapRle8 : kBitmapRle4;
      im->layout = kBitmapIndexed; im->bits = 8; im->stride = (uint32_t)W;
      *plane_bytes = (W * H + 15) & ~15ll;
    } else {
      const int64_t pitch = ((W * (bpp == 15 ? 16 : bpp) + 7) / 8 + 3) & ~3ll;
      if (H * pitch > (int64_t)(n - begin)) return bad("truncated pixel data");
      end = begin + (size_t)(H * pitch);
      im->stride = (uint32_t)pitch;
      if (bpp <= 8) { im->layout = kBitmapIndexed; im->bits = bpp; }
      else if (bpp == 15 || bpp == 16) im->layout = bpp == 15 ? kBitmap555 : kBitmap565;
      else { im->layout = kBitmapBytes; im->px_bytes = bpp / 8; im->sample_bytes = 1; im->channels = 3; im->bgr = 1; }
    }
    info->components = bpp <= 8 && !colour ? 1 : bpp == 32 && comp == 3 ? 4 : 3;
  } else {
    const int kind = p[1] - '0';
    uint32_t pos = 2;
    int32_t w = 0, h = 0, maxval = 1;
    const uint32_t hn = (uint32_t)std::min<size_t>(n, 0xFFFFFFFFu);   // the header lies in the first 4 GiB
    if (!pnm_read_number(p, hn, pos, 0, w) || !pnm_read_number(p, hn, pos, 0, h) ||
        (kind != 1 && kind != 4 && !pnm_read_number(p, hn, pos, 0, maxval)))
      return bad("malformed header");
    if (maxval > 65535) return unsupported("maxval above 65535 is not supported");
    if (w <= 0 || h <= 0 || maxval <= 0) return bad("bad image size or maxval");
    W = w; H = h;
    if (W > kBitmapMaxSide || H > kBitmapMaxSide || W * H > kBitmapMaxPixels)
      return unsupported("images wider or taller than 2^20 pixels or larger than 2^30 pixels are not supported (OpenCV's limit)");
    begin = pos;
    im->width = w; im->height = h;
    const int ch = kind == 3 || kind == 6 ? 3 : 1;
    if (kind == 1 || kind == 4) {                            // bit 1 is black
      im->pal[0][0] = im->pal[0][1] = im->pal[0][2] = 255;
      im->layout = kBitmapIndexed;
    }
    if (kind <= 3) {
      im->unpack = kBitmapAscii; im->ascii_channels = ch; im->ascii_bits = kind == 1; im->maxval = maxval;
      if (kind == 1) im->bits = 8;
      else { im->layout = kBitmapBytes; im->px_bytes = ch; im->sample_bytes = 1; im->channels = ch; }
      im->stride = (uint32_t)(W * ch);
      *plane_bytes = (W * H * ch + 15) & ~15ll;
    } else {
      const int sb = maxval > 255 ? 2 : 1;
      const int64_t pitch = kind == 4 ? (W + 7) / 8 : W * ch * sb;
      if (H * pitch > (int64_t)(n - begin)) return bad("truncated raster");
      end = begin + (size_t)(H * pitch);
      im->stride = (uint32_t)pitch;
      if (kind == 4) im->bits = 1;
      else { im->layout = kBitmapBytes; im->px_bytes = ch * sb; im->sample_bytes = sb; im->channels = ch; }
    }
    info->components = ch;
  }
  if (end - begin >= (1ull << 32)) return unsupported("image data of 4 GiB or more is not supported");
  im->plane_off = plane_base;
  im->raw_len = (uint32_t)(end - begin);
  info->stage_begin = begin; info->stage_end = end;
  info->width = (int)W; info->height = (int)H;
  return DALIB200_SUCCESS;
}

}  // namespace dalib200
#endif  // DALI_B200_CSRC_BITMAP_PLAN_H_
