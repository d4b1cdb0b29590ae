// dali_b200/csrc/png_plan.h -- host-side planning of a PNG stream inside the image decoder plan: the chunk walk (headers only, no
// per-byte work on the image data), IHDR / PLTE validation, the eXIf orientation, the zlib header, and the (offset, length) of every
// IDAT payload.  Plain C++ (no CUDA types): jpeg.cu calls it from JpegGetInfo / JpegPlanSetup, tools/emul/png_emul.cc from the CPU
// tests.
//
// What is checked here follows what libpng (behind cv2.imdecode) rejects: a bad CRC of a critical chunk (IHDR, PLTE; the IDAT CRCs are
// checked on the device by png_crc), an unknown critical chunk, IDAT chunks that are not consecutive (libpng stops at the first gap and
// runs out of image data), a stream without IEND.  An ancillary chunk with a bad CRC is ignored, as libpng discards it; that matters
// only for eXIf, whose orientation cv2 applies wherever the chunk sits.
#ifndef DALI_B200_CSRC_PNG_PLAN_H_
#define DALI_B200_CSRC_PNG_PLAN_H_
#include <cstring>
#include <string>
#include <vector>
#include "../../include/dali_b200.h"
#include "exif.h"
#include "png_core.h"
#include "stream_info.h"

namespace dalib200 {

inline bool IsPngStream(const uint8_t *p, size_t n) { return n >= 8 && !memcmp(p, "\x89PNG\r\n\x1a\n", 8); }

inline uint32_t PngCrc32(const uint8_t *p, size_t n) {
  struct Table { uint32_t v[256]; };
  static const Table table = [] { Table t; for (uint32_t i = 0; i < 256; i++) t.v[i] = png_crc_table_entry(i); return t; }();
  uint32_t c = 0xFFFFFFFFu;
  for (size_t i = 0; i < n; i++) c = table.v[(c ^ p[i]) & 255] ^ (c >> 8);
  return c ^ 0xFFFFFFFFu;
}

// libpng's default user limit on either side (png_set_user_limits: PNG_USER_WIDTH_MAX / PNG_USER_HEIGHT_MAX): cv2 rejects larger images.
// It also keeps every row size and pixel offset of png_core.h far inside 32 bits.
constexpr uint32_t kPngMaxSide = 1000000;

// Plans image `image` (its chunks are appended to `chunks`, offsets relative to stage_begin).  The staged bytes, info->stage_begin ..
// stage_end, run from the first IDAT's type field to the last IDAT's CRC.  Returns a DALIB200 status.
inline int PlanPng(const uint8_t *p, size_t n, int image, PngImage *im, std::vector<PngChunk> &chunks, StreamInfo *info, std::string *err) {
  auto bad = [&](const char *m) { if (err) *err = std::string("PNG: ") + m; return DALIB200_ERROR_BAD_DATA; };
  auto be32 = [](const uint8_t *q) { return ((uint32_t)q[0] << 24) | ((uint32_t)q[1] << 16) | ((uint32_t)q[2] << 8) | q[3]; };
  if (!IsPngStream(p, n)) return bad("missing signature");
  memset(im, 0, sizeof(*im));
  *info = StreamInfo();
  const int first_chunk = (int)chunks.size();
  bool have_ihdr = false, have_iend = false;
  int idat_state = 0;                                   // 0: none yet, 1: in the IDAT run, 2: behind it
  int npal = 0;
  size_t pos = 8;
  while (pos + 12 <= n) {
    const uint32_t len = be32(p + pos);
    const uint8_t *type = p + pos + 4, *data = p + pos + 8;
    if (len > 0x7FFFFFFFu || len > n - pos - 12) return bad("truncated chunk");
    // the CRC of the chunks the planner reads (IHDR, PLTE, eXIf); the IDAT CRCs are the device's (png_crc), not a host pass over the data
    auto crc_ok = [&] { return PngCrc32(type, (size_t)len + 4) == be32(data + len); };
    if (!have_ihdr && memcmp(type, "IHDR", 4)) return bad("IHDR must be the first chunk");
    if (!memcmp(type, "IDAT", 4)) {
      if (idat_state == 2) return bad("IDAT chunks are not consecutive");
      if (idat_state == 0) { info->stage_begin = pos + 4; idat_state = 1; }
      PngChunk c;
      c.off = (uint32_t)(pos + 8 - info->stage_begin); c.len = len; c.image = image;
      chunks.push_back(c);
      info->stage_end = pos + 12 + len;
      if (info->stage_end - info->stage_begin >= (1ull << 32)) return bad("image data exceeds 4 GiB");
    } else {
      if (idat_state == 1) idat_state = 2;
      if (!memcmp(type, "IHDR", 4)) {
        if (have_ihdr) return bad("second IHDR");
        if (len != 13 || !crc_ok()) return bad("bad IHDR");
        const uint32_t w = be32(data), h = be32(data + 4);
        const int depth = data[8], ct = data[9];
        if (w == 0 || h == 0 || w > 0x7FFFFFFFu || h > 0x7FFFFFFFu) return bad("bad image size");
        if (w > kPngMaxSide || h > kPngMaxSide) {
          if (err) *err = "PNG: images wider or taller than 1000000 pixels are not supported (libpng's limit)";
          return DALIB200_ERROR_UNSUPPORTED;
        }
        const bool legal = (ct == kPngGray && (depth == 1 || depth == 2 || depth == 4 || depth == 8 || depth == 16)) ||
                           (ct == kPngPalette && (depth == 1 || depth == 2 || depth == 4 || depth == 8)) ||
                           ((ct == kPngRGB || ct == kPngGrayAlpha || ct == kPngRGBA) && (depth == 8 || depth == 16));
        if (!legal) return bad("illegal bit depth / colour type");
        if (data[10] != 0 || data[11] != 0 || data[12] > 1) return bad("unknown compression, filter or interlace method");
        if ((uint64_t)w * h >= (1ull << 31)) {
          if (err) *err = "PNG: images of 2^31 pixels or more are not supported";
          return DALIB200_ERROR_UNSUPPORTED;
        }
        im->width = (int)w; im->height = (int)h; im->depth = depth; im->ctype = ct; im->interlace = data[12];
        im->spp = ct == kPngRGB ? 3 : ct == kPngGrayAlpha ? 2 : ct == kPngRGBA ? 4 : 1;
        have_ihdr = true;
      } else if (!memcmp(type, "PLTE", 4)) {
        if (!crc_ok()) return bad("PLTE CRC error");
        if (im->ctype == kPngPalette) {
          if (len % 3 || len == 0 || len > 768) return bad("invalid palette length");
          npal = (int)len / 3;
          memcpy(im->pal, data, len);
        }
      } else if (!memcmp(type, "eXIf", 4)) {
        if (crc_ok()) info->orientation = ParseExifOrientation(data, (int)len);
      } else if (!memcmp(type, "IEND", 4)) {
        have_iend = true;
        break;
      } else if (!(type[0] & 0x20)) {
        return bad("unknown critical chunk");
      }
    }
    pos += 12 + (size_t)len;
  }
  if (!have_ihdr) return bad("no IHDR");
  if (!have_iend) return bad("no IEND (truncated stream)");
  if (idat_state == 0) return bad("no IDAT");
  if (im->ctype == kPngPalette && npal == 0) return bad("missing PLTE");
  // zlib header (RFC 1950): deflate, window <= 32 KiB, check bits, no preset dictionary -- the first two bytes of the IDAT data
  uint8_t zh[2];
  int got = 0;
  for (size_t k = first_chunk; k < chunks.size() && got < 2; k++)
    for (uint32_t i = 0; i < chunks[k].len && got < 2; i++) zh[got++] = p[info->stage_begin + chunks[k].off + i];
  if (got < 2) return bad("IDAT data ends inside the zlib header");
  if (!zlib_header_ok(zh[0], zh[1])) return bad("bad zlib header");
  // scanline layout, pass by pass
  int64_t off = 0;
  for (int ps = 0; ps < (im->interlace ? 7 : 1); ps++) {
    int x0, y0, dx, dy;
    png_pass_geom(im->interlace, ps, x0, y0, dx, dy);
    const int64_t pw = im->width > x0 ? (im->width - x0 + dx - 1) / dx : 0, ph = im->height > y0 ? (im->height - y0 + dy - 1) / dy : 0;
    im->pass_off[ps] = off;
    if (pw == 0 || ph == 0) continue;
    im->pass_row[ps] = (int32_t)(1 + (pw * im->spp * im->depth + 7) / 8);
    off += ph * im->pass_row[ps];
  }
  im->scan_bytes = off;
  im->chunk_begin = first_chunk; im->chunk_end = (int)chunks.size();
  info->width = im->width; info->height = im->height;
  info->components = im->ctype == kPngPalette ? 3 : im->spp;
  return DALIB200_SUCCESS;
}

}  // namespace dalib200
#endif  // DALI_B200_CSRC_PNG_PLAN_H_
