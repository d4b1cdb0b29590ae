// dali_b200/csrc/tiff_plan.h -- host-side planning of a TIFF stream inside the image decoder plan: the walk of the first IFD, the
// validation of every tag the decode reads (type, count, offsets inside the stream), the segment table (one strip or tile of one plane
// each: its byte range, its decoded size), the ColorMap and the orientation.  No per-byte work on the image data beyond the first two
// bytes of each LZW segment (the old-style LZW test).  Plain C++ (no CUDA types): jpeg.cu calls it from JpegGetInfo / JpegPlanSetup,
// tools/emul/tiff_emul.cc from the CPU tests.
//
// Classic TIFF in either byte order, first IFD only (as cv2.imdecode).  Supported: strips or tiles, PlanarConfiguration 1 or 2;
// compression none (strips only), LZW (the MSB-first variant), Deflate (8 and 32946), PackBits; Predictor 1 or 2 (8- and 16-bit
// samples); MinIsWhite and MinIsBlack at 1/8/16 bits (one extra sample at 8 and 16; no 16-bit tiles without it), RGB at 8/16 bits with
// at most one extra sample, Palette at 1/4/8 bits.  Everything else is DALIB200_ERROR_UNSUPPORTED with a message; a malformed IFD or segment table is
// DALIB200_ERROR_BAD_DATA.
#ifndef DALI_B200_CSRC_TIFF_PLAN_H_
#define DALI_B200_CSRC_TIFF_PLAN_H_
#include <algorithm>
#include <cstring>
#include <string>
#include <vector>
#include "../../include/dali_b200.h"
#include "stream_info.h"
#include "tiff_core.h"

namespace dalib200 {

inline bool IsTiffStream(const uint8_t *p, size_t n) {
  return n >= 4 && (!memcmp(p, "II*\0", 4) || !memcmp(p, "MM\0*", 4) || !memcmp(p, "II+\0", 4) || !memcmp(p, "MM\0+", 4));
}

// OpenCV's validateInputImageSize (imgcodecs/src/loadsave.cpp): at most 2^20 pixels on a side and 2^30 pixels in all, by default.
// Every row size, segment size and pixel offset of tiff_core.h then stays inside 32 bits.
constexpr uint32_t kTiffMaxSide = 1u << 20;
constexpr uint64_t kTiffMaxPixels = 1ull << 30;
constexpr uint32_t kTiffMaxTile = 512;      // tile side allowed beyond the image's (rounded up to 16)

// Plans image `image`: its segments are appended to `segs`, offsets relative to stage_begin, decoded bytes from `dec_base` on in the
// scratch buffer (16-byte aligned each); *dec_bytes receives the image's decoded size.  The staged bytes, info->stage_begin ..
// stage_end, are the span of the segments.  Returns a DALIB200 status.
inline int PlanTiff(const uint8_t *p, size_t n, int image, TiffImage *im, std::vector<TiffSeg> &segs, int64_t dec_base, int64_t *dec_bytes,
                    StreamInfo *info, std::string *err) {
  auto fail = [&](int rc, const std::string &m) { if (err) *err = "TIFF: " + m; return rc; };
  auto bad = [&](const std::string &m) { return fail(DALIB200_ERROR_BAD_DATA, m); };
  auto unsupported = [&](const std::string &m) { return fail(DALIB200_ERROR_UNSUPPORTED, m); };
  if (!IsTiffStream(p, n)) return bad("missing header");
  if (p[2] == '+' || p[3] == '+') return unsupported("BigTIFF is not supported");
  const bool be = p[0] == 'M';
  auto u16 = [&](size_t o) -> uint32_t { return be ? (p[o] << 8) | p[o + 1] : (p[o + 1] << 8) | p[o]; };
  auto u32 = [&](size_t o) -> uint32_t {
    return be ? ((uint32_t)p[o] << 24) | ((uint32_t)p[o + 1] << 16) | ((uint32_t)p[o + 2] << 8) | p[o + 3]
              : ((uint32_t)p[o + 3] << 24) | ((uint32_t)p[o + 2] << 16) | ((uint32_t)p[o + 1] << 8) | p[o];
  };
  memset(im, 0, sizeof(*im));
  *info = StreamInfo();
  if (n < 8) return bad("truncated header");
  const uint32_t ifd = u32(4);
  if (ifd < 8 || (uint64_t)ifd + 2 > n) return bad("IFD offset outside the stream");
  const uint32_t nent = u16(ifd);
  if (nent == 0 || (uint64_t)ifd + 2 + 12ull * nent > n) return bad("IFD outside the stream");

  struct Tag { uint32_t type = 0, count = 0; size_t data = 0; bool present = false; };
  enum { kWidth, kHeight, kBps, kCompression, kPhotometric, kFillOrder, kStripOffsets, kOrientation, kSpp, kRowsPerStrip,
         kStripByteCounts, kPlanar, kPredictor, kColorMap, kTileWidth, kTileLength, kTileOffsets, kTileByteCounts, kExtraSamples,
         kSampleFormat, kNumTags };
  static const uint16_t kIds[kNumTags] = { 256, 257, 258, 259, 262, 266, 273, 274, 277, 278, 279, 284, 317, 320, 322, 323, 324, 325,
                                           338, 339 };
  Tag tags[kNumTags];
  for (uint32_t e = 0; e < nent; e++) {
    const size_t o = ifd + 2 + 12 * (size_t)e;
    const uint32_t id = u16(o);
    int t = -1;
    for (int k = 0; k < kNumTags; k++) if (kIds[k] == id) t = k;
    if (t < 0) continue;
    Tag &g = tags[t];
    g.type = u16(o + 2); g.count = u32(o + 4);
    if (g.type != 3 && g.type != 4) return bad("tag " + std::to_string(id) + " has type " + std::to_string(g.type) + " (SHORT or LONG expected)");
    const uint64_t bytes = (uint64_t)g.count * (g.type == 3 ? 2 : 4);
    if (g.count == 0) return bad("tag " + std::to_string(id) + " has no value");
    if (bytes <= 4) {
      g.data = o + 8;
    } else {
      g.data = u32(o + 8);
      if (g.data > n || bytes > n - g.data) return bad("values of tag " + std::to_string(id) + " lie outside the stream");
    }
    g.present = true;
  }
  auto val = [&](int t, uint32_t i) -> uint32_t { const Tag &g = tags[t]; return g.type == 3 ? u16(g.data + 2 * i) : u32(g.data + 4 * i); };
  auto one = [&](int t, uint32_t dflt) -> uint32_t { return tags[t].present ? val(t, 0) : dflt; };
  if (!tags[kWidth].present || !tags[kHeight].present) return bad("missing ImageWidth / ImageLength");
  const uint32_t W = val(kWidth, 0), H = val(kHeight, 0);
  if (W == 0 || H == 0) return bad("zero image size");
  if (W > kTiffMaxSide || H > kTiffMaxSide || (uint64_t)W * H > kTiffMaxPixels)
    return unsupported("images wider or taller than 2^20 pixels or larger than 2^30 pixels are not supported (OpenCV's limit)");
  const uint32_t spp = one(kSpp, 1);
  if (spp == 0) return bad("SamplesPerPixel is 0");
  const uint32_t bps = one(kBps, 1);
  if (tags[kBps].present) {
    if (tags[kBps].count < spp) return bad("BitsPerSample has fewer values than SamplesPerPixel");
    for (uint32_t i = 1; i < spp; i++) if (val(kBps, i) != bps) return unsupported("samples of different bit depths are not supported");
  }
  if (tags[kSampleFormat].present) {
    if (tags[kSampleFormat].count < spp) return bad("SampleFormat has fewer values than SamplesPerPixel");
    for (uint32_t i = 0; i < spp; i++) if (val(kSampleFormat, i) != 1) return unsupported("signed or floating-point samples are not supported");
  }
  const uint32_t compression = one(kCompression, 1);
  switch (compression) {
    case 1: case 5: case 8: case 32946: case 32773: break;
    case 6: case 7: return unsupported("JPEG compression is not supported");
    case 2: case 3: case 4: return unsupported("CCITT compression is not supported");
    case 34925: return unsupported("LZMA compression is not supported");
    case 50000: return unsupported("ZSTD compression is not supported");
    case 50001: return unsupported("WebP compression is not supported");
    default: return unsupported("compression " + std::to_string(compression) + " is not supported");
  }
  if (one(kFillOrder, 1) != 1) return unsupported("FillOrder 2 is not supported");
  // libtiff applies Predictor to LZW and Deflate only
  const uint32_t predictor = compression == 1 || compression == 32773 ? 1 : one(kPredictor, 1);
  if (predictor != 1 && predictor != 2) return unsupported("Predictor " + std::to_string(predictor) + " is not supported");
  if (predictor == 2 && bps != 8 && bps != 16) return unsupported("Predictor 2 is supported for 8- and 16-bit samples only");
  const uint32_t planar = one(kPlanar, 1);
  if (planar != 1 && planar != 2) return bad("bad PlanarConfiguration");
  if (!tags[kPhotometric].present) return unsupported("a stream without Photometric is not supported");
  const uint32_t photometric = val(kPhotometric, 0);
  const uint32_t nextra = tags[kExtraSamples].present ? tags[kExtraSamples].count : 0;
  bool ok = false;
  uint32_t colour = 1;
  if (photometric == kTiffMinIsWhite || photometric == kTiffMinIsBlack) {
    // 2- and 4-bit gray: cv2 4.13 rejects these streams
    ok = (spp == 1 && (bps == 1 || bps == 8 || bps == 16)) || (spp == 2 && (bps == 8 || bps == 16));
  } else if (photometric == kTiffRGB) {
    colour = 3;
    ok = (spp == 3 || spp == 4) && (bps == 8 || bps == 16);
  } else if (photometric == kTiffPalette) {
    ok = spp == 1 && (bps == 1 || bps == 4 || bps == 8);           // 2-bit palette: cv2 4.13 rejects it
  } else {
    return unsupported("Photometric " + std::to_string(photometric) + " is not supported (MinIsWhite, MinIsBlack, RGB, Palette)");
  }
  if (!ok) return unsupported("Photometric " + std::to_string(photometric) + " with " + std::to_string(spp) + " samples of " +
                              std::to_string(bps) + " bits is not supported");
  if (nextra > spp - colour) return bad("ExtraSamples names more samples than there are");
  // libtiff's RGBA reader premultiplies only an extra sample marked as unassociated alpha
  const bool premultiply = nextra >= 1 && val(kExtraSamples, 0) == 2;

  im->width = (int)W; im->height = (int)H; im->bps = (int)bps; im->spp = (int)spp; im->photometric = (int)photometric;
  im->planar = spp == 1 ? 1 : (int)planar; im->compression = compression == 32946 ? kTiffDeflate : (int)compression;
  im->predictor = (int)predictor; im->big_endian = be; im->premultiply = premultiply;
  if (photometric == kTiffPalette) {
    const uint32_t ne = 1u << bps;
    if (!tags[kColorMap].present || tags[kColorMap].type != 3 || tags[kColorMap].count != 3 * ne) return bad("missing or bad ColorMap");
    bool wide = false;                                      // libtiff: a map whose entries all lie below 256 is an 8-bit map
    for (uint32_t i = 0; i < 3 * ne; i++) if (val(kColorMap, i) >= 256) wide = true;
    for (uint32_t i = 0; i < ne; i++)
      for (int c = 0; c < 3; c++) { const uint32_t v = val(kColorMap, c * ne + i); im->pal[i][c] = (uint8_t)(wide ? v >> 8 : v); }
  }
  const int o = (int)one(kOrientation, 1);
  info->orientation = o >= 1 && o <= 8 ? o : 1;

  // segment table
  const bool tiled = tags[kTileWidth].present || tags[kTileLength].present || tags[kTileOffsets].present;
  const int ot = tiled ? kTileOffsets : kStripOffsets, ct = tiled ? kTileByteCounts : kStripByteCounts;
  uint32_t sw, sh;
  if (tiled) {
    if (!tags[kTileWidth].present || !tags[kTileLength].present) return bad("missing TileWidth / TileLength");
    sw = val(kTileWidth, 0); sh = val(kTileLength, 0);
    if (sw == 0 || sh == 0) return bad("bad tile size");
    // a tile wider or taller than the image (rounded up to 16, TIFF's tile granule) decodes only padding; beyond 512 pixels that lets
    // a stream of a few bytes claim gigabytes of decode scratch, so such tiles are refused
    if (sw > std::max(kTiffMaxTile, (W + 15) & ~15u) || sh > std::max(kTiffMaxTile, (H + 15) & ~15u))
      return unsupported("tiles larger than both the image and 512 pixels on a side are not supported");
    // cv2 4.13 rejects uncompressed tiles, and reads 16-bit gray tiles otherwise than libtiff's RGBA rules (not matched here)
    if (compression == 1) return unsupported("uncompressed tiles are not supported");
    if (bps == 16 && photometric != kTiffRGB && spp == 1) return unsupported("16-bit gray tiles are not supported");
  } else {
    sw = W; sh = one(kRowsPerStrip, 0xFFFFFFFFu);
    if (sh == 0) return bad("RowsPerStrip is 0");
    if (sh > H) sh = H;
  }
  const uint32_t planes = im->planar == 2 ? spp : 1;
  const uint64_t row_bytes = ((uint64_t)sw * (planes == 1 ? spp : 1) * bps + 7) / 8;
  if (row_bytes * sh >= (1ull << 31)) return unsupported("segments of 2 GiB or more are not supported");
  const uint32_t across = (W + sw - 1) / sw, down = (H + sh - 1) / sh;
  const uint64_t nseg = (uint64_t)across * down * planes;
  if (!tags[ot].present || !tags[ct].present) return bad(tiled ? "missing TileOffsets / TileByteCounts" : "missing StripOffsets / StripByteCounts");
  if (tags[ot].count != nseg || tags[ct].count != nseg) return bad("the segment table does not match the image layout");
  im->seg_w = (int)sw; im->seg_h = (int)sh; im->segs_across = (int)across; im->segs_per_plane = (int)(across * down);
  im->row_bytes = (uint32_t)row_bytes;
  const size_t first = segs.size();
  size_t lo = n, hi = 0;
  int64_t dec = 0;
  for (uint64_t k = 0; k < nseg; k++) {
    const uint32_t so = val(ot, (uint32_t)k), sl = val(ct, (uint32_t)k);
    if (so > n || sl > n - so) return bad("segment " + std::to_string(k) + " lies outside the stream");
    if (im->compression == kTiffLzw && sl >= 2 && p[so] == 0 && (p[so + 1] & 1)) return unsupported("old-style (LSB-first) LZW is not supported");
    TiffSeg s;
    s.off = so; s.len = sl; s.image = image;
    const uint32_t row0 = (uint32_t)((k % im->segs_per_plane) / across) * sh;
    s.rows = tiled ? sh : std::min(sh, H - row0);
    s.dec_off = dec_base + dec;
    dec += ((int64_t)s.rows * row_bytes + 15) & ~(int64_t)15;
    segs.push_back(s);
    if (sl) { lo = std::min(lo, (size_t)so); hi = std::max(hi, (size_t)so + sl); }
  }
  if (lo >= hi) lo = hi = 0;
  if (hi - lo >= (1ull << 32)) return unsupported("image data spanning 4 GiB or more is not supported");
  for (size_t k = first; k < segs.size(); k++) segs[k].off = segs[k].len ? segs[k].off - (uint32_t)lo : 0;
  im->seg_begin = (int)first; im->seg_end = (int)segs.size();
  *dec_bytes = dec;
  info->stage_begin = lo; info->stage_end = hi;
  info->width = (int)W; info->height = (int)H;
  info->components = photometric == kTiffPalette ? 3 : (int)spp;
  return DALIB200_SUCCESS;
}

}  // namespace dalib200
#endif  // DALI_B200_CSRC_TIFF_PLAN_H_
