// dali_b200/csrc/webp_core.h -- lossy WebP (VP8 key frame) decoding written once for device and host: the boolean decoder, the entropy
// decode of one image (webp_entropy), the reconstruction (webp_recon_mb) and loop filter (webp_filter_mb) of one macroblock, and the
// conversion of one output pixel (webp_pixel).
//
// Parity target: cv2.imdecode (OpenCV 4.13 / libwebp), i.e. libwebp's WebPDecodeBGRInto.  The functions restate libwebp's integer
// expressions (src/dec/vp8_dec.c, tree_dec.c, frame_dec.c, src/dsp/dec.c, upsampling.c, yuv.h), which for the VP8 stages are those of
// RFC 6386:
//   * entropy: libwebp's ParseIntraMode / ParseResiduals, including the int16 truncation of the dequantised coefficients and of the
//     inverse WHT, and its bit reader's end-of-data rule: the first read past a partition's end feeds one zero byte and sets `eof`,
//     which fails the image once the macroblock row is complete;
//   * reconstruction reads the UNFILTERED neighbours (libwebp keeps its own copy of the top samples from before the loop filter), with
//     127 above the first row, 129 left of the first column, and the top-right samples of a 4x4 block in column 3 taken from the
//     above-right macroblock's bottom row (the replicated last pixel on the right edge);
//   * out-of-range coefficients: the inverse DCT is libwebp's choice per block (frame_dec.c DoTransform / DoUVTransform).  A luma block
//     with a token past zigzag index 2, and all four blocks of a chroma plane in which any block has an AC token, take the full
//     transform, which cv2's x86 build runs in int16 SIMD lanes (dec_sse2.c Transform_SSE2): the vertical pass's outputs and the sums
//     in front of the final >> 3 wrap to int16.  The other blocks take TransformAC3 / TransformDC in int.  The two agree until the
//     dequantised coefficients near the int16 limit, i.e. at high quantizer indices (cv2 quality-100 streams re-quantised at 127);
//   * the loop filter is a separate pass over the finished planes, in libwebp's order per macroblock: left edge, inner vertical edges,
//     top edge, inner horizontal edges;
//   * colour: libwebp's fancy upsampler (UpsampleRgbLinePair) and VP8YUVToR/G/B; GRAY is cv2's BGR2GRAY of the colour decode.
// The same functions compiled by a host compiler are what tools/emul/webp_emul.cc runs to pin them against cv2 without a GPU.
#ifndef DALI_B200_CSRC_WEBP_CORE_H_
#define DALI_B200_CSRC_WEBP_CORE_H_
#include <stdint.h>
#include "host_device.h"

namespace dalib200 {

// intra modes, libwebp's numbering (the 16x16 and chroma modes are the first four)
enum WebpMode : int { kWebpDC = 0, kWebpTM = 1, kWebpVE = 2, kWebpHE = 3, kWebpRD = 4, kWebpVR = 5, kWebpLD = 6, kWebpVL = 7,
                      kWebpHD = 8, kWebpHU = 9 };

struct WebpBitState {          // a boolean decoder, as byte offsets into the image's staged bytes
  uint32_t pos, end;           // next byte, end of the partition
  uint32_t value, range;       // range is stored minus one (libwebp's range_)
  int32_t bits, eof;
};

struct WebpMb {                // one macroblock, written by webp_entropy
  uint32_t nz;                 // bit n: block n has a residual (0-15: Y in raster order, 16-19: U, 20-23: V)
  uint32_t wrap;               // bit n: block n takes libwebp's full inverse DCT, whose intermediate sums are int16 (webp_idct_add)
  uint8_t segment, i4, uvmode, inner;   // inner: the loop filter runs on the inner edges
  uint8_t modes[16];           // i4: the 4x4 modes in raster order; 16x16: modes[0]
};

struct WebpImage {
  int64_t raw_off;             // byte offset of the image's staged bytes: the VP8 chunk payload behind the 10-byte frame header
  int64_t coef_off, mb_off, plane_off, ctx_off;   // byte offsets of the image's ranges in the WebP scratch buffer
  int32_t sample;              // batch index (status word)
  int32_t width, height, mb_w, mb_h;
  int32_t nparts;              // 1, 2, 4 or 8 token partitions
  uint32_t part_off[8], part_len[8];
  WebpBitState br0;            // partition 0 at the first macroblock
  int32_t update_map, use_skip;
  uint8_t seg_p[3], skip_p;
  int16_t dq[4][6];            // per segment: Y1 DC, Y1 AC, Y2 DC, Y2 AC, UV DC, UV AC
  int32_t filter_type;         // 0 none, 1 simple, 2 normal
  uint8_t f_limit[4][2], f_ilevel[4][2], f_hev[4][2];   // per segment and 16x16 / 4x4 (libwebp's fstrengths_)
  uint8_t proba[4][8][3][11];  // token probabilities after the frame's updates
  // output, filled at launch: the window [win_x0, win_x0 + win_w) x [win_y0, win_y0 + win_h) of the image goes to `out` as a tight
  // win_h x win_w x C buffer, C = 1 for GRAY (cv2 IMREAD_GRAYSCALE), 3 for RGB / BGR (IMREAD_COLOR)
  uint8_t *out;
  int32_t win_x0, win_y0, win_w, win_h, out_type;
  int64_t first_px;            // prefix of window pixels over the WebP images (webp_color's sample search)
};

// the padded planes of an image: Y (16 mb_w x 16 mb_h), then U and V (8 mb_w x 8 mb_h each)
DB_HD uint8_t *webp_plane(const WebpImage &im, uint8_t *scratch, int c) {
  uint8_t *y = scratch + im.plane_off;
  const int64_t ny = (int64_t)im.mb_w * im.mb_h * 256;
  return c == 0 ? y : y + ny + (c - 1) * (ny >> 2);
}

// ---------------------------------------------------------------------------------------------------------------------------------
// constants (RFC 6386; libwebp's numbering of the 4x4 modes)
#if defined(__CUDACC__)
#define WEBP_TABLE(T, name, ...) __device__ const T d_##name __VA_ARGS__; static const T h_##name __VA_ARGS__;
#else
#define WEBP_TABLE(T, name, ...) static const T h_##name __VA_ARGS__;
#endif
#if defined(__CUDA_ARCH__)
#define WEBP_T(name) d_##name
#else
#define WEBP_T(name) h_##name
#endif
WEBP_TABLE(uint8_t, webp_zigzag[16], = { 0, 1, 4, 8, 5, 2, 3, 6, 9, 12, 13, 10, 7, 11, 14, 15 })
WEBP_TABLE(uint8_t, webp_bands[17], = { 0, 1, 2, 3, 6, 4, 5, 6, 6, 6, 6, 6, 6, 6, 6, 7, 0 })
WEBP_TABLE(uint8_t, webp_cat[4][12], = { { 173, 148, 140, 0 }, { 176, 155, 140, 135, 0 }, { 180, 157, 141, 134, 130, 0 },
                                         { 254, 254, 243, 230, 196, 177, 153, 140, 133, 130, 129, 0 } })
WEBP_TABLE(int8_t, webp_ymodes4_tree[18], = { -kWebpDC, 1, -kWebpTM, 2, -kWebpVE, 3, 4, 6, -kWebpHE, 5, -kWebpRD, -kWebpVR, -kWebpLD, 7,
                                              -kWebpVL, 8, -kWebpHD, -kWebpHU })
// key-frame probabilities of the 4x4 modes, [top mode][left mode]
WEBP_TABLE(uint8_t, webp_bmodes_proba[10][10][9], = {
  { { 231, 120,  48,  89, 115, 113, 120, 152, 112 }, { 152, 179,  64, 126, 170, 118,  46,  70,  95 }, { 175,  69, 143,  80,  85,  82,  72, 155, 103 }, {  56,  58,  10, 171, 218, 189,  17,  13, 152 }, { 114,  26,  17, 163,  44, 195,  21,  10, 173 },
    { 121,  24,  80, 195,  26,  62,  44,  64,  85 }, { 144,  71,  10,  38, 171, 213, 144,  34,  26 }, { 170,  46,  55,  19, 136, 160,  33, 206,  71 }, {  63,  20,   8, 114, 114, 208,  12,   9, 226 }, {  81,  40,  11,  96, 182,  84,  29,  16,  36 } },
  { { 134, 183,  89, 137,  98, 101, 106, 165, 148 }, {  72, 187, 100, 130, 157, 111,  32,  75,  80 }, {  66, 102, 167,  99,  74,  62,  40, 234, 128 }, {  41,  53,   9, 178, 241, 141,  26,   8, 107 }, {  74,  43,  26, 146,  73, 166,  49,  23, 157 },
    {  65,  38, 105, 160,  51,  52,  31, 115, 128 }, { 104,  79,  12,  27, 217, 255,  87,  17,   7 }, {  87,  68,  71,  44, 114,  51,  15, 186,  23 }, {  47,  41,  14, 110, 182, 183,  21,  17, 194 }, {  66,  45,  25, 102, 197, 189,  23,  18,  22 } },
  { {  88,  88, 147, 150,  42,  46,  45, 196, 205 }, {  43,  97, 183, 117,  85,  38,  35, 179,  61 }, {  39,  53, 200,  87,  26,  21,  43, 232, 171 }, {  56,  34,  51, 104, 114, 102,  29,  93,  77 }, {  39,  28,  85, 171,  58, 165,  90,  98,  64 },
    {  34,  22, 116, 206,  23,  34,  43, 166,  73 }, { 107,  54,  32,  26,  51,   1,  81,  43,  31 }, {  68,  25, 106,  22,  64, 171,  36, 225, 114 }, {  34,  19,  21, 102, 132, 188,  16,  76, 124 }, {  62,  18,  78,  95,  85,  57,  50,  48,  51 } },
  { { 193, 101,  35, 159, 215, 111,  89,  46, 111 }, {  60, 148,  31, 172, 219, 228,  21,  18, 111 }, { 112, 113,  77,  85, 179, 255,  38, 120, 114 }, {  40,  42,   1, 196, 245, 209,  10,  25, 109 }, {  88,  43,  29, 140, 166, 213,  37,  43, 154 },
    {  61,  63,  30, 155,  67,  45,  68,   1, 209 }, { 100,  80,   8,  43, 154,   1,  51,  26,  71 }, { 142,  78,  78,  16, 255, 128,  34, 197, 171 }, {  41,  40,   5, 102, 211, 183,   4,   1, 221 }, {  51,  50,  17, 168, 209, 192,  23,  25,  82 } },
  { { 138,  31,  36, 171,  27, 166,  38,  44, 229 }, {  67,  87,  58, 169,  82, 115,  26,  59, 179 }, {  63,  59,  90, 180,  59, 166,  93,  73, 154 }, {  40,  40,  21, 116, 143, 209,  34,  39, 175 }, {  47,  15,  16, 183,  34, 223,  49,  45, 183 },
    {  46,  17,  33, 183,   6,  98,  15,  32, 183 }, {  57,  46,  22,  24, 128,   1,  54,  17,  37 }, {  65,  32,  73, 115,  28, 128,  23, 128, 205 }, {  40,   3,   9, 115,  51, 192,  18,   6, 223 }, {  87,  37,   9, 115,  59,  77,  64,  21,  47 } },
  { { 104,  55,  44, 218,   9,  54,  53, 130, 226 }, {  64,  90,  70, 205,  40,  41,  23,  26,  57 }, {  54,  57, 112, 184,   5,  41,  38, 166, 213 }, {  30,  34,  26, 133, 152, 116,  10,  32, 134 }, {  39,  19,  53, 221,  26, 114,  32,  73, 255 },
    {  31,   9,  65, 234,   2,  15,   1, 118,  73 }, {  75,  32,  12,  51, 192, 255, 160,  43,  51 }, {  88,  31,  35,  67, 102,  85,  55, 186,  85 }, {  56,  21,  23, 111,  59, 205,  45,  37, 192 }, {  55,  38,  70, 124,  73, 102,   1,  34,  98 } },
  { { 125,  98,  42,  88, 104,  85, 117, 175,  82 }, {  95,  84,  53,  89, 128, 100, 113, 101,  45 }, {  75,  79, 123,  47,  51, 128,  81, 171,   1 }, {  57,  17,   5,  71, 102,  57,  53,  41,  49 }, {  38,  33,  13, 121,  57,  73,  26,   1,  85 },
    {  41,  10,  67, 138,  77, 110,  90,  47, 114 }, { 115,  21,   2,  10, 102, 255, 166,  23,   6 }, { 101,  29,  16,  10,  85, 128, 101, 196,  26 }, {  57,  18,  10, 102, 102, 213,  34,  20,  43 }, { 117,  20,  15,  36, 163, 128,  68,   1,  26 } },
  { { 102,  61,  71,  37,  34,  53,  31, 243, 192 }, {  69,  60,  71,  38,  73, 119,  28, 222,  37 }, {  68,  45, 128,  34,   1,  47,  11, 245, 171 }, {  62,  17,  19,  70, 146,  85,  55,  62,  70 }, {  37,  43,  37, 154, 100, 163,  85, 160,   1 },
    {  63,   9,  92, 136,  28,  64,  32, 201,  85 }, {  75,  15,   9,   9,  64, 255, 184, 119,  16 }, {  86,   6,  28,   5,  64, 255,  25, 248,   1 }, {  56,   8,  17, 132, 137, 255,  55, 116, 128 }, {  58,  15,  20,  82, 135,  57,  26, 121,  40 } },
  { { 164,  50,  31, 137, 154, 133,  25,  35, 218 }, {  51, 103,  44, 131, 131, 123,  31,   6, 158 }, {  86,  40,  64, 135, 148, 224,  45, 183, 128 }, {  22,  26,  17, 131, 240, 154,  14,   1, 209 }, {  45,  16,  21,  91,  64, 222,   7,   1, 197 },
    {  56,  21,  39, 155,  60, 138,  23, 102, 213 }, {  83,  12,  13,  54, 192, 255,  68,  47,  28 }, {  85,  26,  85,  85, 128, 128,  32, 146, 171 }, {  18,  11,   7,  63, 144, 171,   4,   4, 246 }, {  35,  27,  10, 146, 174, 171,  12,  26, 128 } },
  { { 190,  80,  35,  99, 180,  80, 126,  54,  45 }, {  85, 126,  47,  87, 176,  51,  41,  20,  32 }, { 101,  75, 128, 139, 118, 146, 116, 128,  85 }, {  56,  41,  15, 176, 236,  85,  37,   9,  62 }, {  71,  30,  17, 119, 118, 255,  17,  18, 138 },
    { 101,  38,  60, 138,  55,  70,  43,  26, 142 }, { 146,  36,  19,  30, 171, 255,  97,  27,  20 }, { 138,  45,  61,  62, 219,   1,  81, 188,  64 }, {  32,  41,  20, 117, 151, 142,  20,  21, 163 }, { 112,  19,  12,  61, 195, 128,  48,   4,  24 } }
})

// ---------------------------------------------------------------------------------------------------------------------------------
// The boolean decoder, as libwebp's VP8BitReader reading one byte at a time (its bulk loads change when bytes enter the value, not the
// bits decoded or when `eof` is set).  `range` is the range minus one.
struct WebpBits {
  const uint8_t *buf, *end;
  uint32_t value, range;
  int bits, eof;
};

DB_HD void webp_bits_load(WebpBits &b) {
  if (b.buf < b.end) { b.bits += 8; b.value = (b.value << 8) | *b.buf++; }
  else if (!b.eof) { b.value <<= 8; b.bits += 8; b.eof = 1; }
  else { b.bits = 0; }
}
DB_HD void webp_bits_init(WebpBits &b, const uint8_t *p, uint32_t n) {
  b.buf = p; b.end = p + n; b.value = 0; b.range = 254; b.bits = -8; b.eof = 0;
  webp_bits_load(b);
}
DB_HD int webp_log2_floor(uint32_t v) {
#if defined(__CUDA_ARCH__)
  return 31 - __clz(v);
#else
  return 31 - __builtin_clz(v);
#endif
}
DB_HD int webp_bit(WebpBits &b, int prob) {
  uint32_t range = b.range;
  if (b.bits < 0) webp_bits_load(b);
  const int pos = b.bits;
  const uint32_t split = (range * (uint32_t)prob) >> 8;
  const uint32_t value = b.value >> pos;
  const int bit = value > split;
  if (bit) { range -= split; b.value -= (split + 1) << pos; }
  else { range = split + 1; }
  const int shift = 7 ^ webp_log2_floor(range);
  range <<= shift;
  b.bits -= shift;
  b.range = range - 1;
  return bit;
}
// VP8GetSigned: the sign bit at probability 1/2, always one bit of shift (the range never is 255 here)
DB_HD int webp_signed(WebpBits &b, int v) {
  if (b.bits < 0) webp_bits_load(b);
  const int pos = b.bits;
  const uint32_t split = b.range >> 1;
  const uint32_t value = b.value >> pos;
  const int32_t mask = (int32_t)(split - value) >> 31;
  b.bits -= 1;
  b.range += (uint32_t)mask;
  b.range |= 1;
  b.value -= ((split + 1) & (uint32_t)mask) << pos;
  return (v ^ mask) - mask;
}
DB_HD uint32_t webp_value(WebpBits &b, int nbits) {
  uint32_t v = 0;
  while (nbits-- > 0) v |= (uint32_t)webp_bit(b, 0x80) << nbits;
  return v;
}
DB_HD int webp_signed_value(WebpBits &b, int nbits) {
  const int v = (int)webp_value(b, nbits);
  return webp_bit(b, 0x80) ? -v : v;
}

// ---------------------------------------------------------------------------------------------------------------------------------
// Entropy decode (libwebp GetCoeffsFast / GetLargeValue).  `bp`: the probabilities of one block type, [band][ctx][11].
DB_HD int webp_large_value(WebpBits &b, const uint8_t *p) {
  int v;
  if (!webp_bit(b, p[3])) {
    v = !webp_bit(b, p[4]) ? 2 : 3 + webp_bit(b, p[5]);
  } else if (!webp_bit(b, p[6])) {
    if (!webp_bit(b, p[7])) { v = 5 + webp_bit(b, 159); }
    else { v = 7 + 2 * webp_bit(b, 165); v += webp_bit(b, 145); }
  } else {
    const int bit1 = webp_bit(b, p[8]);
    const int bit0 = webp_bit(b, p[9 + bit1]);
    const int cat = 2 * bit1 + bit0;
    v = 0;
    for (const uint8_t *tab = WEBP_T(webp_cat)[cat]; *tab; ++tab) v += v + webp_bit(b, *tab);
    v += 3 + (8 << cat);
  }
  return v;
}
// Tokens of one block from coefficient n on into out[16] (zeroed by the caller).  Returns the index behind the last token.
DB_HD int webp_coeffs(WebpBits &b, const uint8_t *bp, int ctx, int dq0, int dq1, int n, int16_t *out) {
  const uint8_t *p = bp + (WEBP_T(webp_bands)[n] * 3 + ctx) * 11;
  for (; n < 16; ++n) {
    if (!webp_bit(b, p[0])) return n;
    while (!webp_bit(b, p[1])) {
      p = bp + WEBP_T(webp_bands)[++n] * 33;
      if (n == 16) return 16;
    }
    const uint8_t *pc = bp + WEBP_T(webp_bands)[n + 1] * 33;
    int v;
    if (!webp_bit(b, p[2])) { v = 1; p = pc + 11; }
    else { v = webp_large_value(b, p); p = pc + 22; }
    out[WEBP_T(webp_zigzag)[n]] = (int16_t)(webp_signed(b, v) * (n > 0 ? dq1 : dq0));
  }
  return 16;
}

// libwebp TransformWHT: the 16 luma DCs of a 16x16 macroblock from its Y2 block, into coefficient 0 of each 4x4 block
DB_HD void webp_wht(const int16_t *in, int16_t *out) {
  int tmp[16];
  for (int i = 0; i < 4; ++i) {
    const int a0 = in[0 + i] + in[12 + i], a1 = in[4 + i] + in[8 + i];
    const int a2 = in[4 + i] - in[8 + i], a3 = in[0 + i] - in[12 + i];
    tmp[0 + i] = a0 + a1; tmp[8 + i] = a0 - a1; tmp[4 + i] = a3 + a2; tmp[12 + i] = a3 - a2;
  }
  for (int i = 0; i < 4; ++i) {
    const int dc = tmp[0 + i * 4] + 3;
    const int a0 = dc + tmp[3 + i * 4], a1 = tmp[1 + i * 4] + tmp[2 + i * 4];
    const int a2 = tmp[1 + i * 4] - tmp[2 + i * 4], a3 = dc - tmp[3 + i * 4];
    out[0] = (int16_t)((a0 + a1) >> 3); out[16] = (int16_t)((a3 + a2) >> 3);
    out[32] = (int16_t)((a0 - a1) >> 3); out[48] = (int16_t)((a3 - a2) >> 3);
    out += 64;
  }
}

DB_HD void webp_bits_restore(WebpBits &b, const WebpBitState &s, const uint8_t *base) {
  b.buf = base + s.pos; b.end = base + s.end; b.value = s.value; b.range = s.range; b.bits = s.bits; b.eof = s.eof;
}

// Decodes every macroblock of one image, row by row: intra modes from partition 0, tokens from partition (row mod nparts).  Writes the
// macroblock records and the dequantised coefficients (384 per macroblock, zero-filled; not written for a skipped macroblock).
// `top`: mb_w words of per-column context (bits 0-15: the four 4x4 modes of the bottom row, 16-23: non-zero flags, 24: Y2 non-zero).
// Returns 0, or 1 when a partition ran out of data (libwebp: "Premature end-of-partition0" / "Premature end-of-file").
DB_HD int webp_entropy(const WebpImage &im, const uint8_t *raw, WebpMb *mbs, int16_t *coef, uint32_t *top) {
  const uint8_t *base = raw + im.raw_off;
  WebpBits br;
  webp_bits_restore(br, im.br0, base);
  WebpBits parts[8];
  for (int p = 0; p < im.nparts; p++) webp_bits_init(parts[p], base + im.part_off[p], im.part_len[p]);
  for (int x = 0; x < im.mb_w; x++) top[x] = 0;
  for (int mby = 0; mby < im.mb_h; mby++) {
    WebpBits tb = parts[mby & (im.nparts - 1)];
    uint32_t lmodes = 0, lnz = 0, lnz_dc = 0;              // left context: the four modes of the right column, non-zero flags
    for (int mbx = 0; mbx < im.mb_w; mbx++) {
      const int64_t m = (int64_t)mby * im.mb_w + mbx;
      uint32_t t = top[mbx];
      WebpMb mb;
      // ---- intra modes (libwebp ParseIntraMode)
      int seg = 0;
      if (im.update_map) seg = !webp_bit(br, im.seg_p[0]) ? webp_bit(br, im.seg_p[1]) : webp_bit(br, im.seg_p[2]) + 2;
      const int skip = im.use_skip ? webp_bit(br, im.skip_p) : 0;
      const int i4 = !webp_bit(br, 145);
      uint32_t tmodes = t & 0xFFFF;
      if (!i4) {
        const int ymode = webp_bit(br, 156) ? (webp_bit(br, 128) ? kWebpTM : kWebpHE) : (webp_bit(br, 163) ? kWebpVE : kWebpDC);
        mb.modes[0] = (uint8_t)ymode;
        for (int k = 1; k < 16; k++) mb.modes[k] = 0;
        tmodes = lmodes = (uint32_t)ymode * 0x1111u;
      } else {
        for (int yy = 0; yy < 4; ++yy) {
          int ymode = (lmodes >> (4 * yy)) & 15;
          for (int xx = 0; xx < 4; ++xx) {
            const uint8_t *prob = WEBP_T(webp_bmodes_proba)[(tmodes >> (4 * xx)) & 15][ymode];
            int i = WEBP_T(webp_ymodes4_tree)[webp_bit(br, prob[0])];
            while (i > 0) i = WEBP_T(webp_ymodes4_tree)[2 * i + webp_bit(br, prob[i])];
            ymode = -i;
            tmodes = (tmodes & ~(15u << (4 * xx))) | ((uint32_t)ymode << (4 * xx));
            mb.modes[4 * yy + xx] = (uint8_t)ymode;
          }
          lmodes = (lmodes & ~(15u << (4 * yy))) | ((uint32_t)ymode << (4 * yy));
        }
      }
      mb.uvmode = !webp_bit(br, 142) ? kWebpDC : !webp_bit(br, 114) ? kWebpVE : webp_bit(br, 183) ? kWebpTM : kWebpHE;
      mb.segment = (uint8_t)seg; mb.i4 = (uint8_t)i4;
      // ---- residuals (libwebp ParseResiduals)
      uint32_t tnz_all = (t >> 16) & 0xFF, tnz_dc = (t >> 24) & 1;
      uint32_t nzmask = 0, wrap = 0;
      if (!skip) {
        int16_t *dst = coef + m * 384;
        for (int k = 0; k < 384; k++) dst[k] = 0;
        const int16_t *q = im.dq[seg];
        const uint8_t *bands = &im.proba[0][0][0][0];
        int first;
        const uint8_t *ac_proba;
        if (!i4) {
          int16_t dc[16];
          for (int k = 0; k < 16; k++) dc[k] = 0;
          const int nz = webp_coeffs(tb, bands + 1 * 264, (int)(tnz_dc + lnz_dc), q[2], q[3], 0, dc);
          tnz_dc = lnz_dc = nz > 0;
          if (nz > 1) {
            webp_wht(dc, dst);
          } else {
            const int dc0 = (dc[0] + 3) >> 3;
            for (int k = 0; k < 256; k += 16) dst[k] = (int16_t)dc0;
          }
          first = 1;
          ac_proba = bands;
        } else {
          first = 0;
          ac_proba = bands + 3 * 264;
        }
        uint32_t tnz = tnz_all & 0x0f, lnzy = lnz & 0x0f;
        for (int y = 0; y < 4; ++y) {
          int l = lnzy & 1;
          for (int x = 0; x < 4; ++x) {
            const int ctx = l + (int)(tnz & 1);
            int16_t *blk = dst + (4 * y + x) * 16;
            const int nz = webp_coeffs(tb, ac_proba, ctx, q[0], q[1], first, blk);
            l = nz > first;
            tnz = (tnz >> 1) | ((uint32_t)l << 7);
            if (nz > 1 || blk[0] != 0) nzmask |= 1u << (4 * y + x);
            if (nz > 3) wrap |= 1u << (4 * y + x);              // libwebp's DoTransform: full transform past zigzag index 2
          }
          tnz >>= 4;
          lnzy = (lnzy >> 1) | ((uint32_t)l << 7);
        }
        uint32_t out_t = tnz, out_l = lnzy >> 4;
        for (int ch = 0; ch < 4; ch += 2) {
          uint32_t tc = tnz_all >> (4 + ch), lc = lnz >> (4 + ch);
          for (int y = 0; y < 2; ++y) {
            int l = lc & 1;
            for (int x = 0; x < 2; ++x) {
              const int ctx = l + (int)(tc & 1);
              const int b = 16 + 2 * ch + 2 * y + x;
              int16_t *blk = dst + b * 16;
              const int nz = webp_coeffs(tb, bands + 2 * 264, ctx, q[4], q[5], 0, blk);
              l = nz > 0;
              tc = (tc >> 1) | ((uint32_t)l << 3);
              if (nz > 1 || blk[0] != 0) nzmask |= 1u << b;
              if (nz > 1) wrap |= 0xFu << (16 + 2 * ch);   // libwebp's DoUVTransform: an AC coefficient sends all 4 blocks
            }
            tc >>= 2;
            lc = (lc >> 1) | ((uint32_t)l << 5);
          }
          out_t |= (tc << 4) << ch;
          out_l |= (lc & 0xf0) << ch;
        }
        tnz_all = out_t & 0xFF;
        lnz = out_l & 0xFF;
      } else {
        tnz_all = 0; lnz = 0;
        if (!i4) tnz_dc = lnz_dc = 0;
      }
      mb.nz = nzmask;
      mb.wrap = wrap;
      mb.inner = (uint8_t)(i4 || nzmask != 0);
      mbs[m] = mb;
      top[mbx] = tmodes | (tnz_all << 16) | (tnz_dc << 24);
    }
    parts[mby & (im.nparts - 1)] = tb;
    if (br.eof || tb.eof) return 1;
  }
  return 0;
}

// ---------------------------------------------------------------------------------------------------------------------------------
// Reconstruction (libwebp ReconstructRow): prediction from the unfiltered neighbours, then the inverse DCT added block by block.
DB_HD uint8_t webp_clip8(int v) { return (uint8_t)(v < 0 ? 0 : v > 255 ? 255 : v); }
DB_HD int webp_mul1(int a) { return ((a * 20091) >> 16) + a; }
DB_HD int webp_mul2(int a) { return (a * 35468) >> 16; }

// libwebp TransformOne / TransformAC3 / TransformDC: adds the inverse DCT of `in` to the 4x4 block at dst.  `wrap`: the block takes
// libwebp's full transform (VP8Transform), which cv2's x86 build runs as Transform_SSE2 in int16 lanes: each output of the vertical
// pass and each sum in front of the final >> 3 is truncated to int16.  Those wrap only for dequantised coefficients near the int16
// limit (high quantizer indices); below it both forms agree.  TransformAC3 and TransformDC run in int.
DB_HD int webp_wrap16(int v, bool wrap) { return wrap ? (int)(int16_t)v : v; }
DB_HD void webp_idct_add(const int16_t *in, uint8_t *dst, int stride, bool wrap) {
  int C[16];
  int *tmp = C;
  for (int i = 0; i < 4; ++i) {
    const int a = in[0] + in[8], b = in[0] - in[8];
    const int c = webp_mul2(in[4]) - webp_mul1(in[12]), d = webp_mul1(in[4]) + webp_mul2(in[12]);
    tmp[0] = webp_wrap16(a + d, wrap); tmp[1] = webp_wrap16(b + c, wrap);
    tmp[2] = webp_wrap16(b - c, wrap); tmp[3] = webp_wrap16(a - d, wrap);
    tmp += 4; in++;
  }
  tmp = C;
  for (int i = 0; i < 4; ++i) {
    const int dc = tmp[0] + 4;
    const int a = dc + tmp[8], b = dc - tmp[8];
    const int c = webp_mul2(tmp[4]) - webp_mul1(tmp[12]), d = webp_mul1(tmp[4]) + webp_mul2(tmp[12]);
    dst[0] = webp_clip8(dst[0] + (webp_wrap16(a + d, wrap) >> 3));
    dst[1] = webp_clip8(dst[1] + (webp_wrap16(b + c, wrap) >> 3));
    dst[2] = webp_clip8(dst[2] + (webp_wrap16(b - c, wrap) >> 3));
    dst[3] = webp_clip8(dst[3] + (webp_wrap16(a - d, wrap) >> 3));
    tmp++; dst += stride;
  }
}

DB_HD uint8_t webp_avg3(int a, int b, int c) { return (uint8_t)((a + 2 * b + c + 2) >> 2); }
DB_HD uint8_t webp_avg2(int a, int b) { return (uint8_t)((a + b + 1) >> 1); }

// libwebp's 4x4 predictors.  T[0]: top-left, T[1..8]: the 8 samples above (4 above, 4 above-right), L[0..3]: left.
DB_HD void webp_pred4(int mode, const uint8_t *T, const uint8_t *L, uint8_t *d /* 4x4, stride 4 */) {
  const int X = T[0], A = T[1], B = T[2], C = T[3], D = T[4], E = T[5], F = T[6], G = T[7], H = T[8];
  const int I = L[0], J = L[1], K = L[2], Lq = L[3];
#define DST(x, y) d[(x) + (y) * 4]
  switch (mode) {
    case kWebpDC: {
      uint32_t dc = 4;
      for (int i = 0; i < 4; ++i) dc += T[1 + i] + L[i];
      dc >>= 3;
      for (int i = 0; i < 16; ++i) d[i] = (uint8_t)dc;
      break;
    }
    case kWebpTM:
      for (int y = 0; y < 4; ++y) for (int x = 0; x < 4; ++x) DST(x, y) = webp_clip8(T[1 + x] + L[y] - X);
      break;
    case kWebpVE: {
      const uint8_t v[4] = { webp_avg3(X, A, B), webp_avg3(A, B, C), webp_avg3(B, C, D), webp_avg3(C, D, E) };
      for (int y = 0; y < 4; ++y) for (int x = 0; x < 4; ++x) DST(x, y) = v[x];
      break;
    }
    case kWebpHE: {
      const uint8_t v[4] = { webp_avg3(X, I, J), webp_avg3(I, J, K), webp_avg3(J, K, Lq), webp_avg3(K, Lq, Lq) };
      for (int y = 0; y < 4; ++y) for (int x = 0; x < 4; ++x) DST(x, y) = v[y];
      break;
    }
    case kWebpRD:
      DST(0, 3) = webp_avg3(J, K, Lq);
      DST(1, 3) = DST(0, 2) = webp_avg3(I, J, K);
      DST(2, 3) = DST(1, 2) = DST(0, 1) = webp_avg3(X, I, J);
      DST(3, 3) = DST(2, 2) = DST(1, 1) = DST(0, 0) = webp_avg3(A, X, I);
      DST(3, 2) = DST(2, 1) = DST(1, 0) = webp_avg3(B, A, X);
      DST(3, 1) = DST(2, 0) = webp_avg3(C, B, A);
      DST(3, 0) = webp_avg3(D, C, B);
      break;
    case kWebpLD:
      DST(0, 0) = webp_avg3(A, B, C);
      DST(1, 0) = DST(0, 1) = webp_avg3(B, C, D);
      DST(2, 0) = DST(1, 1) = DST(0, 2) = webp_avg3(C, D, E);
      DST(3, 0) = DST(2, 1) = DST(1, 2) = DST(0, 3) = webp_avg3(D, E, F);
      DST(3, 1) = DST(2, 2) = DST(1, 3) = webp_avg3(E, F, G);
      DST(3, 2) = DST(2, 3) = webp_avg3(F, G, H);
      DST(3, 3) = webp_avg3(G, H, H);
      break;
    case kWebpVR:
      DST(0, 0) = DST(1, 2) = webp_avg2(X, A);
      DST(1, 0) = DST(2, 2) = webp_avg2(A, B);
      DST(2, 0) = DST(3, 2) = webp_avg2(B, C);
      DST(3, 0) = webp_avg2(C, D);
      DST(0, 3) = webp_avg3(K, J, I);
      DST(0, 2) = webp_avg3(J, I, X);
      DST(0, 1) = DST(1, 3) = webp_avg3(I, X, A);
      DST(1, 1) = DST(2, 3) = webp_avg3(X, A, B);
      DST(2, 1) = DST(3, 3) = webp_avg3(A, B, C);
      DST(3, 1) = webp_avg3(B, C, D);
      break;
    case kWebpVL:
      DST(0, 0) = webp_avg2(A, B);
      DST(1, 0) = DST(0, 2) = webp_avg2(B, C);
      DST(2, 0) = DST(1, 2) = webp_avg2(C, D);
      DST(3, 0) = DST(2, 2) = webp_avg2(D, E);
      DST(0, 1) = webp_avg3(A, B, C);
      DST(1, 1) = DST(0, 3) = webp_avg3(B, C, D);
      DST(2, 1) = DST(1, 3) = webp_avg3(C, D, E);
      DST(3, 1) = DST(2, 3) = webp_avg3(D, E, F);
      DST(3, 2) = webp_avg3(E, F, G);
      DST(3, 3) = webp_avg3(F, G, H);
      break;
    case kWebpHD:
      DST(0, 0) = DST(2, 1) = webp_avg2(I, X);
      DST(0, 1) = DST(2, 2) = webp_avg2(J, I);
      DST(0, 2) = DST(2, 3) = webp_avg2(K, J);
      DST(0, 3) = webp_avg2(Lq, K);
      DST(3, 0) = webp_avg3(A, B, C);
      DST(2, 0) = webp_avg3(X, A, B);
      DST(1, 0) = DST(3, 1) = webp_avg3(I, X, A);
      DST(1, 1) = DST(3, 2) = webp_avg3(X, I, J);
      DST(1, 2) = DST(3, 3) = webp_avg3(I, J, K);
      DST(1, 3) = webp_avg3(J, K, Lq);
      break;
    default:  // kWebpHU
      DST(0, 0) = webp_avg2(I, J);
      DST(2, 0) = DST(0, 1) = webp_avg2(J, K);
      DST(2, 1) = DST(0, 2) = webp_avg2(K, Lq);
      DST(1, 0) = webp_avg3(I, J, K);
      DST(3, 0) = DST(1, 1) = webp_avg3(J, K, Lq);
      DST(3, 1) = DST(1, 2) = webp_avg3(K, Lq, Lq);
      DST(3, 2) = DST(2, 2) = DST(0, 3) = DST(1, 3) = DST(2, 3) = DST(3, 3) = (uint8_t)Lq;
      break;
  }
#undef DST
}

// 16x16 or 8x8 prediction into dst (libwebp's VP8PredLuma16 / VP8PredChroma8 after CheckMode: DC without top and / or left samples).
// top[0]: top-left, top[1..n]: above; left[0..n-1].
DB_HD void webp_pred_block(int mode, int n, int mbx, int mby, const uint8_t *top, const uint8_t *left, uint8_t *dst, int stride) {
  const int sh = n == 16 ? 4 : 3;
  int dc = 0;
  if (mode == kWebpDC) {
    int s = 0;
    if (mbx > 0 && mby > 0) {
      for (int i = 0; i < n; i++) s += top[1 + i] + left[i];
      dc = (s + n) >> (sh + 1);
    } else if (mby > 0) {
      for (int i = 0; i < n; i++) s += top[1 + i];
      dc = (s + (n >> 1)) >> sh;
    } else if (mbx > 0) {
      for (int i = 0; i < n; i++) s += left[i];
      dc = (s + (n >> 1)) >> sh;
    } else {
      dc = 0x80;
    }
  }
  for (int y = 0; y < n; y++) {
    uint8_t *row = dst + (int64_t)y * stride;
    for (int x = 0; x < n; x++) {
      row[x] = mode == kWebpDC ? (uint8_t)dc : mode == kWebpTM ? webp_clip8(top[1 + x] + left[y] - top[0])
             : mode == kWebpVE ? top[1 + x] : left[y];
    }
  }
}

// Reconstructs macroblock (mbx, mby) into the padded planes.  Reads the unfiltered left, top and top-right macroblocks: the caller
// orders the macroblocks so that (mbx - 1, mby), (mbx, mby - 1) and (mbx + 1, mby - 1) are complete.
DB_HD void webp_recon_mb(const WebpImage &im, const WebpMb *mbs, const int16_t *coef, uint8_t *scratch, int mbx, int mby) {
  const int64_t m = (int64_t)mby * im.mb_w + mbx;
  const WebpMb mb = mbs[m];
  const int16_t *c = coef + m * 384;
  // ---- luma
  {
    const int ys = 16 * im.mb_w;
    uint8_t *Y = webp_plane(im, scratch, 0) + (int64_t)16 * mby * ys + 16 * mbx;
    uint8_t top[21], left[16];                     // top[0]: top-left, [1..16]: above, [17..20]: above-right
    const uint8_t *up = Y - ys;
    top[0] = mby == 0 ? 127 : mbx == 0 ? 129 : up[-1];
    for (int i = 0; i < 16; i++) top[1 + i] = mby == 0 ? 127 : up[i];
    for (int i = 0; i < 4; i++) top[17 + i] = mby == 0 ? 127 : mbx == im.mb_w - 1 ? up[15] : up[16 + i];
    for (int j = 0; j < 16; j++) left[j] = mbx == 0 ? 129 : Y[(int64_t)j * ys - 1];
    if (!mb.i4) {
      webp_pred_block(mb.modes[0], 16, mbx, mby, top, left, Y, ys);
      for (int n = 0; n < 16; n++)
        if (mb.nz & (1u << n)) webp_idct_add(c + n * 16, Y + (int64_t)4 * (n >> 2) * ys + 4 * (n & 3), ys, (mb.wrap >> n) & 1);
    } else {
      for (int n = 0; n < 16; n++) {
        const int bx = 4 * (n & 3), by = 4 * (n >> 2);
        uint8_t *d = Y + (int64_t)by * ys + bx;
        uint8_t T[9], L[4], P[16];
        // samples of the macroblock's own pixels (already reconstructed), or its border
        T[0] = by == 0 ? top[bx] : bx == 0 ? left[by - 1] : d[-ys - 1];
        for (int i = 0; i < 4; i++) T[1 + i] = by == 0 ? top[1 + bx + i] : d[-ys + i];
        for (int i = 0; i < 4; i++) T[5 + i] = bx == 12 ? top[17 + i] : by == 0 ? top[5 + bx + i] : d[-ys + 4 + i];
        for (int j = 0; j < 4; j++) L[j] = bx == 0 ? left[by + j] : d[(int64_t)j * ys - 1];
        webp_pred4(mb.modes[n], T, L, P);
        for (int y = 0; y < 4; y++) for (int x = 0; x < 4; x++) d[(int64_t)y * ys + x] = P[4 * y + x];
        if (mb.nz & (1u << n)) webp_idct_add(c + n * 16, d, ys, (mb.wrap >> n) & 1);
      }
    }
  }
  // ---- chroma
  const int cs = 8 * im.mb_w;
  for (int ch = 1; ch <= 2; ch++) {
    uint8_t *U = webp_plane(im, scratch, ch) + (int64_t)8 * mby * cs + 8 * mbx;
    const uint8_t *up = U - cs;
    uint8_t top[9], left[8];
    top[0] = mby == 0 ? 127 : mbx == 0 ? 129 : up[-1];
    for (int i = 0; i < 8; i++) top[1 + i] = mby == 0 ? 127 : up[i];
    for (int j = 0; j < 8; j++) left[j] = mbx == 0 ? 129 : U[(int64_t)j * cs - 1];
    webp_pred_block(mb.uvmode, 8, mbx, mby, top, left, U, cs);
    for (int k = 0; k < 4; k++) {
      const int b = 16 + 4 * (ch - 1) + k;
      if (mb.nz & (1u << b)) webp_idct_add(c + b * 16, U + (int64_t)4 * (k >> 1) * cs + 4 * (k & 1), cs, (mb.wrap >> b) & 1);
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------------------------
// Loop filter (libwebp DoFilter and the dsp/dec.c filters), in place on the padded planes
DB_HD int webp_sclip1(int v) { return v < -128 ? -128 : v > 127 ? 127 : v; }
DB_HD int webp_sclip2(int v) { return v < -16 ? -16 : v > 15 ? 15 : v; }
DB_HD int webp_abs(int v) { return v < 0 ? -v : v; }

DB_HD void webp_do_filter2(uint8_t *p, int step) {
  const int p1 = p[-2 * step], p0 = p[-step], q0 = p[0], q1 = p[step];
  const int a = 3 * (q0 - p0) + webp_sclip1(p1 - q1);
  const int a1 = webp_sclip2((a + 4) >> 3), a2 = webp_sclip2((a + 3) >> 3);
  p[-step] = webp_clip8(p0 + a2);
  p[0] = webp_clip8(q0 - a1);
}
DB_HD void webp_do_filter4(uint8_t *p, int step) {
  const int p1 = p[-2 * step], p0 = p[-step], q0 = p[0], q1 = p[step];
  const int a = 3 * (q0 - p0);
  const int a1 = webp_sclip2((a + 4) >> 3), a2 = webp_sclip2((a + 3) >> 3);
  const int a3 = (a1 + 1) >> 1;
  p[-2 * step] = webp_clip8(p1 + a3);
  p[-step] = webp_clip8(p0 + a2);
  p[0] = webp_clip8(q0 - a1);
  p[step] = webp_clip8(q1 - a3);
}
DB_HD void webp_do_filter6(uint8_t *p, int step) {
  const int p2 = p[-3 * step], p1 = p[-2 * step], p0 = p[-step], q0 = p[0], q1 = p[step], q2 = p[2 * step];
  const int a = webp_sclip1(3 * (q0 - p0) + webp_sclip1(p1 - q1));
  const int a1 = (27 * a + 63) >> 7, a2 = (18 * a + 63) >> 7, a3 = (9 * a + 63) >> 7;
  p[-3 * step] = webp_clip8(p2 + a3);
  p[-2 * step] = webp_clip8(p1 + a2);
  p[-step] = webp_clip8(p0 + a1);
  p[0] = webp_clip8(q0 - a1);
  p[step] = webp_clip8(q1 - a2);
  p[2 * step] = webp_clip8(q2 - a3);
}
DB_HD bool webp_hev(const uint8_t *p, int step, int thresh) {
  const int p1 = p[-2 * step], p0 = p[-step], q0 = p[0], q1 = p[step];
  return webp_abs(p1 - p0) > thresh || webp_abs(q1 - q0) > thresh;
}
DB_HD bool webp_needs_filter(const uint8_t *p, int step, int t) {
  const int p1 = p[-2 * step], p0 = p[-step], q0 = p[0], q1 = p[step];
  return 4 * webp_abs(p0 - q0) + webp_abs(p1 - q1) <= t;
}
DB_HD bool webp_needs_filter2(const uint8_t *p, int step, int t, int it) {
  const int p3 = p[-4 * step], p2 = p[-3 * step], p1 = p[-2 * step], p0 = p[-step];
  const int q0 = p[0], q1 = p[step], q2 = p[2 * step], q3 = p[3 * step];
  if (4 * webp_abs(p0 - q0) + webp_abs(p1 - q1) > t) return false;
  return webp_abs(p3 - p2) <= it && webp_abs(p2 - p1) <= it && webp_abs(p1 - p0) <= it && webp_abs(q3 - q2) <= it &&
         webp_abs(q2 - q1) <= it && webp_abs(q1 - q0) <= it;
}
// simple filter across one edge of `size` pixels: hstride steps across the edge, vstride along it
DB_HD void webp_simple_edge(uint8_t *p, int hstride, int vstride, int thresh) {
  const int t2 = 2 * thresh + 1;
  for (int i = 0; i < 16; ++i, p += vstride)
    if (webp_needs_filter(p, hstride, t2)) webp_do_filter2(p, hstride);
}
// normal filter: 6-tap on macroblock edges (mb_edge), 4-tap on inner edges
DB_HD void webp_normal_edge(uint8_t *p, int hstride, int vstride, int size, int thresh, int ithresh, int hev_thresh, bool mb_edge) {
  const int t2 = 2 * thresh + 1;
  for (int i = 0; i < size; ++i, p += vstride) {
    if (!webp_needs_filter2(p, hstride, t2, ithresh)) continue;
    if (webp_hev(p, hstride, hev_thresh)) webp_do_filter2(p, hstride);
    else if (mb_edge) webp_do_filter6(p, hstride);
    else webp_do_filter4(p, hstride);
  }
}

// Filters macroblock (mbx, mby) in place.  The caller orders the macroblocks so that (mbx - 1, mby) and (mbx + 1, mby - 1) -- whose
// left edge wrote pixels this top edge reads -- are complete; two macroblocks on one diagonal mbx + 2 mby touch disjoint pixels.
DB_HD void webp_filter_mb(const WebpImage &im, const WebpMb *mbs, uint8_t *scratch, int mbx, int mby) {
  if (im.filter_type == 0) return;
  const WebpMb mb = mbs[(int64_t)mby * im.mb_w + mbx];
  const int limit = im.f_limit[mb.segment][mb.i4];
  if (limit == 0) return;
  const int ilevel = im.f_ilevel[mb.segment][mb.i4], hev = im.f_hev[mb.segment][mb.i4];
  const int ys = 16 * im.mb_w;
  uint8_t *y = webp_plane(im, scratch, 0) + (int64_t)16 * mby * ys + 16 * mbx;
  if (im.filter_type == 1) {
    if (mbx > 0) webp_simple_edge(y, 1, ys, limit + 4);
    if (mb.inner) for (int k = 4; k < 16; k += 4) webp_simple_edge(y + k, 1, ys, limit);
    if (mby > 0) webp_simple_edge(y, ys, 1, limit + 4);
    if (mb.inner) for (int k = 4; k < 16; k += 4) webp_simple_edge(y + (int64_t)k * ys, ys, 1, limit);
    return;
  }
  const int cs = 8 * im.mb_w;
  uint8_t *u = webp_plane(im, scratch, 1) + (int64_t)8 * mby * cs + 8 * mbx;
  uint8_t *v = webp_plane(im, scratch, 2) + (int64_t)8 * mby * cs + 8 * mbx;
  if (mbx > 0) {
    webp_normal_edge(y, 1, ys, 16, limit + 4, ilevel, hev, true);
    webp_normal_edge(u, 1, cs, 8, limit + 4, ilevel, hev, true);
    webp_normal_edge(v, 1, cs, 8, limit + 4, ilevel, hev, true);
  }
  if (mb.inner) {
    for (int k = 4; k < 16; k += 4) webp_normal_edge(y + k, 1, ys, 16, limit, ilevel, hev, false);
    webp_normal_edge(u + 4, 1, cs, 8, limit, ilevel, hev, false);
    webp_normal_edge(v + 4, 1, cs, 8, limit, ilevel, hev, false);
  }
  if (mby > 0) {
    webp_normal_edge(y, ys, 1, 16, limit + 4, ilevel, hev, true);
    webp_normal_edge(u, cs, 1, 8, limit + 4, ilevel, hev, true);
    webp_normal_edge(v, cs, 1, 8, limit + 4, ilevel, hev, true);
  }
  if (mb.inner) {
    for (int k = 4; k < 16; k += 4) webp_normal_edge(y + (int64_t)k * ys, ys, 1, 16, limit, ilevel, hev, false);
    webp_normal_edge(u + (int64_t)4 * cs, cs, 1, 8, limit, ilevel, hev, false);
    webp_normal_edge(v + (int64_t)4 * cs, cs, 1, 8, limit, ilevel, hev, false);
  }
}

// ---------------------------------------------------------------------------------------------------------------------------------
// One output pixel of the window (lx, ly): libwebp's fancy upsampling (UpsampleRgbLinePair, restated per pixel) and VP8YUVToR/G/B.
// Row r takes its chroma from the "near" chroma row with weight 3 and the "far" one with weight 1: row 0 and, for an even height, the
// last row use one chroma row for both.  Column 0 and, for an even width, the last column use one chroma column.
DB_HD int webp_mult_hi(int v, int coeff) { return (v * coeff) >> 8; }
DB_HD int webp_clip_yuv(int v) { return (v & ~16383) == 0 ? (v >> 6) : v < 0 ? 0 : 255; }

DB_HD void webp_pixel(const WebpImage &im, uint8_t *scratch, int lx, int ly) {
  const int x = im.win_x0 + lx, r = im.win_y0 + ly;
  const int W = im.width, H = im.height;
  const int ys = 16 * im.mb_w, cs = 8 * im.mb_w;
  const uint8_t *Y = webp_plane(im, scratch, 0), *U = webp_plane(im, scratch, 1), *V = webp_plane(im, scratch, 2);
  int near_row, far_row;
  if (r == 0) { near_row = far_row = 0; }
  else if (r & 1) { near_row = (r - 1) >> 1; far_row = r == H - 1 ? near_row : (r + 1) >> 1; }
  else { near_row = r >> 1; far_row = near_row - 1; }
  int cu, cv;
  const uint8_t *nu = U + (int64_t)near_row * cs, *fu = U + (int64_t)far_row * cs;
  const uint8_t *nv = V + (int64_t)near_row * cs, *fv = V + (int64_t)far_row * cs;
  if (x == 0 || (x == W - 1 && !(W & 1))) {
    const int j = x >> 1;
    cu = (3 * nu[j] + fu[j] + 2) >> 2;
    cv = (3 * nv[j] + fv[j] + 2) >> 2;
  } else {
    const int j = (x + 1) >> 1;                                   // chroma columns j - 1 and j
    const int au = nu[j - 1] + nu[j] + fu[j - 1] + fu[j] + 8, av = nv[j - 1] + nv[j] + fv[j - 1] + fv[j] + 8;
    if (x & 1) {
      cu = (((au + 2 * (nu[j] + fu[j - 1])) >> 3) + nu[j - 1]) >> 1;
      cv = (((av + 2 * (nv[j] + fv[j - 1])) >> 3) + nv[j - 1]) >> 1;
    } else {
      cu = (((au + 2 * (nu[j - 1] + fu[j])) >> 3) + nu[j]) >> 1;
      cv = (((av + 2 * (nv[j - 1] + fv[j])) >> 3) + nv[j]) >> 1;
    }
  }
  const int yy = Y[(int64_t)r * ys + x];
  const int R = webp_clip_yuv(webp_mult_hi(yy, 19077) + webp_mult_hi(cv, 26149) - 14234);
  const int G = webp_clip_yuv(webp_mult_hi(yy, 19077) - webp_mult_hi(cu, 6419) - webp_mult_hi(cv, 13320) + 8708);
  const int B = webp_clip_yuv(webp_mult_hi(yy, 19077) + webp_mult_hi(cu, 33050) - 17685);
  const int64_t o = (int64_t)ly * im.win_w + lx;
  if (im.out_type == 2 /* DALIB200_GRAY */) { im.out[o] = (uint8_t)((9798 * R + 19235 * G + 3735 * B + 16384) >> 15); return; }
  uint8_t *d = im.out + o * 3;
  if (im.out_type == 1 /* DALIB200_BGR */) { d[0] = (uint8_t)B; d[1] = (uint8_t)G; d[2] = (uint8_t)R; }
  else { d[0] = (uint8_t)R; d[1] = (uint8_t)G; d[2] = (uint8_t)B; }
}

}  // namespace dalib200
#endif  // DALI_B200_CSRC_WEBP_CORE_H_
