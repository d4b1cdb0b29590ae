// dali_b200/csrc/jpeg_distort_core.h -- the encode half of fn.jpeg_compression_distortion, written once for device and host: RGB ->
// YCbCr, 2x2 chroma downsampling, islow forward DCT and quantisation of one MCU strip into the decoder's coefficient layout.
//
// Parity target: cv2.imencode(".jpg", IMWRITE_JPEG_QUALITY q) (libjpeg-turbo, 8-bit, 4:2:0, islow) followed by cv2.imdecode.  The
// decoded pixels depend only on the quantised DCT coefficients, so no entropy coder is needed: these functions restate
//   * jccolor.c rgb_ycc_convert (SCALEBITS 16; Cb / Cr round with 2^15 - 1);
//   * jcprepct.c / jcsample.c h2v2_downsample + expand_right_edge: luma row and column indices clamp to the image; chroma is the mean of
//     2x2 pixels with the bias 1, 2, 1, 2, ... along a row, its pixel rows padded to an even count with the last one and its pixel
//     columns clamped to W - 1; chroma rows at or beyond ceil(H / 2) repeat chroma row ceil(H / 2) - 1;
//   * jfdctint.c jpeg_fdct_islow on samples centred by 128 (CONST_BITS 13, PASS1_BITS 2);
//   * jcdctmgr.c quantize: (c + d / 2) / d with d = 8 q, by magnitude;
//   * jccoefct.c compress_data's dummy blocks: a luma block right of the last real block column is zero with the DC of its left
//     neighbour, a luma block row below the last real one is zero with the DC of the MCU's block above-right (Y01).
// The coefficients go to the arenas the decoder's reconstruct kernels read (jpeg_recon.h): MCU order, blocks Y00 Y01 Y10 Y11 Cb Cr,
// natural order in each block, and the absolute DC of every block in the compact DC array.
// The same functions compiled by a host compiler are what tools/emul/jpeg_distort_emul.cc runs to pin them against cv2 without a GPU.
#ifndef DALI_B200_CSRC_JPEG_DISTORT_CORE_H_
#define DALI_B200_CSRC_JPEG_DISTORT_CORE_H_
#include <stdint.h>
#include "jpeg_recon.h"
#include "host_device.h"

namespace dalib200 {

constexpr int kJdMcus = 16;                  // MCU columns per strip: one CTA transforms one MCU row of a strip
constexpr int kJdThreads = 128;              // >= 6 * kJdMcus blocks: one forward DCT per thread
constexpr int kJdStripW = 16 * kJdMcus;      // luma columns of a strip

struct JdImage {
  const uint8_t *in;                         // HWC RGB u8, filled at launch
  int32_t width, height, mcux, mcuy;
  int32_t quant_set;                         // QuantSet: q[0] luma, q[1] chroma
  int32_t strips_x;                          // strips per MCU row
  int64_t blk0;                              // first block of the image in the coefficient / DC arenas
};

// one strip's samples (shared memory on the device): luma rows 16 my .. 16 my + 15, chroma rows 8 my .. 8 my + 7
struct JdStrip {
  alignas(16) uint8_t y[16][kJdStripW];
  alignas(16) uint8_t c[2][8][kJdStripW / 2];
  int32_t dc[kJdMcus][4];                    // quantised DC of the real luma blocks (for the dummy blocks)
};

DB_HD void jd_rgb_ycc(int r, int g, int b, int &y, int &cb, int &cr) {
  y = (19595 * r + 38470 * g + 7471 * b + 32768) >> 16;
  cb = (-11059 * r - 21709 * g + 32768 * b + (128 << 16) + 32767) >> 16;
  cr = (32768 * r - 27439 * g - 5329 * b + (128 << 16) + 32767) >> 16;
}

// strip li of image im: MCU row my, first MCU column mx0, nt MCU columns
DB_HD void jd_strip(const JdImage &im, int64_t li, int &my, int &mx0, int &nt) {
  my = (int)(li / im.strips_x);
  mx0 = (int)(li - (int64_t)my * im.strips_x) * kJdMcus;
  nt = im.mcux - mx0 < kJdMcus ? im.mcux - mx0 : kJdMcus;
}

// 2x2 pixel quad e (row-major over 8 x 8 nt quads) of the strip: its four luma samples and one chroma sample of each component
DB_HD void jd_convert_quad(const JdImage &im, int my, int mx0, int nt, int e, JdStrip &t) {
  const int W = im.width, H = im.height, qw = 8 * nt;
  const int qy = e / qw, qx = e - qy * qw;
  const int x0 = 16 * mx0 + 2 * qx, y0 = 16 * my + 2 * qy;
  const int xa = x0 < W - 1 ? x0 : W - 1, xb = x0 + 1 < W - 1 ? x0 + 1 : W - 1;
  int ya = y0 < H - 1 ? y0 : H - 1, yb = y0 + 1 < H - 1 ? y0 + 1 : H - 1;
  const uint8_t *in = im.in;
  int cs[2] = { 0, 0 };
  for (int pass = 0; pass < 2; pass++) {
    const uint8_t *ra = in + ((int64_t)ya * W) * 3, *rb = in + ((int64_t)yb * W) * 3;
    int yv[4], cbv[4], crv[4];
    jd_rgb_ycc(ra[3 * xa], ra[3 * xa + 1], ra[3 * xa + 2], yv[0], cbv[0], crv[0]);
    jd_rgb_ycc(ra[3 * xb], ra[3 * xb + 1], ra[3 * xb + 2], yv[1], cbv[1], crv[1]);
    jd_rgb_ycc(rb[3 * xa], rb[3 * xa + 1], rb[3 * xa + 2], yv[2], cbv[2], crv[2]);
    jd_rgb_ycc(rb[3 * xb], rb[3 * xb + 1], rb[3 * xb + 2], yv[3], cbv[3], crv[3]);
    if (pass == 0) {
      t.y[2 * qy][2 * qx] = (uint8_t)yv[0]; t.y[2 * qy][2 * qx + 1] = (uint8_t)yv[1];
      t.y[2 * qy + 1][2 * qx] = (uint8_t)yv[2]; t.y[2 * qy + 1][2 * qx + 1] = (uint8_t)yv[3];
    }
    cs[0] = cbv[0] + cbv[1] + cbv[2] + cbv[3];
    cs[1] = crv[0] + crv[1] + crv[2] + crv[3];
    // chroma rows at or beyond ceil(H / 2) repeat the last real one, whose pixel rows differ from the clamped luma rows
    const int ch = (H + 1) >> 1, ci = 8 * my + qy;
    if (pass == 1 || ci < ch) break;
    ya = 2 * (ch - 1); yb = ya + 1 < H - 1 ? ya + 1 : H - 1;
  }
  const int bias = 1 + (qx & 1);             // the chroma column 8 mx0 + qx has the parity of qx
  t.c[0][qy][qx] = (uint8_t)((cs[0] + bias) >> 2);
  t.c[1][qy][qx] = (uint8_t)((cs[1] + bias) >> 2);
}

// jpeg_fdct_islow + quantize of the 8 x 8 samples at src (row pitch `pitch`, 8-byte aligned rows); out: 64 coefficients, natural order
DB_HD void jd_fdct_quant(const uint8_t *src, int pitch, const uint16_t *q, int *out) {
  int d[64];
#pragma unroll
  for (int r = 0; r < 8; r++) {              // pass 1: rows
    const uint64_t w = *reinterpret_cast<const uint64_t *>(src + r * pitch);
    int s[8];
#pragma unroll
    for (int k = 0; k < 8; k++) s[k] = (int)((w >> (8 * k)) & 0xFF) - 128;
    int tmp0 = s[0] + s[7], tmp7 = s[0] - s[7], tmp1 = s[1] + s[6], tmp6 = s[1] - s[6];
    int tmp2 = s[2] + s[5], tmp5 = s[2] - s[5], tmp3 = s[3] + s[4], tmp4 = s[3] - s[4];
    const int tmp10 = tmp0 + tmp3, tmp13 = tmp0 - tmp3, tmp11 = tmp1 + tmp2, tmp12 = tmp1 - tmp2;
    int *o = d + 8 * r;
    o[0] = (tmp10 + tmp11) * 4;
    o[4] = (tmp10 - tmp11) * 4;
    int z1 = (tmp12 + tmp13) * 4433;
    o[2] = (z1 + tmp13 * 6270 + (1 << 10)) >> 11;
    o[6] = (z1 - tmp12 * 15137 + (1 << 10)) >> 11;
    z1 = tmp4 + tmp7;
    int z2 = tmp5 + tmp6, z3 = tmp4 + tmp6, z4 = tmp5 + tmp7;
    const int z5 = (z3 + z4) * 9633;
    tmp4 *= 2446; tmp5 *= 16819; tmp6 *= 25172; tmp7 *= 12299;
    z1 *= -7373; z2 *= -20995; z3 *= -16069; z4 *= -3196;
    z3 += z5; z4 += z5;
    o[7] = (tmp4 + z1 + z3 + (1 << 10)) >> 11;
    o[5] = (tmp5 + z2 + z4 + (1 << 10)) >> 11;
    o[3] = (tmp6 + z2 + z3 + (1 << 10)) >> 11;
    o[1] = (tmp7 + z1 + z4 + (1 << 10)) >> 11;
  }
#pragma unroll
  for (int c = 0; c < 8; c++) {              // pass 2: columns
    int *o = d + c;
    int tmp0 = o[0] + o[56], tmp7 = o[0] - o[56], tmp1 = o[8] + o[48], tmp6 = o[8] - o[48];
    int tmp2 = o[16] + o[40], tmp5 = o[16] - o[40], tmp3 = o[24] + o[32], tmp4 = o[24] - o[32];
    const int tmp10 = tmp0 + tmp3, tmp13 = tmp0 - tmp3, tmp11 = tmp1 + tmp2, tmp12 = tmp1 - tmp2;
    o[0] = (tmp10 + tmp11 + 2) >> 2;
    o[32] = (tmp10 - tmp11 + 2) >> 2;
    int z1 = (tmp12 + tmp13) * 4433;
    o[16] = (z1 + tmp13 * 6270 + (1 << 14)) >> 15;
    o[48] = (z1 - tmp12 * 15137 + (1 << 14)) >> 15;
    z1 = tmp4 + tmp7;
    int z2 = tmp5 + tmp6, z3 = tmp4 + tmp6, z4 = tmp5 + tmp7;
    const int z5 = (z3 + z4) * 9633;
    tmp4 *= 2446; tmp5 *= 16819; tmp6 *= 25172; tmp7 *= 12299;
    z1 *= -7373; z2 *= -20995; z3 *= -16069; z4 *= -3196;
    z3 += z5; z4 += z5;
    o[56] = (tmp4 + z1 + z3 + (1 << 14)) >> 15;
    o[40] = (tmp5 + z2 + z4 + (1 << 14)) >> 15;
    o[24] = (tmp6 + z2 + z3 + (1 << 14)) >> 15;
    o[8] = (tmp7 + z1 + z4 + (1 << 14)) >> 15;
  }
#pragma unroll
  for (int k = 0; k < 64; k++) {
    const uint32_t dv = 8u * q[k], a = (uint32_t)(d[k] < 0 ? -d[k] : d[k]);
    const int v = (int)((a + (dv >> 1)) / dv);
    out[k] = d[k] < 0 ? -v : v;
  }
}

DB_HD void jd_store_block(int16_t *dst, const int *c) {
#if defined(__CUDA_ARCH__)
  uint4 *d4 = reinterpret_cast<uint4 *>(dst);
#pragma unroll
  for (int r = 0; r < 8; r++) {
    const int *v = c + 8 * r;
    d4[r] = make_uint4((uint32_t)(v[0] & 0xFFFF) | ((uint32_t)v[1] << 16), (uint32_t)(v[2] & 0xFFFF) | ((uint32_t)v[3] << 16),
                       (uint32_t)(v[4] & 0xFFFF) | ((uint32_t)v[5] << 16), (uint32_t)(v[6] & 0xFFFF) | ((uint32_t)v[7] << 16));
  }
#else
  for (int k = 0; k < 64; k++) dst[k] = (int16_t)c[k];
#endif
}

// Block j (MCU j / 6 of the strip, block j % 6 of the MCU) of the strip.  pass 0 transforms the real blocks and records the luma DCs
// in t.dc; pass 1 (after every pass-0 block of the strip) writes the dummy blocks from them.
DB_HD void jd_block(const JdImage &im, const QuantSet &qs, int my, int mx0, int j, int pass, JdStrip &t, int16_t *coef, int16_t *dc) {
  const int m = j / 6, b = j - 6 * m;
  const int64_t gb = im.blk0 + ((int64_t)my * im.mcux + mx0 + m) * 6 + b;
  const int wb = (im.width + 7) >> 3, hb = (im.height + 7) >> 3;      // real luma block columns / rows
  const int bx = 2 * (mx0 + m) + (b & 1), by = 2 * my + (b >> 1);
  const bool dummy = b < 4 && (bx >= wb || by >= hb);
  int c[64];
  if (pass == 0) {
    if (dummy) return;
    if (b < 4) jd_fdct_quant(&t.y[8 * (b >> 1)][16 * m + 8 * (b & 1)], kJdStripW, qs.q[0], c);
    else jd_fdct_quant(&t.c[b - 4][0][8 * m], kJdStripW / 2, qs.q[1], c);
    if (b < 4) t.dc[m][b] = c[0];
  } else {
    if (!dummy) return;
    for (int k = 1; k < 64; k++) c[k] = 0;
    if (by >= hb) c[0] = 2 * (mx0 + m) + 1 < wb ? t.dc[m][1] : t.dc[m][0];     // below: the DC of Y01 (itself a dummy: of Y00)
    else c[0] = t.dc[m][b - 1];                                                 // right: the DC of the left neighbour
  }
  jd_store_block(coef + gb * 64, c);
  dc[gb] = (int16_t)c[0];
}

}  // namespace dalib200
#endif  // DALI_B200_CSRC_JPEG_DISTORT_CORE_H_
