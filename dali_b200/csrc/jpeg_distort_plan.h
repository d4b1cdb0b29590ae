// dali_b200/csrc/jpeg_distort_plan.h -- host planning of fn.jpeg_compression_distortion (plain C++, also compiled by
// tools/emul/jpeg_distort_emul.cc): argument checks, libjpeg's quantisation tables for a quality, and the descriptors of one image for
// the forward kernel (JdImage) and for the decoder's reconstruct kernels (JpegImage).
#ifndef DALI_B200_CSRC_JPEG_DISTORT_PLAN_H_
#define DALI_B200_CSRC_JPEG_DISTORT_PLAN_H_
#include <cstdio>
#include <cstring>
#include "common.cuh"
#include "jpeg_distort_core.h"
#include "jpeg_recon.h"

namespace dalib200 {

constexpr int kJdMaxSide = 65500;            // libjpeg's JPEG_MAX_DIMENSION: cv2.imencode fails above it

// ITU-T T.81 Annex K tables, natural order (jcparam.c std_luminance_quant_tbl / std_chrominance_quant_tbl)
static const uint8_t kJdLumaBase[64] = {
  16, 11, 10, 16, 24, 40, 51, 61, 12, 12, 14, 19, 26, 58, 60, 55, 14, 13, 16, 24, 40, 57, 69, 56, 14, 17, 22, 29, 51, 87, 80, 62,
  18, 22, 37, 56, 68, 109, 103, 77, 24, 35, 55, 64, 81, 104, 113, 92, 49, 64, 78, 87, 103, 121, 120, 101, 72, 92, 95, 98, 112, 100, 103, 99 };
static const uint8_t kJdChromaBase[64] = {
  17, 18, 24, 47, 99, 99, 99, 99, 18, 21, 26, 66, 99, 99, 99, 99, 24, 26, 56, 99, 99, 99, 99, 99, 47, 66, 99, 99, 99, 99, 99, 99,
  99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99 };

// jpeg_set_quality(quality, force_baseline = TRUE): q[0] luma, q[1] chroma (natural order); q[2], q[3] unused
inline void JdQuantTables(int quality, QuantSet &qs) {
  memset(&qs, 0, sizeof(qs));
  const long scale = quality < 50 ? 5000 / quality : 200 - 2 * quality;
  for (int k = 0; k < 64; k++) {
    const long l = (kJdLumaBase[k] * scale + 50) / 100, c = (kJdChromaBase[k] * scale + 50) / 100;
    qs.q[0][k] = (uint16_t)(l < 1 ? 1 : l > 255 ? 255 : l);
    qs.q[1][k] = (uint16_t)(c < 1 ? 1 : c > 255 ? 255 : c);
  }
}

// 0 when the sample can be distorted, else a DALIB200 status with the reason in `msg`
inline int JdCheckSample(int i, int height, int width, int quality, char *msg, size_t msg_len) {
  if (quality < 1 || quality > 100) {
    snprintf(msg, msg_len, "jpeg_compression_distortion: sample %d: quality %d is outside [1, 100]", i, quality);
    return DALIB200_ERROR_INVALID_ARGUMENT;
  }
  if (height < 1 || width < 1 || height > kJdMaxSide || width > kJdMaxSide) {
    snprintf(msg, msg_len, "jpeg_compression_distortion: sample %d: %d x %d image; each side must be in [1, %d] (the JPEG size limit)",
             i, height, width, kJdMaxSide);
    return DALIB200_ERROR_INVALID_ARGUMENT;
  }
  if (!ElementsFit31(height, width, 3)) {
    snprintf(msg, msg_len, "jpeg_compression_distortion: sample %d: %d x %d x 3 image has 2^31 or more elements", i, height, width);
    return DALIB200_ERROR_INVALID_ARGUMENT;
  }
  return 0;
}

inline int64_t JdBlocks(int height, int width) { return (int64_t)((width + 15) / 16) * ((height + 15) / 16) * 6; }

// descriptors of one image whose blocks start at blk0: the forward kernel's, and the decoder's (4:2:0 YCbCr, fancy upsampling, RGB
// output, the whole image as window).  The plane fields are left to the caller.
inline void JdPlanImage(int height, int width, int quant_set, int64_t blk0, JdImage &d, JpegImage &im) {
  memset(&d, 0, sizeof(d));
  d.width = width; d.height = height; d.mcux = (width + 15) / 16; d.mcuy = (height + 15) / 16;
  d.quant_set = quant_set; d.strips_x = (d.mcux + kJdMcus - 1) / kJdMcus; d.blk0 = blk0;
  memset(&im, 0, sizeof(im));
  im.width = width; im.height = height; im.ncomp = 3;
  im.hs[0] = im.vs[0] = 2; im.hs[1] = im.vs[1] = im.hs[2] = im.vs[2] = 1;
  im.hmax = im.vmax = 2;
  im.mcux = d.mcux; im.mcuy = d.mcuy; im.bpm = 6;
  static const int comp[6] = { 0, 0, 0, 0, 1, 2 }, bx[6] = { 0, 1, 0, 1, 0, 0 }, by[6] = { 0, 0, 1, 1, 0, 0 };
  for (int b = 0; b < 6; b++) { im.blk_comp[b] = comp[b]; im.blk_x[b] = bx[b]; im.blk_y[b] = by[b]; }
  im.tq[0] = 0; im.tq[1] = im.tq[2] = 1;
  im.quant_set = quant_set;
  im.coef_off = blk0 * 64;
  im.out_type = DALIB200_RGB; im.fancy = 1; im.color = kColorYCbCr;
  im.win_x0 = 0; im.win_y0 = 0; im.win_w = width; im.win_h = height;
  im.mcu_x0 = 0; im.mcu_y0 = 0; im.mcu_nx = im.mcux; im.mcu_ny = im.mcuy;
}

}  // namespace dalib200
#endif  // DALI_B200_CSRC_JPEG_DISTORT_PLAN_H_
