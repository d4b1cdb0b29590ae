// tools/emul/webp_emul.cc -- TEST INFRASTRUCTURE.  Runs the WebP decode of the product on the host.
//
// The device kernels webp_entropy / webp_recon / webp_filter / webp_color (dali_b200/csrc/webp.cu) are thin wrappers around
// webp_entropy(), webp_recon_mb(), webp_filter_mb() and webp_pixel() (dali_b200/csrc/webp_core.h); the planner (webp_plan.h) is plain
// C++.  This file compiles them with the host compiler and runs them on one stream -- macroblocks in raster order -- so that
// tests/test_webp_cpu.py can compare the decode with cv2.imdecode on a machine without a GPU, and run mutated streams under ASan +
// UBSan.  The staged bytes and the scratch are heap buffers of exactly the sizes the plan gives the device: any access past them is a
// sanitizer report.
//   g++ -std=c++17 -O2 -shared -fPIC -I/usr/local/cuda/include tools/emul/webp_emul.cc
#include <cstdlib>
#include <string>
#include <vector>
#include "../../dali_b200/csrc/webp_plan.h"

using namespace dalib200;

// info: { width, height, components, orientation }.  out (width * height * C, C = 1 for out_type GRAY, else 3) may be NULL: plan only.
// Returns the planner's DALIB200 status (non-zero: rejected at plan set-up), or -1 when the device stage would set the sample's
// status (a partition that runs out of data).
extern "C" int emul_webp_decode(const uint8_t *data, size_t len, int out_type, uint8_t *out, int *info) {
  WebpImage im;
  StreamInfo wi;
  int64_t scratch_bytes = 0;
  std::string err;
  const int rc = PlanWebp(data, len, 0, &im, 0, &scratch_bytes, &wi, &err);
  if (rc) return rc;
  info[0] = wi.width; info[1] = wi.height; info[2] = wi.components; info[3] = wi.orientation;
  if (!out) return 0;
  const size_t span = wi.stage_end - wi.stage_begin;
  uint8_t *staged = static_cast<uint8_t *>(malloc(span ? span : 1));
  memcpy(staged, data + wi.stage_begin, span);
  uint8_t *scratch = static_cast<uint8_t *>(malloc(scratch_bytes));
  memset(scratch, 0xA5, scratch_bytes);
  WebpMb *mbs = reinterpret_cast<WebpMb *>(scratch + im.mb_off);
  int16_t *coef = reinterpret_cast<int16_t *>(scratch + im.coef_off);
  int status = webp_entropy(im, staged, mbs, coef, reinterpret_cast<uint32_t *>(scratch + im.ctx_off)) ? -1 : 0;
  if (!status) {
    for (int y = 0; y < im.mb_h; y++)
      for (int x = 0; x < im.mb_w; x++) webp_recon_mb(im, mbs, coef, scratch, x, y);
    for (int y = 0; y < im.mb_h; y++)
      for (int x = 0; x < im.mb_w; x++) webp_filter_mb(im, mbs, scratch, x, y);
    im.out = out; im.out_type = out_type;
    im.win_x0 = 0; im.win_y0 = 0; im.win_w = im.width; im.win_h = im.height;
    for (int y = 0; y < im.height; y++)
      for (int x = 0; x < im.width; x++) webp_pixel(im, scratch, x, y);
  }
  free(scratch);
  free(staged);
  return status;
}

// The frame header as the planner read it, and what the entropy decode found, for the corpus checks of tests/test_webp_cpu.py:
// h = { token partitions, filter type, sharpness-limited inner level of segment 0 (16x16), segment map present, skip probability
// used, number of 4x4-predicted macroblocks, number of distinct segments used }.  Returns the planner's status, or -1.
extern "C" int emul_webp_header(const uint8_t *data, size_t len, int *h) {
  WebpImage im;
  StreamInfo wi;
  int64_t scratch_bytes = 0;
  const int rc = PlanWebp(data, len, 0, &im, 0, &scratch_bytes, &wi, nullptr);
  if (rc) return rc;
  std::vector<uint8_t> scratch(scratch_bytes);
  WebpMb *mbs = reinterpret_cast<WebpMb *>(scratch.data() + im.mb_off);
  if (webp_entropy(im, data + wi.stage_begin, mbs, reinterpret_cast<int16_t *>(scratch.data() + im.coef_off),
                   reinterpret_cast<uint32_t *>(scratch.data() + im.ctx_off)))
    return -1;
  int i4 = 0, segs = 0;
  for (int64_t m = 0; m < (int64_t)im.mb_w * im.mb_h; m++) { i4 += mbs[m].i4; segs |= 1 << mbs[m].segment; }
  h[0] = im.nparts; h[1] = im.filter_type; h[2] = im.f_ilevel[0][0]; h[3] = im.update_map; h[4] = im.use_skip; h[5] = i4;
  h[6] = __builtin_popcount(segs);
  return 0;
}
