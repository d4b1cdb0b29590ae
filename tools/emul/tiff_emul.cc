// tools/emul/tiff_emul.cc -- TEST INFRASTRUCTURE.  Runs the TIFF decode of the product on the host.
//
// The device kernels tiff_segment / tiff_color (dali_b200/csrc/tiff.cu) are thin wrappers around tiff_decode_segment() and
// tiff_pixel() (dali_b200/csrc/tiff_core.h); the planner (tiff_plan.h) is plain C++.  This file compiles them with the host compiler
// and runs them on one stream the way a launch does, so that tests/test_tiff_cpu.py can compare the decode with tests/tiff_oracle.py
// (pinned to cv2.imdecode) on a machine without a GPU, and run mutated streams under ASan + UBSan.  The staged bytes, the decoded
// segments and the working slot are heap buffers of exactly the sizes the plan gives the device: any access past them is a sanitizer
// report.
//   g++ -std=c++17 -O2 -shared -fPIC -I/usr/local/cuda/include tools/emul/tiff_emul.cc
#include <cstdlib>
#include <string>
#include <vector>
#include "../../dali_b200/csrc/tiff_plan.h"

using namespace dalib200;

// info: { width, height, components, orientation }.  out (width * height * C, C = 1 for out_type GRAY, else 3) may be NULL: plan only.
// Returns the planner's DALIB200 status (non-zero: rejected at plan set-up), or -1 when the device stage would set the sample's
// status (a corrupt segment).
extern "C" int emul_tiff_decode(const uint8_t *data, size_t len, int out_type, uint8_t *out, int *info) {
  TiffImage im;
  std::vector<TiffSeg> segs;
  StreamInfo ti;
  int64_t dec_bytes = 0;
  std::string err;
  const int rc = PlanTiff(data, len, 0, &im, segs, 0, &dec_bytes, &ti, &err);
  if (rc) return rc;
  info[0] = ti.width; info[1] = ti.height; info[2] = ti.components; info[3] = ti.orientation;
  if (!out) return 0;
  const size_t span = ti.stage_end - ti.stage_begin;
  uint8_t *staged = static_cast<uint8_t *>(malloc(span ? span : 1));
  memcpy(staged, data + ti.stage_begin, span);
  uint8_t *dec = static_cast<uint8_t *>(malloc(dec_bytes ? dec_bytes : 1));
  void *slot = malloc(kTiffSlotBytes);
  int status = 0;
  for (const TiffSeg &s : segs)                                       // tiff_segment_kernel: one lane per segment
    if (!status && tiff_decode_segment(im, s, staged, dec + s.dec_off, slot)) status = -1;
  im.out = out; im.out_type = out_type;
  im.win_x0 = 0; im.win_y0 = 0; im.win_w = im.width; im.win_h = im.height;
  if (!status)
    for (int y = 0; y < im.height; y++)
      for (int x = 0; x < im.width; x++) tiff_pixel(im, segs.data(), dec, x, y);   // tiff_color_kernel: one thread per pixel
  free(slot);
  free(dec);
  free(staged);
  return status;
}
