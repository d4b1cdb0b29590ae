// tools/emul/bitmap_emul.cc -- TEST INFRASTRUCTURE.  Runs the BMP / PNM decode of the product on the host.
//
// The device kernels bitmap_unpack / bitmap_color (dali_b200/csrc/bitmap.cu) are thin wrappers around bitmap_unpack() and
// bitmap_group() (dali_b200/csrc/bitmap_core.h); the planner (bitmap_plan.h) is plain C++.  This file compiles them with the host
// compiler and runs them the way a launch does, so that tests/test_bitmap_cpu.py can compare the decode with cv2.imdecode on a machine
// without a GPU, and run mutated streams under ASan + UBSan.  The staged bytes and the plane are heap buffers of exactly the sizes the
// plan gives the device: any access past them is a sanitizer report.
//   g++ -std=c++17 -O2 -ffp-contract=off -shared -fPIC -I/usr/local/cuda/include tools/emul/bitmap_emul.cc
#include <cstdlib>
#include <string>
#include "../../dali_b200/csrc/bitmap_plan.h"

using namespace dalib200;

// info: { width, height, components, orientation, unpack, layout, bits, bottom_up, stride, px_bytes, channels, maxval }.  out
// (width * height * C, C = 1 for out_type GRAY, else 3) may be NULL: plan only.  Returns the planner's DALIB200 status (non-zero:
// rejected at plan set-up), or -1 when the device stage would set the sample's status (corrupt RLE or ASCII data).
extern "C" int emul_bitmap_decode(const uint8_t *data, size_t len, int out_type, uint8_t *out, int *info) {
  BitmapImage im;
  StreamInfo si;
  int64_t plane_bytes = 0;
  std::string err;
  const int rc = PlanBitmap(data, len, &im, 0, &plane_bytes, &si, &err);
  if (rc) return rc;
  const int fields[] = { si.width, si.height, si.components, si.orientation, im.unpack, im.layout, im.bits, im.bottom_up,
                         (int)im.stride, im.px_bytes, im.channels, im.maxval };
  for (int k = 0; k < 12; k++) info[k] = fields[k];
  if (!out) return 0;
  const size_t span = si.stage_end - si.stage_begin;
  uint8_t *staged = static_cast<uint8_t *>(malloc(span ? span : 1));
  memcpy(staged, data + si.stage_begin, span);
  uint8_t *plane = plane_bytes ? static_cast<uint8_t *>(malloc((size_t)im.width * im.height * (im.ascii_channels ? im.ascii_channels : 1))) : nullptr;
  int status = 0;
  if (im.unpack != kBitmapDirect && bitmap_unpack(im, staged, plane)) status = -1;   // bitmap_unpack_kernel: one lane per image
  im.out = out; im.out_type = out_type;
  im.win_x0 = 0; im.win_y0 = 0; im.win_w = im.width; im.win_h = im.height;
  if (!status) {
    const int64_t groups = ((int64_t)im.width * im.height + kBitmapGroup - 1) / kBitmapGroup;
    for (int64_t g = 0; g < groups; g++) bitmap_group(im, plane ? plane : staged, g);  // bitmap_color_kernel: one thread per group
  }
  free(plane);
  free(staged);
  return status;
}
