// tools/emul/png_emul.cc -- TEST INFRASTRUCTURE.  Runs the PNG decode of the product on the host.
//
// The device kernels png_crc / png_inflate / png_color (dali_b200/csrc/png.cu) are thin wrappers around png_chunk_crc_ok(),
// png_inflate_unfilter() and png_pixel() (dali_b200/csrc/png_core.h); the planner (png_plan.h) is plain C++.  This file compiles them
// with the host compiler and runs them on one stream the way a launch does, so that tests/test_png_cpu.py can compare the decode with
// tests/png_oracle.py (pinned to cv2.imdecode) on a machine without a GPU, and run mutated streams under ASan + UBSan.  The staged
// bytes and the scanline scratch are heap buffers of exactly the sizes the plan gives the device: any read or write past them is a
// sanitizer report.
//   g++ -std=c++17 -O2 -shared -fPIC -I/usr/local/cuda/include tools/emul/png_emul.cc
#include <cstdlib>
#include <string>
#include <vector>
#include "../../dali_b200/csrc/png_plan.h"

using namespace dalib200;

// info: { width, height, components, orientation }.  out (width * height * C, C = 1 for out_type GRAY, else 3) may be NULL: plan only.
// Returns the planner's DALIB200 status (non-zero: rejected at plan set-up), or -1 when the device stage would set the sample's
// status (CRC, inflate or filter error).
extern "C" int emul_png_decode(const uint8_t *data, size_t len, int out_type, uint8_t *out, int *info) {
  PngImage im;
  std::vector<PngChunk> chunks;
  StreamInfo pi;
  std::string err;
  const int rc = PlanPng(data, len, 0, &im, chunks, &pi, &err);
  if (rc) return rc;
  info[0] = pi.width; info[1] = pi.height; info[2] = pi.components; info[3] = pi.orientation;
  if (!out) return 0;
  uint8_t *staged = static_cast<uint8_t *>(malloc(pi.stage_end - pi.stage_begin));
  memcpy(staged, data + pi.stage_begin, pi.stage_end - pi.stage_begin);
  uint8_t *scan = static_cast<uint8_t *>(malloc(im.scan_bytes ? im.scan_bytes : 1));
  uint32_t table[256];
  for (uint32_t i = 0; i < 256; i++) table[i] = png_crc_table_entry(i);
  int status = 0;
  for (const PngChunk &c : chunks)                                    // png_crc_kernel: one thread per chunk
    if (!png_chunk_crc_ok(staged + im.raw_off + c.off - 4, c.len, table)) status = -1;
  InflateWork *w = new InflateWork;
  if (!status && png_inflate_unfilter(im, chunks.data(), staged, scan, *w)) status = -1;
  delete w;
  im.out = out; im.out_type = out_type;
  im.win_x0 = 0; im.win_y0 = 0; im.win_w = im.width; im.win_h = im.height;
  if (!status)
    for (int y = 0; y < im.height; y++)
      for (int x = 0; x < im.width; x++) png_pixel(im, scan, x, y);   // png_color_kernel: one thread per pixel
  free(scan);
  free(staged);
  return status;
}
