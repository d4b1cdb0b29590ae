// tools/emul/jpeg_distort_emul.cc -- TEST INFRASTRUCTURE.  Runs the encode half of fn.jpeg_compression_distortion on the host.
//
// The device kernel jpeg_distort_fdct (dali_b200/csrc/jpeg_distort.cu) is a thin wrapper around jd_strip(), jd_convert_quad() and
// jd_block() (dali_b200/csrc/jpeg_distort_core.h); the planner (jpeg_distort_plan.h) is plain C++.  This file compiles them with the
// host compiler and runs every strip of an image -- the quads, then the real blocks, then the dummy blocks, as the kernel's barriers
// order them -- so that tests/test_jpeg_distort_cpu.py can compare the coefficients with the ones cv2.imencode writes, on a machine
// without a GPU.  The coefficient and DC arenas are heap buffers of exactly the planned sizes.
//   g++ -std=c++17 -O2 -shared -fPIC -I/usr/local/cuda/include tools/emul/jpeg_distort_emul.cc
#include <cstdlib>
#include <vector>
#include "../../dali_b200/csrc/jpeg_distort_plan.h"

namespace dalib200 {
void SetLastError(const char *, ...) {}
}  // namespace dalib200

using namespace dalib200;

// rgb: height x width x 3.  coef (JdBlocks(height, width) * 64 int16, MCU order, natural order per block, absolute DC) and qt (2 x 64,
// luma then chroma, natural order) may be NULL.  Returns the planner's status.
extern "C" int emul_jd_coefficients(const uint8_t *rgb, int height, int width, int quality, int16_t *coef, uint16_t *qt) {
  char msg[256];
  const int rc = JdCheckSample(0, height, width, quality, msg, sizeof(msg));
  if (rc) return rc;
  QuantSet qs;
  JdQuantTables(quality, qs);
  if (qt) for (int k = 0; k < 64; k++) { qt[k] = qs.q[0][k]; qt[64 + k] = qs.q[1][k]; }
  if (!coef) return 0;
  JdImage d;
  JpegImage im;
  JdPlanImage(height, width, 0, 0, d, im);
  d.in = rgb;
  const int64_t nblk = JdBlocks(height, width);
  int16_t *arena = static_cast<int16_t *>(malloc(sizeof(int16_t) * nblk * 64));
  int16_t *dc = static_cast<int16_t *>(malloc(sizeof(int16_t) * nblk));
  JdStrip *t = new JdStrip;
  for (int64_t li = 0; li < (int64_t)d.mcuy * d.strips_x; li++) {
    int my, mx0, nt;
    jd_strip(d, li, my, mx0, nt);
    memset(t, 0xA5, sizeof(*t));
    for (int e = 0; e < 64 * nt; e++) jd_convert_quad(d, my, mx0, nt, e, *t);
    for (int pass = 0; pass < 2; pass++)
      for (int j = 0; j < 6 * nt; j++) jd_block(d, qs, my, mx0, j, pass, *t, arena, dc);
  }
  for (int64_t b = 0; b < nblk; b++) {
    memcpy(coef + b * 64, arena + b * 64, sizeof(int16_t) * 64);
    coef[b * 64] = dc[b];
  }
  delete t;
  free(dc);
  free(arena);
  return 0;
}
