// tools/emul/jpeg_idct_emul.cc -- TEST INFRASTRUCTURE.  Runs the reconstruct arithmetic of the JPEG kernels on the host.
//
// idct_kernel and idct_color_420 (dali_b200/csrc/jpeg.cu) load their operands and call idct_block_words(), halo_pass1() /
// halo_pass2() and color_unit16() (dali_b200/csrc/jpeg_idct_core.h).  This file compiles those with the host compiler, so that
// tests/test_jpeg_idct_core_cpu.py can compare them with the numpy statement of the IDCT (tests/jpeg_idct16.py) and with libjpeg's
// upsampling and colour formulas, on a machine without a GPU.
//   g++ -std=c++17 -O2 -shared -fPIC tools/emul/jpeg_idct_emul.cc
#include <cstring>
#include "../../dali_b200/csrc/jpeg_idct_core.h"

using namespace dalib200;

// coef, q: n blocks of 64 (natural order, coef[0] = the absolute DC); out: n x 64 samples
extern "C" void emul_idct_blocks(const int16_t *coef, const uint16_t *q, int n, uint8_t *out) {
  for (int i = 0; i < n; i++) {
    int w[32];
    uint32_t qw[32], rows[16];
    memcpy(w, coef + 64 * i, sizeof(w));
    memcpy(qw, q + 64 * i, sizeof(qw));
    w[0] = (int)(((uint32_t)w[0] & 0xFFFF0000u) | 0x5A5Au);      // the arena's DC slot is not the DC
    idct_block_words(w, qw, coef[64 * i], rows);
    memcpy(out + 64 * i, rows, 64);
  }
}

// the same blocks through idct_color_420's halo path: out = n x 16, column 0 of block i's 8 rows, then its column 7
extern "C" void emul_idct_halo(const int16_t *coef, const uint16_t *q, int n, uint8_t *out) {
  for (int i = 0; i < n; i++) {
    const int16_t *c = coef + 64 * i;
    const uint16_t *qq = q + 64 * i;
    uint32_t ac = 0;
    for (int k = 8; k < 64; k++) ac |= (uint32_t)(int)c[k];
    int ws[8][8];                                        // [row][column], as the kernel's shared workspace
    for (int x = 0; x < 8; x++) {                        // lane x
      int in[8], col[8];
      for (int y = 0; y < 8; y++) in[y] = wrap16(c[8 * y + x] * (int)qq[8 * y + x]);
      halo_pass1(in, ac == 0, col);
      for (int y = 0; y < 8; y++) ws[y][x] = col[y];
    }
    for (int y = 0; y < 8; y++) {                        // lane y
      out[16 * i + y] = (uint8_t)halo_pass2(ws[y], false);
      out[16 * i + 8 + y] = (uint8_t)halo_pass2(ws[y], true);
    }
  }
}

// n colour units: tiles = n x 4 x 10 bytes (channel-0 chroma near / far row, channel-2 chroma near / far row; byte k = chroma column
// i0 - 1 + k), y = n x 16 luma samples, out = n x 48 bytes
extern "C" void emul_color_units(const uint8_t *tiles, const uint8_t *y, int n, int bgr, uint8_t *out) {
  const ColorK k = color_k(bgr != 0);
  for (int i = 0; i < n; i++) {
    alignas(16) uint8_t t[4][24];                        // as the kernel's tile rows: chroma column i0 at byte 8
    uint32_t yw[4], w[12];
    for (int r = 0; r < 4; r++) memcpy(&t[r][7], tiles + 40 * i + 10 * r, 10);
    memcpy(yw, y + 16 * i, 16);
    color_unit16(yw, t[0], t[1], t[2], t[3], 8, k, w);
    memcpy(out + 48 * i, w, 48);
  }
}
