// dali_b200/csrc/jpeg_idct_core.h -- the arithmetic of the JPEG reconstruct kernels (jpeg.cu): dequantisation + islow IDCT of a
// block (idct_kernel, idct_color_420, and the decode half of fn.jpeg_compression_distortion), the one-column IDCT of
// idct_color_420's halo blocks, and its 16-pixel h2v2 fancy upsampling + YCbCr -> RGB / BGR unit.  Plain functions of values, with
// no memory access of their own except the unit's chroma tile reads, so that tests/test_jpeg_idct_core_cpu.py runs them on the host.
//
// The IDCT is that of libjpeg-turbo's x86 SIMD kernels (jidctint-sse2 / -avx2), which cv2.imdecode and the reference's CPU decoder
// run; it equals the C jidctint on natural streams and parts from it where coefficients are far out of range (damaged or hostile
// streams, 16-bit DQT): dequantised words and the sums i0 +- i4, i7 + i3, i5 + i1 wrap to 16 bits, the multiply-adds are exact in 32
// bits, each pass saturates its output to int16 and the result to [-128, 127].  Restated in oracle/jpeg_oracle.c and tests/jpeg_idct16.py.
#ifndef DALI_B200_CSRC_JPEG_IDCT_CORE_H_
#define DALI_B200_CSRC_JPEG_IDCT_CORE_H_
#include <stdint.h>
#include "host_device.h"

#if defined(__CUDACC__)
#define JPEG_IDCT_UNROLL _Pragma("unroll")
#else
#define JPEG_IDCT_UNROLL
#endif

namespace dalib200 {

DB_HD int wrap16(int x) { return (int)(int16_t)x; }

// __byte_perm: byte k of the result is byte (s >> 4k) & 7 of the pair {b:a} (a = bytes 0..3)
DB_HD uint32_t prmt(uint32_t a, uint32_t b, uint32_t s) {
#if defined(__CUDA_ARCH__)
  return __byte_perm(a, b, s);
#else
  const uint64_t v = ((uint64_t)b << 32) | a;
  uint32_t r = 0;
  for (int k = 0; k < 4; k++) r |= (uint32_t)((v >> (8 * ((s >> (4 * k)) & 7))) & 0xFF) << (8 * k);
  return r;
#endif
}

// four ints -> four saturated bytes of one word (byte 0 = p0): two cvt.pack.sat instead of eight min/max and three merges
DB_HD uint32_t pack4_sat_u8(int p0, int p1, int p2, int p3) {
#if defined(__CUDA_ARCH__)
  uint32_t hi, w;
  asm("cvt.pack.sat.u8.s32.b32 %0, %1, %2, %3;" : "=r"(hi) : "r"(p3), "r"(p2), "r"(0));
  asm("cvt.pack.sat.u8.s32.b32 %0, %1, %2, %3;" : "=r"(w) : "r"(p1), "r"(p0), "r"(hi));
  return w;
#else
  const int p[4] = { p0, p1, p2, p3 };
  uint32_t w = 0;
  for (int k = 0; k < 4; k++) w |= (uint32_t)(p[k] < 0 ? 0 : p[k] > 255 ? 255 : p[k]) << (8 * k);
  return w;
#endif
}

DB_HD int sat16(int x) { return x < -32768 ? -32768 : x > 32767 ? 32767 : x; }     // packssdw

// One 1-D pass over int16 inputs: the descaled 32-bit results; the caller saturates.  No sum leaves 32 bits for int16 inputs:
// |t1x| <= 2^28 + 32768 * (10703 + 4433), |o_k| <= 32768 * (20995 + 4177 + 6436 + 9633), and with pass 2's rounding constant 2^17 the
// largest sum is 2 115 960 832 < 2^31 (tests/test_jpeg_idct_core_cpu.py).  That leaves no room to fold pass 2's + 128 into the
// rounding constant (128 << 18 would take the sum past 2^31), so the output packs to signed bytes and flips their sign bits.
template <int SHIFT>
DB_HD void idct8(int i0, int i1, int i2, int i3, int i4, int i5, int i6, int i7, int *o) {
  const int tmp3 = i2 * 10703 + i6 * 4433, tmp2 = i2 * 4433 - i6 * 10704;
  const int tmp0 = wrap16(i0 + i4) * 8192, tmp1 = wrap16(i0 - i4) * 8192;
  const int r = 1 << (SHIFT - 1);
  const int t10 = tmp0 + tmp3 + r, t13 = tmp0 - tmp3 + r, t11 = tmp1 + tmp2 + r, t12 = tmp1 - tmp2 + r;
  const int z3 = wrap16(i7 + i3), z4 = wrap16(i5 + i1);
  const int Z3 = z3 * -6436 + z4 * 9633, Z4 = z3 * 9633 + z4 * 6437;
  const int o0 = i7 * -4927 + i1 * -7373 + Z3, o3 = i7 * -7373 + i1 * 4926 + Z4;
  const int o1 = i5 * -4176 + i3 * -20995 + Z4, o2 = i5 * -20995 + i3 * 4177 + Z3;
  o[0] = (t10 + o3) >> SHIFT; o[7] = (t10 - o3) >> SHIFT;
  o[1] = (t11 + o2) >> SHIFT; o[6] = (t11 - o2) >> SHIFT;
  o[2] = (t12 + o1) >> SHIFT; o[5] = (t12 - o1) >> SHIFT;
  o[3] = (t13 + o0) >> SHIFT; o[4] = (t13 - o0) >> SHIFT;
}

// packsswb + 128 of four pass-2 outputs: four bytes saturated to [-128, 127], each + 128 (= its sign bit flipped)
DB_HD uint32_t pack4_pixels(int p0, int p1, int p2, int p3) {
#if defined(__CUDA_ARCH__)
  uint32_t hi, w;
  asm("cvt.pack.sat.s8.s32.b32 %0, %1, %2, %3;" : "=r"(hi) : "r"(p3), "r"(p2), "r"(0));
  asm("cvt.pack.sat.s8.s32.b32 %0, %1, %2, %3;" : "=r"(w) : "r"(p1), "r"(p0), "r"(hi));
  return w ^ 0x80808080u;
#else
  return pack4_sat_u8(p0 + 128, p1 + 128, p2 + 128, p3 + 128);
#endif
}

// Dequantised coefficient: the low 16 bits of coef * q (pmullw).  For a word w holding two coefficients and a word qw holding their
// two table entries, the low half is wrap16(w * qw) (the high halves only add multiples of 2^16) and the high half is
// wrap16((w >> 16) * (qw >> 16)).
DB_HD int dequant_lo(int w, uint32_t qw) { return wrap16(w * (int)qw); }
DB_HD int dequant_hi(int w, uint32_t qw) { return wrap16((w >> 16) * (int)(qw >> 16)); }

// The coefficients of rows 1..7 all zero (rows0only): the SIMD kernels skip pass 1 and shift row 0 left by PASS1_BITS in 16 bits,
// which wraps where the full pass (whose outputs are then exactly in[x] << 2) saturates.  wrap16(in[x] << 2) is a multiple of 4, so
// feeding the full pass a quarter of it yields the wrapped value unsaturated.
DB_HD int row0_only(int v) { return wrap16(v * 4) >> 2; }

// A whole block: w = its 32 coefficient words (row r = words 4r .. 4r + 3, natural order, the arena's DC slot ignored), qw = the
// table's 32 words, dc = the block's absolute DC.  rows[2y], rows[2y + 1] = output row y, byte k = column k.
DB_HD void idct_block_words(const int *w, const uint32_t *qw, int dc, uint32_t *rows) {
  int ws[64];
  {
    int in[64];
    uint32_t ac_rows = 0;
JPEG_IDCT_UNROLL
    for (int k = 4; k < 32; k++) ac_rows |= (uint32_t)w[k];
JPEG_IDCT_UNROLL
    for (int k = 0; k < 32; k++) { in[2 * k] = dequant_lo(w[k], qw[k]); in[2 * k + 1] = dequant_hi(w[k], qw[k]); }
    in[0] = wrap16(dc * (int)(qw[0] & 0xFFFFu));     // DC lives in the compact array (after prediction)
    if (ac_rows == 0) {
JPEG_IDCT_UNROLL
      for (int x = 0; x < 8; x++) in[x] = row0_only(in[x]);
    }
JPEG_IDCT_UNROLL
    for (int x = 0; x < 8; x++) {       // pass 1: columns
      int o[8];
      idct8<11>(in[x], in[8 + x], in[16 + x], in[24 + x], in[32 + x], in[40 + x], in[48 + x], in[56 + x], o);
JPEG_IDCT_UNROLL
      for (int y = 0; y < 8; y++) ws[y * 8 + x] = sat16(o[y]);
    }
  }
JPEG_IDCT_UNROLL
  for (int y = 0; y < 8; y++) {         // pass 2: rows
    int o[8];
    idct8<18>(ws[y * 8], ws[y * 8 + 1], ws[y * 8 + 2], ws[y * 8 + 3], ws[y * 8 + 4], ws[y * 8 + 5], ws[y * 8 + 6], ws[y * 8 + 7], o);
    rows[2 * y] = pack4_pixels(o[0], o[1], o[2], o[3]);
    rows[2 * y + 1] = pack4_pixels(o[4], o[5], o[6], o[7]);
  }
}

// The one-column IDCT of a block of which only column 0 or 7 is needed (idct_color_420's halo), split over 8 lanes: lane x runs
// pass 1 on column x (halo_pass1: in[y] = dequantised coefficient (y, x), the DC included; ws[y] = workspace (y, x)), lane y then
// runs pass 2 on row y for the one output it needs (halo_pass2: ws = workspace row y; returns the sample of column 7 if last, else
// of column 0).  rows0only is the whole block's, as in idct_block_words.
DB_HD void halo_pass1(int *in, bool rows0only, int *ws) {
  if (rows0only) in[0] = row0_only(in[0]);
  int o[8];
  idct8<11>(in[0], in[1], in[2], in[3], in[4], in[5], in[6], in[7], o);
JPEG_IDCT_UNROLL
  for (int y = 0; y < 8; y++) ws[y] = sat16(o[y]);
}

DB_HD uint32_t halo_pass2(const int *ws, bool last) {
  int o[8];
  idct8<18>(ws[0], ws[1], ws[2], ws[3], ws[4], ws[5], ws[6], ws[7], o);
  const int v = last ? o[7] : o[0];
  return (uint32_t)((v < -128 ? -128 : v > 127 ? 127 : v) + 128);
}

// ---------------------------------------------------------------------------------------------
// idct_color_420's colour unit: 16 pixels of one luma row.  libjpeg's h2v2 fancy upsampling (jdsample.c): from the vertical sums
// cs = 3 * near + far of the chroma rows, the outputs 2i and 2i + 1 of chroma column i are (3 cs[i] + cs[i - 1] + 8) >> 4 and
// (3 cs[i] + cs[i + 1] + 7) >> 4; then jdcolor.c's fixed-point YCbCr -> RGB (SCALEBITS 16), saturated by the byte packs
// (range_limit).
//
// The sums run in 16-bit lanes, two chroma columns per word: 3 * near + far <= 1020 and 3 cs + cs' + 8 <= 4088, so no lane carries
// into the next.  The unit reads the tile bytes c - 1 .. c + 8 of the near and far rows (c = the byte of chroma column i0); libjpeg
// takes the missing neighbour of the image's first and last chroma column to be the column itself, so at the image's edges the
// kernel stores a copy of the edge column there (fancy_edge_col) and the unit has no edge case.

// The colour constants of one output order, uniform over the kernel's CTA: channel 0 = Y + a * (s0 - 128), channel 2 = Y + b * (s2
// - 128), channel 1 = Y + g0 * (s0 - 128) + g2 * (s2 - 128), where s0 / s2 are the Cr / Cb samples for RGB and the Cb / Cr samples for
// BGR.  The - 128 and jdcolor.c's ONE_HALF are folded into the additive constants, once as is (samples in a word's high lane, taken
// as v = lane >> 4) and once times 16 (samples in the low lane, taken as 16 v = lane & 0xFF0, descaled by 20 bits instead of 16).
struct ColorK {
  int a, b, g0, g2;
  int ca, cb, cg, ca16, cb16, cg16;
};

DB_HD ColorK color_k(bool bgr) {
  const int kr = 91881, kb = 116130, kgb = -22554, kgr = -46802;       // R: Cr, B: Cb, G: Cb and Cr
  ColorK k;
  k.a = bgr ? kb : kr; k.b = bgr ? kr : kb;
  k.g0 = bgr ? kgb : kgr; k.g2 = bgr ? kgr : kgb;
  k.ca = 32768 - 128 * k.a; k.cb = 32768 - 128 * k.b; k.cg = 32768 - 128 * (k.g0 + k.g2);
  k.ca16 = 16 * k.ca; k.cb16 = 16 * k.cb; k.cg16 = 16 * k.cg;
  return k;
}

// the upsampled chroma of the unit in 16-bit lanes, each lane 16 times the sample plus 4 bits below it: u[q] holds the samples of
// pixels 8 (q >> 2) + (q & 3) (low lane) and 4 more (high lane); near / far: the tile rows, c: the byte of chroma column i0 (8-aligned)
DB_HD void fancy_unit16(const uint8_t *near, const uint8_t *far, int c, uint32_t *u) {
  const uint64_t nw = *reinterpret_cast<const uint64_t *>(near + c), fw = *reinterpret_cast<const uint64_t *>(far + c);
  const uint32_t n0 = (uint32_t)nw, n1 = (uint32_t)(nw >> 32), f0 = (uint32_t)fw, f1 = (uint32_t)(fw >> 32);
  const uint32_t csl = 3u * near[c - 1] + far[c - 1], csr = 3u * near[c + 8] + far[c + 8];
  // E = (cs[i], cs[i + 2]) for i = 0 / 4, O = (cs[i + 1], cs[i + 3])
  const uint32_t e0 = 3u * prmt(n0, 0, 0x4240) + prmt(f0, 0, 0x4240), o0 = 3u * prmt(n0, 0, 0x4341) + prmt(f0, 0, 0x4341);
  const uint32_t e1 = 3u * prmt(n1, 0, 0x4240) + prmt(f1, 0, 0x4240), o1 = 3u * prmt(n1, 0, 0x4341) + prmt(f1, 0, 0x4341);
  const uint32_t p0 = prmt(csl, o0, 0x5410), p1 = prmt(o0, o1, 0x5432);      // cs[i - 1] of the E lanes
  const uint32_t n0x = prmt(e0, e1, 0x5432), n1x = prmt(e1, csr, 0x5432);    // cs[i + 1] of the O lanes
  // chroma column i: outputs 2i (even, + 8) and 2i + 1 (odd, + 7)
  u[0] = 3u * e0 + p0 + 0x00080008u;  u[1] = 3u * e0 + o0 + 0x00070007u;   // i = 0, 2: pixels 0, 1 | 4, 5
  u[2] = 3u * o0 + e0 + 0x00080008u;  u[3] = 3u * o0 + n0x + 0x00070007u;  // i = 1, 3: pixels 2, 3 | 6, 7
  u[4] = 3u * e1 + p1 + 0x00080008u;  u[5] = 3u * e1 + o1 + 0x00070007u;   // i = 4, 6: pixels 8, 9 | 12, 13
  u[6] = 3u * o1 + e1 + 0x00080008u;  u[7] = 3u * o1 + n1x + 0x00070007u;  // i = 5, 7: pixels 10, 11 | 14, 15
}

// yw: the unit's 16 luma samples (byte k of yw[k >> 2] = pixel k); s0n / s0f, s2n / s2f: near / far tile rows of the chroma of
// channel 0 and 2 (ColorK); out: 48 bytes, 3 per pixel
DB_HD void color_unit16(const uint32_t *yw, const uint8_t *s0n, const uint8_t *s0f, const uint8_t *s2n, const uint8_t *s2f, int c,
                               const ColorK &k, uint32_t *out) {
  uint32_t u0[8], u2[8];
  fancy_unit16(s0n, s0f, c, u0);
  fancy_unit16(s2n, s2f, c, u2);
  int px[48];
JPEG_IDCT_UNROLL
  for (int q = 0; q < 8; q++) {
JPEG_IDCT_UNROLL
    for (int hi = 0; hi < 2; hi++) {
      const int p = 8 * (q >> 2) + (q & 3) + 4 * hi;          // pixel of lane hi of word q
      const int yy = (int)((yw[p >> 2] >> (8 * (p & 3))) & 0xFFu);
      int c0, c1, c2;
      if (hi) {
        const int v0 = (int)(u0[q] >> 20), v2 = (int)(u2[q] >> 20);
        c0 = (k.a * v0 + k.ca) >> 16; c2 = (k.b * v2 + k.cb) >> 16; c1 = (k.g0 * v0 + k.g2 * v2 + k.cg) >> 16;
      } else {
        const int v0 = (int)(u0[q] & 0xFF0u), v2 = (int)(u2[q] & 0xFF0u);
        c0 = (k.a * v0 + k.ca16) >> 20; c2 = (k.b * v2 + k.cb16) >> 20; c1 = (k.g0 * v0 + k.g2 * v2 + k.cg16) >> 20;
      }
      px[3 * p] = yy + c0; px[3 * p + 1] = yy + c1; px[3 * p + 2] = yy + c2;
    }
  }
JPEG_IDCT_UNROLL
  for (int t = 0; t < 12; t++) out[t] = pack4_sat_u8(px[4 * t], px[4 * t + 1], px[4 * t + 2], px[4 * t + 3]);
}

}  // namespace dalib200
#endif  // DALI_B200_CSRC_JPEG_IDCT_CORE_H_
