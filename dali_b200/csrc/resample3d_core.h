// dali_b200/csrc/resample3d_core.h -- one pass of the 3-D (DHWC) separable resampler, written once for device and host.
//
// The body of resample3d_pass_kernel (resample3d.cu) is r3_element(): one output element per call, no cooperation between threads.
// The same function compiled by a host compiler is what tools/emul/resample3d_emul.cc runs over every element to check the planner
// and the arithmetic against the reference's SeparableResampleCPU<.., 3> without a GPU (tests/test_resample3d_emul_cpu.py).
// Arithmetic: separable_cpu.h:149-249 -> resampling_impl_cpu.h (ResampleHorz / ResampleVert / ResampleDepth / ResampleNN): products
// and sums rounded separately (the reference is built without FMA), taps in ascending order, u8 stores rounded half-to-even where the
// reference's SSE path stores and half-away in its scalar remainders.
#ifndef DALI_B200_CSRC_RESAMPLE3D_CORE_H_
#define DALI_B200_CSRC_RESAMPLE3D_CORE_H_
#include <stdint.h>
#include "host_device.h"

#if !defined(__CUDACC__)
#include <math.h>
#endif

namespace dalib200 {

// One pass of one sample.  Output: contiguous [z][y][x][c] of extent osz; input: a strided view (the first pass reads the caller's volume
// cropped to the filter footprint, later passes read a contiguous float temporary).  Vec order: [0] = x, [1] = y, [2] = z.
struct R3Pass {
  const void *in;
  void *out;
  int64_t in_offset;             // elements
  int64_t in_stride[3];          // elements; in_stride[0] == C
  int64_t total;                 // output elements
  int32_t osz[3], isz[3];        // isz: extents of the input view = clamp limits
  int32_t C;
  int32_t in_u8, out_u8;         // element types: 1 = uint8, 0 = float
  int32_t axis;                  // FIR pass: the resampled axis; -1 = gather (nearest-neighbour pass: source index maps on all three axes)
  int32_t idx_off, coef_off, support;      // FIR tables (offsets into the int32 table arena; coefficients are float bits)
  int32_t map_off[3];            // gather: per-axis source indices, already clamped
  int32_t flags_off;             // u8 output, axis 0: per-column byte flags, 1 = half-to-even
  uint32_t simd_end;             // u8 output, axis 1 / 2: stores whose flat index (inside the fused row) is below this round half-to-even
};

#if defined(__CUDA_ARCH__)
DB_HD float r3_mul(float a, float b) { return __fmul_rn(a, b); }
DB_HD float r3_add(float a, float b) { return __fadd_rn(a, b); }
DB_HD uint8_t r3_u8_away(float v) { return sat_u8_half_away(v); }
DB_HD uint8_t r3_u8_even(float v) { return sat_u8_half_even(v); }
#else
// host build: compile with -ffp-contract=off (no FMA contraction), default rounding mode
DB_HD float r3_mul(float a, float b) { return a * b; }
DB_HD float r3_add(float a, float b) { return a + b; }
DB_HD uint8_t r3_u8_away(float v) { float r = roundf(v); return (uint8_t)(r <= 0.0f ? 0 : r >= 255.0f ? 255 : (int)r); }
DB_HD uint8_t r3_u8_even(float v) { float r = nearbyintf(v); return (uint8_t)(r <= 0.0f ? 0 : r >= 255.0f ? 255 : (int)r); }
#endif

DB_HD float r3_load(const R3Pass &p, int64_t i) {
  return p.in_u8 ? (float)static_cast<const uint8_t *>(p.in)[i] : static_cast<const float *>(p.in)[i];
}

DB_HD void r3_element(const R3Pass &p, const int32_t *tab, int64_t e) {
  // a pass has fewer than 2^31 output elements (the planner checks): 32-bit index arithmetic (a 64-bit division costs ~100 instructions)
  const uint32_t C = (uint32_t)p.C, X = (uint32_t)p.osz[0], Y = (uint32_t)p.osz[1];
  uint32_t t = (uint32_t)e;
  const int c = (int)(t % C); t /= C;
  const int x = (int)(t % X); t /= X;
  const int y = (int)(t % Y);
  const int z = (int)(t / Y);
  if (p.axis < 0) {             // gather: ResampleNN (resampling_impl_cpu.h:522-629); values are copied, not computed
    const int sx = tab[p.map_off[0] + x], sy = tab[p.map_off[1] + y], sz = tab[p.map_off[2] + z];
    const int64_t i = p.in_offset + sz * p.in_stride[2] + sy * p.in_stride[1] + sx * p.in_stride[0] + c;
    if (p.in_u8) {
      const uint8_t v = static_cast<const uint8_t *>(p.in)[i];
      if (p.out_u8) static_cast<uint8_t *>(p.out)[e] = v; else static_cast<float *>(p.out)[e] = (float)v;
    } else {
      const float v = static_cast<const float *>(p.in)[i];
      if (p.out_u8) static_cast<uint8_t *>(p.out)[e] = r3_u8_away(v); else static_cast<float *>(p.out)[e] = v;
    }
    return;
  }
  const int a = p.axis;
  const int o = a == 0 ? x : a == 1 ? y : z;
  // selects instead of indexing the descriptor with `a`: the struct stays in registers / constant bank instead of a local-memory copy
  const int lim = (a == 0 ? p.isz[0] : a == 1 ? p.isz[1] : p.isz[2]) - 1;
  int64_t base = p.in_offset + c;
  if (a != 0) base += x * p.in_stride[0];
  if (a != 1) base += y * p.in_stride[1];
  if (a != 2) base += z * p.in_stride[2];
  const int64_t step = a == 0 ? p.in_stride[0] : a == 1 ? p.in_stride[1] : p.in_stride[2];
  const int i0 = tab[p.idx_off + o];
  const int32_t *cf = tab + p.coef_off + (int64_t)o * p.support;
  float sum = 0.0f;
  for (int k = 0; k < p.support; k++) {
    int s = i0 + k;
    s = s < 0 ? 0 : s;
    s = s > lim ? lim : s;
    union { int32_t i; float f; } w;
    w.i = cf[k];
    sum = r3_add(sum, r3_mul(w.f, r3_load(p, base + s * step)));
  }
  if (!p.out_u8) { static_cast<float *>(p.out)[e] = sum; return; }
  bool even;
  if (a == 0) even = reinterpret_cast<const uint8_t *>(tab + p.flags_off)[x] != 0;
  else if (a == 1) even = (uint32_t)x * C + (uint32_t)c < p.simd_end;
  else even = ((uint32_t)y * X + (uint32_t)x) * C + (uint32_t)c < p.simd_end;
  static_cast<uint8_t *>(p.out)[e] = even ? r3_u8_even(sum) : r3_u8_away(sum);
}

}  // namespace dalib200
#endif  // DALI_B200_CSRC_RESAMPLE3D_CORE_H_
