// dali_b200/csrc/resample_axis.h -- the per-axis host setup of the separable resampler (filter choice, scale / origin, ROI footprint,
// pass order, index + coefficient tables), shared by the 2-D plan (resample.cu) and the 3-D plan (resample3d_plan.h).
// Plain C++: no CUDA types, so the 3-D planner can be compiled by a host compiler for the CPU emulation test (tools/emul).
#ifndef DALI_B200_CSRC_RESAMPLE_AXIS_H_
#define DALI_B200_CSRC_RESAMPLE_AXIS_H_
#include <stdint.h>
#include <algorithm>
#include <cmath>
#include <cstring>
#include <vector>
#include "../../include/dali_b200.h"

namespace dalib200 {

// Tables are addressed with 32-bit offsets and live in one host / device arena: requests beyond 2^26 words (256 MB) are refused (e.g. a
// 2^31-wide source minified with antialiasing = millions of taps per output) instead of exhausting memory.
constexpr int64_t kMaxTableWords = int64_t{1} << 26;

inline bool FilterDescValid(const dalib200FilterDesc &f) {
  return f.type >= DALIB200_FILTER_NN && f.type <= DALIB200_FILTER_LANCZOS3 && f.radius >= 0 && f.radius <= 1e6f;
}
inline bool RoiFinite(float start, float end) {
  return std::isfinite(start) && std::isfinite(end) && std::fabs(start) <= 1e9f && std::fabs(end) <= 1e9f;
}

// ---------------------------------------------------------------------------------------------
// filters (resampling_filters.cuh / .cu restated for the host-side table builder)
struct RFilter {
  const float *coeffs; int num_coeffs; float anchor; float scale;
  void rescale(float support) { float old = scale; scale = (num_coeffs - 1) / support; anchor = anchor * old / scale; }
  int support() const { return (int)ceilf((num_coeffs - 1) / scale); }
  float operator()(float x) const {
    if (!(x > -1)) return 0;
    if (x >= num_coeffs) return 0;
    int x0 = (int)std::floor(x), x1 = x0 + 1;
    float d = x - x0;
    float f0 = x0 < 0.0f ? 0 : coeffs[x0];
    float f1 = x1 >= num_coeffs ? 0.0f : coeffs[x1];
    float t = f1 - f0;
    float m = d * t;
    return f0 + m;
  }
};

struct FilterBank {
  float tri[3], gauss[65], lanczos[193], cubic[129];
  RFilter base[4];
  FilterBank() {
    tri[0] = 0; tri[1] = 1; tri[2] = 0;
    for (int i = 0; i < 65; i++) { float x = 4 * (i - 64 * 0.5f) / 64; gauss[i] = expf(-x * x); }
    auto sinc = [](float x) { x = (float)(x * M_PI); if (std::fabs(x) < 1e-5f) return 1.0f - x * x * (1.0f / 6); return sinf(x) / x; };
    for (int i = 0; i < 193; i++) {
      float x = 2 * 3.0f * (i - 192 * 0.5f) / 192;
      lanczos[i] = std::fabs(x) >= 3.0f ? 0.0f : sinc(x) * sinc(x / 3.0f);
    }
    for (int i = 0; i < 129; i++) {
      float x = std::fabs(4 * (i - 128 * 0.5f) / 128), v;
      if (x >= 2) v = 0;
      else { float x2 = x * x, x3 = x2 * x; v = x > 1 ? -0.5f * x3 + 2.5f * x2 - 4.0f * x + 2.0f : 1.5f * x3 - 2.5f * x2 + 1.0f; }
      cubic[i] = v;
    }
    base[0] = { tri, 3, 1, 1.0f };
    base[1] = { gauss, 65, 1, 32.0f };
    base[2] = { lanczos, 193, 1, 96.0f };
    base[3] = { cubic, 129, 1, 64.0f };
    base[2].rescale(6);
    base[3].rescale(4);
  }
  RFilter get(int type, float radius) const {
    RFilter f;
    switch (type) {
      case DALIB200_FILTER_LINEAR:     f = base[0]; f.rescale(std::max(1.0f, 2 * 1.0f)); return f;
      case DALIB200_FILTER_TRIANGULAR: f = base[0]; f.rescale(std::max(1.0f, 2 * radius)); return f;
      case DALIB200_FILTER_GAUSSIAN: { float sigma = (float)(radius * 0.5f / M_SQRT2);
                                       f = base[1]; f.rescale(std::max(1.0f, static_cast<float>(4 * M_SQRT2) * sigma)); return f; }
      case DALIB200_FILTER_CUBIC:      f = base[3]; f.rescale(2.0f * std::max(2.0f, radius)); return f;
      case DALIB200_FILTER_LANCZOS3:   f = base[2]; f.rescale(2.0f * std::max(3.0f, radius)); return f;
      default:                         f = { nullptr, 0, 0, 1 }; return f;
    }
  }
};
// one bank per process: the filters' coefficient tables outlive every plan that points into them
inline const FilterBank &Filters() { static FilterBank fb; return fb; }

inline float DefaultRadius(int type, bool antialias, float in_size, float out_size) {
  antialias = antialias && in_size > out_size;
  switch (type) {
    case DALIB200_FILTER_TRIANGULAR: return antialias ? in_size / out_size : 1;
    case DALIB200_FILTER_GAUSSIAN:   return antialias ? in_size / out_size : 1;
    case DALIB200_FILTER_CUBIC:      return antialias ? (2 * in_size / out_size) : 2;
    case DALIB200_FILTER_LANCZOS3:   return antialias ? (3 * in_size / out_size) : 3;
    default: return 1;
  }
}

// One axis of one sample after setup.  Axis 0 = x (width), 1 = y (height), 2 = z (depth) -- the reference's vec order.
struct AxisSetup {
  int in_size, out_size;
  int ftype;
  RFilter filter;
  float origin, scale;       // origin already shifted by roi_lo when the axis is cropped
  int roi_lo, roi_hi;
  int base, extent;          // absolute source index = base + clamp(idx, 0, extent-1)
  int support;               // >= 1 (NN -> 1)
};

struct AxisTableRef { int idx_off, coef_off, support; };

// resampling_setup.cc:47-122 for one axis
inline int SetupAxis(AxisSetup &a, int in_size, int out_size, bool use_roi, float roi_start, float roi_end,
                     dalib200FilterDesc minf, dalib200FilterDesc magf) {
  a.in_size = in_size; a.out_size = out_size;
  float fin = use_roi ? std::abs(roi_end - roi_start) : (float)in_size;
  dalib200FilterDesc fd = out_size < fin ? minf : magf;
  if (fd.antialias && fd.type == DALIB200_FILTER_LINEAR) fd.type = DALIB200_FILTER_TRIANGULAR;
  else if (!fd.antialias && fd.type == DALIB200_FILTER_TRIANGULAR) fd.type = DALIB200_FILTER_LINEAR;
  if (fd.radius == 0) fd.radius = DefaultRadius(fd.type, fd.antialias != 0, fin, (float)out_size);
  a.ftype = fd.type;
  a.filter = Filters().get(fd.type, fd.radius);
  float rs = use_roi ? roi_start : 0, re = use_roi ? roi_end : (float)in_size;
  a.origin = rs;
  a.scale = (re - rs) / out_size;
  int support = a.filter.num_coeffs ? a.filter.support() : 1;
  if (support > 8192) a.filter.rescale(8192);
  float lo, hi;
  if (rs <= re) { lo = rs - a.filter.anchor; hi = re - a.filter.anchor + support; }
  else          { lo = re - a.filter.anchor; hi = rs - a.filter.anchor + support; }
  a.roi_lo = std::max<int>(0, std::min<int>(in_size, (int)std::floor(lo)));
  a.roi_hi = std::max<int>(0, std::min<int>(in_size, (int)std::ceil(hi)));
  a.support = std::max(1, a.filter.num_coeffs ? a.filter.support() : 1);
  return 0;
}

// The first pass reads the whole input along its axis; the input of the later passes is cropped to the filter footprint along theirs,
// with the origin moved to match (resampling_setup.cc:323-336).  Sets base / extent; an empty extent is the caller's error to report.
inline void CropAxis(AxisSetup &a, bool first_pass) {
  if (first_pass) {
    a.base = 0; a.extent = a.in_size;
  } else {
    a.origin -= a.roi_lo;
    a.base = a.roi_lo; a.extent = a.roi_hi - a.roi_lo;
  }
}

// resampling_setup.cc:131-192 for ndim = 2 or 3 axes: the pass order of least estimated cost, order[0] = the first pass's axis.
// Depth-first over the orders in lexicographic order; a branch is abandoned as soon as it is not cheaper than the best complete order.
inline void ProcessingOrder(const AxisSetup *ax, int ndim, int *order) {
  float best = 1e+30f;
  int seq[3] = { 0, 1, 2 };
  std::copy(seq, seq + ndim, order);
  do {
    int64_t sz[3] = { 1, 1, 1 };
    for (int a = 0; a < ndim; a++) sz[a] = ax[a].roi_hi - ax[a].roi_lo;
    float total = 0;
    bool ok = true;
    for (int p = 0; p < ndim; p++) {
      if (total >= best) { ok = false; break; }
      const int a = seq[p];
      sz[a] = ax[a].out_size;
      const int64_t vol = sz[0] * sz[1] * sz[2];
      const float mul = a == 0 ? 1.4f : a == 1 ? 1.0f : 1.2f;
      total += mul * (float)(ax[a].support * vol) + vol * 3.0f;
    }
    if (ok && !(total >= best)) { best = total; std::copy(seq, seq + ndim, order); }
  } while (std::next_permutation(seq, seq + ndim));
}

// Nearest-neighbour source indices of one axis, unclamped (resampling_impl_cpu.h:522-606): x is computed per element, the other axes'
// coordinate is accumulated incrementally as the reference does.
inline void NNIndices(int32_t *idx, int n, float origin, float scale, int axis) {
  if (axis != 0) {
    float src = origin + 0.5f * scale;
    for (int i = 0; i < n; i++, src += scale) idx[i] = (int)std::floor(src);
  } else if (scale == 1) {
    const int sx0 = (int)std::floor(origin + 0.5f);
    for (int x = 0; x < n; x++) idx[x] = sx0 + x;
  } else {
    for (int x = 0; x < n; x++) idx[x] = (int)std::floor(origin + (x + 0.5f) * scale);
  }
}

// Coefficient / index table of one axis, appended to `arena`: idx[out_size], then coef[out_size * support] as float bits.
// FIR: resampling_impl_cpu.cc:22-47.  NN: NNIndices with weight 1.
inline void BuildTable(std::vector<int32_t> &arena, AxisTableRef &ref, const AxisSetup &a, int axis) {
  const int n = a.out_size, S = a.support;
  ref.support = S;
  ref.idx_off = (int)arena.size();
  arena.resize(arena.size() + n);
  ref.coef_off = (int)arena.size();
  arena.resize(arena.size() + (size_t)n * S);
  int32_t *idx = arena.data() + ref.idx_off;
  float *coef = reinterpret_cast<float *>(arena.data() + ref.coef_off);
  if (a.ftype == DALIB200_FILTER_NN) {
    NNIndices(idx, n, a.origin, a.scale, axis);
    for (int x = 0; x < n; x++) coef[x] = 1.0f;
    return;
  }
  const RFilter &f = a.filter;
  float s0 = a.origin;
  s0 += 0.5f * a.scale - 0.5f - f.anchor;
  for (int x = 0; x < n; x++) {
    float sx0f = x * a.scale + s0;
    int sx0 = (int)ceilf(sx0f);
    idx[x] = sx0;
    const float f0 = sx0 - sx0f;
    float sum = 0;
    for (int k = 0; k < S; k++) {
      float c = f((f0 + k) * f.scale);
      coef[(size_t)S * x + k] = c;
      sum += c;
    }
    if (sum) for (int k = 0; k < S; k++) coef[(size_t)S * x + k] /= sum;
  }
}

// Which output columns does the reference's horizontal pass compute in its 16-lane SSE path?
// (resampling_impl_cpu.h:126-222,225-336) -- those round half-to-even when storing u8.  Appends (ow + 3) / 4 words of flag bytes
// (1 = half to even, zero-padded) to `arena` and returns their offset.
inline int BuildHorzFlags(std::vector<int32_t> &arena, int idx_off, int ow, int iw, int support) {
  int off = (int)arena.size();
  arena.resize(arena.size() + (ow + 3) / 4);
  const int32_t *idx = arena.data() + idx_off;      // after the resize: the arena may have moved
  uint8_t *fl = reinterpret_cast<uint8_t *>(arena.data() + off);
  memset(fl, 0, (size_t)((ow + 3) / 4) * 4);
  bool flipped = idx[ow - 1] < idx[0];
  int first = 0, last = ow - 1;
  if (flipped) {
    while (first < ow && idx[first] + support > iw) first++;
    while (last >= 0 && idx[last] < 0) last--;
  } else {
    while (first < ow && idx[first] < 0) first++;
    while (last >= 0 && idx[last] + support > iw) last--;
  }
  int bounds[4] = { std::min(first, last + 1), first, last + 1, ow };
  int x = 0;
  for (int r = 0; r < 4; r++) {
    int ox1 = bounds[r];
    for (; x + 16 <= ox1; x += 16) memset(fl + x, 1, 16);
    for (; x < ox1; x++) fl[x] = 0;
  }
  return off;
}

}  // namespace dalib200
#endif  // DALI_B200_CSRC_RESAMPLE_AXIS_H_
