// dali_b200/csrc/filter_plan.h -- host-only planner of fn.experimental.filter (plain C++, no CUDA: tools/emul/filter_emul.cc compiles
// it with g++).  It checks the data, filter, fill and argument rules of DESIGN.md section 2, resolves each sample's layout into frames
// of H x (W * C) elements, and cuts every output frame into strips (csrc/filter_core.h): one flat list of work items across the batch.
// Whatever it refuses, it refuses with a message naming the sample.
#ifndef DALI_B200_CSRC_FILTER_PLAN_H_
#define DALI_B200_CSRC_FILTER_PLAN_H_

#include <cstdarg>
#include <cstdio>
#include <algorithm>
#include <cstring>
#include <string>
#include <vector>
#include "filter_core.h"

namespace dalib200 {

// The accepted layouts; an empty layout takes the one with the input's rank (2: HW, 3: HWC, 4: FHWC).
constexpr const char *kFltLayouts[] = { "HW", "HWC", "FHW", "FHWC" };
constexpr int kFltNumLayouts = 4;
constexpr int64_t kFltMaxPlane = ((int64_t)1 << 31) - 1;
enum : int { kFltSame = 0, kFltValid = 1 };

inline bool FltFail(std::string *err, const char *fmt, ...) __attribute__((format(printf, 2, 3)));
inline bool FltFail(std::string *err, const char *fmt, ...) {
  char buf[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  *err = buf;
  return false;
}

inline std::string FltShapeStr(const int64_t *s, int nd) {
  std::string r = "[";
  for (int a = 0; a < nd; a++) r += (a ? ", " : "") + std::to_string(s[a]);
  return r + "]";
}

inline const char *FltTypeName(int t) {
  static const char *const names[] = { "UINT8", "UINT16", "UINT32", "UINT64", "INT8", "INT16", "INT32", "INT64", "FLOAT16", "FLOAT",
                                       "FLOAT64", "BOOL" };
  return t >= 0 && t <= 11 ? names[t] : "an unknown type";
}

inline int FltTypeSize(int t) { return t == kAU8 || t == kAI8 ? 1 : t == kAF32 ? 4 : 2; }

// The index in kFltLayouts of `layout` for an input of `ndim` dimensions, or -1 with a message.
inline int FltResolveLayout(const char *layout, int ndim, std::string *err) {
  if (!layout || !*layout) {
    for (int k = 0; k < kFltNumLayouts; k++)
      if ((int)strlen(kFltLayouts[k]) == ndim && strcmp(kFltLayouts[k], "FHW")) return k;
    FltFail(err, "experimental.Filter: cannot infer the layout of %d-dimensional input 0; give it one of HW, HWC, FHW, FHWC", ndim);
    return -1;
  }
  for (int k = 0; k < kFltNumLayouts; k++)
    if (!strcmp(layout, kFltLayouts[k])) {
      if ((int)strlen(layout) == ndim) return k;
      FltFail(err, "experimental.Filter: input 0 has layout \"%s\" but %d dimensions", layout, ndim);
      return -1;
    }
  if (strchr(layout, 'D'))
    FltFail(err, "experimental.Filter: layout \"%s\" of input 0 is volumetric; only 2-D data is supported (HW, HWC, FHW, FHWC)", layout);
  else if (strchr(layout, 'C') && strchr(layout, 'H') && strchr(layout, 'C') < strchr(layout, 'H'))
    FltFail(err, "experimental.Filter: layout \"%s\" of input 0 is channel-first; only channel-last data is supported (HW, HWC, FHW, FHWC)",
            layout);
  else
    FltFail(err, "experimental.Filter: layout \"%s\" of input 0 is not supported; expected one of HW, HWC, FHW, FHWC", layout);
  return -1;
}

// Everything a set-up decides: one FltSample per sample (pointers unbound), the element counts of each sample's filter and fill value,
// the launch's work items and the shared memory it needs.
struct FltPlanData {
  int n = 0, in_type = 0, out_type = 0, border = 0;
  bool has_fill = false;
  std::vector<FltSample> samples;
  std::vector<int64_t> filter_elems, fill_elems;
  int64_t items = 0;
  int row_floats = 0, smem_taps = 0;           // the largest window row, the largest filter read from shared memory
  int chunk = 1;                               // window rows loaded between two barriers
  size_t smem_bytes() const { return (size_t)(chunk * row_floats + smem_taps) * sizeof(float); }
};

// in_shapes, out_shapes: n x ndim.  out_type: -1 for the input's type.  filter_shapes: n x filter_ndim.  anchors: n x 2 (row, column),
// -1 for the centre.  fill_type: -1 without a fill input; fill_counts: the elements of each sample's fill value.
inline bool FltSetup(FltPlanData *p, int in_type, int out_type, int n, int ndim, const int64_t *in_shapes, const char *layout,
                     int filter_type, int filter_ndim, const int64_t *filter_shapes, const int32_t *anchors, int border, int mode,
                     int fill_type, const int64_t *fill_counts, int64_t *out_shapes, std::string *err) {
  const int types[] = { kAU8, kAI8, kAU16, kAI16, kAF16, kAF32 };
  bool known = false;
  for (int t : types) known |= in_type == t;
  if (!known)
    return FltFail(err, "experimental.Filter: input 0 must be UINT8, INT8, UINT16, INT16, FLOAT16 or FLOAT, got %s (type %d)",
                   FltTypeName(in_type), in_type);
  if (out_type < 0) out_type = in_type;
  if (out_type != in_type && out_type != kAF32)
    return FltFail(err, "experimental.Filter: dtype must be the input's type (%s) or FLOAT, got %s (type %d)", FltTypeName(in_type),
                   FltTypeName(out_type), out_type);
  if (border < kFltReflect101 || border > kFltConstant) return FltFail(err, "experimental.Filter: unknown border mode %d", border);
  if (mode != kFltSame && mode != kFltValid) return FltFail(err, "experimental.Filter: unknown mode %d", mode);
  if (n > 0 && filter_type != kAF32)
    return FltFail(err, "experimental.Filter: input 1 (the filter) must be FLOAT, got %s (type %d)", FltTypeName(filter_type), filter_type);
  if (n > 0 && filter_ndim != 2)
    return FltFail(err, "experimental.Filter: input 1 (the filter) must be 2-dimensional (HW), got %d dimensions", filter_ndim);
  if (fill_type >= 0 && fill_type != in_type)
    return FltFail(err, "experimental.Filter: input 2 (fill_value) must have the type of input 0 (%s), got %s (type %d)",
                   FltTypeName(in_type), FltTypeName(fill_type), fill_type);
  const int li = FltResolveLayout(layout, ndim, err);
  if (li < 0) return false;
  const char *lay = kFltLayouts[li];
  const bool has_f = lay[0] == 'F', has_c = lay[strlen(lay) - 1] == 'C';
  const int ah = has_f ? 1 : 0;
  p->n = n;
  p->in_type = in_type;
  p->out_type = out_type;
  p->border = border;
  p->has_fill = fill_type >= 0;
  p->samples.assign(n, FltSample());
  p->filter_elems.assign(n, 0);
  p->fill_elems.assign(n, 0);
  p->row_floats = p->smem_taps = 0;
  int64_t items = 0;
  int max_rows = 1;
  for (int i = 0; i < n; i++) {
    const int64_t *s = in_shapes + (size_t)i * ndim, *fs = filter_shapes + (size_t)i * 2;
    for (int a = 0; a < ndim; a++)
      if (s[a] < 0) return FltFail(err, "experimental.Filter: sample %d of input 0 has a negative extent %s", i, FltShapeStr(s, ndim).c_str());
    const int64_t F = has_f ? s[0] : 1, H = s[ah], W = s[ah + 1], C = has_c ? s[ah + 2] : 1;
    if (fs[0] < 1 || fs[0] > kFltMaxExtent || fs[1] < 1 || fs[1] > kFltMaxExtent)
      return FltFail(err, "experimental.Filter: sample %d of input 1 (the filter) has extents %s; each must be 1 to %d", i,
                     FltShapeStr(fs, 2).c_str(), kFltMaxExtent);
    if (C > kFltMaxChannels)
      return FltFail(err, "experimental.Filter: sample %d of input 0 has %lld channels %s; at most %d are supported", i, (long long)C,
                     FltShapeStr(s, ndim).c_str(), kFltMaxChannels);
    if (H > 0 && W > 0 && C > 0 && (W > kFltMaxPlane / C || W * C > kFltMaxPlane / H))
      return FltFail(err, "experimental.Filter: sample %d of input 0 has a frame of %lld x %lld x %lld elements %s; at most 2^31 - 1 are "
                     "supported", i, (long long)H, (long long)W, (long long)C, FltShapeStr(s, ndim).c_str());
    const int64_t plane = H * W * C;
    if (F > 0 && plane > (((int64_t)1 << 50) / F))
      return FltFail(err, "experimental.Filter: sample %d of input 0 has too many elements %s", i, FltShapeStr(s, ndim).c_str());
    const int fh = (int)fs[0], fw = (int)fs[1];
    int ar = anchors ? anchors[2 * i] : -1, ac = anchors ? anchors[2 * i + 1] : -1;
    if (mode == kFltValid) {
      if (H < fh || W < fw)
        return FltFail(err, "experimental.Filter: sample %d of input 0 %s is smaller than its %d x %d filter in \"valid\" mode", i,
                       FltShapeStr(s, ndim).c_str(), fh, fw);
      ar = ac = 0;
    } else {
      if (ar < -1 || ar >= fh || ac < -1 || ac >= fw)
        return FltFail(err, "experimental.Filter: sample %d: anchor (%d, %d) is outside its %d x %d filter; each value must be -1 or in "
                       "[0, extent - 1]", i, ar, ac, fh, fw);
      if (ar < 0) ar = fh / 2;
      if (ac < 0) ac = fw / 2;
    }
    if (fill_type >= 0 && fill_counts[i] != 1 && !(has_f && fill_counts[i] == F))
      return FltFail(err, "experimental.Filter: sample %d of input 2 (fill_value) has %lld values; expected 1%s", i,
                     (long long)fill_counts[i], has_f ? " or one per frame" : "");
    const int64_t Ho = mode == kFltValid ? H - fh + 1 : H, Wo = mode == kFltValid ? W - fw + 1 : W;
    int64_t *os = out_shapes + (size_t)i * ndim;
    for (int a = 0; a < ndim; a++) os[a] = s[a];
    os[ah] = Ho;
    os[ah + 1] = Wo;
    FltSample &d = p->samples[i];
    d.in_frame = plane;
    d.out_frame = Ho * Wo * C;
    d.H = (int32_t)H; d.W = (int32_t)W; d.C = (int32_t)C; d.Ho = (int32_t)Ho; d.Wo = (int32_t)Wo;
    d.fh = fh; d.fw = fw; d.ar = ar; d.ac = ac;
    d.border = border;
    d.in_type = in_type;
    d.out_type = out_type;
    d.fill_n = fill_type >= 0 ? (int32_t)fill_counts[i] : 0;
    d.first_item = items;
    p->filter_elems[i] = (int64_t)fh * fw;
    p->fill_elems[i] = fill_type >= 0 ? fill_counts[i] : 0;
    if (F == 0 || d.out_frame == 0) continue;                // an empty sample or empty frames: nothing to read or write
    d.sx = (int32_t)((Wo * C + kFltSpan - 1) / kFltSpan);
    d.ipf = (int32_t)((Ho + kFltRows - 1) / kFltRows) * d.sx;
    d.items = F * d.ipf;
    items += d.items;
    const int rf = flt_row_floats(fw, (int)C);
    if (rf > p->row_floats) p->row_floats = rf;
    if (fh * fw <= kFltSmemTaps && fh * fw > p->smem_taps) p->smem_taps = fh * fw;
    if (kFltRows + fh - 1 > max_rows) max_rows = kFltRows + fh - 1;
  }
  p->items = items;
  p->chunk = p->row_floats ? std::max(1, std::min({ kFltMaxChunk, max_rows, kFltChunkFloats / p->row_floats })) : 1;
  return true;
}

// The launch of filter_kernel run on the host (tools/emul): work items in reverse order, the threads of each CTA in reverse order, each
// phase of a chunk of window rows in every thread before the next, as the barriers order them on the device.
inline void FltRunOnHost(const FltSample *descs, int n, int64_t total, int row_floats, int chunk) {
  std::vector<float> mem((size_t)chunk * row_floats + 4);
  float *const rows = mem.data() + ((16 - ((uintptr_t)mem.data() & 15)) & 15) / sizeof(float);   // 16-byte aligned as on the device
  std::vector<float> acc((size_t)kFltThreads * kFltRows * kFltElems);
  FltRowMap maps[kFltMaxChunk];
  auto acc_of = [&](int t) -> float (&)[kFltRows][kFltElems] {
    return *reinterpret_cast<float (*)[kFltRows][kFltElems]>(acc.data() + (size_t)t * kFltRows * kFltElems);
  };
  for (int64_t item = total - 1; item >= 0; item--) {
    const FltSample &d = descs[last_at_most(descs, 0, n - 1, item, [](const FltSample &e) { return e.first_item; })];
    const FltStrip st = flt_strip(d, item - d.first_item);
    flt_dispatch(d.in_type, d.out_type, [&](auto ti, auto to) {
      typedef decltype(ti) TI;
      typedef decltype(to) TO;
      std::fill(acc.begin(), acc.end(), 0.0f);
      const int nrows = std::min(kFltRows, d.Ho - st.y0) + d.fh - 1;
      for (int j0 = 0; j0 < nrows; j0 += chunk) {
        const int kn = std::min(chunk, nrows - j0);
        for (int q = kn - 1; q >= 0; q--) maps[q] = flt_row_map<TI>(d, st, j0 + q);
        for (int t = kFltThreads - 1; t >= 0; t--) flt_load_groups<TI>(d, st, maps, kn, rows, row_floats, t);
        for (int t = kFltThreads - 1; t >= 0; t--) flt_load_edges<TI>(d, st, maps, kn, rows, row_floats, t);
        for (int t = kFltThreads - 1; t >= 0; t--)
          for (int q = 0; q < kn; q++) flt_accum_row(d, d.filter, j0 + q, rows + q * row_floats + maps[q].sh, acc_of(t), t);
      }
      for (int t = kFltThreads - 1; t >= 0; t--) flt_store<TO>(d, st, acc_of(t), t);
    });
  }
}

}  // namespace dalib200

#endif  // DALI_B200_CSRC_FILTER_PLAN_H_
