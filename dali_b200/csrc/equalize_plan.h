// dali_b200/csrc/equalize_plan.h -- host-only planner of fn.experimental.equalize (plain C++, no CUDA: tools/emul/equalize_emul.cc
// compiles it with g++).  It resolves each sample's layout into frames, channels and the channel stride, cuts every frame into work
// items of kEqChunk bytes (csrc/equalize_core.h), places each frame's C x 256 bins in the batch histogram, and refuses what the kernels
// cannot take with a message naming the sample.
#ifndef DALI_B200_CSRC_EQUALIZE_PLAN_H_
#define DALI_B200_CSRC_EQUALIZE_PLAN_H_

#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>
#include "equalize_core.h"

namespace dalib200 {

// The accepted layouts; an empty layout takes the first of them with the input's rank (2: HW, 3: HWC, 4: FHWC).
constexpr const char *kEqLayouts[] = { "HW", "HWC", "CHW", "FHW", "FHWC", "FCHW" };
constexpr int kEqNumLayouts = 6;
constexpr int64_t kEqMaxPlane = ((int64_t)1 << 31) - 1;    // cv2.equalizeHist counts a plane's pixels in an int

inline bool EqFail(std::string *err, const char *fmt, ...) __attribute__((format(printf, 2, 3)));
inline bool EqFail(std::string *err, const char *fmt, ...) {
  char buf[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  *err = buf;
  return false;
}

inline std::string EqShapeStr(const int64_t *s, int nd) {
  std::string r = "[";
  for (int a = 0; a < nd; a++) r += (a ? ", " : "") + std::to_string(s[a]);
  return r + "]";
}

inline const char *EqTypeName(int t) {
  static const char *const names[] = { "UINT8", "UINT16", "UINT32", "UINT64", "INT8", "INT16", "INT32", "INT64", "FLOAT16", "FLOAT",
                                       "FLOAT64", "BOOL" };
  return t >= 0 && t <= 11 ? names[t] : "an unknown type";
}

// The index in kEqLayouts of `layout` for an input of `ndim` dimensions, or -1 with a message.
inline int EqResolveLayout(const char *layout, int ndim, std::string *err) {
  if (!layout || !*layout) {
    for (int k = 0; k < kEqNumLayouts; k++)
      if ((int)strlen(kEqLayouts[k]) == ndim) return k;
    EqFail(err, "experimental.Equalize: cannot infer the layout of %d-dimensional input 0; give it one of HW, HWC, CHW, FHW, FHWC, FCHW", ndim);
    return -1;
  }
  for (int k = 0; k < kEqNumLayouts; k++)
    if (!strcmp(layout, kEqLayouts[k])) {
      if ((int)strlen(layout) == ndim) return k;
      EqFail(err, "experimental.Equalize: input 0 has layout \"%s\" but %d dimensions", layout, ndim);
      return -1;
    }
  EqFail(err, "experimental.Equalize: layout \"%s\" of input 0 is not supported; expected one of HW, HWC, CHW, FHW, FHWC, FCHW", layout);
  return -1;
}

// Everything a setup decides: one EqSample per sample (pointers unbound), the launch's items and the histogram's u32 words.
struct EqPlanData {
  int n = 0;
  std::vector<EqSample> samples;
  int64_t items = 0, hist_words = 0;
};

inline bool EqSetup(EqPlanData *p, int in_type, int n, int ndim, const int64_t *in_shapes, const char *layout, std::string *err) {
  if (in_type != 0)
    return EqFail(err, "experimental.Equalize: input 0 must be UINT8, got %s (type %d)", EqTypeName(in_type), in_type);
  const int li = EqResolveLayout(layout, ndim, err);
  if (li < 0) return false;
  const char *lay = kEqLayouts[li];
  const char *hp = strchr(lay, 'H'), *cp = strchr(lay, 'C');
  const int ah = (int)(hp - lay), ac = cp ? (int)(cp - lay) : -1;
  const bool has_f = lay[0] == 'F', chw = cp && ac < ah;
  p->n = n;
  p->samples.assign(n, EqSample());
  int64_t items = 0, hist = 0;
  for (int i = 0; i < n; i++) {
    const int64_t *s = in_shapes + (size_t)i * ndim;
    for (int a = 0; a < ndim; a++)
      if (s[a] < 0) return EqFail(err, "experimental.Equalize: sample %d of input 0 has a negative extent %s", i, EqShapeStr(s, ndim).c_str());
    const int64_t F = has_f ? s[0] : 1, H = s[ah], W = s[ah + 1], C = cp ? s[ac] : 1;
    if (C > kEqMaxChannels)
      return EqFail(err, "experimental.Equalize: sample %d of input 0 has %lld channels %s; at most %d are supported", i, (long long)C,
                    EqShapeStr(s, ndim).c_str(), kEqMaxChannels);
    if (H > 0 && W > kEqMaxPlane / H)
      return EqFail(err, "experimental.Equalize: sample %d of input 0 has a plane of %lld x %lld pixels %s; at most 2^31 - 1 are supported",
                    i, (long long)H, (long long)W, EqShapeStr(s, ndim).c_str());
    const int64_t plane = H * W, frame = plane * C;         // < 2^35
    if (F > 0 && frame > (((int64_t)1 << 50) / F))
      return EqFail(err, "experimental.Equalize: sample %d of input 0 has too many elements %s", i, EqShapeStr(s, ndim).c_str());
    EqSample &d = p->samples[i];
    d.frame_bytes = frame;
    d.plane = (uint32_t)plane;
    d.stride = chw ? (uint32_t)plane : 1;
    d.C = (int32_t)(C > 0 ? C : 1);
    d.nsub = kEqSmemWords / (d.C * 256) < kEqMaxSub ? kEqSmemWords / (d.C * 256) : kEqMaxSub;
    d.skip_cb = (kEqSkip % (uint32_t)d.C) << 8;
    d.first_item = items;
    if (frame == 0 || F == 0) continue;                      // an empty sample or empty frames: nothing to read or write
    d.ipf = (frame + kEqChunk - 1) / kEqChunk;
    d.items = F * d.ipf;
    d.hist_off = hist;
    items += d.items;
    hist += F * C * 256;
  }
  p->items = items;
  p->hist_words = hist;
  return true;
}

inline void EqBind(EqSample &d, const void *in, void *out) {
  d.in = static_cast<const uint8_t *>(in);
  d.out = static_cast<uint8_t *>(out);
}

}  // namespace dalib200

#endif  // DALI_B200_CSRC_EQUALIZE_PLAN_H_
