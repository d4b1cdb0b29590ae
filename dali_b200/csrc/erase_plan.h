// dali_b200/csrc/erase_plan.h -- host-only planner of fn.erase (plain C++, no CUDA: tools/emul/erase_emul.cc compiles it with g++).
// It checks the type, layout, axis, region and fill rules of DESIGN.md section 2, turns each sample's regions into clipped boxes,
// reduces the sample to rows x an inner run, cuts the rows' key space into bands with their interval lists (csrc/erase_core.h),
// converts the fill values to the data type, and cuts every sample into work items of 16-byte slots: one flat list across the batch.
// Whatever it refuses, it refuses with a message naming the sample and the argument.
#ifndef DALI_B200_CSRC_ERASE_PLAN_H_
#define DALI_B200_CSRC_ERASE_PLAN_H_

#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <algorithm>
#include <cstring>
#include <string>
#include <vector>
#include "erase_core.h"
#include "arith_core.h"

namespace dalib200 {

inline bool ErFail(std::string *err, const char *fmt, ...) __attribute__((format(printf, 2, 3)));
inline bool ErFail(std::string *err, const char *fmt, ...) {
  char buf[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  *err = buf;
  return false;
}

inline std::string ErShapeStr(const int64_t *s, int nd) {
  std::string r = "[";
  for (int a = 0; a < nd; a++) r += (a ? ", " : "") + std::to_string(s[a]);
  return r + "]";
}

// Everything a set-up decides: one ErSample per sample (pointers unbound), the samples' bands and intervals back to back, the fill
// table (ErFillTable) and the launch's work items.
struct ErPlanData {
  int n = 0, type = 0, esz = 1, nfill = 1;
  std::vector<ErSample> samples;
  std::vector<ErBand> bands;
  std::vector<ErIval> ivals;
  std::vector<int64_t> band_off, ival_off;     // per sample, into bands / ivals
  std::vector<uint8_t> fill;                   // the fill table, er_rot_off(nfill, esz) + 32 nfill bytes
  int64_t items = 0;
};

// The fill table: the values converted with ConvertSat (tests/arith_ref.py), then the rotated patterns and the broadcasts.
inline void ErFillTable(const float *vals, int nfill, int type, std::vector<uint8_t> *t) {
  const int esz = arith_size(type), V = 16 / esz;
  const int64_t rot = er_rot_off(nfill, esz);
  t->assign((size_t)(rot + 32 * (int64_t)nfill), 0);
  std::vector<uint64_t> bits(nfill);
  for (int c = 0; c < nfill; c++) {
    bits[c] = arith_to_bits(arith_cast(arith_uf(vals[c]), kAF32, type), type);
    memcpy(t->data() + (size_t)c * esz, &bits[c], esz);                    // little-endian: the low esz bytes
  }
  for (int p = 0; p < nfill; p++)
    for (int k = 0; k < V; k++) {
      memcpy(t->data() + rot + 16 * p + k * esz, &bits[(p + k) % nfill], esz);
      memcpy(t->data() + rot + 16 * (nfill + p) + k * esz, &bits[p], esz);
    }
}

// One region after the coordinate rules: [b[a], e[a]) per dimension a (erased dimensions only), clipped, non-empty.
struct ErBox { int64_t b[kErMaxDim], e[kErMaxDim]; };

struct ErBandBuilder {
  const int64_t *s;
  std::vector<int> ed;                         // the erased outer dimensions, outermost first
  std::vector<int64_t> kstride;                // their strides in the key space
  int q;                                       // the innermost erased dimension
  int64_t unit;                                // elements per step of dimension q
  const std::vector<ErBox> *boxes;
  std::vector<ErIval> *ivals;
  int64_t ival_base;

  static void push(std::vector<ErBand> *out, int64_t key, int64_t off, int64_t cnt) {
    if (!out->empty() && out->back().off == off && out->back().cnt == cnt) return;      // the band before goes on
    out->push_back(ErBand{ key, off, cnt });
  }

  // the bands of the key sub-space of ed[l..], keys relative to it, for the regions in act (non-empty)
  std::vector<ErBand> pattern(size_t l, const std::vector<int> &act) {
    std::vector<ErBand> out;
    if (l == ed.size()) {
      std::vector<ErIval> iv;
      for (int r : act) iv.push_back(ErIval{ (*boxes)[r].b[q] * unit, (*boxes)[r].e[q] * unit });
      std::sort(iv.begin(), iv.end(), [](const ErIval &x, const ErIval &y) { return x.lo < y.lo; });
      const int64_t off = (int64_t)ivals->size() - ival_base;
      for (const ErIval &v : iv) {
        if (ivals->size() > (size_t)(off + ival_base) && ivals->back().hi >= v.lo) ivals->back().hi = std::max(ivals->back().hi, v.hi);
        else ivals->push_back(v);
      }
      out.push_back(ErBand{ 0, off, (int64_t)ivals->size() - ival_base - off });
      return out;
    }
    const int a = ed[l];
    std::vector<int64_t> cuts = { 0, s[a] };
    for (int r : act) cuts.push_back((*boxes)[r].b[a]), cuts.push_back((*boxes)[r].e[a]);
    std::sort(cuts.begin(), cuts.end());
    cuts.erase(std::unique(cuts.begin(), cuts.end()), cuts.end());
    for (size_t k = 0; k + 1 < cuts.size(); k++) {
      const int64_t p0 = cuts[k], p1 = cuts[k + 1];
      std::vector<int> inside;
      for (int r : act)
        if ((*boxes)[r].b[a] <= p0 && (*boxes)[r].e[a] >= p1) inside.push_back(r);
      if (inside.empty()) { push(&out, p0 * kstride[l], 0, 0); continue; }
      const std::vector<ErBand> sub = pattern(l + 1, inside);
      if (sub.size() == 1) { push(&out, p0 * kstride[l], sub[0].off, sub[0].cnt); continue; }
      for (int64_t p = p0; p < p1; p++)
        for (const ErBand &b : sub) push(&out, p * kstride[l] + b.key, b.off, b.cnt);
    }
    return out;
  }
};

// shapes: n x ndim.  axis_names: the erased axes as layout characters, or NULL to take axes (naxes dimension indices).  anchors,
// shapes_arg: the values of every sample back to back, anchor_counts / shape_counts of them per sample.  fill: nfill values.
inline bool ErSetup(ErPlanData *p, int type, int n, int ndim, const int64_t *shapes, const char *layout, const char *axis_names,
                    const int32_t *axes, int naxes, const float *anchors, const int64_t *anchor_counts, const float *shapes_arg,
                    const int64_t *shape_counts, int norm_anchor, int norm_shape, int centered, const float *fill, int nfill,
                    std::string *err) {
  if (type < 0 || type > 11) return ErFail(err, "erase: input 0 has an unsupported type (code %d)", type);
  if (ndim < 1 || ndim > kErMaxDim) return ErFail(err, "erase: input 0 has %d dimensions; 1 to %d are supported", ndim, kErMaxDim);
  const size_t lay_len = layout ? strlen(layout) : 0;
  if (lay_len && (int)lay_len != ndim) return ErFail(err, "erase: input 0 has layout \"%s\" but %d dimensions", layout, ndim);
  for (size_t a = 0; a < lay_len; a++)
    if (strchr(layout + a + 1, layout[a]))
      return ErFail(err, "erase: layout \"%s\" of input 0 repeats the axis '%c'", layout, layout[a]);
  // the erased dimensions, in the order of the anchor and shape values
  std::vector<int> dims;
  if (axis_names) {
    if (!lay_len)
      return ErFail(err, "erase: axis_names \"%s\" needs a layout, and input 0 has none; give the axes as dimension indices (axes)",
                    axis_names);
    for (const char *c = axis_names; *c; c++) {
      const char *at = strchr(layout, *c);
      if (!at) return ErFail(err, "erase: axis_names \"%s\": '%c' is not an axis of the layout \"%s\"", axis_names, *c, layout);
      dims.push_back((int)(at - layout));
    }
  } else {
    for (int k = 0; k < naxes; k++) {
      if (axes[k] < 0 || axes[k] >= ndim)
        return ErFail(err, "erase: axes: %d is not a dimension of the %d-dimensional input 0", axes[k], ndim);
      dims.push_back(axes[k]);
    }
  }
  const char *what = axis_names ? "axis_names" : "axes";
  if (dims.empty()) return ErFail(err, "erase: %s names no axis", what);
  uint32_t mask = 0;
  for (int a : dims) {
    if (mask >> a & 1u) return ErFail(err, "erase: %s names the dimension %d twice", what, a);
    mask |= 1u << a;
  }
  const int nax = (int)dims.size(), q = *std::max_element(dims.begin(), dims.end());
  // fill values: one, or one per channel of a C axis that is not erased
  if (nfill < 1) return ErFail(err, "erase: fill_value has no value");
  const char *cpos = lay_len ? strchr(layout, 'C') : nullptr;
  const int cdim = cpos ? (int)(cpos - layout) : -1;
  if (nfill > 1 && cdim < 0)
    return ErFail(err, "erase: fill_value has %d values; more than one needs a C axis in the layout of input 0 (\"%s\")", nfill,
                  lay_len ? layout : "");
  if (nfill > 1 && (mask >> cdim & 1u))
    return ErFail(err, "erase: fill_value has %d values, one per channel, but the C axis is erased", nfill);
  p->n = n;
  p->type = type;
  p->esz = arith_size(type);
  p->nfill = nfill;
  p->samples.assign(n, ErSample());
  p->bands.clear();
  p->ivals.clear();
  p->band_off.assign(n, 0);
  p->ival_off.assign(n, 0);
  ErFillTable(fill, nfill, type, &p->fill);
  int64_t items = 0, vpos = 0;
  const int V = 16 / p->esz;
  std::vector<ErBox> boxes;
  for (int i = 0; i < n; i++) {
    const int64_t *s = shapes + (size_t)i * ndim;
    for (int a = 0; a < ndim; a++)
      if (s[a] < 0) return ErFail(err, "erase: sample %d of input 0 has a negative extent %s", i, ErShapeStr(s, ndim).c_str());
    int64_t vol = 1;
    for (int a = 0; a < ndim; a++) {
      if (s[a] > 0 && vol > ((int64_t)1 << 50) / s[a])
        return ErFail(err, "erase: sample %d of input 0 has too many elements %s", i, ErShapeStr(s, ndim).c_str());
      vol *= s[a];
    }
    if (nfill > 1 && s[cdim] != nfill)
      return ErFail(err, "erase: sample %d: fill_value has %d values, but the C axis of input 0 has %lld channels %s", i, nfill,
                    (long long)s[cdim], ErShapeStr(s, ndim).c_str());
    const int64_t na = anchor_counts[i], ns = shape_counts[i];
    if (na != ns)
      return ErFail(err, "erase: sample %d: anchor has %lld values and shape %lld; they must have as many", i, (long long)na,
                    (long long)ns);
    if (na % nax)
      return ErFail(err, "erase: sample %d: anchor and shape have %lld values, not a multiple of the %d erased axes", i,
                    (long long)na, nax);
    boxes.clear();
    for (int64_t r = 0; r < na / nax; r++) {
      ErBox box;
      bool empty = false;
      for (int k = 0; k < nax; k++) {
        const int a = dims[k];
        const float fa = anchors[vpos + r * nax + k], fs = shapes_arg[vpos + r * nax + k];
        if (!std::isfinite(fa)) return ErFail(err, "erase: sample %d: anchor value %g is not finite", i, (double)fa);
        if (!std::isfinite(fs)) return ErFail(err, "erase: sample %d: shape value %g is not finite", i, (double)fs);
        if (fs < 0) return ErFail(err, "erase: sample %d: shape value %g is a negative extent", i, (double)fs);
        double x = fa, w = fs;
        if (norm_anchor) x *= (double)s[a];
        if (norm_shape) w *= (double)s[a];
        if (centered) x -= w / 2;
        const double lim = 4.0e18;                                          // llround's range; beyond it the clip decides anyway
        const int64_t b = std::llround(std::min(std::max(x, -lim), lim)), e = std::llround(std::min(std::max(x + w, -lim), lim));
        box.b[a] = std::min(std::max(b, (int64_t)0), s[a]);
        box.e[a] = std::min(std::max(e, (int64_t)0), s[a]);
        empty |= box.e[a] <= box.b[a];
      }
      if (!empty) boxes.push_back(box);
    }
    vpos += na;
    ErSample &d = p->samples[i];
    d.n = vol;
    d.esz = p->esz;
    d.first_item = items;
    d.run = 1;
    for (int a = q; a < ndim; a++) d.run *= s[a];
    d.cstride = 1;
    if (nfill > 1)
      for (int a = cdim + 1; a < ndim; a++) d.cstride *= s[a];
    // the outer dimensions in groups of like ones, and the key strides of the erased groups
    d.ngroups = 0;
    d.gfirst = -1;
    for (int a = 0; a < q; a++) {
      const bool er = mask >> a & 1u;
      if (d.ngroups && (d.kst[d.ngroups - 1] != 0) == er) {
        d.ext[d.ngroups - 1] *= s[a];
      } else {
        d.ext[d.ngroups] = s[a];
        d.kst[d.ngroups++] = er;                                            // 1 marks an erased group until the strides are set
      }
    }
    int64_t kmul = 1;
    for (int g = d.ngroups - 1; g >= 0; g--)
      if (d.kst[g]) { d.kst[g] = kmul; kmul *= d.ext[g]; d.gfirst = g; }
    if (vol == 0) continue;                                                 // an empty sample: nothing to read or write
    d.items = ((vol + 2 * V - 2) / V + kErSlotsPerItem - 1) / kErSlotsPerItem;
    items += d.items;
    ErBandBuilder bb;
    bb.s = s;
    bb.q = q;
    bb.unit = 1;
    for (int a = q + 1; a < ndim; a++) bb.unit *= s[a];
    for (int a = 0; a < q; a++)
      if (mask >> a & 1u) bb.ed.push_back(a);
    bb.kstride.assign(bb.ed.size(), 1);
    for (int l = (int)bb.ed.size() - 2; l >= 0; l--) bb.kstride[l] = bb.kstride[l + 1] * s[bb.ed[l + 1]];
    bb.boxes = &boxes;
    bb.ivals = &p->ivals;
    bb.ival_base = p->ival_off[i] = (int64_t)p->ivals.size();
    p->band_off[i] = (int64_t)p->bands.size();
    std::vector<int> all(boxes.size());
    for (size_t r = 0; r < boxes.size(); r++) all[r] = (int)r;
    const std::vector<ErBand> bands = all.empty() ? std::vector<ErBand>{ ErBand{ 0, 0, 0 } } : bb.pattern(0, all);
    p->bands.insert(p->bands.end(), bands.begin(), bands.end());
    d.nbands = (int32_t)bands.size();
  }
  p->items = items;
  return true;
}

// f(ErElem<element size>())
template <typename F> void er_dispatch(int esz, F &&f) {
  switch (esz) {
    case 1: f(ErElem<1>()); break;
    case 2: f(ErElem<2>()); break;
    case 4: f(ErElem<4>()); break;
    default: f(ErElem<8>()); break;
  }
}

// The launch of erase_kernel run on the host (tools/emul): work items in reverse order, the threads of each CTA in reverse order.
inline void ErRunOnHost(const ErSample *descs, int n, int64_t total, const uint8_t *fill, int nfill) {
  for (int64_t item = total - 1; item >= 0; item--) {
    const ErSample &d = descs[last_at_most(descs, 0, n - 1, item, [](const ErSample &e) { return e.first_item; })];
    er_dispatch(d.esz, [&](auto t) {
      constexpr int ESZ = (int)sizeof(typename decltype(t)::T);
      for (int tid = kErThreads - 1; tid >= 0; tid--) er_item<ESZ>(d, fill, nfill, item - d.first_item, tid);
    });
  }
}

}  // namespace dalib200

#endif  // DALI_B200_CSRC_ERASE_PLAN_H_
