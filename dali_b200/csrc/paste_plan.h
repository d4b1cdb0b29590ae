// dali_b200/csrc/paste_plan.h -- host-only planner of fn.multi_paste and fn.paste (plain C++, no CUDA: tools/emul/paste_emul.cc
// compiles it with g++).  It checks the type, layout, shape, region and fill rules of DESIGN.md section 2, resolves each output's
// regions to pixel rectangles, cuts each output's rows into bands at the regions' y-edges, resolves the visible segments of a row in
// every band (a later region on top of an earlier one, the fill where none is), builds the fill table in the output type, and cuts
// every output into work items of 16-byte slots: one flat list across the batch.  fn.paste is one region per output on a canvas
// filled with a per-channel value; PsCanvasSetup states its geometry and hands it to the same builder.  Whatever the planner refuses,
// it refuses with a message naming the sample, the region and the argument.
#ifndef DALI_B200_CSRC_PASTE_PLAN_H_
#define DALI_B200_CSRC_PASTE_PLAN_H_

#include <cmath>
#include <algorithm>
#include <string>
#include <type_traits>
#include <vector>
#include "paste_core.h"
#include "erase_plan.h"

namespace dalib200 {

// The region arguments of multi_paste, in the order of dalib200PasteSetup's args / arg_counts.
enum : int { kPsInAnchors, kPsInAnchorsRel, kPsShapes, kPsShapesRel, kPsOutAnchors, kPsOutAnchorsRel, kPsNumArgs };
inline const char *PsArgName(int a) {
  static const char *const names[kPsNumArgs] = { "in_anchors", "in_anchors_rel", "shapes", "shapes_rel", "out_anchors", "out_anchors_rel" };
  return names[a];
}

// Everything a set-up decides: one PsSample per output (pointers unbound), the outputs' bands and segments back to back, the fill
// table, which inputs some segment reads, the output shapes and the launch's work items.
struct PsPlanData {
  int n = 0, nsrc = 0, in_type = 0, out_type = 0, osz = 1, nfill = 1;
  std::vector<PsSample> samples;
  std::vector<PsBand> bands;
  std::vector<PsSeg> segs;
  std::vector<int64_t> band_off, seg_off;     // per output, into bands / segs
  std::vector<uint8_t> fill;                  // ErFillTable in the output type
  std::vector<uint8_t> used;                  // per input pointer: read by some segment
  std::vector<int64_t> out_shapes;            // n x 3 (H, W, C)
  int64_t items = 0;
};

// One region in pixels: source src (an index into the input pointers), its rectangle there and its place in the output.
struct PsRegion { int32_t src; int64_t iy, ix, h, w, oy, ox; };

// The bands and segments of one output of H x W pixels of C channels; regs in paste order (later on top), none empty.
// Host work O(K^2) for K regions: at most 2K + 1 bands, and per band one pass over the 2K + 1 column cells in which each region
// paints the cells not yet painted by a later one (a disjoint-set "next unpainted cell" walk).
inline void PsBuildOutput(PsPlanData *p, int i, int64_t H, int64_t W, int64_t C, const std::vector<PsRegion> &regs, const int64_t *in_shapes) {
  PsSample &d = p->samples[i];
  d.n = H * W * C;
  d.run = W * C;
  d.first_item = p->items;
  p->band_off[i] = (int64_t)p->bands.size();
  p->seg_off[i] = (int64_t)p->segs.size();
  if (d.n == 0) return;                                                  // an empty output: nothing to read or write
  const int V = 16 / p->osz;
  d.items = ((d.n + 2 * V - 2) / V + kPsSlotsPerItem - 1) / kPsSlotsPerItem;
  p->items += d.items;
  std::vector<int64_t> xs = { 0, W }, ys = { 0, H };
  for (const PsRegion &r : regs) {
    xs.push_back(r.ox), xs.push_back(r.ox + r.w);
    ys.push_back(r.oy), ys.push_back(r.oy + r.h);
  }
  std::sort(xs.begin(), xs.end());
  xs.erase(std::unique(xs.begin(), xs.end()), xs.end());
  std::sort(ys.begin(), ys.end());
  ys.erase(std::unique(ys.begin(), ys.end()), ys.end());
  const int K = (int)regs.size(), ncell = (int)xs.size() - 1;
  std::vector<int> ca(K), cb(K), owner(ncell), nxt(ncell + 1);
  for (int r = 0; r < K; r++) {
    ca[r] = (int)(std::lower_bound(xs.begin(), xs.end(), regs[r].ox) - xs.begin());
    cb[r] = (int)(std::lower_bound(xs.begin(), xs.end(), regs[r].ox + regs[r].w) - xs.begin());
  }
  auto find = [&](int c) {
    int root = c;
    while (nxt[root] != root) root = nxt[root];
    while (nxt[c] != root) { const int t = nxt[c]; nxt[c] = root; c = t; }
    return root;
  };
  std::vector<PsSeg> row;
  int64_t prev_off = -1, prev_cnt = 0;
  for (size_t b = 0; b + 1 < ys.size(); b++) {
    const int64_t y0 = ys[b], y1 = ys[b + 1];
    for (int c = 0; c <= ncell; c++) nxt[c] = c;
    std::fill(owner.begin(), owner.end(), -1);
    for (int r = K - 1; r >= 0; r--) {
      if (regs[r].oy > y0 || regs[r].oy + regs[r].h < y1) continue;       // the y-cuts make a region cover a band or miss it
      for (int c = find(ca[r]); c < cb[r]; c = find(c + 1)) { owner[c] = r; nxt[c] = c + 1; }
    }
    row.clear();
    for (int c = 0; c < ncell; c++) {
      PsSeg s = { xs[c] * C, 0, 0, -1, 0 };
      if (owner[c] >= 0) {
        const PsRegion &r = regs[owner[c]];
        s.src = r.src;
        s.pitch = in_shapes[(size_t)r.src * 3 + 1] * C;
        s.base = (r.iy - r.oy) * s.pitch + (r.ix - r.ox) * C;
      }
      if (!row.empty() && row.back().src == s.src && row.back().base == s.base && row.back().pitch == s.pitch) continue;
      row.push_back(s);
      if (s.src >= 0) p->used[s.src] = 1;
    }
    // a band whose segments equal the band before it continues that band
    if (prev_off >= 0 && prev_cnt == (int64_t)row.size() &&
        std::equal(row.begin(), row.end(), p->segs.begin() + prev_off, [](const PsSeg &x, const PsSeg &y) {
          return x.lo == y.lo && x.base == y.base && x.pitch == y.pitch && x.src == y.src;
        }))
      continue;
    prev_off = (int64_t)p->segs.size() - p->seg_off[i];
    prev_cnt = (int64_t)row.size();
    p->bands.push_back(PsBand{ y0, prev_off, prev_cnt });
    p->segs.insert(p->segs.end(), row.begin(), row.end());
    prev_off += p->seg_off[i];
  }
  d.nbands = (int32_t)((int64_t)p->bands.size() - p->band_off[i]);
}

inline bool PsCheckTypes(const char *op, int in_type, int *out_type, std::string *err) {
  if (in_type < 0 || in_type > 11) return ErFail(err, "%s: the input has an unsupported type (code %d)", op, in_type);
  if (*out_type < 0) *out_type = in_type;
  if (*out_type > 11) return ErFail(err, "%s: dtype has an unsupported type (code %d)", op, *out_type);
  return true;
}

// The inputs' layouts, ranks and shapes: HWC (or no layout and rank 3), one channel count, no negative extent.
inline bool PsCheckInputs(const char *op, int ninputs, int n, const int *ndims, const char *const *layouts, const int64_t *in_shapes,
                          int64_t *channels, std::string *err) {
  for (int k = 0; k < ninputs; k++) {
    const char *lay = layouts ? layouts[k] : nullptr;
    if (lay && *lay && strcmp(lay, "HWC"))
      return ErFail(err, "%s: input %d has layout \"%s\"; only HWC images (or no layout and rank 3) are supported", op, k, lay);
    if (ndims[k] != 3) return ErFail(err, "%s: input %d has %d dimensions; HWC images of rank 3 are supported", op, k, ndims[k]);
  }
  *channels = n > 0 ? in_shapes[2] : 0;
  for (int s = 0; s < ninputs * n; s++) {
    const int64_t *sh = in_shapes + (size_t)s * 3;
    if (sh[0] < 0 || sh[1] < 0 || sh[2] < 0)
      return ErFail(err, "%s: sample %d of input %d has a negative extent %s", op, s % n, s / n, ErShapeStr(sh, 3).c_str());
    if ((sh[0] && sh[1] > ((int64_t)1 << 50) / sh[0]) || (sh[0] * sh[1] && sh[2] > ((int64_t)1 << 50) / (sh[0] * sh[1])))
      return ErFail(err, "%s: sample %d of input %d has too many elements %s", op, s % n, s / n, ErShapeStr(sh, 3).c_str());
    if (sh[2] != *channels)
      return ErFail(err, "%s: sample %d of input %d has %lld channels, sample 0 of input 0 has %lld; all samples must have one channel count",
                    op, s % n, s / n, (long long)sh[2], (long long)*channels);
  }
  return true;
}

inline bool PsStart(PsPlanData *p, int n, int nsrc, int in_type, int out_type, int64_t C, const float *fill, int nfill, const char *op,
                    std::string *err) {
  if (nfill < 1) return ErFail(err, "%s: fill_value has no value", op);
  if (n > 0 && nfill != 1 && nfill != C)
    return ErFail(err, "%s: fill_value has %d values; one, or one per channel (%lld), is needed", op, nfill, (long long)C);
  p->n = n;
  p->nsrc = nsrc;
  p->in_type = in_type;
  p->out_type = out_type;
  p->osz = arith_size(out_type);
  p->nfill = nfill;
  p->samples.assign(n, PsSample());
  p->bands.clear();
  p->segs.clear();
  p->band_off.assign(n, 0);
  p->seg_off.assign(n, 0);
  p->used.assign(nsrc, 0);
  p->out_shapes.assign((size_t)n * 3, 0);
  p->items = 0;
  ErFillTable(fill, nfill, out_type, &p->fill);
  return true;
}

// One coordinate of a region argument: an absolute value must be an integer; a relative one is llround(value * extent) in double.
inline bool PsCoord(const char *op, int i, int k, int a, double v, int64_t extent, int64_t *out, std::string *err) {
  if (!std::isfinite(v)) return ErFail(err, "%s: sample %d, region %d: %s value %g is not finite", op, i, k, PsArgName(a), v);
  const bool rel = a & 1;
  if (!rel && v != std::floor(v)) return ErFail(err, "%s: sample %d, region %d: %s value %g is not an integer", op, i, k, PsArgName(a), v);
  const double x = rel ? v * (double)extent : v, lim = 4.0e18;               // beyond lim the placement checks refuse it anyway
  *out = std::llround(std::min(std::max(x, -lim), lim));
  return true;
}

// multi_paste.  in_shapes: ninputs x n samples (input-major) x (H, W, C); ndims, layouts: per input.  in_ids: NULL for the multi-input
// form, else in_id_counts[i] source indices per output, back to back.  args[a] (NULL: not given) holds arg_counts[a][i] values per
// output, (y, x) pairs region by region.  out_sizes: NULL, or n x (H, W).
inline bool PsSetup(PsPlanData *p, int in_type, int out_type, int ninputs, int n, const int *ndims, const char *const *layouts,
                    const int64_t *in_shapes, const int32_t *in_ids, const int64_t *in_id_counts, const double *const *args,
                    const int64_t *const *arg_counts, const int64_t *out_sizes, const float *fill, int nfill, std::string *err) {
  const char *op = "multi_paste";
  if (!PsCheckTypes(op, in_type, &out_type, err)) return false;
  if (in_ids && ninputs != 1) return ErFail(err, "%s: in_ids is given, so exactly one input is allowed; got %d", op, ninputs);
  if (ninputs < 1 || ninputs > kPsMaxInputs) return ErFail(err, "%s: %d inputs; 1 to %d are supported", op, ninputs, kPsMaxInputs);
  int64_t C = 0;
  if (!PsCheckInputs(op, ninputs, n, ndims, layouts, in_shapes, &C, err)) return false;
  for (int a = 0; a < kPsNumArgs; a += 2)
    if (args[a] && args[a + 1]) return ErFail(err, "%s: both %s and %s are given; give one of them", op, PsArgName(a), PsArgName(a + 1));
  if (!out_sizes)
    for (int s = 1; s < ninputs * n; s++)
      if (in_shapes[(size_t)s * 3] != in_shapes[0] || in_shapes[(size_t)s * 3 + 1] != in_shapes[1])
        return ErFail(err, "%s: output_size is not given, and sample %d of input %d has the shape %s where sample 0 of input 0 has %s; "
                      "without output_size every input sample must have one shape", op, s % n, s / n, ErShapeStr(in_shapes + (size_t)s * 3, 3).c_str(),
                      ErShapeStr(in_shapes, 3).c_str());
  if (!PsStart(p, n, ninputs * n, in_type, out_type, C, fill, nfill, op, err)) return false;
  std::vector<int64_t> voff(kPsNumArgs, 0);
  int64_t idoff = 0;
  std::vector<PsRegion> regs;
  for (int i = 0; i < n; i++) {
    const int64_t H = out_sizes ? out_sizes[2 * i] : in_shapes[0], W = out_sizes ? out_sizes[2 * i + 1] : in_shapes[1];
    if (H < 0 || W < 0) return ErFail(err, "%s: sample %d: output_size (%lld, %lld) has a negative extent", op, i, (long long)H, (long long)W);
    if (H && (W > ((int64_t)1 << 50) / H || (W && C > ((int64_t)1 << 50) / (H * W))))
      return ErFail(err, "%s: sample %d: output_size (%lld, %lld) has too many elements", op, i, (long long)H, (long long)W);
    const int64_t K = in_ids ? in_id_counts[i] : ninputs;
    for (int a = 0; a < kPsNumArgs; a++)
      if (args[a] && arg_counts[a][i] != 2 * K)
        return ErFail(err, "%s: sample %d: %s has %lld values; its %lld regions need %lld (a [%lld, 2] tensor)", op, i, PsArgName(a),
                      (long long)arg_counts[a][i], (long long)K, (long long)(2 * K), (long long)K);
    regs.clear();
    for (int64_t k = 0; k < K; k++) {
      int64_t src = in_ids ? in_ids[idoff + k] : k * n + i;
      if (in_ids && (src < 0 || src >= n))
        return ErFail(err, "%s: sample %d, region %d: in_ids %lld is not a sample of the batch of %d", op, i, (int)k, (long long)src, n);
      const int64_t Hs = in_shapes[(size_t)src * 3], Ws = in_shapes[(size_t)src * 3 + 1];
      int64_t v[3][2] = { { 0, 0 }, { 0, 0 }, { 0, 0 } };                 // in anchor, shape, out anchor: (y, x)
      int given[3] = { -1, -1, -1 };
      for (int g = 0; g < 3; g++)
        for (int a = 2 * g; a < 2 * g + 2; a++) {
          if (!args[a]) continue;
          given[g] = a;
          for (int c = 0; c < 2; c++) {
            const int64_t ext = g == 2 ? (c ? W : H) : (c ? Ws : Hs);
            if (!PsCoord(op, i, (int)k, a, args[a][voff[a] + 2 * k + c], ext, &v[g][c], err)) return false;
          }
        }
      if (given[1] < 0) v[1][0] = Hs - v[0][0], v[1][1] = Ws - v[0][1];
      const char *ina = given[0] >= 0 ? PsArgName(given[0]) : "in_anchors (default)";
      const char *shp = given[1] >= 0 ? PsArgName(given[1]) : "shapes (default)";
      const char *outa = given[2] >= 0 ? PsArgName(given[2]) : "out_anchors (default)";
      if (v[1][0] < 0 || v[1][1] < 0)
        return ErFail(err, "%s: sample %d, region %d: %s gives the extent (%lld, %lld), which is negative", op, i, (int)k, shp,
                      (long long)v[1][0], (long long)v[1][1]);
      if (v[1][0] == 0 || v[1][1] == 0) continue;                          // a zero-size region does nothing
      if (v[0][0] < 0 || v[0][1] < 0 || v[0][0] + v[1][0] > Hs || v[0][1] + v[1][1] > Ws)
        return ErFail(err, "%s: sample %d, region %d: %s (%lld, %lld) and %s (%lld, %lld) leave the source, sample %lld of input %lld (%lld x %lld)",
                      op, i, (int)k, ina, (long long)v[0][0], (long long)v[0][1], shp, (long long)v[1][0], (long long)v[1][1],
                      (long long)(src % n), (long long)(src / n), (long long)Hs, (long long)Ws);
      if (v[2][0] < 0 || v[2][1] < 0 || v[2][0] + v[1][0] > H || v[2][1] + v[1][1] > W)
        return ErFail(err, "%s: sample %d, region %d: %s (%lld, %lld) and %s (%lld, %lld) leave the output (%lld x %lld)", op, i, (int)k,
                      outa, (long long)v[2][0], (long long)v[2][1], shp, (long long)v[1][0], (long long)v[1][1], (long long)H, (long long)W);
      regs.push_back(PsRegion{ (int32_t)src, v[0][0], v[0][1], v[1][0], v[1][1], v[2][0], v[2][1] });
    }
    for (int a = 0; a < kPsNumArgs; a++)
      if (args[a]) voff[a] += arg_counts[a][i];
    if (in_ids) idoff += in_id_counts[i];
    p->out_shapes[(size_t)i * 3] = H;
    p->out_shapes[(size_t)i * 3 + 1] = W;
    p->out_shapes[(size_t)i * 3 + 2] = C;
    PsBuildOutput(p, i, H, W, C, regs, in_shapes);
  }
  return true;
}

// paste: each uint8 HWC image of n_channels channels on a canvas of H' = max(int(ratio * H), int(min_canvas_size)) rows (W' the same
// way, float products truncated), at (int(paste_y * (H' - H)), int(paste_x * (W' - W))); the rest of the canvas is fill_value.
// ratio, paste_x, paste_y, min_canvas_size: one value per sample.
inline bool PsCanvasSetup(PsPlanData *p, int in_type, int n, int ndim, const char *layout, const int64_t *in_shapes, int n_channels,
                          const float *ratio, const float *paste_x, const float *paste_y, const float *min_canvas, const float *fill,
                          int nfill, std::string *err) {
  const char *op = "paste";
  if (in_type != kAU8) return ErFail(err, "%s: the input has type code %d; paste takes UINT8 images", op, in_type);
  if (n_channels < 1) return ErFail(err, "%s: n_channels is %d; at least 1 is needed", op, n_channels);
  if (nfill != 1 && nfill != n_channels)
    return ErFail(err, "%s: fill_value has %d values; one per channel (%d), or one for all, is needed", op, nfill, n_channels);
  int64_t C = 0;
  const char *const lays[1] = { layout };
  if (!PsCheckInputs(op, 1, n, &ndim, lays, in_shapes, &C, err)) return false;
  if (n > 0 && C != n_channels) return ErFail(err, "%s: sample 0 has %lld channels, but n_channels is %d", op, (long long)C, n_channels);
  if (!PsStart(p, n, n, in_type, in_type, C, fill, nfill, op, err)) return false;
  for (int i = 0; i < n; i++) {
    const float r = ratio[i], px = paste_x[i], py = paste_y[i], mc = min_canvas[i];
    if (!(r >= 1.0f)) return ErFail(err, "%s: sample %d: ratio %g is less than 1", op, i, (double)r);
    if (!(px >= 0.0f && px <= 1.0f)) return ErFail(err, "%s: sample %d: paste_x %g is not in [0, 1]", op, i, (double)px);
    if (!(py >= 0.0f && py <= 1.0f)) return ErFail(err, "%s: sample %d: paste_y %g is not in [0, 1]", op, i, (double)py);
    if (!(mc >= 0.0f)) return ErFail(err, "%s: sample %d: min_canvas_size %g is negative", op, i, (double)mc);
    const int64_t H = in_shapes[(size_t)i * 3], W = in_shapes[(size_t)i * 3 + 1];
    const float fh = r * (float)H, fw = r * (float)W;                    // float products, as the reference computes them
    if (!(fh < 2147483648.0f && fw < 2147483648.0f && mc < 2147483648.0f))
      return ErFail(err, "%s: sample %d: the canvas of ratio %g over %lld x %lld (min_canvas_size %g) does not fit in an int", op, i, (double)r,
                    (long long)H, (long long)W, (double)mc);
    const int64_t Ho = std::max((int64_t)(int)fh, (int64_t)(int)mc), Wo = std::max((int64_t)(int)fw, (int64_t)(int)mc);
    if (Ho && (Wo > ((int64_t)1 << 50) / Ho || (Wo && C > ((int64_t)1 << 50) / (Ho * Wo))))
      return ErFail(err, "%s: sample %d: the canvas %lld x %lld has too many elements", op, i, (long long)Ho, (long long)Wo);
    if (Ho < H || Wo < W)                                                  // float rounding of a product above 2^24
      return ErFail(err, "%s: sample %d: the canvas %lld x %lld is smaller than the image %lld x %lld", op, i, (long long)Ho, (long long)Wo,
                    (long long)H, (long long)W);
    const int64_t oy = (int)(py * (float)(Ho - H)), ox = (int)(px * (float)(Wo - W));
    std::vector<PsRegion> regs;
    if (H > 0 && W > 0) regs.push_back(PsRegion{ i, 0, 0, H, W, oy, ox });
    p->out_shapes[(size_t)i * 3] = Ho;
    p->out_shapes[(size_t)i * 3 + 1] = Wo;
    p->out_shapes[(size_t)i * 3 + 2] = C;
    PsBuildOutput(p, i, Ho, Wo, C, regs, in_shapes);
  }
  return true;
}

// f(ErElem<output element size>(), std::integral_constant<bool, converting>())
template <typename F> void ps_dispatch(int osz, bool cvt, F &&f) {
  auto g = [&](auto t) {
    if (cvt) f(t, std::true_type());
    else f(t, std::false_type());
  };
  switch (osz) {
    case 1: g(ErElem<1>()); break;
    case 2: g(ErElem<2>()); break;
    case 4: g(ErElem<4>()); break;
    default: g(ErElem<8>()); break;
  }
}

// The launch of paste_kernel run on the host (tools/emul): work items in reverse order, the threads of each CTA in reverse order.
inline void PsRunOnHost(const PsSample *descs, int n, int64_t total, const PsBatch &B) {
  ps_dispatch(arith_size(B.out_type), B.in_type != B.out_type, [&](auto t, auto cvt) {
    constexpr int OSZ = (int)sizeof(typename decltype(t)::T);
    for (int64_t item = total - 1; item >= 0; item--) {
      const PsSample &d = descs[last_at_most(descs, 0, n - 1, item, [](const PsSample &e) { return e.first_item; })];
      for (int tid = kPsThreads - 1; tid >= 0; tid--) ps_item<OSZ, decltype(cvt)::value>(d, B, item - d.first_item, tid);
    }
  });
}

}  // namespace dalib200

#endif  // DALI_B200_CSRC_PASTE_PLAN_H_
