// dali_b200/csrc/resample3d_plan.h -- host-side planning of the 3-D (DHWC) separable resampler: per sample the three passes
// (or one gather for pure nearest-neighbour), their tables and the float temporaries.  No CUDA types: resample3d.cu uploads what this
// produces; tools/emul/resample3d_emul.cc runs the same plan through resample3d_core.h on the host.
//
// Restates SeparableResamplingSetup<3>::SetupSample (dali/kernels/imgproc/resample/resampling_setup.cc:271-337): filters and ROI per
// axis (:47-122), pass order by the reference's cost search (:131-192), temporaries (:296-307), input cropped to the filter footprint
// along the non-first axes (:323-336); the passes follow SeparableResampleCPU<.., 3> (separable_cpu.h:149-249), the parity target.
// The per-axis steps (filters, ROI, pass order, crop, tables) are the 2-D plan's, from resample_axis.h.
#ifndef DALI_B200_CSRC_RESAMPLE3D_PLAN_H_
#define DALI_B200_CSRC_RESAMPLE3D_PLAN_H_
#include <cstring>
#include <string>
#include <vector>
#include "resample_axis.h"
#include "resample3d_core.h"

namespace dalib200 {

struct R3SamplePlan {
  int order[3] = { 0, 1, 2 };    // pass axes in vec numbering (0 = x, 1 = y, 2 = z)
  int npass = 0;                 // 0 (empty output), 1 (pure nearest neighbour) or 3
  R3Pass pass[3];                // in / out pointers are filled at launch
  int64_t tmp_floats[2] = { 0, 0 };   // temporaries written by pass 0 / pass 1
};

namespace r3detail {
inline bool Fit31(int64_t a, int64_t b, int64_t c, int64_t d) {
  const int64_t lim = (int64_t{1} << 31) - 1;
  int64_t v = 1;
  for (int64_t f : { a, b, c, d }) {
    if (f < 0) return false;
    if (f == 0) return true;
    if (v > lim / f) return false;
    v *= f;
  }
  return true;
}
inline int ClampIdx(int v, int n) { return v < 0 ? 0 : v > n - 1 ? n - 1 : v; }
}  // namespace r3detail

// Plans one sample; appends its tables to `tables` (int32 words; float coefficients as bits).  Returns 0 or a DALIB200_ERROR_* with `err`.
inline int PlanResample3D(const dalib200Resample3DSample &s, int in_dtype, int out_dtype, std::vector<int32_t> &tables,
                          R3SamplePlan *sp, std::string *err) {
  using namespace r3detail;
  auto fail = [&](const char *m) { if (err) *err = m; return DALIB200_ERROR_INVALID_ARGUMENT; };
  *sp = R3SamplePlan();
  memset(sp->pass, 0, sizeof(sp->pass));
  const int C = s.channels;
  if (!(s.in_shape[0] > 0 && s.in_shape[1] > 0 && s.in_shape[2] > 0 && C >= 1 && C <= 16)) return fail("unsupported input shape (extents > 0, 1..16 channels)");
  if (s.out_shape[0] < 0 || s.out_shape[1] < 0 || s.out_shape[2] < 0) return fail("negative output size");
  if (!Fit31(s.in_shape[0], s.in_shape[1], s.in_shape[2], C) || !Fit31(s.out_shape[0], s.out_shape[1], s.out_shape[2], C))
    return fail("volumes of 2^31 elements or more are not supported");
  for (int d = 0; d < 3; d++) {
    for (const dalib200FilterDesc *f : { &s.min_filter[d], &s.mag_filter[d] })
      if (!FilterDescValid(*f)) return fail("invalid filter");
    if (s.use_roi[d] && !RoiFinite(s.roi_start[d], s.roi_end[d])) return fail("the region of interest must be finite");
  }
  if (s.out_shape[0] == 0 || s.out_shape[1] == 0 || s.out_shape[2] == 0) return DALIB200_SUCCESS;
  AxisSetup ax[3];
  for (int a = 0; a < 3; a++) {          // vec axis a <- shape / params index 2 - a
    const int d = 2 - a;
    SetupAxis(ax[a], s.in_shape[d], s.out_shape[d], s.use_roi[d] != 0, s.roi_start[d], s.roi_end[d], s.min_filter[d], s.mag_filter[d]);
  }
  ProcessingOrder(ax, 3, sp->order);
  for (int a = 0; a < 3; a++) {
    CropAxis(ax[a], a == sp->order[0]);
    if (ax[a].extent <= 0) return fail("empty region of interest");
  }
  const int64_t vstride[3] = { C, (int64_t)s.in_shape[2] * C, (int64_t)s.in_shape[1] * s.in_shape[2] * C };
  const int osz[3] = { s.out_shape[2], s.out_shape[1], s.out_shape[0] };
  auto nn_map = [&](int a, float scale, int n_out, int n_in) {      // resampling_impl_cpu.h:534,552-557 (x), :550,594 (y), :623-626 (z)
    const int o = (int)tables.size();
    tables.resize(tables.size() + n_out);
    int32_t *m = tables.data() + o;
    NNIndices(m, n_out, ax[a].origin, scale, a);
    for (int i = 0; i < n_out; i++) m[i] = ClampIdx(m[i], n_in);
    return o;
  };
  const bool pure_nn = ax[0].ftype == DALIB200_FILTER_NN && ax[1].ftype == DALIB200_FILTER_NN && ax[2].ftype == DALIB200_FILTER_NN;
  auto common = [&](R3Pass &p, const int in_sz[3], const int out_sz[3]) {
    for (int a = 0; a < 3; a++) { p.osz[a] = out_sz[a]; p.isz[a] = in_sz[a]; }
    p.C = C;
    p.total = (int64_t)out_sz[0] * out_sz[1] * out_sz[2] * C;
    p.flags_off = -1; p.simd_end = 0; p.idx_off = p.coef_off = 0; p.support = 1;
  };
  int cur[3] = { ax[0].extent, ax[1].extent, ax[2].extent };
  if (pure_nn) {
    R3Pass &p = sp->pass[0];
    common(p, cur, osz);
    p.axis = -1;
    p.in_u8 = in_dtype == DALIB200_UINT8; p.out_u8 = out_dtype == DALIB200_UINT8;
    for (int a = 0; a < 3; a++) { p.in_stride[a] = vstride[a]; p.in_offset += ax[a].base * vstride[a]; }
    for (int a = 0; a < 3; a++) p.map_off[a] = nn_map(a, ax[a].scale, osz[a], cur[a]);
    sp->npass = 1;
    return DALIB200_SUCCESS;
  }
  for (int stage = 0; stage < 3; stage++) {
    const int a = sp->order[stage];
    int nxt[3] = { cur[0], cur[1], cur[2] };
    nxt[a] = osz[a];
    if (!Fit31(nxt[0], nxt[1], nxt[2], C)) return fail("an intermediate volume has 2^31 elements or more");
    R3Pass &p = sp->pass[stage];
    common(p, cur, nxt);
    p.in_u8 = stage == 0 && in_dtype == DALIB200_UINT8;
    p.out_u8 = stage == 2 && out_dtype == DALIB200_UINT8;
    if (stage == 0) { for (int b = 0; b < 3; b++) { p.in_stride[b] = vstride[b]; p.in_offset += ax[b].base * vstride[b]; } }
    else { p.in_stride[0] = C; p.in_stride[1] = (int64_t)cur[0] * C; p.in_stride[2] = (int64_t)cur[0] * cur[1] * C; }
    if (stage < 2) sp->tmp_floats[stage] = p.total;
    if (ax[a].ftype == DALIB200_FILTER_NN) {       // separable_cpu.h:219-227: ResampleNN with the other scales forced to 1
      p.axis = -1;
      for (int b = 0; b < 3; b++) p.map_off[b] = nn_map(b, b == a ? ax[b].scale : 1.0f, nxt[b], cur[b]);
    } else {
      p.axis = a;
      const int64_t words = (int64_t)osz[a] * (ax[a].support + 1);
      if (words + (int64_t)tables.size() >= kMaxTableWords) return fail("the filter tables would exceed 256 MB");
      AxisTableRef ref;
      BuildTable(tables, ref, ax[a], a);
      p.support = ref.support; p.idx_off = ref.idx_off; p.coef_off = ref.coef_off;
      if (p.out_u8) {
        if (a == 0) {
          p.flags_off = BuildHorzFlags(tables, p.idx_off, osz[0], cur[0], p.support);
        } else {
          // ResampleVert stores rows of X * C (per slice); ResampleDepth fuses x and y of the (contiguous) temporary and output
          const int64_t flat_w = a == 1 ? (int64_t)nxt[0] * C : (int64_t)nxt[0] * nxt[1] * C;
          p.simd_end = (uint32_t)(flat_w / 16 * 16);
        }
      }
    }
    cur[0] = nxt[0]; cur[1] = nxt[1]; cur[2] = nxt[2];
  }
  sp->npass = 3;
  return DALIB200_SUCCESS;
}

}  // namespace dalib200
#endif  // DALI_B200_CSRC_RESAMPLE3D_PLAN_H_
