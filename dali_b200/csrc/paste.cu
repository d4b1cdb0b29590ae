// dali_b200/csrc/paste.cu -- fn.multi_paste and fn.paste: each output built from rectangles of input samples, later ones on top, the
// rest a fill (0 for multi_paste, one value per channel for paste).  One launch per batch, paste_kernel<output element size,
// converting>: each CTA takes work items (16-byte output slots, csrc/paste_core.h) of the whole batch.  The descriptors, the input
// pointers, the fill table and the bands and segments of the planner (csrc/paste_plan.h) go up in one upload through the descriptor
// arena.
#include "common.cuh"
#include "paste_plan.h"
#include <algorithm>

namespace dalib200 {

template <int OSZ, bool CVT>
__global__ void __launch_bounds__(kPsThreads, 4) paste_kernel(const PsSample *__restrict__ descs, int n, int64_t total, PsBatch batch) {
  for (int64_t item = blockIdx.x; item < total; item += gridDim.x) {
    const PsSample &d = descs[last_at_most(descs, 0, n - 1, item, [](const PsSample &s) { return s.first_item; })];
    ps_item<OSZ, CVT>(d, batch, item - d.first_item, threadIdx.x);
  }
}

}  // namespace dalib200

using namespace dalib200;  // NOLINT

struct dalib200PastePlan {
  int max_samples = 0;
  bool ready = false;
  PsPlanData data;
  DescArena arena;
};

extern "C" {

int dalib200PastePlanCreate(dalib200PastePlan **plan, int max_samples) try {
  DB_CHECK_ARG(plan && max_samples > 0, "PastePlanCreate: bad arguments");
  auto *p = new dalib200PastePlan();
  p->max_samples = max_samples;
  *plan = p;
  return DALIB200_SUCCESS;
} DB_API_CATCH

int dalib200PastePlanDestroy(dalib200PastePlan *p) try {
  if (!p) return DALIB200_SUCCESS;
  p->arena.Free();
  delete p;
  return DALIB200_SUCCESS;
} DB_API_CATCH

int dalib200PasteSetup(dalib200PastePlan *p, int in_type, int out_type, int ninputs, int n, const int *ndims, const char *const *layouts,
                       const int64_t *in_shapes, const int32_t *in_ids, const int64_t *in_id_counts, const double *const *region_args,
                       const int64_t *const *region_counts, const int64_t *output_sizes, const float *fill, int nfill,
                       int64_t *out_shapes) try {
  DB_CHECK_ARG(p && n >= 0 && n <= p->max_samples && ninputs >= 1 && ndims && region_args && region_counts && (nfill <= 0 || fill) &&
               (n == 0 || (in_shapes && out_shapes)) && (!in_ids || in_id_counts),
               "PasteSetup: bad arguments (%d samples for a plan of %d)", n, p ? p->max_samples : 0);
  p->ready = false;
  for (int a = 0; a < kPsNumArgs; a++) DB_CHECK_ARG(!region_args[a] || region_counts[a], "PasteSetup: bad arguments (%s needs its counts)", PsArgName(a));
  for (int i = 0; i < n; i++) {
    DB_CHECK_ARG(!in_ids || in_id_counts[i] >= 0, "multi_paste: sample %d: negative in_ids count", i);
    for (int a = 0; a < kPsNumArgs; a++) DB_CHECK_ARG(!region_args[a] || region_counts[a][i] >= 0, "multi_paste: sample %d: negative %s count", i, PsArgName(a));
  }
  std::string err;
  if (!PsSetup(&p->data, in_type, out_type, ninputs, n, ndims, layouts, in_shapes, in_ids, in_id_counts, region_args, region_counts,
               output_sizes, fill, nfill, &err)) {
    SetLastError("%s", err.c_str());
    return DALIB200_ERROR_INVALID_ARGUMENT;
  }
  std::copy(p->data.out_shapes.begin(), p->data.out_shapes.end(), out_shapes);
  p->ready = true;
  return DALIB200_SUCCESS;
} DB_API_CATCH

int dalib200PasteCanvasSetup(dalib200PastePlan *p, int in_type, int n, int ndim, const char *layout, const int64_t *in_shapes, int n_channels,
                             const float *ratio, const float *paste_x, const float *paste_y, const float *min_canvas_size, const float *fill,
                             int nfill, int64_t *out_shapes) try {
  DB_CHECK_ARG(p && n >= 0 && n <= p->max_samples && (nfill <= 0 || fill) &&
               (n == 0 || (in_shapes && ratio && paste_x && paste_y && min_canvas_size && out_shapes)),
               "PasteCanvasSetup: bad arguments (%d samples for a plan of %d)", n, p ? p->max_samples : 0);
  p->ready = false;
  std::string err;
  if (!PsCanvasSetup(&p->data, in_type, n, ndim, layout, in_shapes, n_channels, ratio, paste_x, paste_y, min_canvas_size, fill, nfill,
                     &err)) {
    SetLastError("%s", err.c_str());
    return DALIB200_ERROR_INVALID_ARGUMENT;
  }
  std::copy(p->data.out_shapes.begin(), p->data.out_shapes.end(), out_shapes);
  p->ready = true;
  return DALIB200_SUCCESS;
} DB_API_CATCH

int dalib200PasteLaunch(dalib200PastePlan *p, const void *const *in_ptrs, void *const *out_ptrs, dalib200Stream_t stream) try {
  DB_CHECK_ARG(p && p->ready, "PasteLaunch: call PasteSetup first");
  PsPlanData &pd = p->data;
  const int n = pd.n;
  if (pd.items == 0) return DALIB200_SUCCESS;
  DB_CHECK_ARG(in_ptrs && out_ptrs, "PasteLaunch: bad arguments (input and output pointers are needed)");
  // the kernel reads and writes whole elements: a device address must be a multiple of its element's size
  const size_t isz = (size_t)arith_size(pd.in_type), osz = (size_t)pd.osz;
  for (int s = 0; s < pd.nsrc; s++) {
    if (!pd.used[s]) continue;
    DB_CHECK_ARG(in_ptrs[s], "paste: sample %d of input %d: null input pointer", s % n, s / n);
    DB_CHECK_ARG((uintptr_t)in_ptrs[s] % isz == 0, "paste: sample %d of input %d: the input pointer is not aligned to its element size",
                 s % n, s / n);
  }
  for (int i = 0; i < n; i++) {
    if (pd.samples[i].items == 0) continue;
    DB_CHECK_ARG(out_ptrs[i], "paste: sample %d: null output pointer", i);
    DB_CHECK_ARG((uintptr_t)out_ptrs[i] % osz == 0, "paste: sample %d: the output pointer is not aligned to its element size", i);
  }
  // one upload: the descriptors, the input pointers, the fill table, the bands and the segments, each at a 16-byte boundary
  const size_t srcs_at = Align(sizeof(PsSample) * (size_t)n, 16), fill_at = Align(srcs_at + sizeof(void *) * (size_t)pd.nsrc, 16),
               bands_at = Align(fill_at + pd.fill.size(), 16), segs_at = Align(bands_at + sizeof(PsBand) * pd.bands.size(), 16),
               bytes = segs_at + sizeof(PsSeg) * pd.segs.size();
  uint8_t *h;
  int rc = p->arena.Stage(bytes, &h);
  if (rc) return rc;
  memcpy(h + srcs_at, in_ptrs, sizeof(void *) * (size_t)pd.nsrc);
  memcpy(h + fill_at, pd.fill.data(), pd.fill.size());
  memcpy(h + bands_at, pd.bands.data(), sizeof(PsBand) * pd.bands.size());
  memcpy(h + segs_at, pd.segs.data(), sizeof(PsSeg) * pd.segs.size());
  PsSample *hd = reinterpret_cast<PsSample *>(h);
  for (int i = 0; i < n; i++) {
    hd[i] = pd.samples[i];
    if (!hd[i].items) continue;
    hd[i].out = out_ptrs[i];
    hd[i].bands = reinterpret_cast<const PsBand *>(p->arena.dev + bands_at) + pd.band_off[i];
    hd[i].segs = reinterpret_cast<const PsSeg *>(p->arena.dev + segs_at) + pd.seg_off[i];
  }
  if ((rc = p->arena.Upload(bytes, stream))) return rc;
  const PsSample *d = reinterpret_cast<const PsSample *>(p->arena.dev);
  PsBatch batch;
  batch.srcs = reinterpret_cast<const void *const *>(p->arena.dev + srcs_at);
  batch.fill = p->arena.dev + fill_at;
  batch.nfill = pd.nfill;
  batch.in_type = pd.in_type;
  batch.out_type = pd.out_type;
  batch.pad = 0;
  bool ok = true;
  ps_dispatch(pd.osz, pd.in_type != pd.out_type, [&](auto t, auto cvt) {
    constexpr int OSZ = (int)sizeof(typename decltype(t)::T);
    auto kernel = paste_kernel<OSZ, decltype(cvt)::value>;
    int per_sm = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, kPsThreads, 0) != cudaSuccess) { ok = false; return; }
    const int grid = (int)std::min<int64_t>(pd.items, (int64_t)NumSMs() * std::max(per_sm, 1));
    Launch("paste", kernel, grid, kPsThreads, 0, stream, d, n, pd.items, batch);
  });
  DB_CHECK_ARG(ok, "paste: cannot query the kernel's occupancy");
  DB_CUDA(cudaGetLastError());
  return DALIB200_SUCCESS;
} DB_API_CATCH

}  // extern "C"
