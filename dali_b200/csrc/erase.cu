// dali_b200/csrc/erase.cu -- fn.erase: rectangular regions of images, sequences, volumes and spectrograms filled with a value (or one
// value per channel), everything else copied bit for bit.  One launch per batch, erase_kernel<element size>: each CTA takes work
// items (16-byte output slots, csrc/erase_core.h) of the whole batch.  The descriptors, the bands and interval lists of the planner
// (csrc/erase_plan.h) and the fill table go up in one upload through the descriptor arena.
#include "common.cuh"
#include "erase_plan.h"
#include <algorithm>

namespace dalib200 {

template <int ESZ>
__global__ void __launch_bounds__(kErThreads) erase_kernel(const ErSample *__restrict__ descs, int n, int64_t total,
                                                          const uint8_t *__restrict__ fill, int nfill) {
  for (int64_t item = blockIdx.x; item < total; item += gridDim.x) {
    const ErSample &d = descs[last_at_most(descs, 0, n - 1, item, [](const ErSample &s) { return s.first_item; })];
    er_item<ESZ>(d, fill, nfill, item - d.first_item, threadIdx.x);
  }
}

}  // namespace dalib200

using namespace dalib200;  // NOLINT

struct dalib200ErasePlan {
  int max_samples = 0;
  bool ready = false;
  ErPlanData data;
  DescArena arena;
};

extern "C" {

int dalib200ErasePlanCreate(dalib200ErasePlan **plan, int max_samples) try {
  DB_CHECK_ARG(plan && max_samples > 0, "ErasePlanCreate: bad arguments");
  auto *p = new dalib200ErasePlan();
  p->max_samples = max_samples;
  *plan = p;
  return DALIB200_SUCCESS;
} DB_API_CATCH

int dalib200ErasePlanDestroy(dalib200ErasePlan *p) try {
  if (!p) return DALIB200_SUCCESS;
  p->arena.Free();
  delete p;
  return DALIB200_SUCCESS;
} DB_API_CATCH

int dalib200EraseSetup(dalib200ErasePlan *p, int type, int n, int ndim, const int64_t *shapes, const char *layout, const char *axis_names,
                       const int32_t *axes, int naxes, const float *anchors, const int64_t *anchor_counts, const float *region_shapes,
                       const int64_t *shape_counts, int normalized_anchor, int normalized_shape, int centered_anchor, const float *fill,
                       int nfill) try {
  DB_CHECK_ARG(p && n >= 0 && n <= p->max_samples && (n == 0 || (shapes && anchor_counts && shape_counts)) &&
               (axis_names || naxes <= 0 || axes) && (nfill <= 0 || fill),
               "EraseSetup: bad arguments (%d samples for a plan of %d)", n, p ? p->max_samples : 0);
  p->ready = false;
  int64_t values = 0;
  for (int i = 0; i < n; i++) {
    DB_CHECK_ARG(anchor_counts[i] >= 0 && shape_counts[i] >= 0, "erase: sample %d: negative anchor or shape count", i);
    values += std::max(anchor_counts[i], shape_counts[i]);
  }
  DB_CHECK_ARG(values == 0 || (anchors && region_shapes), "EraseSetup: bad arguments (anchor and shape values are needed)");
  std::string err;
  if (!ErSetup(&p->data, type, n, ndim, shapes, layout, axis_names, axes, naxes, anchors, anchor_counts, region_shapes, shape_counts,
               normalized_anchor, normalized_shape, centered_anchor, fill, nfill, &err)) {
    SetLastError("%s", err.c_str());
    return DALIB200_ERROR_INVALID_ARGUMENT;
  }
  p->ready = true;
  return DALIB200_SUCCESS;
} DB_API_CATCH

int dalib200EraseLaunch(dalib200ErasePlan *p, const void *const *in_ptrs, void *const *out_ptrs, dalib200Stream_t stream) try {
  DB_CHECK_ARG(p && p->ready, "EraseLaunch: call EraseSetup first");
  ErPlanData &pd = p->data;
  const int n = pd.n;
  if (pd.items == 0) return DALIB200_SUCCESS;
  DB_CHECK_ARG(in_ptrs && out_ptrs, "EraseLaunch: bad arguments (input and output pointers are needed)");
  const size_t esz = (size_t)pd.esz;
  for (int i = 0; i < n; i++) {
    if (pd.samples[i].items == 0) continue;
    DB_CHECK_ARG(in_ptrs[i] && out_ptrs[i], "erase: sample %d: null input or output pointer", i);
    // the kernel reads and writes whole elements: a device address must be a multiple of its element's size
    DB_CHECK_ARG((uintptr_t)in_ptrs[i] % esz == 0 && (uintptr_t)out_ptrs[i] % esz == 0,
                 "erase: sample %d: a device pointer is not aligned to its element size", i);
  }
  // one upload: the descriptors, the fill table, the bands and the intervals, each at a 16-byte boundary
  const size_t fill_at = Align(sizeof(ErSample) * (size_t)n, 16), bands_at = Align(fill_at + pd.fill.size(), 16),
               ivals_at = Align(bands_at + sizeof(ErBand) * pd.bands.size(), 16), bytes = ivals_at + sizeof(ErIval) * pd.ivals.size();
  uint8_t *h;
  int rc = p->arena.Stage(bytes, &h);
  if (rc) return rc;
  memcpy(h + fill_at, pd.fill.data(), pd.fill.size());
  if (!pd.bands.empty()) memcpy(h + bands_at, pd.bands.data(), sizeof(ErBand) * pd.bands.size());
  if (!pd.ivals.empty()) memcpy(h + ivals_at, pd.ivals.data(), sizeof(ErIval) * pd.ivals.size());
  ErSample *hd = reinterpret_cast<ErSample *>(h);
  for (int i = 0; i < n; i++) {
    hd[i] = pd.samples[i];
    if (!hd[i].items) continue;
    hd[i].in = in_ptrs[i];
    hd[i].out = out_ptrs[i];
    hd[i].bands = reinterpret_cast<const ErBand *>(p->arena.dev + bands_at) + pd.band_off[i];
    hd[i].ivals = reinterpret_cast<const ErIval *>(p->arena.dev + ivals_at) + pd.ival_off[i];
  }
  if ((rc = p->arena.Upload(bytes, stream))) return rc;
  const ErSample *d = reinterpret_cast<const ErSample *>(p->arena.dev);
  const uint8_t *fill = p->arena.dev + fill_at;
  bool ok = true;
  er_dispatch(pd.esz, [&](auto t) {
    constexpr int ESZ = (int)sizeof(typename decltype(t)::T);
    auto kernel = erase_kernel<ESZ>;
    int per_sm = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, kErThreads, 0) != cudaSuccess) { ok = false; return; }
    const int grid = (int)std::min<int64_t>(pd.items, (int64_t)NumSMs() * std::max(per_sm, 1));
    Launch("erase", kernel, grid, kErThreads, 0, stream, d, n, pd.items, fill, pd.nfill);
  });
  DB_CHECK_ARG(ok, "erase: cannot query the kernel's occupancy");
  DB_CUDA(cudaGetLastError());
  return DALIB200_SUCCESS;
} DB_API_CATCH

}  // extern "C"
