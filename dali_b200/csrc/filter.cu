// dali_b200/csrc/filter.cu -- fn.experimental.filter: batched 2-D correlation of images and sequences with one float32 filter per sample,
// every border mode and both output modes.  One launch per batch, filter_kernel<input type, output type>: each CTA takes work items
// (output strips, csrc/filter_core.h) of the whole batch, loads the input rows of its strip into shared memory and accumulates
// kFltRows x kFltElems outputs per thread.  The descriptors, and the filters and fill values given in host memory, go up in one upload
// through the descriptor arena; filters and fill values in device memory are read in place.
#include "common.cuh"
#include "filter_plan.h"
#include <algorithm>

namespace dalib200 {

static_assert(DALIB200_FILTER_BORDER_REFLECT_101 == kFltReflect101 && DALIB200_FILTER_BORDER_REFLECT_1001 == kFltReflect1001 &&
              DALIB200_FILTER_BORDER_WRAP == kFltWrap && DALIB200_FILTER_BORDER_CLAMP == kFltClamp &&
              DALIB200_FILTER_BORDER_CONSTANT == kFltConstant && DALIB200_FILTER_SAME == kFltSame && DALIB200_FILTER_VALID == kFltValid,
              "the C-ABI's filter enums are the planner's");

template <typename TI, typename TO>
__global__ void __launch_bounds__(kFltThreads) filter_kernel(const FltSample *__restrict__ descs, int n, int64_t total, int row_floats,
                                                             int chunk) {
  extern __shared__ __align__(16) float flt_smem[];
  __shared__ FltRowMap maps[kFltMaxChunk];
  float *const taps_sh = flt_smem + chunk * row_floats;
  const int tid = threadIdx.x;
  for (int64_t item = blockIdx.x; item < total; item += gridDim.x) {
    const FltSample &d = descs[last_at_most(descs, 0, n - 1, item, [](const FltSample &s) { return s.first_item; })];
    const FltStrip st = flt_strip(d, item - d.first_item);
    const int ntaps = d.fh * d.fw;
    const float *taps = d.filter;
    if (ntaps <= kFltSmemTaps) {
      for (int k = tid; k < ntaps; k += kFltThreads) taps_sh[k] = __ldg(d.filter + k);
      taps = taps_sh;
    }
    float acc[kFltRows][kFltElems];
#pragma unroll
    for (int t = 0; t < kFltRows; t++)
#pragma unroll
      for (int k = 0; k < kFltElems; k++) acc[t][k] = 0.0f;
    const int nrows = min(kFltRows, d.Ho - st.y0) + d.fh - 1;
    for (int j0 = 0; j0 < nrows; j0 += chunk) {              // one chunk for small filters: every load of the strip in flight at once
      const int kn = min(chunk, nrows - j0);
      if (tid < kn) maps[tid] = flt_row_map<TI>(d, st, j0 + tid);
      __syncthreads();
      flt_load_groups<TI>(d, st, maps, kn, flt_smem, row_floats, tid);
      flt_load_edges<TI>(d, st, maps, kn, flt_smem, row_floats, tid);
      __syncthreads();
      for (int q = 0; q < kn; q++) flt_accum_row(d, taps, j0 + q, flt_smem + q * row_floats + maps[q].sh, acc, tid);
      __syncthreads();                                        // before the next chunk or item overwrites the rows, maps and taps
    }
    flt_store<TO>(d, st, acc, tid);
  }
}

}  // namespace dalib200

using namespace dalib200;  // NOLINT

struct dalib200FilterPlan {
  int max_samples = 0;
  bool ready = false;
  FltPlanData data;
  DescArena arena;
};

extern "C" {

int dalib200FilterPlanCreate(dalib200FilterPlan **plan, int max_samples) try {
  DB_CHECK_ARG(plan && max_samples > 0, "FilterPlanCreate: bad arguments");
  auto *p = new dalib200FilterPlan();
  p->max_samples = max_samples;
  *plan = p;
  return DALIB200_SUCCESS;
} DB_API_CATCH

int dalib200FilterPlanDestroy(dalib200FilterPlan *p) try {
  if (!p) return DALIB200_SUCCESS;
  p->arena.Free();
  delete p;
  return DALIB200_SUCCESS;
} DB_API_CATCH

int dalib200FilterSetup(dalib200FilterPlan *p, int in_type, int out_type, int n, int ndim, const int64_t *in_shapes, const char *layout,
                        int filter_type, int filter_ndim, const int64_t *filter_shapes, const int32_t *anchors, int border, int mode,
                        int fill_type, const int64_t *fill_counts, int64_t *out_shapes) try {
  DB_CHECK_ARG(p && n >= 0 && n <= p->max_samples && (n == 0 || (in_shapes && filter_shapes && out_shapes)) &&
               (fill_type < 0 || n == 0 || fill_counts),
               "FilterSetup: bad arguments (%d samples for a plan of %d)", n, p ? p->max_samples : 0);
  p->ready = false;
  std::string err;
  if (!FltSetup(&p->data, in_type, out_type, n, ndim, in_shapes, layout, filter_type, filter_ndim, filter_shapes, anchors, border, mode,
                fill_type, fill_counts, out_shapes, &err)) {
    SetLastError("%s", err.c_str());
    return DALIB200_ERROR_INVALID_ARGUMENT;
  }
  p->ready = true;
  return DALIB200_SUCCESS;
} DB_API_CATCH

int dalib200FilterLaunch(dalib200FilterPlan *p, const void *const *in_ptrs, const void *const *filters, int filters_on_device,
                         const void *const *fills, int fills_on_device, void *const *out_ptrs, dalib200Stream_t stream) try {
  DB_CHECK_ARG(p && p->ready, "FilterLaunch: call FilterSetup first");
  FltPlanData &pd = p->data;
  const int n = pd.n;
  if (pd.items == 0) return DALIB200_SUCCESS;
  DB_CHECK_ARG(in_ptrs && out_ptrs && filters, "FilterLaunch: bad arguments (input, filter and output pointers are needed)");
  DB_CHECK_ARG(!pd.has_fill || fills, "FilterLaunch: the plan was set up with fill values, but none are given");
  const size_t esz = (size_t)FltTypeSize(pd.in_type), osz = (size_t)FltTypeSize(pd.out_type);
  for (int i = 0; i < n; i++) {
    if (pd.samples[i].items == 0) continue;
    DB_CHECK_ARG(in_ptrs[i] && out_ptrs[i] && filters[i] && (!pd.has_fill || fills[i]),
                 "experimental.Filter: sample %d: null input, filter, fill or output pointer", i);
    // the kernel reads and writes whole elements: a device address must be a multiple of its element's size
    DB_CHECK_ARG((uintptr_t)in_ptrs[i] % esz == 0 && (uintptr_t)out_ptrs[i] % osz == 0 &&
                 (!filters_on_device || (uintptr_t)filters[i] % sizeof(float) == 0) &&
                 (!pd.has_fill || !fills_on_device || (uintptr_t)fills[i] % esz == 0),
                 "experimental.Filter: sample %d: a device pointer is not aligned to its element size", i);
  }
  // one upload: the descriptors, then the filters and fill values that are in host memory, each at a 16-byte boundary
  size_t bytes = Align(sizeof(FltSample) * (size_t)n, 16);
  std::vector<size_t> foff(n, 0), voff(n, 0);
  for (int i = 0; i < n; i++) {
    if (!pd.samples[i].items) continue;
    if (!filters_on_device) { foff[i] = bytes; bytes = Align(bytes + sizeof(float) * (size_t)pd.filter_elems[i], 16); }
    if (pd.has_fill && !fills_on_device) { voff[i] = bytes; bytes = Align(bytes + esz * (size_t)pd.fill_elems[i], 16); }
  }
  uint8_t *h;
  int rc = p->arena.Stage(bytes, &h);
  if (rc) return rc;
  FltSample *hd = reinterpret_cast<FltSample *>(h);
  for (int i = 0; i < n; i++) {
    hd[i] = pd.samples[i];
    if (!hd[i].items) continue;
    hd[i].in = in_ptrs[i];
    hd[i].out = out_ptrs[i];
    if (filters_on_device) {
      hd[i].filter = static_cast<const float *>(filters[i]);
    } else {
      memcpy(h + foff[i], filters[i], sizeof(float) * (size_t)pd.filter_elems[i]);
      hd[i].filter = reinterpret_cast<const float *>(p->arena.dev + foff[i]);
    }
    if (pd.has_fill && fills_on_device) {
      hd[i].fill = fills[i];
    } else if (pd.has_fill) {
      memcpy(h + voff[i], fills[i], esz * (size_t)pd.fill_elems[i]);
      hd[i].fill = p->arena.dev + voff[i];
    }
  }
  if ((rc = p->arena.Upload(bytes, stream))) return rc;
  const FltSample *d = reinterpret_cast<const FltSample *>(p->arena.dev);
  const size_t smem = pd.smem_bytes();
  bool ok = true;
  flt_dispatch(pd.in_type, pd.out_type, [&](auto ti, auto to) {
    auto kernel = filter_kernel<decltype(ti), decltype(to)>;
    int per_sm = 0;
    if (smem > 48 * 1024 && cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) ok = false;
    if (ok && cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, kFltThreads, smem) != cudaSuccess) ok = false;
    if (!ok) return;
    const int grid = (int)std::min<int64_t>(pd.items, (int64_t)NumSMs() * std::max(per_sm, 1));
    Launch("filter", kernel, grid, kFltThreads, smem, stream, d, n, pd.items, pd.row_floats, pd.chunk);
  });
  DB_CHECK_ARG(ok, "experimental.Filter: cannot launch with %zu bytes of shared memory", smem);
  DB_CUDA(cudaGetLastError());
  return DALIB200_SUCCESS;
} DB_API_CATCH

}  // extern "C"
