// dali_b200/csrc/equalize.cu -- fn.experimental.equalize: per-channel histogram equalization of uint8 images and sequences, the
// table of cv2.equalizeHist for every (sample, frame, channel) plane.  Per batch: the histogram scratch is zeroed, then two launches,
// equalize_hist (every work item's bytes into its frame's histogram) and equalize_apply (each item builds its frame's tables from the
// histogram and maps its bytes).  The per-thread bodies are host/device functions in equalize_core.h; the descriptors go up in one
// upload through the descriptor arena.
#include "common.cuh"
#include "equalize_plan.h"
#include <algorithm>

namespace dalib200 {

__global__ void __launch_bounds__(kEqThreads) equalize_hist_kernel(const EqSample *__restrict__ descs, int n, int64_t total,
                                                                   uint32_t *__restrict__ hist) {
  __shared__ uint32_t sh[kEqSmemWords];
  const int tid = threadIdx.x;
  for (int64_t item = blockIdx.x; item < total; item += gridDim.x) {
    const EqSample &d = descs[last_at_most(descs, 0, n - 1, item, [](const EqSample &s) { return s.first_item; })];
    const int64_t local = item - d.first_item;
    const int words = d.nsub * d.C * 256;
    for (int k = tid; k < words; k += kEqThreads) sh[k] = 0;
    __syncthreads();
    eq_hist_thread(d, local, sh + ((tid >> 5) % d.nsub) * d.C * 256, tid);
    __syncthreads();
    eq_hist_flush(d, local, sh, hist, tid);
    __syncthreads();
  }
}

__global__ void __launch_bounds__(kEqThreads) equalize_apply_kernel(const EqSample *__restrict__ descs, int n, int64_t total,
                                                                    const uint32_t *__restrict__ hist) {
  __shared__ __align__(16) uint8_t lut[kEqMaxChannels * 256];
  const int tid = threadIdx.x, lane = tid & 31;
  for (int64_t item = blockIdx.x; item < total; item += gridDim.x) {
    const EqSample &d = descs[last_at_most(descs, 0, n - 1, item, [](const EqSample &s) { return s.first_item; })];
    const int64_t local = item - d.first_item;
    const int64_t frame = eq_item(d, local).frame;
    for (int c = tid >> 5; c < d.C; c += kEqThreads / 32) {     // one warp per plane: lane l scans bins 8 l ... 8 l + 7
      const uint32_t *h = hist + d.hist_off + (frame * d.C + c) * 256;
      uint32_t s = 0;
      for (int k = 0; k < 8; k++) s += h[8 * lane + k];
      uint32_t incl = s;
      for (int off = 1; off < 32; off <<= 1) {
        const uint32_t o = __shfl_up_sync(0xFFFFFFFFu, incl, off);
        if (lane >= off) incl += o;
      }
      const uint32_t nz = __ballot_sync(0xFFFFFFFFu, s != 0);    // a plane with items has pixels: some lane holds a count
      const int fl = __ffs(nz) - 1;
      const uint32_t first = __shfl_sync(0xFFFFFFFFu, 8 * lane + eq_first_in_lane(h, lane), fl);
      eq_lut_lane(h, lane, first, h[first], d.plane, incl - s, lut + c * 256);
    }
    __syncthreads();
    eq_apply_thread(d, local, lut, tid);
    __syncthreads();
  }
}

}  // namespace dalib200

using namespace dalib200;  // NOLINT

struct dalib200EqualizePlan {
  int max_samples = 0;
  bool ready = false;
  int hist_ctas = 0, apply_ctas = 0;     // resident CTAs per SM of each kernel (at the first launch): a grid of one wave
  EqPlanData data;
  DescArena arena;
  uint32_t *hist = nullptr;
  size_t hist_cap = 0;
};

extern "C" {

int dalib200EqualizePlanCreate(dalib200EqualizePlan **plan, int max_samples) try {
  DB_CHECK_ARG(plan && max_samples > 0, "EqualizePlanCreate: bad arguments");
  auto *p = new dalib200EqualizePlan();
  p->max_samples = max_samples;
  *plan = p;
  return DALIB200_SUCCESS;
} DB_API_CATCH

int dalib200EqualizePlanDestroy(dalib200EqualizePlan *p) try {
  if (!p) return DALIB200_SUCCESS;
  p->arena.Free();
  if (p->hist) cudaFree(p->hist);
  delete p;
  return DALIB200_SUCCESS;
} DB_API_CATCH

int dalib200EqualizeSetup(dalib200EqualizePlan *p, int in_type, int n, int ndim, const int64_t *in_shapes, const char *layout) try {
  DB_CHECK_ARG(p && n >= 0 && n <= p->max_samples && (n == 0 || in_shapes),
               "EqualizeSetup: bad arguments (%d samples for a plan of %d)", n, p ? p->max_samples : 0);
  p->ready = false;
  std::string err;
  if (!EqSetup(&p->data, in_type, n, ndim, in_shapes, layout, &err)) {
    SetLastError("%s", err.c_str());
    return DALIB200_ERROR_INVALID_ARGUMENT;
  }
  p->ready = true;
  return DALIB200_SUCCESS;
} DB_API_CATCH

int dalib200EqualizeLaunch(dalib200EqualizePlan *p, const void *const *in_ptrs, void *const *out_ptrs, dalib200Stream_t stream) try {
  DB_CHECK_ARG(p && p->ready, "EqualizeLaunch: call EqualizeSetup first");
  EqPlanData &pd = p->data;
  const int n = pd.n;
  if (pd.items == 0) return DALIB200_SUCCESS;
  DB_CHECK_ARG(in_ptrs && out_ptrs, "EqualizeLaunch: bad arguments (input and output pointers are needed)");
  for (int i = 0; i < n; i++)
    DB_CHECK_ARG(pd.samples[i].items == 0 || (in_ptrs[i] && out_ptrs[i]), "experimental.Equalize: sample %d: null input or output pointer", i);
  if (p->hist_ctas == 0) {
    int h = 0, a = 0;
    DB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&h, equalize_hist_kernel, kEqThreads, 0));
    DB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&a, equalize_apply_kernel, kEqThreads, 0));
    p->hist_ctas = std::max(h, 1);
    p->apply_ctas = std::max(a, 1);
  }
  int rc = GrowDevice(p->hist, p->hist_cap, (size_t)pd.hist_words);
  if (rc) return rc;
  const size_t bytes = sizeof(EqSample) * (size_t)n;
  EqSample *h;
  if ((rc = p->arena.Stage(bytes, &h))) return rc;
  for (int i = 0; i < n; i++) {
    h[i] = pd.samples[i];
    if (h[i].items) EqBind(h[i], in_ptrs[i], out_ptrs[i]);
  }
  if ((rc = p->arena.Upload(bytes, stream))) return rc;
  const EqSample *d = reinterpret_cast<const EqSample *>(p->arena.dev);
  DB_CUDA(cudaMemsetAsync(p->hist, 0, (size_t)pd.hist_words * sizeof(uint32_t), stream));
  Launch("equalize_hist", equalize_hist_kernel, (int)std::min<int64_t>(pd.items, (int64_t)NumSMs() * p->hist_ctas), kEqThreads, 0, stream, d, n,
         pd.items, p->hist);
  DB_CUDA(cudaGetLastError());
  Launch("equalize_apply", equalize_apply_kernel, (int)std::min<int64_t>(pd.items, (int64_t)NumSMs() * p->apply_ctas), kEqThreads, 0, stream, d, n,
         pd.items, p->hist);
  DB_CUDA(cudaGetLastError());
  return DALIB200_SUCCESS;
} DB_API_CATCH

}  // extern "C"
