// dali_b200/csrc/reduce.cu -- fn.reductions.* (the reference's reductions.Min / Max / Sum / Mean / MeanSquare / RMS / StdDev /
// Variance): one batched axis reduction per operator and batch.  The planner (reduce_plan.h) turns every sample into at most three
// passes; each pass is one launch for the whole batch, followed by a combine launch when any sample of it is split.  The per-thread
// bodies are host/device functions in reduce_core.h.  All passes' descriptors go up in one upload through the descriptor arena.
#include "common.cuh"
#include "reduce_plan.h"
#include <algorithm>

namespace dalib200 {

template <typename T, typename A, int E>
__global__ void __launch_bounds__(kRedThreads) reduce_pass_kernel(const RedPass *__restrict__ descs, int n, int64_t total, RedFinal f) {
  __shared__ __align__(16) uint8_t smem[kRedSmemBytes];
  A *sm = reinterpret_cast<A *>(smem);
  A *sm2 = reinterpret_cast<A *>(smem + kRedThreads * 16 * 8);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (int64_t item = blockIdx.x; item < total; item += gridDim.x) {
    const RedPass &d = descs[last_at_most(descs, 0, n - 1, item, [](const RedPass &p) { return p.first_item; })];
    const int64_t local = item - d.first_item;
    if (d.path == kRedPathColumns) {
      red_columns<T, A, E>(d, f, local, tid);
      continue;
    }
    const RedRun u = red_run<T>(d, local);
    red_inner_fold<T, A, E>(d, u, sm, tid);
    __syncthreads();
    red_inner_slices<T, A, E>(d, u, sm, sm2, tid);
    __syncthreads();
    for (int i = warp; i < d.I; i += kRedThreads / 32) {
      A v = red_inner_lane<A, E>(d, sm2, i, lane);
      for (int off = 16; off > 0; off >>= 1) {       // the butterfly of red_tree32: lane l folds lane l + off
        const A o = __shfl_down_sync(0xFFFFFFFFu, v, off);
        v = red_comb<E, A>(v, o);
      }
      if (lane == 0) red_store(d, f, u.ch, u.o * d.I + i, v);
    }
    __syncthreads();
  }
}

template <typename A, int E>
__global__ void __launch_bounds__(kRedThreads) reduce_combine_kernel(const RedPass *__restrict__ descs, int n, int64_t total, RedFinal f) {
  for (int64_t item = blockIdx.x; item < total; item += gridDim.x) {
    const RedPass &d = descs[last_at_most(descs, 0, n - 1, item, [](const RedPass &p) { return p.cfirst; })];
    red_combine<A, E>(d, f, item - d.cfirst, threadIdx.x);
  }
}

}  // namespace dalib200

using namespace dalib200;  // NOLINT

struct dalib200ReducePlan {
  int max_samples = 0;
  bool ready = false;
  RedPlanData data;
  DescArena arena;
  uint8_t *scratch = nullptr;
  size_t scratch_cap = 0;
};

extern "C" {

int dalib200ReducePlanCreate(dalib200ReducePlan **plan, int max_samples) try {
  DB_CHECK_ARG(plan && max_samples > 0, "ReducePlanCreate: bad arguments");
  auto *p = new dalib200ReducePlan();
  p->max_samples = max_samples;
  *plan = p;
  return DALIB200_SUCCESS;
} DB_API_CATCH

int dalib200ReducePlanDestroy(dalib200ReducePlan *p) try {
  if (!p) return DALIB200_SUCCESS;
  p->arena.Free();
  if (p->scratch) cudaFree(p->scratch);
  delete p;
  return DALIB200_SUCCESS;
} DB_API_CATCH

int dalib200ReduceSetup(dalib200ReducePlan *p, int op, int in_type, int32_t *out_type, int n, int ndim, const int64_t *in_shapes,
                        uint32_t axis_mask, int keep_dims, int ddof, int64_t *out_shapes) try {
  DB_CHECK_ARG(p && out_type && n >= 0 && n <= p->max_samples && (n == 0 || ndim <= 0 || (in_shapes && out_shapes)),
               "ReduceSetup: bad arguments (%d samples for a plan of %d)", n, p ? p->max_samples : 0);
  p->ready = false;
  std::string err;
  if (!RedSetup(&p->data, op, in_type, *out_type, n, ndim, in_shapes, axis_mask, keep_dims != 0, ddof, out_shapes, &err)) {
    SetLastError("%s", err.c_str());
    return DALIB200_ERROR_INVALID_ARGUMENT;
  }
  *out_type = p->data.out_type;
  p->ready = true;
  return DALIB200_SUCCESS;
} DB_API_CATCH

int dalib200ReduceLaunch(dalib200ReducePlan *p, const void *const *in_ptrs, const void *const *mean_ptrs, void *const *out_ptrs,
                         dalib200Stream_t stream) try {
  DB_CHECK_ARG(p && p->ready, "ReduceLaunch: call ReduceSetup first");
  RedPlanData &pd = p->data;
  const int n = pd.n;
  if (pd.npass == 0) return DALIB200_SUCCESS;
  DB_CHECK_ARG(in_ptrs && out_ptrs && (pd.elem != kElemSqDev || mean_ptrs), "ReduceLaunch: bad arguments (%s needs data%s and output pointers)",
               RedOpName(pd.op), pd.elem == kElemSqDev ? ", mean" : "");
  const int es = RedTypeSize(pd.in_type);
  for (int i = 0; i < n; i++)
    DB_CHECK_ARG(pd.passes[0][i].items == 0 || ((uintptr_t)in_ptrs[i] % es == 0 && in_ptrs[i] && out_ptrs[i]),
                 "%s: sample %d: the input pointer must be a non-null multiple of the element size", RedOpName(pd.op), i);
  if (pd.scratch_bytes > 0) {
    int rc = GrowDevice(p->scratch, p->scratch_cap, (size_t)pd.scratch_bytes);
    if (rc) return rc;
  }
  const size_t bytes = sizeof(RedPass) * (size_t)n * pd.npass;
  RedPass *h;
  int rc = p->arena.Stage(bytes, &h);
  if (rc) return rc;
  for (int q = 0; q < pd.npass; q++)
    for (int i = 0; i < n; i++) {
      RedPass &d = h[(size_t)q * n + i];
      d = pd.passes[q][i];
      if (d.items) RedBind(d, q, in_ptrs[i], mean_ptrs ? mean_ptrs[i] : nullptr, out_ptrs[i], p->scratch);
    }
  if ((rc = p->arena.Upload(bytes, stream))) return rc;
  const RedFinal f = { pd.op, pd.out_type, pd.ddof, 0 };
  const int cap = NumSMs() * 8;
  static const char *const names[] = { "reduce_columns", "reduce_inner", "reduce_split" };
  for (int q = 0; q < pd.npass; q++) {
    const RedPass *d = reinterpret_cast<const RedPass *>(p->arena.dev) + (size_t)q * n;
    if (pd.items[q] > 0) {
      int kinds = 0;
      for (int i = 0; i < n; i++) if (pd.kinds[(size_t)i * kRedMaxPasses + q] >= 0) kinds |= 1 << pd.kinds[(size_t)i * kRedMaxPasses + q];
      const char *name = kinds == 1 ? names[0] : kinds == 2 ? names[1] : kinds == 4 ? names[2] : "reduce_mixed";
      const int grid = (int)std::min<int64_t>(pd.items[q], cap);
      const auto launch = [&](auto t, auto a, auto e) {
        Launch(name, reduce_pass_kernel<decltype(t), decltype(a), decltype(e)::value>, grid, kRedThreads, 0, stream, d, n, pd.items[q], f);
      };
      if (q == 0) red_dispatch(pd.in_type, pd.acc, pd.elem, launch);
      else red_dispatch(pd.acc == kAccI64 ? kRedI64 : pd.acc == kAccU64 ? kRedU64 : pd.acc == kAccF32 ? kRedF32 : kRedF64, pd.acc,
                        RedCombineElem(pd.elem), launch);
      DB_CUDA(cudaGetLastError());
    }
    if (pd.citems[q] > 0) {
      const int grid = (int)std::min<int64_t>(pd.citems[q], cap);
      const auto launch = [&](auto, auto a, auto e) {
        Launch("reduce_combine", reduce_combine_kernel<decltype(a), decltype(e)::value>, grid, kRedThreads, 0, stream, d, n, pd.citems[q], f);
      };
      red_dispatch(pd.acc == kAccI64 ? kRedI64 : pd.acc == kAccU64 ? kRedU64 : pd.acc == kAccF32 ? kRedF32 : kRedF64, pd.acc,
                   RedCombineElem(pd.elem), launch);
      DB_CUDA(cudaGetLastError());
    }
  }
  return DALIB200_SUCCESS;
} DB_API_CATCH

// the path of every (sample, pass) of the last setup (kinds: n x 3, kRedKind*: 0 columns, 1 inner, 2 split, -1 no pass) and the
// depth of each sample's floating-point accumulation tree (depths: n, may be NULL), for tests and the benchmark
int dalib200ReducePlanGetPaths(const dalib200ReducePlan *p, int32_t *kinds, int32_t *depths, int cap) try {
  DB_CHECK_ARG(p && p->ready && kinds && cap >= p->data.n, "ReducePlanGetPaths: bad arguments");
  for (size_t k = 0; k < p->data.kinds.size(); k++) kinds[k] = p->data.kinds[k];
  if (depths)
    for (int i = 0; i < p->data.n; i++) depths[i] = (int32_t)std::min<int64_t>(p->data.depths[i], INT32_MAX);
  return DALIB200_SUCCESS;
} DB_API_CATCH

}  // extern "C"
