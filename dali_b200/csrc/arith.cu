// dali_b200/csrc/arith.cu -- arithmetic expressions on DataNodes (the reference's ArithmeticGenericOp<GPUBackend>, and fn.cast) in
// one launch per expression and batch.  The planner (arith_plan.h) turns the expression into a short program; the per-element bodies
// are host/device functions in arith_core.h.  Work items of kArithItem output elements are spread over the samples as generic.cu
// spreads them; the program is copied to shared memory once per block, and the instruction switch is uniform across the block.  A thread evaluates
// kArithEpt consecutive elements with its values in registers; operands with the output's shape and the output move with one vector
// access per thread (16 bytes for 4-byte types).
#include "common.cuh"
#include "arith_plan.h"
#include <algorithm>
#include <cstring>

namespace dalib200 {

constexpr int kArithThreads = 256;

// kWide = prog.wide: programs without 64-bit values keep a 32-bit value file (fewer registers per thread)
template <bool kWide>
__global__ void __launch_bounds__(kArithThreads) arith_kernel(const ArithProgram prog, const ArithSample *__restrict__ samples, int n,
                                                               int64_t total_items) {
  __shared__ ArithProgram p;
  for (int k = threadIdx.x; k < (int)(sizeof(ArithProgram) / 4); k += blockDim.x)
    reinterpret_cast<uint32_t *>(&p)[k] = reinterpret_cast<const uint32_t *>(&prog)[k];
  __syncthreads();
  for (int64_t item = blockIdx.x; item < total_items; item += gridDim.x) {
    const ArithSample &d = samples[last_at_most(samples, 0, n - 1, item, [](const ArithSample &s) { return s.first_item; })];
    const int64_t e0 = (item - d.first_item) * kArithItem, e1 = min(d.n, e0 + kArithItem);
    for (int64_t base = e0; base < e1; base += (int64_t)kArithEpt * blockDim.x)
      arith_elements<kWide>(p, d, base, e1, threadIdx.x);
  }
}

}  // namespace dalib200

using namespace dalib200;  // NOLINT

struct dalib200ArithPlan {
  int max_batch = 0, n = 0;
  bool compiled = false, ready = false;
  ArithCompiled c;
  std::vector<ArithSample> samples;
  int64_t total_items = 0;
  DescArena arena;
};

extern "C" {

int dalib200ArithPlanCreate(dalib200ArithPlan **plan, int max_batch) try {
  DB_CHECK_ARG(plan && max_batch > 0, "ArithPlanCreate: bad arguments");
  auto *p = new dalib200ArithPlan();
  p->max_batch = max_batch;
  *plan = p;
  return DALIB200_SUCCESS;
} DB_API_CATCH

int dalib200ArithPlanDestroy(dalib200ArithPlan *p) try {
  if (!p) return DALIB200_SUCCESS;
  p->arena.Free();
  delete p;
  return DALIB200_SUCCESS;
} DB_API_CATCH

int dalib200ArithCompile(dalib200ArithPlan *p, const char *desc, int ninputs, const int32_t *in_types, const uint8_t *in_scalar,
                         const int64_t *int_consts, int nint, const double *real_consts, int nreal, int32_t *out_type) try {
  DB_CHECK_ARG(p && desc && out_type && (ninputs == 0 || in_types) && (nint == 0 || int_consts) && (nreal == 0 || real_consts),
               "ArithCompile: bad arguments");
  p->compiled = p->ready = false;
  std::string err;
  if (!ArithCompile(desc, ninputs, in_types, in_scalar, int_consts, nint, real_consts, nreal, &p->c, &err)) {
    SetLastError("arithmetic expression: %s", err.c_str());
    return DALIB200_ERROR_INVALID_ARGUMENT;
  }
  *out_type = p->c.prog.out_type;
  p->compiled = true;
  return DALIB200_SUCCESS;
} DB_API_CATCH

int dalib200ArithSetup(dalib200ArithPlan *p, int n, const int32_t *ndims, const int64_t *shapes, const void *const *scalars,
                       int64_t *out_shapes, int32_t *out_ndim) try {
  DB_CHECK_ARG(p && p->compiled && n >= 0 && n <= p->max_batch && out_shapes && out_ndim && (p->c.nin == 0 || ndims) &&
               (n == 0 || shapes), "ArithSetup: bad arguments (compile the expression first)");
  p->ready = false;
  std::string err;
  int nd = 0;
  if (!ArithSetupSamples(p->c, n, ndims, shapes, scalars, &p->samples, out_shapes, &nd, &p->total_items, &err)) {
    SetLastError("arithmetic expression: %s", err.c_str());
    return DALIB200_ERROR_INVALID_ARGUMENT;
  }
  *out_ndim = nd;
  p->n = n;
  p->ready = true;
  return DALIB200_SUCCESS;
} DB_API_CATCH

int dalib200ArithLaunch(dalib200ArithPlan *p, const void *const *in_ptrs, void *const *out_ptrs, dalib200Stream_t stream) try {
  DB_CHECK_ARG(p && p->ready && (p->n == 0 || (out_ptrs && (p->c.nin == 0 || in_ptrs))), "ArithLaunch: call ArithSetup first");
  if (p->n == 0 || p->total_items == 0) return DALIB200_SUCCESS;
  ArithSample *h;
  int rc = p->arena.Stage(sizeof(ArithSample) * p->n, &h);
  if (rc) return rc;
  for (int i = 0; i < p->n; i++) {
    h[i] = p->samples[i];
    for (int k = 0; k < p->c.nin; k++) h[i].in[k] = p->c.scalar_slot[k] >= 0 ? nullptr : in_ptrs[(size_t)i * p->c.nin + k];
    h[i].out = out_ptrs[i];
  }
  if ((rc = p->arena.Upload(sizeof(ArithSample) * p->n, stream))) return rc;
  const ArithSample *d = reinterpret_cast<const ArithSample *>(p->arena.dev);
  const int grid = (int)std::min<int64_t>(p->total_items, (int64_t)NumSMs() * 8);
  Launch("arith", p->c.prog.wide ? arith_kernel<true> : arith_kernel<false>, grid, kArithThreads, 0, stream, p->c.prog, d, p->n, p->total_items);
  DB_CUDA(cudaGetLastError());
  return DALIB200_SUCCESS;
} DB_API_CATCH

}  // extern "C"
