// dali_b200/csrc/resample3d.cu -- separable resampling of volumes (DHWC): fn.resize on 3-D data (SURVEY.md 8f rank 4).
//
// Replaces the spatial_ndim = 3 instances of the reference's GPU resampler (dali/kernels/imgproc/resample/separable_impl.h:110-203,
// resampling_batch.cu) behind ResizeBase<GPUBackend>.  Structure: the planner (resample3d_plan.h, plain C++) turns each sample into
// three passes (or one gather for pure nearest-neighbour); one launch per stage processes that stage of every sample of the batch, an
// output element per thread (resample3d_core.h: the same function the host emulation test runs), float temporaries between the stages
// in a grow-only device buffer owned by the plan.  HBM-bound streaming work: an element is read `support` times through L1/L2 (its
// neighbours along x, y or z) and written once; consecutive threads write consecutive elements.
#include "common.cuh"
#include "resample3d_plan.h"
#include <algorithm>

namespace dalib200 {

constexpr int kR3Threads = 256;

// grid: x = chunks of the largest sample of the stage (grid-stride), y = sample
__global__ void __launch_bounds__(kR3Threads) resample3d_pass_kernel(const R3Pass *__restrict__ passes, const int32_t *__restrict__ tab, int stage_stride) {
  const R3Pass p = passes[(int64_t)blockIdx.y * stage_stride];
  const int64_t step = (int64_t)gridDim.x * kR3Threads;
  for (int64_t e = (int64_t)blockIdx.x * kR3Threads + threadIdx.x; e < p.total; e += step) r3_element(p, tab, e);
}

}  // namespace dalib200

using namespace dalib200;

struct dalib200Resample3DPlan {
  int max_batch = 0, n = 0;
  int in_dtype = DALIB200_UINT8, out_dtype = DALIB200_UINT8;
  std::vector<R3SamplePlan> samples;
  std::vector<int32_t> tables;
  DescArena pass_arena, table_arena;
  float *tmp = nullptr;            // device temporaries of the whole batch
  size_t tmp_cap = 0;              // floats
  bool tables_dirty = true;
};

extern "C" {

int dalib200Resample3DPlanCreate(dalib200Resample3DPlan **plan, int max_batch) try {
  DB_CHECK_ARG(plan && max_batch > 0 && max_batch <= 65535, "Resample3DPlanCreate: bad arguments (1..65535 samples)");
  auto *p = new dalib200Resample3DPlan();
  p->max_batch = max_batch;
  *plan = p;
  return DALIB200_SUCCESS;
} DB_API_CATCH

int dalib200Resample3DPlanDestroy(dalib200Resample3DPlan *p) try {
  if (!p) return DALIB200_SUCCESS;
  p->pass_arena.Free(); p->table_arena.Free();
  if (p->tmp) cudaFree(p->tmp);
  delete p;
  return DALIB200_SUCCESS;
} DB_API_CATCH

int dalib200Resample3DPlanGetOrder(const dalib200Resample3DPlan *p, int sample, int32_t order[3]) try {
  if (!p || !order || sample < 0 || sample >= p->n) return -1;
  for (int k = 0; k < 3; k++) order[k] = p->samples[sample].order[k];
  return DALIB200_SUCCESS;
} DB_API_CATCH

int dalib200Resample3DPlanSetup(dalib200Resample3DPlan *p, int n, const dalib200Resample3DSample *samples, int in_dtype, int out_dtype) try {
  DB_CHECK_ARG(p && n >= 0 && (n == 0 || samples), "Resample3DPlanSetup: null argument");
  DB_CHECK_ARG(n <= p->max_batch, "Resample3DPlanSetup: batch %d exceeds plan capacity %d", n, p->max_batch);
  DB_CHECK_ARG((in_dtype == DALIB200_UINT8 && (out_dtype == DALIB200_UINT8 || out_dtype == DALIB200_FLOAT)) ||
               (in_dtype == DALIB200_FLOAT && out_dtype == DALIB200_FLOAT),
               "Resize (3-D): unsupported type combination in=%d out=%d (u8->u8, u8->f32, f32->f32)", in_dtype, out_dtype);
  p->n = 0;
  p->samples.assign(n, R3SamplePlan());
  p->tables.clear();
  p->tables_dirty = true;
  for (int i = 0; i < n; i++) {
    std::string err;
    int rc = PlanResample3D(samples[i], in_dtype, out_dtype, p->tables, &p->samples[i], &err);
    if (rc != DALIB200_SUCCESS) { SetLastError("Resize (3-D): sample %d: %s", i, err.c_str()); return rc; }
  }
  p->in_dtype = in_dtype; p->out_dtype = out_dtype;
  p->n = n;
  return DALIB200_SUCCESS;
} DB_API_CATCH

int dalib200Resample3DLaunch(dalib200Resample3DPlan *p, const void *const *in_ptrs, void *const *out_ptrs, dalib200Stream_t stream) try {
  DB_CHECK_ARG(p && (p->n == 0 || (in_ptrs && out_ptrs)), "Resample3DLaunch: null argument");
  const int n = p->n;
  if (n == 0) return DALIB200_SUCCESS;
  // temporaries: sample i owns [tmp_off, tmp_off + tmp_floats[0] + tmp_floats[1])
  size_t need = 0;
  for (const auto &s : p->samples) need += (size_t)s.tmp_floats[0] + (size_t)s.tmp_floats[1];
  int rc = GrowDevice(p->tmp, p->tmp_cap, need);
  if (rc) return rc;
  R3Pass *hp;
  if ((rc = p->pass_arena.Stage(sizeof(R3Pass) * 3 * (size_t)n, &hp))) return rc;
  size_t tmp_off = 0;
  int64_t stage_max[3] = { 0, 0, 0 };
  for (int i = 0; i < n; i++) {
    const R3SamplePlan &s = p->samples[i];
    float *t0 = p->tmp + tmp_off, *t1 = t0 + s.tmp_floats[0];
    tmp_off += (size_t)s.tmp_floats[0] + (size_t)s.tmp_floats[1];
    for (int k = 0; k < 3; k++) {
      R3Pass &d = hp[(size_t)i * 3 + k];
      if (k >= s.npass) { memset(&d, 0, sizeof(d)); continue; }       // total = 0: the CTAs of this sample return at once
      d = s.pass[k];
      DB_CHECK_ARG(in_ptrs[i] && out_ptrs[i], "Resample3DLaunch: sample %d: null pointer", i);
      d.in = k == 0 ? in_ptrs[i] : k == 1 ? static_cast<const void *>(t0) : static_cast<const void *>(t1);
      d.out = k == s.npass - 1 ? out_ptrs[i] : k == 0 ? static_cast<void *>(t0) : static_cast<void *>(t1);
      stage_max[k] = std::max(stage_max[k], d.total);
    }
  }
  if ((rc = p->pass_arena.Upload(sizeof(R3Pass) * 3 * (size_t)n, stream))) return rc;
  if (p->tables_dirty) {
    const size_t bytes = p->tables.size() * sizeof(int32_t);
    int32_t *ht;
    if ((rc = p->table_arena.Stage(std::max<size_t>(bytes, 16), &ht))) return rc;
    if (bytes) memcpy(ht, p->tables.data(), bytes);
    if ((rc = p->table_arena.Upload(bytes, stream))) return rc;
    p->tables_dirty = false;
  }
  const R3Pass *dp = reinterpret_cast<const R3Pass *>(p->pass_arena.dev);
  const int32_t *dt = reinterpret_cast<const int32_t *>(p->table_arena.dev);
  for (int k = 0; k < 3; k++) {
    if (stage_max[k] == 0) continue;
    const int64_t chunks = (stage_max[k] + kR3Threads - 1) / kR3Threads;
    const int gx = (int)std::min<int64_t>(chunks, std::max<int64_t>(1, (int64_t)NumSMs() * 8 / n) * 4);
    Launch("resample3d_pass", resample3d_pass_kernel, dim3(gx, n), kR3Threads, 0, stream, dp + k, dt, 3);
    DB_CUDA(cudaGetLastError());
  }
  return DALIB200_SUCCESS;
} DB_API_CATCH

}  // extern "C"
