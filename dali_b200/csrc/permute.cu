// dali_b200/csrc/permute.cu -- fn.transpose, fn.cat and fn.stack (the reference's Transpose, Cat and Stack operators): one batched
// N-D strided copy, launched once per operator and batch.  The planner (permute_plan.h) turns every (sample, input) into one copy
// descriptor; the per-thread bodies are host/device functions in permute_core.h.  Work items (whole rows or shared-memory tiles) are
// spread over the descriptors as generic.cu spreads them, found by binary search over their first items.
#include "common.cuh"
#include "permute_plan.h"
#include <algorithm>

namespace dalib200 {

__global__ void __launch_bounds__(kPermThreads) permute_kernel(const PermDesc *__restrict__ descs, int n, int64_t total_items) {
  __shared__ __align__(16) uint8_t sm[kPermSmemBytes];
  for (int64_t item = blockIdx.x; item < total_items; item += gridDim.x) {
    const PermDesc &d = descs[last_at_most(descs, 0, n - 1, item, [](const PermDesc &p) { return p.first_item; })];
    const int64_t local = item - d.first_item;
    if (d.path == kPermPathRow) {
      const PermRowItem it = perm_row_item(d, local);
      perm_rows_prepare(d, it, reinterpret_cast<int64_t *>(sm), threadIdx.x, blockDim.x);
      __syncthreads();
      perm_rows_copy(d, it, reinterpret_cast<const int64_t *>(sm), threadIdx.x, blockDim.x);
    } else {
      const PermTile t = perm_tile_at(d, local);
      perm_tile_phase(d, t, sm, threadIdx.x, blockDim.x, false);
      __syncthreads();
      perm_tile_phase(d, t, sm, threadIdx.x, blockDim.x, true);
    }
    __syncthreads();
  }
}

}  // namespace dalib200

using namespace dalib200;  // NOLINT

struct dalib200PermutePlan {
  int max_copies = 0, n = 0, nin = 0;
  bool ready = false;
  std::vector<PermDesc> descs;
  int64_t total_items = 0;
  DescArena arena;
};

extern "C" {

int dalib200PermutePlanCreate(dalib200PermutePlan **plan, int max_copies) try {
  DB_CHECK_ARG(plan && max_copies > 0, "PermutePlanCreate: bad arguments");
  auto *p = new dalib200PermutePlan();
  p->max_copies = max_copies;
  *plan = p;
  return DALIB200_SUCCESS;
} DB_API_CATCH

int dalib200PermutePlanDestroy(dalib200PermutePlan *p) try {
  if (!p) return DALIB200_SUCCESS;
  p->arena.Free();
  delete p;
  return DALIB200_SUCCESS;
} DB_API_CATCH

int dalib200TransposeSetup(dalib200PermutePlan *p, int n, int ndim, int elem_size, const int64_t *in_shapes, const int32_t *perm,
                           int64_t *out_shapes) try {
  DB_CHECK_ARG(p && n >= 0 && n <= p->max_copies && (ndim == 0 || perm) && (n == 0 || ndim == 0 || (in_shapes && out_shapes)),
               "TransposeSetup: bad arguments");
  DB_CHECK_ARG(elem_size == 1 || elem_size == 2 || elem_size == 4 || elem_size == 8, "Transpose: elements of 1, 2, 4 or 8 bytes (got %d)", elem_size);
  p->ready = false;
  std::string err;
  if (!PermTransposeSetup(n, ndim, elem_size, in_shapes, perm, &p->descs, out_shapes, &p->total_items, &err)) {
    SetLastError("Transpose: %s", err.c_str());
    return DALIB200_ERROR_INVALID_ARGUMENT;
  }
  p->n = n; p->nin = 1; p->ready = true;
  return DALIB200_SUCCESS;
} DB_API_CATCH

int dalib200JoinSetup(dalib200PermutePlan *p, int n, int ninputs, int ndim, int elem_size, const int64_t *in_shapes, int axis, int new_axis,
                      int64_t *out_shapes) try {
  const char *op = new_axis ? "Stack" : "Cat";
  DB_CHECK_ARG(p && n >= 0 && ninputs >= 1 && (int64_t)n * ninputs <= p->max_copies && (n == 0 || ((ndim == 0 || in_shapes) && out_shapes)),
               "%s: bad arguments (%d samples x %d inputs for a plan of %d copies)", op, n, ninputs, p ? p->max_copies : 0);
  DB_CHECK_ARG(elem_size == 1 || elem_size == 2 || elem_size == 4 || elem_size == 8, "%s: elements of 1, 2, 4 or 8 bytes (got %d)", op, elem_size);
  p->ready = false;
  std::string err;
  if (!PermJoinSetup(n, ninputs, ndim, elem_size, in_shapes, axis, new_axis != 0, &p->descs, out_shapes, &p->total_items, &err)) {
    SetLastError("%s: %s", op, err.c_str());
    return DALIB200_ERROR_INVALID_ARGUMENT;
  }
  p->n = n; p->nin = ninputs; p->ready = true;
  return DALIB200_SUCCESS;
} DB_API_CATCH

int dalib200PermuteLaunch(dalib200PermutePlan *p, const void *const *in_ptrs, void *const *out_ptrs, dalib200Stream_t stream) try {
  DB_CHECK_ARG(p && p->ready && (p->n == 0 || (in_ptrs && out_ptrs)), "PermuteLaunch: call TransposeSetup or JoinSetup first");
  if (p->total_items == 0) return DALIB200_SUCCESS;
  int live = 0;
  for (const auto &d : p->descs) live += d.items > 0;
  PermDesc *h;
  int rc = p->arena.Stage(sizeof(PermDesc) * live, &h);
  if (rc) return rc;
  int kinds = 0, m = 0;
  for (size_t c = 0; c < p->descs.size(); c++) {
    if (p->descs[c].items == 0) continue;
    h[m] = p->descs[c];
    PermBind(h[m], in_ptrs[c], out_ptrs[c / p->nin]);
    kinds |= 1 << PermKindOf(h[m]);
    m++;
  }
  if ((rc = p->arena.Upload(sizeof(PermDesc) * live, stream))) return rc;
  const PermDesc *d = reinterpret_cast<const PermDesc *>(p->arena.dev);
  const int grid = (int)std::min<int64_t>(p->total_items, (int64_t)NumSMs() * 8);
  const char *name = kinds == 1 << kPermKindRows ? "permute_rows" : kinds == 1 << kPermKindTiled ? "permute_tiled"
                   : kinds == 1 << kPermKindSmall ? "permute_small" : "permute_mixed";
  Launch(name, permute_kernel, grid, kPermThreads, 0, stream, d, live, p->total_items);
  DB_CUDA(cudaGetLastError());
  return DALIB200_SUCCESS;
} DB_API_CATCH

// the path each copy of the last setup takes (kPermKind*: 0 rows, 1 tiled, 2 small), for tests and the benchmark
int dalib200PermutePlanGetPaths(const dalib200PermutePlan *p, int32_t *kinds, int cap) try {
  DB_CHECK_ARG(p && p->ready && kinds && cap >= (int)p->descs.size(), "PermutePlanGetPaths: bad arguments");
  for (size_t c = 0; c < p->descs.size(); c++) kinds[c] = p->descs[c].items == 0 ? -1 : PermKindOf(p->descs[c]);
  return DALIB200_SUCCESS;
} DB_API_CATCH

}  // extern "C"
