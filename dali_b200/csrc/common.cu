// dali_b200/csrc/common.cu -- error state, descriptor arena, launch accounting.
#include "common.cuh"
#include <algorithm>
#include <mutex>
#include <nvtx3/nvToolsExt.h>
#include <cstring>

namespace dalib200 {

static thread_local std::string tls_error;
std::atomic<uint64_t> g_launch_count{0};

void SetLastError(const char *fmt, ...) {
  char buf[1024];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  tls_error = buf;
}

int PinnedStage::Grow(size_t bytes, uint8_t **dev) {
  if (pending_) { DB_CUDA(cudaEventSynchronize(uploaded_)); pending_ = false; }
  if (bytes <= cap_) return DALIB200_SUCCESS;
  size_t ncap = cap_ ? cap_ : 4096;
  while (ncap < bytes) ncap *= 2;
  uint8_t *nh = nullptr, *nd = nullptr;
  DB_CUDA(cudaMallocHost(reinterpret_cast<void **>(&nh), ncap));
  if (dev) {
    cudaError_t e = cudaMalloc(reinterpret_cast<void **>(&nd), ncap);
    if (e != cudaSuccess) { cudaFreeHost(nh); DB_CUDA(e); }
    // NOTE: a previous launch may still be reading the old device arena; cudaFree synchronises the
    // device implicitly, so growing is safe (it only happens while shapes are still warming up).
    if (*dev) cudaFree(*dev);
    *dev = nd;
  }
  if (host_) cudaFreeHost(host_);
  host_ = nh; cap_ = ncap;
  return DALIB200_SUCCESS;
}

int PinnedStage::Record(cudaStream_t s) {
  cudaError_t e = uploaded_ ? cudaSuccess : cudaEventCreateWithFlags(&uploaded_, cudaEventDisableTiming);
  if (e == cudaSuccess) e = cudaEventRecord(uploaded_, s);
  if (e != cudaSuccess) cudaStreamSynchronize(s);       // nothing to wait on later: the copies must be over before the buffer is reused
  DB_CUDA(e);
  pending_ = true;
  return DALIB200_SUCCESS;
}

void PinnedStage::Free() {
  if (uploaded_) { cudaEventSynchronize(uploaded_); cudaEventDestroy(uploaded_); }
  if (host_) cudaFreeHost(host_);
  host_ = nullptr; cap_ = 0; uploaded_ = nullptr; pending_ = false;
}

int DescArena::Upload(size_t bytes, cudaStream_t s) {
  if (bytes == 0) return DALIB200_SUCCESS;
  DB_CUDA(cudaMemcpyAsync(dev, host_, bytes, cudaMemcpyHostToDevice, s));
  return Record(s);
}

void DescArena::Free() {
  PinnedStage::Free();
  if (dev) cudaFree(dev);
  dev = nullptr;
}

int NumSMs() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0)
      n = 132;
  }
  return n;
}

SerialLanes SerialLaneGeometry(int nchains, int max_workers) {
  const int resident = NumSMs() * 32;                         // one-warp CTAs: at most 32 resident per SM
  SerialLanes g;
  g.lanes = std::max(1, std::min(32, (nchains + resident - 1) / resident));
  g.warps = std::max(1, std::min((nchains + g.lanes - 1) / g.lanes, std::min(resident, max_workers / g.lanes)));
  return g;
}

// ---------------------------------------------------------------------------------------------
static bool g_prof_on = false;
struct ProfRec { const char *name; cudaEvent_t a, b; };
static std::vector<ProfRec> g_prof;
static std::vector<cudaEvent_t> g_prof_pool;
static std::mutex g_prof_mutex;                        // several pipelines (one host thread each) may launch concurrently
static thread_local std::vector<size_t> tls_prof_open;  // indices of this thread's open records
static cudaEvent_t ProfEvent() {
  if (!g_prof_pool.empty()) { cudaEvent_t e = g_prof_pool.back(); g_prof_pool.pop_back(); return e; }
  cudaEvent_t e = nullptr;
  cudaEventCreate(&e);
  return e;
}
// NVTX range around every kernel launch (header-only nvtx3: a no-op unless a tool such as nsys / ncu injects the library), like the
// reference's DomainTimeRange around operator Setup / Run (dali/pipeline/executor/executor2/exec_node_task.cc:291,314,
// include/dali/core/nvtx.h:37-100).
void ProfBegin(const char *name, cudaStream_t s) {
  nvtxRangePushA(name);
  if (!g_prof_on) return;
  std::lock_guard<std::mutex> lock(g_prof_mutex);
  ProfRec r{name, ProfEvent(), ProfEvent()};
  cudaEventRecord(r.a, s);
  tls_prof_open.push_back(g_prof.size());
  g_prof.push_back(r);
}
void ProfEnd(cudaStream_t s) {
  nvtxRangePop();
  if (!g_prof_on || tls_prof_open.empty()) return;
  std::lock_guard<std::mutex> lock(g_prof_mutex);
  const size_t i = tls_prof_open.back();
  tls_prof_open.pop_back();
  if (i < g_prof.size()) cudaEventRecord(g_prof[i].b, s);
}

}  // namespace dalib200

namespace dalib200 {
__global__ void half_cvt_check_kernel(unsigned long long *mismatches) {
  unsigned long long bad = 0;
  for (uint64_t v = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; v < (1ull << 32); v += (uint64_t)gridDim.x * blockDim.x) {
    const float f = __uint_as_float((uint32_t)v);
    bad += float2half_ties_away(f) != float2half_ties_away_ref(f);
    // round_u8_bits is used for values in (-0.5, 255.5) only
    if (f > -0.4999f && f < 255.4999f) bad += (round_u8_bits(f) & 0xFFu) != (uint32_t)sat_u8_half_away(f);
  }
  if (bad) atomicAdd(mismatches, bad);
}
}  // namespace dalib200

extern "C" {

// Test hook: compares the hardware-assisted float -> half (ties away) conversion of the kernels with the integer restatement of
// include/dali/util/half.hpp on ALL 2^32 float bit patterns; *mismatches must come back 0.
int dalib200DebugCheckHalfConversion(uint64_t *mismatches) try {
  DB_CHECK_ARG(mismatches, "DebugCheckHalfConversion: null pointer");
  unsigned long long *d = nullptr;
  DB_CUDA(cudaMalloc(reinterpret_cast<void **>(&d), 8));
  DB_CUDA(cudaMemset(d, 0, 8));
  dalib200::Launch("half_cvt_check", dalib200::half_cvt_check_kernel, dalib200::NumSMs() * 8, 256, 0, nullptr, d);
  unsigned long long h = 0;
  const cudaError_t e = cudaMemcpy(&h, d, 8, cudaMemcpyDeviceToHost);
  cudaFree(d);
  DB_CUDA(e);
  *mismatches = h;
  return DALIB200_SUCCESS;
} DB_API_CATCH

int dalib200HostAlloc(void **ptr, size_t bytes) try {
  DB_CHECK_ARG(ptr, "HostAlloc: null pointer");
  *ptr = nullptr;
  if (bytes == 0) return DALIB200_SUCCESS;
  DB_CUDA(cudaHostAlloc(ptr, bytes, cudaHostAllocDefault));
  return DALIB200_SUCCESS;
} DB_API_CATCH

// The same for a caller thread whose current device is not the consumer's (e.g. a reader's read-ahead thread, whose thread-local
// current device is still 0): the allocation is made with `device` current -- no context is created on another GPU as a side effect
// -- and is portable (page-locked for every context).  The thread's current device is restored.
int dalib200HostAllocOnDevice(void **ptr, size_t bytes, int device) try {
  DB_CHECK_ARG(ptr && device >= 0, "HostAllocOnDevice: bad arguments");
  *ptr = nullptr;
  if (bytes == 0) return DALIB200_SUCCESS;
  int prev = -1;
  const bool have_prev = cudaGetDevice(&prev) == cudaSuccess;
  DB_CUDA(cudaSetDevice(device));
  const cudaError_t e = cudaHostAlloc(ptr, bytes, cudaHostAllocPortable);
  if (have_prev && prev != device) cudaSetDevice(prev);
  DB_CUDA(e);
  return DALIB200_SUCCESS;
} DB_API_CATCH

int dalib200HostFree(void *ptr) try {
  if (ptr) DB_CUDA(cudaFreeHost(ptr));
  return DALIB200_SUCCESS;
} DB_API_CATCH

int dalib200ProfilingEnable(int on) { dalib200::g_prof_on = on != 0; return DALIB200_SUCCESS; }
// Synchronises, writes up to `max` records (names: `name_stride` bytes each, NUL terminated) and clears the log.
int dalib200ProfilingCollect(char *names, int name_stride, float *ms, int max, int *count) try {
  using namespace dalib200;  // NOLINT
  std::lock_guard<std::mutex> lock(g_prof_mutex);
  int n = 0;
  for (auto &r : g_prof) {
    cudaEventSynchronize(r.b);
    float t = 0;
    cudaEventElapsedTime(&t, r.a, r.b);
    if (n < max) {
      if (names && name_stride > 0) { snprintf(names + (size_t)n * name_stride, name_stride, "%s", r.name); }
      if (ms) ms[n] = t;
      n++;
    }
    g_prof_pool.push_back(r.a); g_prof_pool.push_back(r.b);
  }
  g_prof.clear();
  if (count) *count = n;
  return DALIB200_SUCCESS;
} DB_API_CATCH
const char *dalib200GetLastError(void) { return dalib200::tls_error.c_str(); }
int dalib200GetVersion(void) { return 100; }
uint64_t dalib200GetLaunchCount(void) { return dalib200::g_launch_count.load(); }
}
