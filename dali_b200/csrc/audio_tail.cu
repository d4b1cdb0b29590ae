// dali_b200/csrc/audio_tail.cu -- the audio tail behind Spectrogram / MelFilterBank (SURVEY.md 8f rank 3): ToDecibels, MFCC
// (DCT + liftering) and Normalize for sm_90a.
//
//   ToDecibels   dali/kernels/signal/decibel/to_decibels_cpu.cc:47-72 + decibel_calculator.h:25-56:
//                out = (mul * log10(2)) * log2(max(min_ratio, in * (1 / s_ref))), s_ref = per-sample maximum when no
//                `reference` is given (0 -> 1).  log2f on the device vs glibc's on the host: <= 2 ulp of the logarithm
//                (stated tolerance of the tests: 1e-5 dB absolute + 1e-6 relative).
//   MFCC         dali/kernels/signal/dct/dct_cpu.cc:76-115 (out[k] = sum_n in[n] * table[k][n], n ascending, mul and add rounded
//                separately), cosine tables table.h:27-112 (double on the host), liftering mfcc.h:36-41, mfcc.cc:52-72.
//                Same order, same tables -> bit-exact.
//   Normalize    dali/operators/math/normalize/normalize.cc: out = (in - mean) * scale / sqrt(var + eps) + shift over the reduced
//                axes of a 2-D sample; the mean / variance sums are tree reductions over the deviations from the group's first
//                element (a constant group gives `shift`), checked against a float64 statement with a per-element bound
//                (tests/audio_tail_f64.py).
//   NonsilentRegion  dali/operators/audio/nonsilence_op.h:60-130 + dali/kernels/signal/moving_mean_square.cc:55-77: moving mean
//                square with a RUNNING float sum (add the new square, emit, subtract the oldest), restarted every `reset_interval`
//                samples; threshold = reference * 10^(cutoff_db / 10) with reference = the maximum of the moving mean square by
//                default; first / last sample at or above it; the start is moved back by window_length - 1.  The running sum
//                is a serial float recurrence: one thread replays one reset interval (bit-exact), intervals and samples in
//                parallel; the reductions behind it are exact (max / min / max index).
//   AudioResample  dali/kernels/signal/resampling_cpu.cc:120-165 (single channel: the SSE2 path, four partial sums over taps
//                i0 + l + 4k, combined as (f0 + f2) + (f1 + f3), then the scalar tail) and :186-230 (multi-channel: scalar, taps in
//                order), window = Hann-windowed sinc looked up with linear interpolation (resampling.h:36-92, built on the host with
//                the same float / double expressions).  The source position is accumulated in float inside blocks of 256 outputs
//                (in_pos += fscale): a serial recurrence, replayed by one thread per block into shared memory; everything else is
//                one thread per output sample with the reference's operation order -> bit-exact.
// Every op is one launch per batch over a per-sample descriptor list (one H2D descriptor copy per launch).
#include "common.cuh"
#include <algorithm>
#include <cmath>
#include <cstring>

namespace dalib200 {

enum { SIG_NONE = 0, SIG_TODB = 1, SIG_MFCC = 2, SIG_NORMALIZE = 3, SIG_NONSILENT = 4, SIG_RESAMPLE = 5 };

struct SigDesc {
  const float *in; float *out;
  int64_t n;                 // elements
  int64_t rows, cols;        // 2-D view (MFCC: rows = nfeat, cols = frames; Normalize)
  int64_t first_item;
};

__device__ __forceinline__ int find_sig(const SigDesc *d, int n, int64_t v) {
  int lo = 0, hi = n - 1;
  while (lo < hi) { int mid = (lo + hi + 1) >> 1; if (d[mid].first_item <= v) lo = mid; else hi = mid - 1; }
  return lo;
}

// ---- AudioResample
struct ArDesc {
  const float *in; float *out;
  int64_t n_in, n_out, first_item;      // items = groups of 4 blocks of 256 outputs
  double scale;                         // in_rate / out_rate
  int32_t channels;
};
struct ArWindow { float scale, center; int lobes; const float *lookup; };

__device__ __forceinline__ float ar_window(const ArWindow &w, float x) {           // resampling.h:59-66 / resampling_cpu.cc:86-99
  const float fi = add_rn(mul_rn(x, w.scale), w.center);
  const float fl = floorf(fi);
  const float di = sub_rn(fi, fl);
  const int i = (int)fl;
  const float c = __ldg(w.lookup + i), nx = __ldg(w.lookup + i + 1);
  return add_rn(c, mul_rn(di, sub_rn(nx, c)));
}

constexpr int kArBlock = 256, kArBlocksPerCta = 4;

__global__ void __launch_bounds__(256) audio_resample_kernel(const ArDesc *__restrict__ descs, int n, int64_t total_items, ArWindow win) {
  __shared__ float s_pos[kArBlocksPerCta][kArBlock];
  __shared__ long long s_blk[kArBlocksPerCta];
  for (int64_t item = blockIdx.x; item < total_items; item += gridDim.x) {
    int lo = 0, hi = n - 1;
    while (lo < hi) { int mid = (lo + hi + 1) >> 1; if (descs[mid].first_item <= item) lo = mid; else hi = mid - 1; }
    const ArDesc &d = descs[lo];
    const int64_t out0 = (item - d.first_item) * (kArBlock * kArBlocksPerCta);
    const float fscale = (float)d.scale;
    // ---- the float source position of every output of the group: one thread replays one block of 256 (resampling_cpu.cc:131-136)
    if (threadIdx.x < kArBlocksPerCta) {
      const int64_t ob = out0 + (int64_t)threadIdx.x * kArBlock;
      if (ob < d.n_out) {
        const double in_block_f = (double)ob * d.scale;
        const long long in_block_i = (long long)floor(in_block_f);
        float in_pos = (float)(in_block_f - (double)in_block_i);
        s_blk[threadIdx.x] = in_block_i;
        const int cnt = (int)min((int64_t)kArBlock, d.n_out - ob);
        for (int j = 0; j < cnt; j++) { s_pos[threadIdx.x][j] = in_pos; in_pos = add_rn(in_pos, fscale); }
      }
    }
    __syncthreads();
    for (int b = 0; b < kArBlocksPerCta; b++) {
      const int64_t op = out0 + (int64_t)b * kArBlock + threadIdx.x;
      if (op >= d.n_out) continue;
      const float in_pos = s_pos[b][threadIdx.x];
      const long long in_block_i = s_blk[b];
      const int xc = (int)ceilf(in_pos);
      int i0 = xc - win.lobes, i1 = xc + win.lobes;
      if (i0 + in_block_i < 0) i0 = (int)(-in_block_i);
      if (i1 + in_block_i > d.n_in) i1 = (int)(d.n_in - in_block_i);
      if (d.channels == 1) {
        const float *__restrict__ inb = d.in + in_block_i;
        int i = i0;
        float f4[4] = {0.f, 0.f, 0.f, 0.f}, x4[4];
#pragma unroll
        for (int l = 0; l < 4; l++) x4[l] = sub_rn((float)(i + l), in_pos);
        for (; i + 3 < i1; i += 4) {
#pragma unroll
          for (int l = 0; l < 4; l++) {
            // evaluate(): truncation instead of floor (cvttps) -- the argument is positive inside the window
            const float fi = add_rn(mul_rn(x4[l], win.scale), win.center);
            const int idx = (int)fi;
            const float di = sub_rn(fi, (float)idx);
            const float c = __ldg(win.lookup + idx), nx = __ldg(win.lookup + idx + 1);
            const float w = add_rn(c, mul_rn(di, sub_rn(nx, c)));
            f4[l] = add_rn(f4[l], mul_rn(__ldg(inb + i + l), w));
            x4[l] = add_rn(x4[l], 4.0f);
          }
        }
        float f = add_rn(add_rn(f4[0], f4[2]), add_rn(f4[1], f4[3]));
        float x = sub_rn((float)i, in_pos);
        for (; i < i1; i++, x = add_rn(x, 1.0f)) f = add_rn(f, mul_rn(__ldg(inb + i), ar_window(win, x)));
        d.out[op] = f;
      } else {
        const int C = d.channels;
        const float *__restrict__ inb = d.in + in_block_i * C;
        float tmp[8];
#pragma unroll
        for (int c = 0; c < 8; c++) tmp[c] = 0.f;
        float x = sub_rn((float)i0, in_pos);
        for (int i = i0; i < i1; i++, x = add_rn(x, 1.0f)) {
          const float w = ar_window(win, x);
#pragma unroll
          for (int c = 0; c < 8; c++) if (c < C) tmp[c] = add_rn(tmp[c], mul_rn(__ldg(inb + (int64_t)i * C + c), w));
        }
#pragma unroll
        for (int c = 0; c < 8; c++) if (c < C) d.out[op * C + c] = tmp[c];
      }
    }
    __syncthreads();
  }
}

// ---- NonsilentRegion
struct NsDesc {
  const float *in; float *mms;          // mms: scratch, one float per input sample
  int32_t *begin, *length;
  int64_t n, first_item;                // items = reset intervals
  float factor, reference;              // threshold = ref * factor, ref = reference > 0 ? reference : max(mms)
  int32_t window, interval;
};

__device__ __forceinline__ int find_ns(const NsDesc *d, int n, int64_t v) {
  int lo = 0, hi = n - 1;
  while (lo < hi) { int mid = (lo + hi + 1) >> 1; if (d[mid].first_item <= v) lo = mid; else hi = mid - 1; }
  return lo;
}

// thread = one reset interval of one sample (moving_mean_square.cc:55-77)
__global__ void __launch_bounds__(128) nonsilent_mms_kernel(const NsDesc *__restrict__ descs, int n, int64_t total_items) {
  const int64_t item = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (item >= total_items) return;
  const NsDesc &d = descs[find_ns(descs, n, item)];
  const int64_t out0 = (item - d.first_item) * d.interval, out1 = min(d.n, out0 + d.interval);
  const float mean_factor = 1.0f / (float)d.window;
  int64_t win_begin = out0 - d.window + 1;
  float sumsq = 0.0f;
  for (int64_t pos = max(win_begin, (int64_t)0); pos < out0; pos++) { const float v = __ldg(d.in + pos); sumsq = add_rn(sumsq, mul_rn(v, v)); }
  for (int64_t pos = out0; pos < out1; pos++, win_begin++) {
    const float v = __ldg(d.in + pos);
    sumsq = add_rn(sumsq, mul_rn(v, v));
    d.mms[pos] = mul_rn(sumsq, mean_factor);
    if (win_begin >= 0) { const float o = __ldg(d.in + win_begin); sumsq = sub_rn(sumsq, mul_rn(o, o)); }
  }
}

// CTA = one sample: maximum of the moving mean square, threshold, first / last index at or above it (nonsilence_op.h:60-130)
__global__ void __launch_bounds__(256) nonsilent_region_kernel(const NsDesc *__restrict__ descs) {
  const NsDesc &d = descs[blockIdx.x];
  __shared__ float s_f[8];
  __shared__ long long s_lo[8], s_hi[8];
  __shared__ float s_ref;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  float ref = d.reference;
  if (!(ref > 0.0f)) {
    float m = -INFINITY;                                  // std::max chain over finite values = exact maximum
    for (int64_t i = threadIdx.x; i < d.n; i += blockDim.x) m = fmaxf(m, d.mms[i]);
    for (int o = 16; o; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if (lane == 0) s_f[warp] = m;
    __syncthreads();
    if (threadIdx.x == 0) { float t = s_f[0]; for (int w = 1; w < 8; w++) t = fmaxf(t, s_f[w]); s_ref = t; }
    __syncthreads();
    ref = s_ref;
  }
  const float cutoff = mul_rn(ref, d.factor);             // s_ref * pow(10, cutoff_db / 10): the power is taken on the host
  long long lo = d.n, hi = -1;
  for (int64_t i = threadIdx.x; i < d.n; i += blockDim.x)
    if (d.mms[i] >= cutoff) { lo = min(lo, (long long)i); hi = max(hi, (long long)i); }
  for (int o = 16; o; o >>= 1) { lo = min(lo, __shfl_xor_sync(0xffffffffu, lo, o)); hi = max(hi, __shfl_xor_sync(0xffffffffu, hi, o)); }
  if (lane == 0) { s_lo[warp] = lo; s_hi[warp] = hi; }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < 8; w++) { lo = min(lo, s_lo[w]); hi = max(hi, s_hi[w]); }
    long long begin = 0, len = 0;
    if (hi >= 0) { begin = lo; len = hi - lo + 1; }
    if (begin != 0 && len != 0) {                         // the non-silent sample sits somewhere inside the window that reported it
      const long long nb = max(begin - (d.window - 1), 0ll);
      len += begin - nb; begin = nb;
    }
    *d.begin = (int32_t)begin; *d.length = (int32_t)len;
  }
}

// ---- ToDecibels
constexpr int kDbItem = 4096;       // elements per work item

__global__ void __launch_bounds__(256) todb_max_kernel(const SigDesc *__restrict__ descs, int n, int64_t total_items, uint32_t *__restrict__ smax) {
  __shared__ float wmax[8];
  for (int64_t item = blockIdx.x; item < total_items; item += gridDim.x) {
    const int s = find_sig(descs, n, item);
    const SigDesc &d = descs[s];
    const int64_t e0 = (item - d.first_item) * kDbItem, e1 = min(d.n, e0 + kDbItem);
    float m = 0.0f;                                    // s_ref starts at 0: only values above it count
    for (int64_t e = e0 + threadIdx.x; e < e1; e += blockDim.x) { const float v = __ldg(d.in + e); if (v > m) m = v; }
    for (int o = 16; o; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((threadIdx.x & 31) == 0) wmax[threadIdx.x >> 5] = m;
    __syncthreads();
    if (threadIdx.x == 0) {
      for (int w = 1; w < 8; w++) m = fmaxf(m, wmax[w]);
      atomicMax(smax + s, __float_as_uint(m));          // m >= 0: the integer order of the bit patterns is the float order
    }
    __syncthreads();
  }
}

__global__ void __launch_bounds__(256) todb_kernel(const SigDesc *__restrict__ descs, int n, int64_t total_items, float mul_log2, float s_ref,
                                                   float min_ratio, const uint32_t *__restrict__ smax) {
  for (int64_t item = blockIdx.x; item < total_items; item += gridDim.x) {
    const int s = find_sig(descs, n, item);
    const SigDesc &d = descs[s];
    float ref = s_ref;
    if (smax) { ref = __uint_as_float(smax[s]); if (ref == 0.0f) ref = 1.0f; }
    const float inv = ref == 1.0f ? 1.0f : __fdiv_rn(1.0f, ref);
    const int64_t e0 = (item - d.first_item) * kDbItem, e1 = min(d.n, e0 + kDbItem);
    for (int64_t e = e0 + threadIdx.x; e < e1; e += blockDim.x)
      d.out[e] = mul_rn(mul_log2, log2f(fmaxf(min_ratio, mul_rn(__ldg(d.in + e), inv))));
  }
}

// ---- MFCC: one thread = one frame (column) x up to 32 coefficients; the table row of a coefficient is read from shared memory
constexpr int kMfccK = 32;
__global__ void __launch_bounds__(128) mfcc_kernel(const SigDesc *__restrict__ descs, int n, int64_t total_items, int nfeat, int ndct,
                                                   const float *__restrict__ table, const float *__restrict__ lifter) {
  extern __shared__ float s_tab[];                      // [ndct][nfeat]
  for (int i = threadIdx.x; i < ndct * nfeat; i += blockDim.x) s_tab[i] = table[i];
  __syncthreads();
  for (int64_t item = blockIdx.x; item < total_items; item += gridDim.x) {
    const int s = find_sig(descs, n, item);
    const SigDesc &d = descs[s];
    const int64_t t = (item - d.first_item) * blockDim.x + threadIdx.x;
    if (t >= d.cols) continue;
    for (int k0 = 0; k0 < ndct; k0 += kMfccK) {
      float acc[kMfccK];
#pragma unroll
      for (int k = 0; k < kMfccK; k++) acc[k] = 0.0f;
      for (int f = 0; f < nfeat; f++) {
        const float v = __ldg(d.in + (int64_t)f * d.cols + t);
#pragma unroll
        for (int k = 0; k < kMfccK; k++)
          if (k0 + k < ndct) acc[k] = add_rn(acc[k], mul_rn(v, s_tab[(k0 + k) * nfeat + f]));
      }
#pragma unroll
      for (int k = 0; k < kMfccK; k++)
        if (k0 + k < ndct) d.out[(int64_t)(k0 + k) * d.cols + t] = lifter ? mul_rn(lifter[k0 + k], acc[k]) : acc[k];
    }
  }
}

// ---- Normalize (2-D samples): mode 0 = over both axes (one mean / stddev per sample), 1 = over axis 1 (per row), 2 = over axis 0
// (per column).  One CTA per (sample, group).
__device__ __forceinline__ float block_sum(float v, float *sh) {
  for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
  __syncthreads();
  float r = 0.0f;
  for (int w = 0; w < (int)(blockDim.x >> 5); w++) r += sh[w];
  return r;
}

__global__ void __launch_bounds__(256) normalize_kernel(const SigDesc *__restrict__ descs, int n, int64_t total_items, int mode, float scale,
                                                        float shift, float eps, int ddof) {
  __shared__ float sh[8];
  for (int64_t item = blockIdx.x; item < total_items; item += gridDim.x) {
    const int s = find_sig(descs, n, item);
    const SigDesc &d = descs[s];
    const int64_t g = item - d.first_item;               // group inside the sample
    int64_t cnt, stride, base;
    if (mode == 0) { cnt = d.rows * d.cols; stride = 1; base = 0; }
    else if (mode == 1) { cnt = d.cols; stride = 1; base = g * d.cols; }
    else { cnt = d.rows; stride = d.cols; base = g; }
    // The sums run over the deviations from the group's first element: a constant group then has mean and variance exactly 0 (a
    // float mean of equal values need not equal them, and (x - mean)^2 > 0 would turn a constant row into +-scale), and an offset
    // shared by the whole group (DC) does not enter the rounding of the sums.
    const float x0 = __ldg(d.in + base);
    float sum = 0.0f;
    for (int64_t e = threadIdx.x; e < cnt; e += blockDim.x) sum += __ldg(d.in + base + e * stride) - x0;
    const float mean = block_sum(sum, sh) / (float)cnt;                 // of the deviations
    float sq = 0.0f;
    for (int64_t e = threadIdx.x; e < cnt; e += blockDim.x) { const float x = (__ldg(d.in + base + e * stride) - x0) - mean; sq += x * x; }
    const float var = block_sum(sq, sh) / (float)max((int64_t)1, cnt - ddof);
    const float sd = sqrtf(var + eps);
    const float mul = sd != 0.0f ? scale / sd : 0.0f;
    for (int64_t e = threadIdx.x; e < cnt; e += blockDim.x) {
      const int64_t i = base + e * stride;
      d.out[i] = ((__ldg(d.in + i) - x0) - mean) * mul + shift;
    }
    __syncthreads();
  }
}

}  // namespace dalib200

using namespace dalib200;  // NOLINT

struct dalib200SignalPlan {
  int max_batch = 0, n = 0, kind = SIG_NONE;
  std::vector<SigDesc> descs;
  int64_t total_items = 0;
  DescArena arena;
  cudaEvent_t uploaded = nullptr;
  bool pending = false;
  // ToDecibels
  float mul_log2 = 0, s_ref = 1, min_ratio = 1e-8f; bool ref_max = false;
  uint32_t *d_max = nullptr; size_t d_max_cap = 0;
  // MFCC
  int nfeat = 0, ndct = 0; bool has_lifter = false;
  float *d_table = nullptr; size_t d_table_cap = 0;     // [ndct * nfeat] + [ndct] lifter
  std::vector<float> h_table;
  bool table_dirty = true;
  // Normalize
  int mode = 0, ddof = 0; float scale = 1, shift = 0, eps = 0;
  // AudioResample
  std::vector<ArDesc> ar;
  std::vector<float> ar_lookup; float *d_lookup = nullptr; size_t d_lookup_cap = 0; bool lookup_dirty = true;
  float ar_scale = 1, ar_center = 1; int ar_lobes = 0; float ar_quality = -1;
  // NonsilentRegion
  std::vector<NsDesc> ns;
  float *d_mms = nullptr; size_t d_mms_cap = 0;
  int64_t mms_total = 0;
};

namespace {
int GrowF(float *&p, size_t &cap, size_t need) {
  if (need <= cap) return DALIB200_SUCCESS;
  if (p) cudaFree(p);
  p = nullptr; cap = 0;
  DB_CUDA(cudaMalloc(reinterpret_cast<void **>(&p), need * sizeof(float)));
  cap = need;
  return DALIB200_SUCCESS;
}

// dali/kernels/signal/dct/table.h:27-112
void FillCosineTable(float *table, int64_t n, int ndct, int type, bool normalize) {
  int64_t idx = 0;
  if (type == 1) {
    const double phase_mul = M_PI / (n - 1);
    for (int64_t k = 0; k < ndct; k++) {
      table[idx++] = 0.5f;
      for (int64_t i = 1; i < n - 1; i++) table[idx++] = static_cast<float>(std::cos(phase_mul * k * i));
      table[idx++] = k % 2 == 0 ? 0.5f : -0.5f;
    }
  } else if (type == 2) {
    const double phase_mul = M_PI / n;
    double f0 = 1, fi = 1;
    if (normalize) { fi = std::sqrt(2.0 / n); f0 = 1.0 / std::sqrt(static_cast<double>(n)); }
    for (int64_t k = 0; k < ndct; k++) {
      const double nf = k == 0 ? f0 : fi;
      for (int64_t i = 0; i < n; i++) table[idx++] = static_cast<float>(nf * std::cos(phase_mul * (i + 0.5) * k));
    }
  } else if (type == 3) {
    const double phase_mul = M_PI / n;
    double f0 = 0.5, fi = 1;
    if (normalize) { fi = std::sqrt(2.0 / n); f0 = 1.0 / std::sqrt(static_cast<double>(n)); }
    for (int64_t k = 0; k < ndct; k++) {
      table[idx++] = static_cast<float>(f0);
      for (int64_t i = 1; i < n; i++) table[idx++] = static_cast<float>(fi * std::cos(phase_mul * i * (k + 0.5)));
    }
  } else {
    const double phase_mul = M_PI / n;
    const double f = normalize ? std::sqrt(2.0 / n) : 1.0;
    for (int64_t k = 0; k < ndct; k++)
      for (int64_t i = 0; i < n; i++) table[idx++] = static_cast<float>(f * std::cos(phase_mul * (i + 0.5) * (k + 0.5)));
  }
}

int UploadDescs(dalib200SignalPlan *p) {
  if (p->pending) { DB_CUDA(cudaEventSynchronize(p->uploaded)); p->pending = false; }
  int rc = p->arena.Reserve(sizeof(SigDesc) * std::max(1, p->n));
  return rc;
}
}  // namespace

extern "C" {

int dalib200SignalPlanCreate(dalib200SignalPlan **plan, int max_batch) try {
  DB_CHECK_ARG(plan && max_batch > 0, "SignalPlanCreate: bad arguments");
  auto *p = new dalib200SignalPlan();
  p->max_batch = max_batch;
  if (cudaEventCreateWithFlags(&p->uploaded, cudaEventDisableTiming) != cudaSuccess) {
    SetLastError("SignalPlanCreate: cudaEventCreate failed"); delete p; return DALIB200_ERROR_CUDA;
  }
  *plan = p;
  return DALIB200_SUCCESS;
} DB_API_CATCH

int dalib200SignalPlanDestroy(dalib200SignalPlan *p) try {
  if (!p) return DALIB200_SUCCESS;
  if (p->uploaded) { cudaEventSynchronize(p->uploaded); cudaEventDestroy(p->uploaded); }
  p->arena.Free();
  if (p->d_max) cudaFree(p->d_max);
  if (p->d_table) cudaFree(p->d_table);
  if (p->d_mms) cudaFree(p->d_mms);
  if (p->d_lookup) cudaFree(p->d_lookup);
  delete p;
  return DALIB200_SUCCESS;
} DB_API_CATCH

int dalib200ToDecibelsSetup(dalib200SignalPlan *p, const dalib200ToDecibelsArgs *a, int n, const int64_t *volumes) try {
  DB_CHECK_ARG(p && a && (n == 0 || volumes) && n >= 0 && n <= p->max_batch, "ToDecibelsSetup: bad arguments");
  DB_CHECK_ARG(a->ref_max || a->reference != 0.0f, "`reference` argument can't be zero");
  p->kind = SIG_TODB; p->n = n;
  // to_decibels_op.h:41-50 and decibel_calculator.h:29-33 (float arithmetic throughout)
  p->mul_log2 = a->multiplier * 0.3010299956639812f;
  p->ref_max = a->ref_max != 0;
  p->s_ref = a->ref_max ? 1.0f : a->reference;
  p->min_ratio = std::pow(10.0f, a->cutoff_db / a->multiplier);
  if (p->min_ratio == 0) p->min_ratio = std::nextafter(0.0f, 1.0f);
  p->descs.assign(n, SigDesc());
  int64_t items = 0;
  for (int i = 0; i < n; i++) {
    DB_CHECK_ARG(volumes[i] >= 0, "ToDecibelsSetup: negative volume");
    p->descs[i].n = volumes[i]; p->descs[i].first_item = items;
    items += (volumes[i] + kDbItem - 1) / kDbItem;
  }
  p->total_items = items;
  return DALIB200_SUCCESS;
} DB_API_CATCH

int dalib200MfccSetup(dalib200SignalPlan *p, const dalib200MfccArgs *a, int n, const int64_t *shapes) try {
  DB_CHECK_ARG(p && a && (n == 0 || shapes) && n >= 0 && n <= p->max_batch, "MfccSetup: bad arguments");
  DB_CHECK_ARG(a->n_mfcc > 0, "number of MFCCs should be > 0");
  DB_CHECK_ARG(a->dct_type >= 1 && a->dct_type <= 4, "Unsupported DCT type: %d. Supported types are: 1, 2, 3, 4.", a->dct_type);
  DB_CHECK_ARG(!(a->normalize && a->dct_type == 1), "Ortho-normalization is not supported for DCT type I.");
  p->kind = SIG_MFCC; p->n = n;
  DB_CHECK_ARG(n == 0 || (shapes[0] >= 1 && shapes[0] <= (1 << 16)), "MFCC: the transformed axis must have 1 .. 65536 elements");
  const int nfeat = n ? (int)shapes[0] : 1;
  int ndct = a->n_mfcc;
  if (ndct > nfeat) ndct = nfeat;                                 // dct_cpu.cc:56-58
  DB_CHECK_ARG(a->dct_type != 1 || nfeat > 1, "DCT type I requires an input length > 1");
  p->descs.assign(n, SigDesc());
  int64_t items = 0;
  for (int i = 0; i < n; i++) {
    DB_CHECK_ARG(shapes[2 * i] == nfeat, "MFCC: all samples of a batch must have the same extent along the transformed axis");
    DB_CHECK_ARG(shapes[2 * i + 1] >= 0 && shapes[2 * i + 1] < (1ll << 31), "MFCC: sample %d has an unsupported number of frames", i);
    p->descs[i].rows = nfeat; p->descs[i].cols = shapes[2 * i + 1]; p->descs[i].n = nfeat * shapes[2 * i + 1];
    p->descs[i].first_item = items;
    items += (shapes[2 * i + 1] + 127) / 128;
  }
  p->total_items = items;
  std::vector<float> tab((size_t)ndct * nfeat + ndct);
  FillCosineTable(tab.data(), nfeat, ndct, a->dct_type, a->normalize != 0);
  p->has_lifter = a->lifter != 0.0f;
  if (p->has_lifter) {                                            // mfcc.h:36-41
    const float ampl_mult = a->lifter / 2, phase_mult = static_cast<float>(M_PI) / a->lifter;
    // all-float arithmetic (the reference's unqualified sin() resolves to sinf there: checked on the compiled header)
    for (int64_t i = 0; i < ndct; i++) tab[(size_t)ndct * nfeat + i] = 1.f + ampl_mult * sinf(phase_mult * (i + 1));
  }
  if (tab != p->h_table || nfeat != p->nfeat || ndct != p->ndct) { p->h_table = tab; p->table_dirty = true; }
  p->nfeat = nfeat; p->ndct = ndct;
  return DALIB200_SUCCESS;
} DB_API_CATCH

int dalib200SignalOutputRows(const dalib200SignalPlan *p) { return p ? p->ndct : 0; }

int dalib200NormalizeSetup(dalib200SignalPlan *p, const dalib200NormalizeArgs *a, int n, const int64_t *shapes) try {
  DB_CHECK_ARG(p && a && (n == 0 || shapes) && n >= 0 && n <= p->max_batch, "NormalizeSetup: bad arguments");
  DB_CHECK_ARG(a->mode >= 0 && a->mode <= 2, "NormalizeSetup: mode must be 0 (all axes), 1 (axis 1) or 2 (axis 0)");
  DB_CHECK_ARG(a->ddof >= 0, "Normalize: ddof must be non-negative");
  p->kind = SIG_NORMALIZE; p->n = n;
  p->mode = a->mode; p->ddof = a->ddof; p->scale = a->scale; p->shift = a->shift; p->eps = a->epsilon;
  p->descs.assign(n, SigDesc());
  int64_t items = 0;
  for (int i = 0; i < n; i++) {
    DB_CHECK_ARG(shapes[2 * i] >= 0 && shapes[2 * i + 1] >= 0 && shapes[2 * i] < (1ll << 31) && shapes[2 * i + 1] < (1ll << 31),
                 "Normalize: sample %d has an unsupported shape", i);
    p->descs[i].rows = shapes[2 * i]; p->descs[i].cols = shapes[2 * i + 1]; p->descs[i].n = shapes[2 * i] * shapes[2 * i + 1];
    p->descs[i].first_item = items;
    items += p->descs[i].n == 0 ? 0 : a->mode == 0 ? 1 : a->mode == 1 ? shapes[2 * i] : shapes[2 * i + 1];
  }
  p->total_items = items;
  return DALIB200_SUCCESS;
} DB_API_CATCH

int dalib200AudioResampleSetup(dalib200SignalPlan *p, int n, const dalib200AudioResampleSample *samples, float quality) try {
  DB_CHECK_ARG(p && n >= 0 && n <= p->max_batch && (n == 0 || samples), "AudioResampleSetup: bad arguments");
  DB_CHECK_ARG(quality >= 0 && quality <= 100, "``quality`` out of range: %g\nValid range is [0..100].", (double)quality);
  p->kind = SIG_RESAMPLE; p->n = n;
  if (quality != p->ar_quality) {
    // ResamplingParams::FromQuality (resampling_params.h:27-30) + windowed_sinc (resampling.h:73-96), same float / double expressions
    const double q = quality;
    const int lobes = (int)std::round(0.007 * q * q - 0.09 * q + 3);
    const int coeffs = lobes * 64 + 1;
    const float scale = 2.0f * lobes / (coeffs - 1);
    const float scale_envelope = 2.0f / coeffs;
    const int center = (int)((coeffs - 1) * 0.5f);
    p->ar_lookup.assign((size_t)coeffs + 5, 0.0f);
    for (int i = 0; i < coeffs; i++) {
      const float x = (i - center) * scale;
      const float y = (i - center) * scale_envelope;
      float sx = x; sx *= M_PI;                                                   // math_util.h:188-193 (float overload)
      const float sinc = std::abs(sx) < 1e-5f ? 1.0f - sx * sx * (1.0f / 6) : std::sin(sx) / sx;
      const double hann = 0.5 * (1 + std::cos((double)y * M_PI));
      const float w = sinc * hann;
      p->ar_lookup[i + 1] = w;
    }
    p->ar_center = (float)(center + 1);
    p->ar_scale = 1 / scale;
    p->ar_lobes = lobes;
    p->ar_quality = quality;
    p->lookup_dirty = true;
  }
  p->ar.assign(n, ArDesc());
  int64_t items = 0;
  for (int i = 0; i < n; i++) {
    const auto &s = samples[i];
    DB_CHECK_ARG(s.in_rate > 0 && s.out_rate > 0, "AudioResample: sample %d: sampling rates must be positive", i);
    DB_CHECK_ARG(s.in_length >= 0 && s.out_length >= 0 && s.channels >= 1 && s.channels <= 8, "AudioResample: sample %d: unsupported shape", i);
    DB_CHECK_ARG(s.in_length < (1ll << 31) && s.out_length < (1ll << 31), "AudioResample: sample %d is too long", i);
    ArDesc &d = p->ar[i];
    memset(&d, 0, sizeof(d));
    d.n_in = s.in_length; d.n_out = s.out_length; d.channels = s.channels;
    d.scale = s.in_rate / s.out_rate;
    d.first_item = items;
    items += (d.n_out + kArBlock * kArBlocksPerCta - 1) / (kArBlock * kArBlocksPerCta);
  }
  p->total_items = items;
  return DALIB200_SUCCESS;
} DB_API_CATCH

int dalib200NonsilentSetup(dalib200SignalPlan *p, int n, const int64_t *lengths, const dalib200NonsilentSample *args, int window_length,
                           int reset_interval) try {
  DB_CHECK_ARG(p && n >= 0 && n <= p->max_batch && (n == 0 || (lengths && args)), "NonsilentSetup: bad arguments");
  DB_CHECK_ARG(window_length > 0, "NonsilentRegion: window_length must be positive, got %d", window_length);
  DB_CHECK_ARG(reset_interval == -1 || (reset_interval > 0 && reset_interval % window_length == 0),
               "`reset_interval` shall be a multiple of `window_length`. Got: reset_interval: %d vs window_length: %d", reset_interval, window_length);
  p->kind = SIG_NONSILENT; p->n = n;
  p->ns.assign(n, NsDesc());
  int64_t items = 0, total = 0;
  for (int i = 0; i < n; i++) {
    DB_CHECK_ARG(lengths[i] > 0, "NonsilentRegion: sample %d is empty", i);
    DB_CHECK_ARG(lengths[i] < (1ll << 31), "NonsilentRegion: sample %d is too long for the int32 outputs", i);
    NsDesc &d = p->ns[i];
    memset(&d, 0, sizeof(d));
    d.n = lengths[i];
    d.window = (int32_t)std::min<int64_t>(window_length, lengths[i]);          // nonsilence_op.cc: min(window_length, num_elements)
    d.interval = reset_interval == -1 ? (int32_t)lengths[i] : reset_interval;
    // DecibelToMagnitude<float>(10.f, ref)(cutoff_db) = ref * pow(10.f, cutoff_db * (1.f / 10.f))   (decibel_calculator.h:60-73)
    d.factor = std::pow(10.0f, args[i].cutoff_db * (1.0f / 10.0f));
    d.reference = args[i].reference_power;
    DB_CHECK_ARG(!(args[i].use_reference_power) || args[i].reference_power > 0, "`reference_power` has to be positive. Got: %g",
                 (double)args[i].reference_power);
    if (!args[i].use_reference_power) d.reference = 0.0f;
    d.first_item = items;
    items += (d.n + d.interval - 1) / d.interval;
    total += d.n;
  }
  p->total_items = items; p->mms_total = total;
  return DALIB200_SUCCESS;
} DB_API_CATCH

int dalib200NonsilentLaunch(dalib200SignalPlan *p, const void *const *in_ptrs, void *const *begin_ptrs, void *const *length_ptrs,
                            dalib200Stream_t stream) try {
  DB_CHECK_ARG(p && p->kind == SIG_NONSILENT && (p->n == 0 || (in_ptrs && begin_ptrs && length_ptrs)), "NonsilentLaunch: call NonsilentSetup first");
  if (p->n == 0) return DALIB200_SUCCESS;
  int rc = GrowF(p->d_mms, p->d_mms_cap, (size_t)p->mms_total);
  if (rc) return rc;
  if (p->pending) { DB_CUDA(cudaEventSynchronize(p->uploaded)); p->pending = false; }
  if ((rc = p->arena.Reserve(sizeof(NsDesc) * p->n))) return rc;
  NsDesc *h = reinterpret_cast<NsDesc *>(p->arena.host);
  int64_t off = 0;
  for (int i = 0; i < p->n; i++) {
    h[i] = p->ns[i];
    h[i].in = static_cast<const float *>(in_ptrs[i]); h[i].mms = p->d_mms + off;
    h[i].begin = static_cast<int32_t *>(begin_ptrs[i]); h[i].length = static_cast<int32_t *>(length_ptrs[i]);
    off += p->ns[i].n;
  }
  if ((rc = p->arena.Upload(sizeof(NsDesc) * p->n, stream))) return rc;
  DB_CUDA(cudaEventRecord(p->uploaded, stream));
  p->pending = true;
  const NsDesc *d = reinterpret_cast<const NsDesc *>(p->arena.dev);
  { ProfScope ps_("nonsilent_mms", stream); nonsilent_mms_kernel<<<(unsigned)((p->total_items + 127) / 128), 128, 0, stream>>>(d, p->n, p->total_items); }
  CountLaunch();
  { ProfScope ps_("nonsilent_region", stream); nonsilent_region_kernel<<<p->n, 256, 0, stream>>>(d); }
  CountLaunch();
  DB_CUDA(cudaGetLastError());
  return DALIB200_SUCCESS;
} DB_API_CATCH

static int AudioResampleLaunch(dalib200SignalPlan *p, const void *const *in_ptrs, void *const *out_ptrs, dalib200Stream_t stream) {
  int rc = GrowF(p->d_lookup, p->d_lookup_cap, p->ar_lookup.size());
  if (rc) return rc;
  if (p->lookup_dirty) {
    DB_CUDA(cudaMemcpyAsync(p->d_lookup, p->ar_lookup.data(), p->ar_lookup.size() * sizeof(float), cudaMemcpyHostToDevice, stream));
    p->lookup_dirty = false;
  }
  if (p->pending) { DB_CUDA(cudaEventSynchronize(p->uploaded)); p->pending = false; }
  if ((rc = p->arena.Reserve(sizeof(ArDesc) * p->n))) return rc;
  ArDesc *h = reinterpret_cast<ArDesc *>(p->arena.host);
  for (int i = 0; i < p->n; i++) { h[i] = p->ar[i]; h[i].in = static_cast<const float *>(in_ptrs[i]); h[i].out = static_cast<float *>(out_ptrs[i]); }
  if ((rc = p->arena.Upload(sizeof(ArDesc) * p->n, stream))) return rc;
  DB_CUDA(cudaEventRecord(p->uploaded, stream));
  p->pending = true;
  ArWindow w{ p->ar_scale, p->ar_center, p->ar_lobes, p->d_lookup };
  const int grid = (int)std::min<int64_t>(p->total_items, (int64_t)NumSMs() * 8);
  ProfScope ps_("audio_resample", stream);
  audio_resample_kernel<<<grid, 256, 0, stream>>>(reinterpret_cast<const ArDesc *>(p->arena.dev), p->n, p->total_items, w);
  CountLaunch();
  DB_CUDA(cudaGetLastError());
  return DALIB200_SUCCESS;
}

int dalib200SignalLaunch(dalib200SignalPlan *p, const void *const *in_ptrs, void *const *out_ptrs, dalib200Stream_t stream) try {
  DB_CHECK_ARG(p && p->kind != SIG_NONE && p->kind != SIG_NONSILENT && (p->n == 0 || (in_ptrs && out_ptrs)),
               "SignalLaunch: call a ...Setup function first (NonsilentRegion has its own launch)");
  if (p->n == 0 || p->total_items == 0) return DALIB200_SUCCESS;
  if (p->kind == SIG_RESAMPLE) return AudioResampleLaunch(p, in_ptrs, out_ptrs, stream);
  int rc = UploadDescs(p);
  if (rc) return rc;
  SigDesc *h = reinterpret_cast<SigDesc *>(p->arena.host);
  for (int i = 0; i < p->n; i++) { h[i] = p->descs[i]; h[i].in = static_cast<const float *>(in_ptrs[i]); h[i].out = static_cast<float *>(out_ptrs[i]); }
  if ((rc = p->arena.Upload(sizeof(SigDesc) * p->n, stream))) return rc;
  DB_CUDA(cudaEventRecord(p->uploaded, stream));
  p->pending = true;
  const SigDesc *d = reinterpret_cast<const SigDesc *>(p->arena.dev);
  const int grid = (int)std::min<int64_t>(p->total_items, (int64_t)NumSMs() * 16);
  if (p->kind == SIG_TODB) {
    const uint32_t *smax = nullptr;
    if (p->ref_max) {
      if ((size_t)p->n > p->d_max_cap) {
        if (p->d_max) cudaFree(p->d_max);
        p->d_max = nullptr; p->d_max_cap = 0;
        DB_CUDA(cudaMalloc(reinterpret_cast<void **>(&p->d_max), sizeof(uint32_t) * p->max_batch));
        p->d_max_cap = p->max_batch;
      }
      DB_CUDA(cudaMemsetAsync(p->d_max, 0, sizeof(uint32_t) * p->n, stream));
      { ProfScope ps_("to_decibels_max", stream); todb_max_kernel<<<grid, 256, 0, stream>>>(d, p->n, p->total_items, p->d_max); }
      CountLaunch();
      smax = p->d_max;
    }
    { ProfScope ps_("to_decibels", stream); todb_kernel<<<grid, 256, 0, stream>>>(d, p->n, p->total_items, p->mul_log2, p->s_ref, p->min_ratio, smax); }
    CountLaunch();
  } else if (p->kind == SIG_MFCC) {
    if ((rc = GrowF(p->d_table, p->d_table_cap, p->h_table.size()))) return rc;
    if (p->table_dirty) {
      // pageable source: the copy is staged by the runtime before the call returns
      DB_CUDA(cudaMemcpyAsync(p->d_table, p->h_table.data(), p->h_table.size() * sizeof(float), cudaMemcpyHostToDevice, stream));
      p->table_dirty = false;
    }
    const size_t smem = (size_t)p->ndct * p->nfeat * sizeof(float);
    DB_CHECK_ARG(smem <= 200 * 1024, "MFCC: the cosine table (%d x %d) does not fit shared memory", p->ndct, p->nfeat);
    if (smem > 48 * 1024) DB_CUDA(cudaFuncSetAttribute(mfcc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    ProfScope ps_("mfcc_dct", stream);
    mfcc_kernel<<<grid, 128, smem, stream>>>(d, p->n, p->total_items, p->nfeat, p->ndct, p->d_table,
                                             p->has_lifter ? p->d_table + (size_t)p->ndct * p->nfeat : nullptr);
    CountLaunch();
  } else {
    ProfScope ps_("normalize", stream);
    normalize_kernel<<<grid, 256, 0, stream>>>(d, p->n, p->total_items, p->mode, p->scale, p->shift, p->eps, p->ddof);
    CountLaunch();
  }
  DB_CUDA(cudaGetLastError());
  return DALIB200_SUCCESS;
} DB_API_CATCH

}  // extern "C"
