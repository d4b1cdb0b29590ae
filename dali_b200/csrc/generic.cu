// dali_b200/csrc/generic.cu -- the remaining per-pixel / geometry operators of SURVEY.md 8f rank 4 that do not need a kernel
// family of their own:
//   * multiply-add  out = ConvertSat<Out>(in * multiplier + addend)        brightness_contrast
//                   (dali/kernels/imgproc/pointwise/multiply_add.h:47-60; mul and add rounded separately like the CPU kernel)
//   * window copy   crop / slice / flip of interleaved u8 images with optional horizontal / vertical flip and out-of-bounds fill
//                   (dali/kernels/slice/slice_cpu.h, dali/operators/generic/flip.h: pure index arithmetic -> bit-exact)
//   * pad           N-D samples of 1-, 2- or 4-byte elements copied to the start of a larger array, the rest filled
//                   (dali/operators/generic/pad*)
// Multiply-add and window copy take u8 HWC inputs; one launch per batch over a per-sample descriptor list.
#include "common.cuh"
#include <algorithm>
#include <cstring>

namespace dalib200 {

struct GenDesc {
  const uint8_t *in; void *out;
  int32_t in_h, in_w, c;
  int32_t anchor_y, anchor_x, out_h, out_w;     // window copy
  int32_t flip_x, flip_y;
  float mul, add;                               // multiply-add
  uint8_t fill[4];
  int64_t n;                                    // output elements
  int64_t first_item;
};

constexpr int kGenItem = 8192;                  // output elements per work item

template <typename Out>
__global__ void __launch_bounds__(256) multiply_add_kernel(const GenDesc *__restrict__ descs, int n, int64_t total_items) {
  for (int64_t item = blockIdx.x; item < total_items; item += gridDim.x) {
    const int s = last_at_most(descs, 0, n - 1, item, [](const GenDesc &d) { return d.first_item; });
    const GenDesc &d = descs[s];
    const int64_t e0 = (item - d.first_item) * kGenItem, e1 = min(d.n, e0 + kGenItem);
    Out *out = static_cast<Out *>(d.out);
    const bool vec = (reinterpret_cast<uintptr_t>(d.in) & 3) == 0 && (reinterpret_cast<uintptr_t>(out) & (4 * sizeof(Out) - 1)) == 0;
    for (int64_t e = e0 + 4 * threadIdx.x; e < e1; e += 4 * blockDim.x) {
      if (vec && e + 4 <= e1) {
        const uint32_t w = __ldg(reinterpret_cast<const uint32_t *>(d.in + e));
        float v[4];
#pragma unroll
        for (int k = 0; k < 4; k++) v[k] = add_rn(mul_rn(u8_to_float((w >> (8 * k)) & 0xFFu), d.mul), d.add);
        if (sizeof(Out) == 1) {
          uint32_t o = 0;
#pragma unroll
          for (int k = 0; k < 4; k++) o |= (uint32_t)sat_u8_half_away(v[k]) << (8 * k);
          *reinterpret_cast<uint32_t *>(reinterpret_cast<uint8_t *>(out) + e) = o;
        } else {
          *reinterpret_cast<float4 *>(reinterpret_cast<float *>(out) + e) = make_float4(v[0], v[1], v[2], v[3]);
        }
      } else {
        for (int64_t q = e; q < min(e1, e + 4); q++) {
          const float v = add_rn(mul_rn((float)d.in[q], d.mul), d.add);
          if (sizeof(Out) == 1) reinterpret_cast<uint8_t *>(out)[q] = sat_u8_half_away(v);
          else reinterpret_cast<float *>(out)[q] = v;
        }
      }
    }
  }
}

// ---- pad.  The trailing axes that are not padded are merged into the innermost padded axis: the output is viewed as
// [outer rows][row_out] elements and the input as [outer rows][row_in], row_in <= row_out.  An output row is the input row's elements
// followed by fill when every outer index lies inside the input, and fill only otherwise.  A thread produces 16 output bytes
// (16 / sizeof(T) elements) and stores them with one 16-byte store when the sample's output is 16-byte aligned.
constexpr int kPadMaxDim = 6;
constexpr int kPadItemBytes = 16384;            // output bytes per work item
struct PadDesc {
  const uint8_t *in; uint8_t *out;
  int64_t out_bytes, first_item;
  int64_t row_in, row_out;                      // elements
  int64_t out_outer[kPadMaxDim], in_outer[kPadMaxDim];      // extents of the outer axes (outermost first)
  int32_t nouter;
};

// input row of output row r, or -1 when r lies in the padding of an outer axis
__device__ __forceinline__ int64_t pad_in_row(const PadDesc &d, int64_t r) {
  int64_t in_r = 0, mul = 1;
  for (int a = d.nouter - 1; a >= 0; a--) {
    const int64_t q = r / d.out_outer[a], idx = r - q * d.out_outer[a];
    if (idx >= d.in_outer[a]) return -1;
    in_r += idx * mul; mul *= d.in_outer[a]; r = q;
  }
  return in_r;
}

template <typename T>
__global__ void __launch_bounds__(256) pad_kernel(const PadDesc *__restrict__ descs, int n, int64_t total_items, T fill) {
  constexpr int V = 16 / sizeof(T);
  for (int64_t item = blockIdx.x; item < total_items; item += gridDim.x) {
    const PadDesc &d = descs[last_at_most(descs, 0, n - 1, item, [](const PadDesc &p) { return p.first_item; })];
    const int64_t b0 = (item - d.first_item) * kPadItemBytes, b1 = min(d.out_bytes, b0 + kPadItemBytes);
    const T *in = reinterpret_cast<const T *>(d.in);
    T *out = reinterpret_cast<T *>(d.out);
    const bool vec = (reinterpret_cast<uintptr_t>(d.out) & 15) == 0;
    for (int64_t b = b0 + 16 * (int64_t)threadIdx.x; b < b1; b += 16 * (int64_t)blockDim.x) {
      const int64_t e0 = b / (int64_t)sizeof(T);
      const int cnt = (int)min((int64_t)V, (b1 - b) / (int64_t)sizeof(T));
      int64_t r = e0 / d.row_out, col = e0 - r * d.row_out;
      int64_t src = pad_in_row(d, r);
      union { uint4 u; T t[V]; } v;
#pragma unroll
      for (int k = 0; k < V; k++) {
        if (k < cnt) {
          v.t[k] = (src >= 0 && col < d.row_in) ? __ldg(in + src * d.row_in + col) : fill;
          if (++col == d.row_out && k + 1 < cnt) { col = 0; r++; src = pad_in_row(d, r); }
        }
      }
      if (vec && cnt == V) *reinterpret_cast<uint4 *>(out + e0) = v.u;
      else for (int k = 0; k < cnt; k++) out[e0 + k] = v.t[k];
    }
  }
}

__global__ void __launch_bounds__(256) window_copy_kernel(const GenDesc *__restrict__ descs, int n, int64_t total_items) {
  for (int64_t item = blockIdx.x; item < total_items; item += gridDim.x) {
    const int s = last_at_most(descs, 0, n - 1, item, [](const GenDesc &d) { return d.first_item; });
    const GenDesc &d = descs[s];
    const int64_t e0 = (item - d.first_item) * kGenItem, e1 = min(d.n, e0 + kGenItem);
    uint8_t *out = static_cast<uint8_t *>(d.out);
    const uint32_t row = (uint32_t)d.out_w * (uint32_t)d.c;          // WindowCopySetup rejects samples of 2^31 elements or more
    for (int64_t e = e0 + threadIdx.x; e < e1; e += blockDim.x) {
      const int oy = (int)((uint32_t)e / row);
      const int r = (int)((uint32_t)e - (uint32_t)oy * row);
      const int ox = r / d.c, ch = r - ox * d.c;
      const int sy = d.anchor_y + (d.flip_y ? d.out_h - 1 - oy : oy), sx = d.anchor_x + (d.flip_x ? d.out_w - 1 - ox : ox);
      uint8_t v = d.fill[min(ch, 3)];
      if (sy >= 0 && sy < d.in_h && sx >= 0 && sx < d.in_w) v = __ldg(d.in + ((int64_t)sy * d.in_w + sx) * d.c + ch);
      out[e] = v;
    }
  }
}

}  // namespace dalib200

using namespace dalib200;  // NOLINT

struct dalib200GenericPlan {
  int max_batch = 0, n = 0, kind = 0, out_dtype = DALIB200_UINT8;      // kind 1 = multiply-add, 2 = window copy, 3 = pad
  std::vector<GenDesc> descs;
  std::vector<PadDesc> pad;
  int pad_elem = 1; uint32_t pad_fill = 0;
  int64_t total_items = 0;
  DescArena arena;
};

extern "C" {

int dalib200GenericPlanCreate(dalib200GenericPlan **plan, int max_batch) try {
  DB_CHECK_ARG(plan && max_batch > 0, "GenericPlanCreate: bad arguments");
  auto *p = new dalib200GenericPlan();
  p->max_batch = max_batch;
  *plan = p;
  return DALIB200_SUCCESS;
} DB_API_CATCH

int dalib200GenericPlanDestroy(dalib200GenericPlan *p) try {
  if (!p) return DALIB200_SUCCESS;
  p->arena.Free();
  delete p;
  return DALIB200_SUCCESS;
} DB_API_CATCH

int dalib200MultiplyAddSetup(dalib200GenericPlan *p, int n, const int64_t *volumes, const float *multipliers, const float *addends, int out_dtype) try {
  DB_CHECK_ARG(p && n >= 0 && n <= p->max_batch && (n == 0 || (volumes && multipliers && addends)), "MultiplyAddSetup: bad arguments");
  DB_CHECK_ARG(out_dtype == DALIB200_UINT8 || out_dtype == DALIB200_FLOAT, "MultiplyAddSetup: output type must be UINT8 or FLOAT");
  p->kind = 1; p->n = n; p->out_dtype = out_dtype;
  p->descs.assign(n, GenDesc());
  int64_t items = 0;
  for (int i = 0; i < n; i++) {
    GenDesc &d = p->descs[i];
    memset(&d, 0, sizeof(d));
    DB_CHECK_ARG(volumes[i] >= 0, "MultiplyAddSetup: sample %d has a negative size", i);
    d.n = volumes[i]; d.mul = multipliers[i]; d.add = addends[i];
    d.first_item = items;
    items += (d.n + kGenItem - 1) / kGenItem;
  }
  p->total_items = items;
  return DALIB200_SUCCESS;
} DB_API_CATCH

int dalib200WindowCopySetup(dalib200GenericPlan *p, int n, const dalib200WindowSample *samples) try {
  DB_CHECK_ARG(p && n >= 0 && n <= p->max_batch && (n == 0 || samples), "WindowCopySetup: bad arguments");
  p->kind = 2; p->n = n; p->out_dtype = DALIB200_UINT8;
  p->descs.assign(n, GenDesc());
  int64_t items = 0;
  for (int i = 0; i < n; i++) {
    const dalib200WindowSample &w = samples[i];
    DB_CHECK_ARG(w.in_h >= 0 && w.in_w >= 0 && w.channels >= 1 && w.out_h >= 0 && w.out_w >= 0, "WindowCopySetup: sample %d: bad shape", i);
    GenDesc &d = p->descs[i];
    memset(&d, 0, sizeof(d));
    d.in_h = w.in_h; d.in_w = w.in_w; d.c = w.channels;
    d.anchor_y = w.anchor_y; d.anchor_x = w.anchor_x; d.out_h = w.out_h; d.out_w = w.out_w;
    d.flip_x = w.flip_x != 0; d.flip_y = w.flip_y != 0;
    for (int k = 0; k < 4; k++) d.fill[k] = w.fill[k];
    DB_CHECK_ARG(ElementsFit31(w.out_h, w.out_w, w.channels) && ElementsFit31(w.in_h, w.in_w, w.channels),
                 "WindowCopySetup: sample %d: images of 2^31 elements or more are not supported", i);
    d.n = (int64_t)w.out_h * w.out_w * w.channels;
    d.first_item = items;
    items += (d.n + kGenItem - 1) / kGenItem;
  }
  p->total_items = items;
  return DALIB200_SUCCESS;
} DB_API_CATCH

int dalib200PadSetup(dalib200GenericPlan *p, int n, int ndim, int elem_size, const int64_t *in_shapes, const int64_t *out_shapes,
                     const void *fill_bytes) try {
  DB_CHECK_ARG(p && n >= 0 && n <= p->max_batch && fill_bytes && (n == 0 || (in_shapes && out_shapes)), "PadSetup: bad arguments");
  DB_CHECK_ARG(ndim >= 1 && ndim <= kPadMaxDim, "Pad: samples of 1 .. %d dimensions are supported (got %d)", kPadMaxDim, ndim);
  DB_CHECK_ARG(elem_size == 1 || elem_size == 2 || elem_size == 4, "Pad: elements of 1, 2 or 4 bytes are supported (got %d)", elem_size);
  p->kind = 3; p->n = n; p->pad_elem = elem_size;
  p->pad_fill = 0;
  memcpy(&p->pad_fill, fill_bytes, elem_size);
  p->pad.assign(n, PadDesc());
  int64_t items = 0;
  for (int i = 0; i < n; i++) {
    const int64_t *is = in_shapes + (size_t)i * ndim, *os = out_shapes + (size_t)i * ndim;
    int last = 0;                                   // innermost padded axis (0 when nothing is padded)
    double vol = 1;
    for (int a = 0; a < ndim; a++) {
      DB_CHECK_ARG(is[a] >= 0 && os[a] >= is[a], "Pad: sample %d axis %d: the output extent (%lld) must not be below the input's (%lld)", i, a,
                   (long long)os[a], (long long)is[a]);
      if (os[a] != is[a]) last = a;
      vol *= (double)os[a];
    }
    DB_CHECK_ARG(vol * elem_size < 9.0e15, "Pad: sample %d is too large", i);
    PadDesc &d = p->pad[i];
    memset(&d, 0, sizeof(d));
    d.row_in = is[last]; d.row_out = os[last];
    for (int a = last + 1; a < ndim; a++) { d.row_in *= is[a]; d.row_out *= os[a]; }
    d.nouter = last;
    int64_t rows = 1;
    for (int a = 0; a < last; a++) { d.out_outer[a] = os[a]; d.in_outer[a] = is[a]; rows *= os[a]; }
    d.out_bytes = rows * d.row_out * elem_size;
    d.first_item = items;
    items += (d.out_bytes + kPadItemBytes - 1) / kPadItemBytes;
  }
  p->total_items = items;
  return DALIB200_SUCCESS;
} DB_API_CATCH

static int PadLaunch(dalib200GenericPlan *p, const void *const *in_ptrs, void *const *out_ptrs, dalib200Stream_t stream) {
  PadDesc *h;
  int rc = p->arena.Stage(sizeof(PadDesc) * p->n, &h);
  if (rc) return rc;
  for (int i = 0; i < p->n; i++) { h[i] = p->pad[i]; h[i].in = static_cast<const uint8_t *>(in_ptrs[i]); h[i].out = static_cast<uint8_t *>(out_ptrs[i]); }
  if ((rc = p->arena.Upload(sizeof(PadDesc) * p->n, stream))) return rc;
  const PadDesc *d = reinterpret_cast<const PadDesc *>(p->arena.dev);
  const int grid = (int)std::min<int64_t>(p->total_items, (int64_t)NumSMs() * 16);
  if (p->pad_elem == 1) Launch("pad", pad_kernel<uint8_t>, grid, 256, 0, stream, d, p->n, p->total_items, (uint8_t)p->pad_fill);
  else if (p->pad_elem == 2) Launch("pad", pad_kernel<uint16_t>, grid, 256, 0, stream, d, p->n, p->total_items, (uint16_t)p->pad_fill);
  else Launch("pad", pad_kernel<uint32_t>, grid, 256, 0, stream, d, p->n, p->total_items, p->pad_fill);
  DB_CUDA(cudaGetLastError());
  return DALIB200_SUCCESS;
}

int dalib200GenericLaunch(dalib200GenericPlan *p, const void *const *in_ptrs, void *const *out_ptrs, dalib200Stream_t stream) try {
  DB_CHECK_ARG(p && p->kind != 0 && (p->n == 0 || (in_ptrs && out_ptrs)), "GenericLaunch: call a ...Setup function first");
  if (p->n == 0 || p->total_items == 0) return DALIB200_SUCCESS;
  if (p->kind == 3) return PadLaunch(p, in_ptrs, out_ptrs, stream);
  GenDesc *h;
  int rc = p->arena.Stage(sizeof(GenDesc) * p->n, &h);
  if (rc) return rc;
  for (int i = 0; i < p->n; i++) { h[i] = p->descs[i]; h[i].in = static_cast<const uint8_t *>(in_ptrs[i]); h[i].out = out_ptrs[i]; }
  if ((rc = p->arena.Upload(sizeof(GenDesc) * p->n, stream))) return rc;
  const GenDesc *d = reinterpret_cast<const GenDesc *>(p->arena.dev);
  const int grid = (int)std::min<int64_t>(p->total_items, (int64_t)NumSMs() * 16);
  if (p->kind == 1)
    Launch("multiply_add", p->out_dtype == DALIB200_UINT8 ? multiply_add_kernel<uint8_t> : multiply_add_kernel<float>, grid, 256, 0, stream, d, p->n,
           p->total_items);
  else
    Launch("window_copy", window_copy_kernel, grid, 256, 0, stream, d, p->n, p->total_items);
  DB_CUDA(cudaGetLastError());
  return DALIB200_SUCCESS;
} DB_API_CATCH

}  // extern "C"
