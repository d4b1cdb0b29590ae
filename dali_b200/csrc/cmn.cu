// dali_b200/csrc/cmn.cu -- CropMirrorNormalize for sm_90a.
//
// Semantics = reference CPU kernel SliceFlipNormalizePermutePadCpu
// (dali/kernels/slice/slice_flip_normalize_permute_pad_cpu.h:37-46):
//     out = ConvertSat<Out>((float(in) - mean[c]) * inv_std[c])     -- sub then mul, two roundings,
// float16 conversion = half_float round-to-nearest ties-away (include/dali/util/half.hpp:233,242).
// (The reference GPU kernel uses fma(in, inv_std, -mean*inv_std): slice_hwc2chw_normalize_gpu.cu:408,791;
// we follow the CPU backend, which is the parity target.)
//
// Fast path (u8 HWC 3-ch window inside the image -> CHW): one warp per 128-pixel row segment.
//   * loads: 3 fully coalesced 128-byte LDG.32 per warp (+ realignment word) through the non-coherent path,
//   * the HWC->CHW regrouping is a register transpose done with warp shuffles (no shared memory),
//   * stores: each lane writes 4 consecutive pixels of one plane -> one 128/256-byte coalesced
//     vector store per plane per warp.
// Everything else (padding, out-of-bounds windows, C != 3, HWC output) takes the generic
// one-thread-per-output-element kernel.
//
// Algorithmic bytes per unit (SURVEY.md 8d): crop_h*crop_w*C read + crop_h*crop_w*out_c*sizeof(Out) written.
#include "common.cuh"
#include <algorithm>
#include <cstring>

namespace dalib200 {

struct CmnDesc {
  const uint8_t *in;
  void *out;
  int32_t in_h, in_w, C;
  int32_t ay, ax, ch, cw;
  int32_t mirror, fast;
  int64_t first_unit;      // first warp-unit (fast) of this sample in the batch
  int64_t first_elem;      // first output element (generic) of this sample in the batch
  float mean[4], inv_std[4], fill[4];
};

template <typename Out>
__device__ __forceinline__ void store4(Out *p, Out a, Out b, Out c, Out d);
template <>
__device__ __forceinline__ void store4<float>(float *p, float a, float b, float c, float d) {
  *reinterpret_cast<float4 *>(p) = make_float4(a, b, c, d);
}
template <>
__device__ __forceinline__ void store4<uint16_t>(uint16_t *p, uint16_t a, uint16_t b, uint16_t c, uint16_t d) {
  *reinterpret_cast<uint2 *>(p) = make_uint2((uint32_t)a | ((uint32_t)b << 16), (uint32_t)c | ((uint32_t)d << 16));
}

// ------------------------------------------------------------------------------------------
// Fast path: u8 HWC (3 ch) -> planar CHW Out, window inside the image.
// A unit = 128 pixels of one row (384 source bytes); a warp works on TWO units per iteration -- all six coalesced word loads are
// issued before the first is consumed, which doubles the bytes each warp keeps in flight (the kernel is latency-bound otherwise).
struct CmnUnit {
  const CmnDesc *d;
  const uint32_t *aw;
  int y, xb, npx, nwords;
  uint32_t sh;
  uint32_t w[3], extra;
};

__device__ __forceinline__ void cmn_unit_open(CmnUnit &c, const CmnDesc &d, int64_t u, int lane) {
  c.d = &d;
  const int upr = (d.cw + 127) >> 7;
  c.y = (int)((uint32_t)u / (uint32_t)upr);            // units of one sample fit 32 bits; a 64-bit division costs ~100 instructions
  c.xb = (int)((uint32_t)u - (uint32_t)c.y * (uint32_t)upr) << 7;
  c.npx = min(128, d.cw - c.xb);
  const int src_px0 = d.mirror ? d.ax + d.cw - c.xb - c.npx : d.ax + c.xb;
  const uint8_t *a = d.in + ((int64_t)(d.ay + c.y) * d.in_w + src_px0) * 3;
  c.sh = (uint32_t)(reinterpret_cast<uintptr_t>(a) & 3);
  c.aw = reinterpret_cast<const uint32_t *>(a - c.sh);
  c.nwords = (int)((c.sh + c.npx * 3 + 3) >> 2);       // aligned words covering the segment
  // coalesced loads: word index = lane + 32 t
#pragma unroll
  for (int t = 0; t < 3; t++) {
    const int i = lane + 32 * t;
    c.w[t] = i < c.nwords ? ld_nc_u32(c.aw + i) : 0u;
  }
  // word 96 for the funnel shift of the last word when the segment is misaligned
  c.extra = (c.sh != 0 && lane == 0 && 96 < c.nwords) ? ld_nc_u32(c.aw + 96) : 0u;
}

template <typename Out>
__device__ __forceinline__ void cmn_unit_finish(const CmnUnit &c, int lane, int out_c) {
  const CmnDesc &d = *c.d;
  const uint32_t extra = __shfl_sync(0xffffffffu, c.extra, 0);
  uint32_t wn[3];
  {
    const uint32_t n0 = __shfl_down_sync(0xffffffffu, c.w[0], 1), n1 = __shfl_down_sync(0xffffffffu, c.w[1], 1),
                   n2 = __shfl_down_sync(0xffffffffu, c.w[2], 1);
    const uint32_t f1 = __shfl_sync(0xffffffffu, c.w[1], 0), f2 = __shfl_sync(0xffffffffu, c.w[2], 0);
    wn[0] = lane == 31 ? f1 : n0;
    wn[1] = lane == 31 ? f2 : n1;
    wn[2] = lane == 31 ? extra : n2;
  }
  uint32_t r[3];
#pragma unroll
  for (int t = 0; t < 3; t++) r[t] = __funnelshift_r(c.w[t], wn[t], c.sh * 8);   // realigned word (lane + 32 t)
  // register transpose: lane l needs realigned words 3l, 3l+1, 3l+2
  uint32_t q[3];
#pragma unroll
  for (int k = 0; k < 3; k++) {
    const int j = 3 * lane + k;
    const int src = j & 31, reg = j >> 5;
    const uint32_t v0 = __shfl_sync(0xffffffffu, r[0], src);
    const uint32_t v1 = __shfl_sync(0xffffffffu, r[1], src);
    const uint32_t v2 = __shfl_sync(0xffffffffu, r[2], src);
    q[k] = reg == 0 ? v0 : reg == 1 ? v1 : v2;
  }
  // 12 bytes = 4 pixels x 3 channels
  const int p0 = lane * 4, npx = c.npx, xb = c.xb;
  if (p0 >= npx) return;
  Out *obase = static_cast<Out *>(d.out);
  const int64_t plane = (int64_t)d.ch * d.cw;
#pragma unroll
  for (int ch = 0; ch < 3; ch++) {
    Out v[4];
#pragma unroll
    for (int p = 0; p < 4; p++) {
      const int bi = 3 * p + ch;
      const uint32_t byte = (q[bi >> 2] >> ((bi & 3) * 8)) & 0xFFu;
      const float f = mul_rn(sub_rn(u8_to_float(byte), d.mean[ch]), d.inv_std[ch]);
      v[p] = OutConv<Out>::cvt(f);
    }
    Out *orow = obase + ch * plane + (int64_t)c.y * d.cw;
    const int valid = min(4, npx - p0);
    if (!d.mirror) {
      Out *o = orow + xb + p0;
      if (valid == 4 && (reinterpret_cast<uintptr_t>(o) & (4 * sizeof(Out) - 1)) == 0) {
        store4<Out>(o, v[0], v[1], v[2], v[3]);
      } else {
        for (int p = 0; p < valid; p++) o[p] = v[p];
      }
    } else {
      // source pixel (src_px0 + p0 + p) lands at output x = xb + npx - 1 - (p0 + p)
      Out *o = orow + xb + npx - 1 - p0 - 3;      // address of the p = 3 pixel
      if (valid == 4 && (reinterpret_cast<uintptr_t>(o) & (4 * sizeof(Out) - 1)) == 0) {
        store4<Out>(o, v[3], v[2], v[1], v[0]);
      } else {
        for (int p = 0; p < valid; p++) orow[xb + npx - 1 - p0 - p] = v[p];
      }
    }
  }
  // padding planes (pad_output): constant fill
  for (int ch = 3; ch < out_c; ch++) {
    const Out fv = OutConv<Out>::cvt(d.fill[ch]);
    Out *orow = obase + ch * plane + (int64_t)c.y * d.cw + xb;
    for (int p = p0; p < min(p0 + 4, npx); p++) orow[p] = fv;
  }
}

template <typename Out>
__global__ void __launch_bounds__(256) cmn_hwc2chw_kernel(const CmnDesc *__restrict__ descs, int n, int64_t total_units,
                                                          int out_c) {
  const int lane = threadIdx.x & 31;
  // every CTA owns one contiguous range of units (its 8 warps interleaved): the sample is searched once per CTA and then only
  // advanced -- a binary search over thousands of frame descriptors per 384-byte unit used to dominate this kernel
  __shared__ int s_first;
  const int wpc = blockDim.x >> 5;
  const int64_t per_cta = ((total_units + gridDim.x - 1) / gridDim.x + 2 * wpc - 1) / (2 * wpc) * (2 * wpc);
  const int64_t u0 = (int64_t)blockIdx.x * per_cta, u1 = min(total_units, u0 + per_cta);
  if (u0 >= u1) return;
  if (threadIdx.x == 0) s_first = last_at_most(descs, 0, n - 1, u0, [](const CmnDesc &d) { return d.first_unit; });
  __syncthreads();
  int s = s_first;
  for (int64_t unit = u0 + (threadIdx.x >> 5); unit < u1; unit += 2 * wpc) {
    while (s + 1 < n && descs[s + 1].first_unit <= unit) s++;
    const int64_t unit2 = unit + wpc;
    int s2 = s;
    const bool two = unit2 < u1;
    if (two) while (s2 + 1 < n && descs[s2 + 1].first_unit <= unit2) s2++;
    const bool go1 = descs[s].fast != 0, go2 = two && descs[s2].fast != 0;       // generic samples own zero units, defensive
    CmnUnit a, b;
    if (go1) cmn_unit_open(a, descs[s], unit - descs[s].first_unit, lane);
    if (go2) cmn_unit_open(b, descs[s2], unit2 - descs[s2].first_unit, lane);
    if (go1) cmn_unit_finish<Out>(a, lane, out_c);
    if (go2) cmn_unit_finish<Out>(b, lane, out_c);
    s = s2;
  }
}

// ------------------------------------------------------------------------------------------
// Generic path: one thread per output element, any C <= 4, HWC or CHW, out-of-bounds -> fill.
template <typename Out>
__global__ void __launch_bounds__(256) cmn_generic_kernel(const CmnDesc *__restrict__ descs, int n, int64_t total_elems,
                                                          int out_c, int chw) {
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total_elems; e += (int64_t)gridDim.x * blockDim.x) {
    const int s = last_at_most(descs, 0, n - 1, e, [](const CmnDesc &d) { return d.first_elem; });
    const CmnDesc &d = descs[s];
    if (d.fast) continue;
    int64_t i = e - d.first_elem;
    int x, y, c;
    if (chw) { x = (int)(i % d.cw); i /= d.cw; y = (int)(i % d.ch); c = (int)(i / d.ch); }
    else { c = (int)(i % out_c); i /= out_c; x = (int)(i % d.cw); y = (int)(i / d.cw); }
    const int sy = d.ay + y;
    const int sx = d.mirror ? d.ax + (d.cw - 1 - x) : d.ax + x;
    Out r;
    if (c >= d.C || sy < 0 || sy >= d.in_h || sx < 0 || sx >= d.in_w) {
      // fill values are static_cast to the output type, no saturation (cpu.h:344-346)
      float fv = d.fill[c];
      if (sizeof(Out) == 2) {
        // static_cast<float16>(float): the half_float conversion without the +-65504 clamp
        uint32_t bits = __float_as_uint(fv);
        uint32_t ex = (bits >> 23) & 0xFFu;
        if (ex >= 143u) {   // overflow / inf / nan -> inf (nan keeps payload top bits)
          uint16_t h = (uint16_t)(((bits >> 16) & 0x8000u) | 0x7C00u | (ex == 255u ? ((bits & 0x7FFFFFu) >> 13) : 0u));
          r = *reinterpret_cast<Out *>(&h);
        } else {
          r = OutConv<Out>::cvt(fv);
        }
      } else {
        r = OutConv<Out>::cvt(fv);
      }
    } else {
      const float f = (float)d.in[((int64_t)sy * d.in_w + sx) * d.C + c];
      r = OutConv<Out>::cvt(mul_rn(sub_rn(f, d.mean[c]), d.inv_std[c]));
    }
    static_cast<Out *>(d.out)[e - d.first_elem] = r;
  }
}

}  // namespace dalib200

using namespace dalib200;  // NOLINT

struct dalib200CmnPlan {
  int max_batch = 0, n = 0;
  int out_dtype = DALIB200_FLOAT, out_layout = DALIB200_LAYOUT_CHW, out_c = 3;
  int64_t total_units = 0, total_elems = 0;
  DescArena arena;
};

extern "C" {

int dalib200CmnPlanCreate(dalib200CmnPlan **plan, int max_batch) try {
  DB_CHECK_ARG(plan && max_batch > 0, "CmnPlanCreate: bad arguments");
  auto *p = new dalib200CmnPlan();
  p->max_batch = max_batch;
  int rc = p->arena.Reserve(sizeof(CmnDesc) * max_batch);
  if (rc) { delete p; return rc; }
  *plan = p;
  return DALIB200_SUCCESS;
} DB_API_CATCH

int dalib200CmnPlanDestroy(dalib200CmnPlan *p) try {
  if (!p) return DALIB200_SUCCESS;
  p->arena.Free();
  delete p;
  return DALIB200_SUCCESS;
} DB_API_CATCH

int dalib200CmnPlanSetup(dalib200CmnPlan *p, int n, const dalib200CmnSample *samples, int out_dtype, int out_layout,
                         int out_channels) try {
  DB_CHECK_ARG(p && samples && n >= 0, "CmnPlanSetup: null argument");
  DB_CHECK_ARG(n <= p->max_batch, "CmnPlanSetup: batch %d exceeds plan capacity %d", n, p->max_batch);
  DB_CHECK_ARG(out_dtype == DALIB200_FLOAT || out_dtype == DALIB200_FLOAT16,
               "CropMirrorNormalize: output type %d not supported (FLOAT, FLOAT16)", out_dtype);
  DB_CHECK_ARG(out_layout == DALIB200_LAYOUT_HWC || out_layout == DALIB200_LAYOUT_CHW, "CropMirrorNormalize: bad layout");
  DB_CHECK_ARG(out_channels >= 1 && out_channels <= 4, "CropMirrorNormalize: 1..4 output channels supported, got %d", out_channels);
  CmnDesc *descs;
  if (int rc = p->arena.Stage(sizeof(CmnDesc) * n, &descs)) return rc;
  int64_t units = 0, elems = 0;
  for (int i = 0; i < n; i++) {
    const auto &s = samples[i];
    DB_CHECK_ARG(s.in_h >= 0 && s.in_w >= 0 && s.channels >= 1 && s.channels <= 4,
                 "CropMirrorNormalize: sample %d has unsupported shape %dx%dx%d", i, s.in_h, s.in_w, s.channels);
    DB_CHECK_ARG(s.crop_h >= 0 && s.crop_w >= 0, "CropMirrorNormalize: sample %d negative crop", i);
    DB_CHECK_ARG(out_channels >= s.channels, "CropMirrorNormalize: out_channels < input channels");
    DB_CHECK_ARG(ElementsFit31(s.in_h, s.in_w, s.channels) && ElementsFit31(s.crop_h, s.crop_w, out_channels),
                 "CropMirrorNormalize: sample %d: inputs / outputs of 2^31 elements or more are not supported", i);
    CmnDesc &d = descs[i];
    memset(&d, 0, sizeof(d));
    d.in_h = s.in_h; d.in_w = s.in_w; d.C = s.channels;
    d.ay = s.anchor_y; d.ax = s.anchor_x; d.ch = s.crop_h; d.cw = s.crop_w;
    d.mirror = s.mirror != 0;
    for (int c = 0; c < 4; c++) { d.mean[c] = s.mean[c]; d.inv_std[c] = s.inv_std[c]; d.fill[c] = s.fill[c]; }
    const bool inside = s.anchor_y >= 0 && s.anchor_x >= 0 && (int64_t)s.anchor_y + s.crop_h <= s.in_h &&
                        (int64_t)s.anchor_x + s.crop_w <= s.in_w;
    d.fast = (s.channels == 3 && out_layout == DALIB200_LAYOUT_CHW && inside && s.crop_h > 0 && s.crop_w > 0) ? 1 : 0;
    d.first_unit = units;
    d.first_elem = elems;
    if (d.fast) units += (int64_t)s.crop_h * ((s.crop_w + 127) / 128);
    else elems += (int64_t)s.crop_h * s.crop_w * out_channels;
  }
  p->n = n; p->out_dtype = out_dtype; p->out_layout = out_layout; p->out_c = out_channels;
  p->total_units = units; p->total_elems = elems;
  return DALIB200_SUCCESS;
} DB_API_CATCH

int dalib200CmnLaunch(dalib200CmnPlan *p, const void *const *in_ptrs, void *const *out_ptrs, dalib200Stream_t stream) try {
  DB_CHECK_ARG(p && in_ptrs && out_ptrs, "CmnLaunch: null argument");
  if (p->n == 0) return DALIB200_SUCCESS;
  CmnDesc *descs;
  if (int rc = p->arena.Stage(sizeof(CmnDesc) * p->n, &descs)) return rc;
  for (int i = 0; i < p->n; i++) {
    descs[i].in = static_cast<const uint8_t *>(in_ptrs[i]);
    descs[i].out = out_ptrs[i];
  }
  int rc = p->arena.Upload(sizeof(CmnDesc) * p->n, stream);
  if (rc) return rc;
  const CmnDesc *dd = reinterpret_cast<const CmnDesc *>(p->arena.dev);
  const int sms = NumSMs();
  if (p->total_units > 0) {
    int64_t blocks = (p->total_units + 7) / 8;
    int grid = (int)std::min<int64_t>(blocks, (int64_t)sms * 8);
    Launch("cmn_hwc2chw", p->out_dtype == DALIB200_FLOAT ? cmn_hwc2chw_kernel<float> : cmn_hwc2chw_kernel<uint16_t>, grid, 256, 0, stream, dd, p->n,
           p->total_units, p->out_c);
  }
  if (p->total_elems > 0) {
    int64_t blocks = (p->total_elems + 255) / 256;
    int grid = (int)std::min<int64_t>(blocks, (int64_t)sms * 16);
    const int chw = p->out_layout == DALIB200_LAYOUT_CHW;
    Launch("cmn_generic", p->out_dtype == DALIB200_FLOAT ? cmn_generic_kernel<float> : cmn_generic_kernel<uint16_t>, grid, 256, 0, stream, dd, p->n,
           p->total_elems, p->out_c, chw);
  }
  DB_CUDA(cudaGetLastError());
  return DALIB200_SUCCESS;
} DB_API_CATCH

}  // extern "C"
