// dali_b200/csrc/pointwise.cu -- per-pixel colour kernels for sm_90a: 3x3 linear transform (Hsv / ColorTwist)
// and ColorSpaceConversion.
//
// Parity targets:
//   * LinearTransformationCpu (dali/kernels/imgproc/pointwise/linear_transformation_cpu.h:57-78):
//       out_c = ConvertSat<Out>( ((m_c0*in_0 + m_c1*in_1) + m_c2*in_2) + t_c )     mul/add unfused (mat.h:283-297)
//     matrix composition on the host: dali/operators/image/color/color_twist.h:50-83,156-170
//   * ColorSpaceConversion CPU (dali/util/ocv.cc:30-158): RGB<->BGR<->GRAY through OpenCV cvtColor (15-bit fixed
//     point: 9798 R + 19235 G + 3735 B, +2^14, >>15), YCbCr through the in-tree BT.601 formulas
//     (dali/kernels/imgproc/color_manipulation/color_space_conversion_impl.h:64-156, bias_scale<u8> = 256).
//
// All samples of a batch are processed by ONE launch (the reference launches ColorSpaceConvKernel once per
// sample: operators/image/color/color_space_conversion.cu:33-39).  Each thread owns 4 consecutive pixels:
// 3 x 32-bit loads / stores when the sample base is 4-byte aligned.
//
// Algorithmic bytes per pixel: in_channels + out_channels * sizeof(Out).
#include "common.cuh"
#include <algorithm>
#include <cmath>
#include <cstring>

namespace dalib200 {

enum { PW_LINEAR = 0, PW_CSC = 1 };

struct PwDesc {
  const uint8_t *in;
  void *out;
  int64_t npix;
  int64_t first_quad;
  float m[9], t[3];
};

template <int NB>
__device__ __forceinline__ void load_bytes(const uint8_t *p, int n, uint8_t *b) {
  if (n == NB && (reinterpret_cast<uintptr_t>(p) & 3) == 0) {
    const uint32_t *w = reinterpret_cast<const uint32_t *>(p);
#pragma unroll
    for (int i = 0; i < NB / 4; i++) {
      const uint32_t v = ld_nc_u32(w + i);
      b[4 * i] = v & 0xFF; b[4 * i + 1] = (v >> 8) & 0xFF; b[4 * i + 2] = (v >> 16) & 0xFF; b[4 * i + 3] = v >> 24;
    }
  } else {
    for (int i = 0; i < n; i++) b[i] = __ldg(p + i);
  }
}
template <int NB>
__device__ __forceinline__ void store_bytes(uint8_t *p, int n, const uint8_t *b) {
  if (n == NB && (reinterpret_cast<uintptr_t>(p) & 3) == 0) {
    uint32_t *w = reinterpret_cast<uint32_t *>(p);
#pragma unroll
    for (int i = 0; i < NB / 4; i++)
      w[i] = (uint32_t)b[4 * i] | ((uint32_t)b[4 * i + 1] << 8) | ((uint32_t)b[4 * i + 2] << 16) | ((uint32_t)b[4 * i + 3] << 24);
  } else {
    for (int i = 0; i < n; i++) p[i] = b[i];
  }
}

// one quad (4 pixels, 12 bytes) of the linear transform
template <typename Out>
__device__ __forceinline__ void lt_quad(const PwDesc &d, int64_t p0, int np) {
  uint8_t b[12];
  load_bytes<12>(d.in + p0 * 3, np * 3, b);
  if (sizeof(Out) == 1) {
    uint8_t o[12];
#pragma unroll
    for (int k = 0; k < 4; k++) {
      const float v0 = u8_to_float(b[3 * k]), v1 = u8_to_float(b[3 * k + 1]), v2 = u8_to_float(b[3 * k + 2]);
#pragma unroll
      for (int c = 0; c < 3; c++) {
        float r = mul_rn(d.m[c * 3], v0);
        r = add_rn(r, mul_rn(d.m[c * 3 + 1], v1));
        r = add_rn(r, mul_rn(d.m[c * 3 + 2], v2));
        r = add_rn(r, d.t[c]);
        o[3 * k + c] = sat_u8_half_away(r);
      }
    }
    store_bytes<12>(static_cast<uint8_t *>(d.out) + p0 * 3, np * 3, o);
  } else {
    float *o = reinterpret_cast<float *>(d.out) + p0 * 3;
    for (int k = 0; k < np; k++) {
      const float v0 = u8_to_float(b[3 * k]), v1 = u8_to_float(b[3 * k + 1]), v2 = u8_to_float(b[3 * k + 2]);
#pragma unroll
      for (int c = 0; c < 3; c++) {
        float r = mul_rn(d.m[c * 3], v0);
        r = add_rn(r, mul_rn(d.m[c * 3 + 1], v1));
        r = add_rn(r, mul_rn(d.m[c * 3 + 2], v2));
        o[3 * k + c] = add_rn(r, d.t[c]);
      }
    }
  }
}

template <typename Out>
__global__ void __launch_bounds__(256) linear_transform_kernel(const PwDesc *__restrict__ descs, int n, int64_t total_quads) {
  // every CTA owns one contiguous range of quads: the sample is searched once per CTA and then only advanced (a per-thread
  // binary search over thousands of frame descriptors costs more than the pixels of work behind it).  A thread takes four
  // consecutive quads = 16 pixels = 48 bytes: three 128-bit loads and stores when they lie in one sample and are 16-byte
  // aligned (more bytes in flight per thread, 4x fewer memory instructions), quad by quad otherwise.
  __shared__ int s_first;
  const int64_t per_cta = ((total_quads + gridDim.x - 1) / gridDim.x + 1023) / 1024 * 1024;
  const int64_t q0 = (int64_t)blockIdx.x * per_cta, q1 = min(total_quads, q0 + per_cta);
  if (q0 >= q1) return;
  if (threadIdx.x == 0) s_first = last_at_most(descs, 0, n - 1, q0, [](const PwDesc &d) { return d.first_quad; });
  __syncthreads();
  int s = s_first;
  for (int64_t gq = q0 + 4 * threadIdx.x; gq < q1; gq += 4 * blockDim.x) {
    while (s + 1 < n && descs[s + 1].first_quad <= gq) s++;
    const PwDesc &d = descs[s];
    const int64_t p0 = (gq - d.first_quad) * 4;
    const uint8_t *ip = d.in + p0 * 3;
    uint8_t *op = static_cast<uint8_t *>(d.out) + p0 * 3;
    const bool one_sample = gq + 3 < q1 && (s + 1 >= n || descs[s + 1].first_quad > gq + 3) && p0 + 16 <= d.npix;
    if (sizeof(Out) == 1 && one_sample && ((reinterpret_cast<uintptr_t>(ip) | reinterpret_cast<uintptr_t>(op)) & 15) == 0) {
      uint32_t w[12], o[12];
      {
        const uint4 *p4 = reinterpret_cast<const uint4 *>(ip);
#pragma unroll
        for (int q = 0; q < 3; q++) { const uint4 v = __ldg(p4 + q); w[4 * q] = v.x; w[4 * q + 1] = v.y; w[4 * q + 2] = v.z; w[4 * q + 3] = v.w; }
      }
      const float m0 = d.m[0], m1 = d.m[1], m2 = d.m[2], m3 = d.m[3], m4 = d.m[4], m5 = d.m[5], m6 = d.m[6], m7 = d.m[7], m8 = d.m[8];
      const float t0 = d.t[0], t1 = d.t[1], t2 = d.t[2];
      uint32_t ob[48];
#pragma unroll
      for (int k = 0; k < 16; k++) {
        float v[3];
#pragma unroll
        for (int c = 0; c < 3; c++) { const int bi = 3 * k + c; v[c] = u8_to_float((w[bi >> 2] >> (8 * (bi & 3))) & 0xFFu); }
        ob[3 * k] = sat_u8_half_away(add_rn(add_rn(add_rn(mul_rn(m0, v[0]), mul_rn(m1, v[1])), mul_rn(m2, v[2])), t0));
        ob[3 * k + 1] = sat_u8_half_away(add_rn(add_rn(add_rn(mul_rn(m3, v[0]), mul_rn(m4, v[1])), mul_rn(m5, v[2])), t1));
        ob[3 * k + 2] = sat_u8_half_away(add_rn(add_rn(add_rn(mul_rn(m6, v[0]), mul_rn(m7, v[1])), mul_rn(m8, v[2])), t2));
      }
#pragma unroll
      for (int q = 0; q < 12; q++) o[q] = ob[4 * q] | (ob[4 * q + 1] << 8) | (ob[4 * q + 2] << 16) | (ob[4 * q + 3] << 24);
      uint4 *o4 = reinterpret_cast<uint4 *>(op);
#pragma unroll
      for (int q = 0; q < 3; q++) o4[q] = make_uint4(o[4 * q], o[4 * q + 1], o[4 * q + 2], o[4 * q + 3]);
    } else {
      int sq = s;
      for (int k = 0; k < 4 && gq + k < q1; k++) {
        while (sq + 1 < n && descs[sq + 1].first_quad <= gq + k) sq++;
        const PwDesc &dq = descs[sq];
        const int64_t pq = (gq + k - dq.first_quad) * 4;
        lt_quad<Out>(dq, pq, (int)min((int64_t)4, dq.npix - pq));
      }
    }
  }
}

__device__ __forceinline__ float dot3(float c0, float c1, float c2, float a, float b, float c) {
  return add_rn(add_rn(mul_rn(c0, a), mul_rn(c1, b)), mul_rn(c2, c));
}

// in_type / out_type: DALIB200_RGB, BGR, GRAY, YCbCr
__global__ void __launch_bounds__(256) csc_kernel(const PwDesc *__restrict__ descs, int n, int64_t total_quads, int in_type,
                                                  int out_type) {
  const int ic = in_type == DALIB200_GRAY ? 1 : 3, oc = out_type == DALIB200_GRAY ? 1 : 3;
  __shared__ int s_first;
  const int64_t per_cta = ((total_quads + gridDim.x - 1) / gridDim.x + 255) / 256 * 256;
  const int64_t q0 = (int64_t)blockIdx.x * per_cta, q1 = min(total_quads, q0 + per_cta);
  if (q0 >= q1) return;
  if (threadIdx.x == 0) s_first = last_at_most(descs, 0, n - 1, q0, [](const PwDesc &d) { return d.first_quad; });
  __syncthreads();
  int s = s_first;
  for (int64_t gq = q0 + threadIdx.x; gq < q1; gq += blockDim.x) {
    while (s + 1 < n && descs[s + 1].first_quad <= gq) s++;
    const PwDesc &d = descs[s];
    const int64_t p0 = (gq - d.first_quad) * 4;
    const int np = (int)min((int64_t)4, d.npix - p0);
    uint8_t b[12], o[12];
    if (ic == 3) load_bytes<12>(d.in + p0 * 3, np * 3, b); else load_bytes<4>(d.in + p0, np, b);
#pragma unroll
    for (int k = 0; k < 4; k++) {
      const uint8_t *i = b + k * ic;
      uint8_t *q = o + k * oc;
      if (in_type == out_type) {
        for (int c = 0; c < ic; c++) q[c] = i[c];
      } else if ((in_type == DALIB200_RGB && out_type == DALIB200_BGR) || (in_type == DALIB200_BGR && out_type == DALIB200_RGB)) {
        q[0] = i[2]; q[1] = i[1]; q[2] = i[0];
      } else if ((in_type == DALIB200_RGB || in_type == DALIB200_BGR) && out_type == DALIB200_GRAY) {
        const int r = in_type == DALIB200_RGB ? i[0] : i[2], g = i[1], bb = in_type == DALIB200_RGB ? i[2] : i[0];
        q[0] = (uint8_t)((r * 9798 + g * 19235 + bb * 3735 + (1 << 14)) >> 15);
      } else if (in_type == DALIB200_GRAY && (out_type == DALIB200_RGB || out_type == DALIB200_BGR)) {
        q[0] = q[1] = q[2] = i[0];
      } else if ((in_type == DALIB200_RGB || in_type == DALIB200_BGR) && out_type == DALIB200_YCbCr) {
        const float r = in_type == DALIB200_RGB ? i[0] : i[2], g = i[1], bb = in_type == DALIB200_RGB ? i[2] : i[0];
        q[0] = sat_u8_half_away(add_rn(dot3(0.25678823529f, 0.50412941176f, 0.09790588235f, r, g, bb), 16.0f));
        q[1] = sat_u8_half_away(add_rn(dot3(-0.14822289945f, -0.29099278682f, 0.43921568627f, r, g, bb), 128.0f));
        q[2] = sat_u8_half_away(add_rn(dot3(0.43921568627f, -0.36778831435f, -0.07142737192f, r, g, bb), 128.0f));
      } else if (in_type == DALIB200_YCbCr && (out_type == DALIB200_RGB || out_type == DALIB200_BGR)) {
        const float ys = mul_rn(mul_rn(sub_rn((float)i[0], 16.0f), 255.0f / 219), 1.0f);
        const float tb = sub_rn((float)i[1], 128.0f), tr = sub_rn((float)i[2], 128.0f);
        const uint8_t R = sat_u8_half_away(add_rn(ys, mul_rn(1.5960267848f, tr)));
        const uint8_t G = sat_u8_half_away(sub_rn(sub_rn(ys, mul_rn(0.39176228842f, tb)), mul_rn(0.81296764538f, tr)));
        const uint8_t B = sat_u8_half_away(add_rn(ys, mul_rn(2.0172321417f, tb)));
        if (out_type == DALIB200_RGB) { q[0] = R; q[1] = G; q[2] = B; } else { q[0] = B; q[1] = G; q[2] = R; }
      } else if (in_type == DALIB200_GRAY && out_type == DALIB200_YCbCr) {
        q[0] = sat_u8_half_away(add_rn(mul_rn((float)i[0], 219 * 1.0f / 255), 16.0f)); q[1] = 128; q[2] = 128;
      } else if (in_type == DALIB200_YCbCr && out_type == DALIB200_GRAY) {
        q[0] = sat_u8_half_away(mul_rn(255 * 1.0f / 219, sub_rn((float)i[0], 16.0f)));
      }
    }
    if (oc == 3) store_bytes<12>(static_cast<uint8_t *>(d.out) + p0 * 3, np * 3, o);
    else store_bytes<4>(static_cast<uint8_t *>(d.out) + p0, np, o);
  }
}

}  // namespace dalib200

using namespace dalib200;  // NOLINT

struct dalib200PointwisePlan {
  int max_batch = 0, n = 0;
  int mode = PW_LINEAR, out_dtype = DALIB200_UINT8, in_type = 0, out_type = 0;
  int64_t total_quads = 0;
  DescArena arena;
};

namespace {
// mat.h:262-280 with dot() = a0*b0 + a1*b1 + a2*b2 accumulated left to right (vec.h:343-348)
void Mat3Mul(const float a[9], const float b[9], float r[9]) {
  float t[9];
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++) {
      volatile float s = a[i * 3] * b[j];
      volatile float p = a[i * 3 + 1] * b[3 + j];
      s = s + p;
      p = a[i * 3 + 2] * b[6 + j];
      s = s + p;
      t[i * 3 + j] = s;
    }
  memcpy(r, t, sizeof(t));
}
// mat.h:552-609: Gauss-Jordan with partial pivoting, updates via fma
void Inverse3(float A[3][3], float O[3][3]) {
  for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) O[i][j] = i == j;
  for (int v = 0; v < 3; v++) {
    float mx = std::fabs(A[v][v]); int mr = v;
    for (int i = v + 1; i < 3; i++) { float q = std::fabs(A[i][v]); if (q > mx) { mx = q; mr = i; } }
    if (!mx) return;
    if (mr != v) for (int j = 0; j < 3; j++) { std::swap(A[v][j], A[mr][j]); std::swap(O[v][j], O[mr][j]); }
    float x = 1.0f / A[v][v];
    A[v][v] = 1;
    for (int j = v + 1; j < 3; j++) A[v][j] *= x;
    for (int j = 0; j < 3; j++) O[v][j] *= x;
    for (int i = 0; i < 3; i++) {
      if (i == v) continue;
      float c = -A[i][v];
      A[i][v] = 0;
      for (int j = v + 1; j < 3; j++) A[i][j] = std::fma(c, A[v][j], A[i][j]);
      for (int j = 0; j < 3; j++) O[i][j] = std::fma(c, O[v][j], O[i][j]);
    }
  }
}
}  // namespace

extern "C" {

void dalib200ColorTwistMatrix(float hue, float saturation, float value, float brightness, float contrast, float half_range,
                              float *M, float *T) {
  const float rgb2yiq[9] = { .299f, .587f, .114f, .596f, -.274f, -.321f, .211f, -.523f, .311f };
  float A[3][3], inv[3][3], yiq2rgb[9];
  for (int i = 0; i < 9; i++) A[i / 3][i % 3] = rgb2yiq[i];
  Inverse3(A, inv);
  for (int i = 0; i < 9; i++) yiq2rgb[i] = inv[i / 3][i % 3];
  const float h_rad = hue * M_PI / 180;
  const float ch = std::cos(h_rad), sh = std::sin(h_rad);      // float overloads, as in the reference TU
  const float hm[9] = { 1, 0, 0, 0, ch, sh, 0, -sh, ch };
  const float sm[9] = { 1, 0, 0, 0, saturation, 0, 0, 0, saturation };
  const float vm[9] = { value, 0, 0, 0, value, 0, 0, 0, value };
  const float bm[9] = { brightness, 0, 0, 0, brightness, 0, 0, 0, brightness };
  const float cm[9] = { contrast, 0, 0, 0, contrast, 0, 0, 0, contrast };
  float r[9];
  Mat3Mul(bm, cm, r); Mat3Mul(r, yiq2rgb, r); Mat3Mul(r, hm, r); Mat3Mul(r, sm, r); Mat3Mul(r, vm, r); Mat3Mul(r, rgb2yiq, r);
  memcpy(M, r, sizeof(r));
  volatile float hc = half_range * contrast;
  const float t = (half_range - hc) * brightness;
  T[0] = T[1] = T[2] = t;
}

int dalib200PointwisePlanCreate(dalib200PointwisePlan **plan, int max_batch) try {
  DB_CHECK_ARG(plan && max_batch > 0, "PointwisePlanCreate: bad arguments");
  auto *p = new dalib200PointwisePlan();
  p->max_batch = max_batch;
  int rc = p->arena.Reserve(sizeof(PwDesc) * max_batch);
  if (rc) { delete p; return rc; }
  *plan = p;
  return DALIB200_SUCCESS;
} DB_API_CATCH

int dalib200PointwisePlanDestroy(dalib200PointwisePlan *p) try {
  if (!p) return DALIB200_SUCCESS;
  p->arena.Free();
  delete p;
  return DALIB200_SUCCESS;
} DB_API_CATCH

int dalib200LinearTransformSetup(dalib200PointwisePlan *p, int n, const dalib200ColorSample *samples, int out_dtype) try {
  DB_CHECK_ARG(p && samples && n >= 0 && n <= p->max_batch, "LinearTransformSetup: bad arguments");
  DB_CHECK_ARG(out_dtype == DALIB200_UINT8 || out_dtype == DALIB200_FLOAT, "Hsv/ColorTwist: output type %d not supported", out_dtype);
  PwDesc *descs;
  if (int rc = p->arena.Stage(sizeof(PwDesc) * n, &descs)) return rc;
  int64_t quads = 0;
  for (int i = 0; i < n; i++) {
    DB_CHECK_ARG(samples[i].num_pixels >= 0, "Hsv/ColorTwist: negative sample size");
    PwDesc &d = descs[i];
    memset(&d, 0, sizeof(d));
    d.npix = samples[i].num_pixels; d.first_quad = quads;
    memcpy(d.m, samples[i].matrix, sizeof(d.m)); memcpy(d.t, samples[i].offset, sizeof(d.t));
    quads += (d.npix + 3) / 4;
  }
  p->n = n; p->mode = PW_LINEAR; p->out_dtype = out_dtype; p->total_quads = quads;
  return DALIB200_SUCCESS;
} DB_API_CATCH

int dalib200ColorSpaceSetup(dalib200PointwisePlan *p, int n, const int64_t *num_pixels, int in_type, int out_type) try {
  DB_CHECK_ARG(p && num_pixels && n >= 0 && n <= p->max_batch, "ColorSpaceSetup: bad arguments");
  DB_CHECK_ARG(in_type >= 0 && in_type <= 3 && out_type >= 0 && out_type <= 3, "ColorSpaceConversion: unknown image type");
  PwDesc *descs;
  if (int rc = p->arena.Stage(sizeof(PwDesc) * n, &descs)) return rc;
  int64_t quads = 0;
  for (int i = 0; i < n; i++) {
    PwDesc &d = descs[i];
    memset(&d, 0, sizeof(d));
    DB_CHECK_ARG(num_pixels[i] >= 0, "ColorSpaceConversion: negative sample size");
    d.npix = num_pixels[i]; d.first_quad = quads;
    quads += (d.npix + 3) / 4;
  }
  p->n = n; p->mode = PW_CSC; p->in_type = in_type; p->out_type = out_type; p->total_quads = quads;
  return DALIB200_SUCCESS;
} DB_API_CATCH

int dalib200PointwiseLaunch(dalib200PointwisePlan *p, const void *const *in_ptrs, void *const *out_ptrs, dalib200Stream_t stream) try {
  DB_CHECK_ARG(p && in_ptrs && out_ptrs, "PointwiseLaunch: null argument");
  if (p->n == 0 || p->total_quads == 0) return DALIB200_SUCCESS;
  PwDesc *descs;
  if (int rc = p->arena.Stage(sizeof(PwDesc) * p->n, &descs)) return rc;
  for (int i = 0; i < p->n; i++) { descs[i].in = static_cast<const uint8_t *>(in_ptrs[i]); descs[i].out = out_ptrs[i]; }
  int rc = p->arena.Upload(sizeof(PwDesc) * p->n, stream);
  if (rc) return rc;
  const auto *dd = reinterpret_cast<const PwDesc *>(p->arena.dev);
  const int grid = (int)std::min<int64_t>((p->total_quads + 255) / 256, (int64_t)NumSMs() * 32);
  if (p->mode == PW_LINEAR)
    Launch("linear_transform", p->out_dtype == DALIB200_UINT8 ? linear_transform_kernel<uint8_t> : linear_transform_kernel<float>, grid, 256, 0, stream,
           dd, p->n, p->total_quads);
  else
    Launch("color_space_conversion", csc_kernel, grid, 256, 0, stream, dd, p->n, p->total_quads, p->in_type, p->out_type);
  DB_CUDA(cudaGetLastError());
  return DALIB200_SUCCESS;
} DB_API_CATCH

}  // extern "C"
