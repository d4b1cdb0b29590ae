// dali_b200/csrc/jpeg_distort.cu -- fn.jpeg_compression_distortion on sm_90a: JPEG compression and decompression of RGB images, bit-exact
// with cv2.imdecode(cv2.imencode(".jpg", img, IMWRITE_JPEG_QUALITY q)).
//
// The decoded pixels depend only on the quantised DCT coefficients, so the operator never writes an entropy-coded stream:
//   jpeg_distort_fdct   one CTA per strip of kJdMcus MCUs of one MCU row: the threads convert the strip's 2x2 pixel quads to Y and
//                       downsampled Cb / Cr in shared memory (each pixel converted once), then one thread per 8x8 block runs the forward
//                       DCT and quantisation (jpeg_distort_core.h) and writes the block to the coefficient arena, its DC to the DC arena.
//   reconstruct         the decoder's own kernels (jpeg_recon.h, jpeg.cu): idct_color_420 for images wider than 4 pixels, else
//                       idct_kernel + color_fast_kernel with libjpeg's box upsampling for chroma widths <= 2.
#include "common.cuh"
#include "jpeg_distort_plan.h"
#include <algorithm>
#include <cstring>
#include <map>

namespace dalib200 {

// items: per image mcuy * strips_x strips, first_strip[i] = first item of image i; one CTA per item
__global__ void __launch_bounds__(kJdThreads) jpeg_distort_fdct_kernel(const JdImage *__restrict__ images, const int64_t *__restrict__ first_strip,
                                                                     int nimages, const QuantSet *__restrict__ quants, int16_t *coef,
                                                                     int16_t *dc) {
  __shared__ JdStrip t;
  __shared__ int s_img;
  if (threadIdx.x == 0) {
    int lo = 0, hi = nimages - 1;
    while (lo < hi) { const int mid = (lo + hi + 1) >> 1; if (first_strip[mid] <= (int64_t)blockIdx.x) lo = mid; else hi = mid - 1; }
    s_img = lo;
  }
  __syncthreads();
  const JdImage &im = images[s_img];
  int my, mx0, nt;
  jd_strip(im, (int64_t)blockIdx.x - first_strip[s_img], my, mx0, nt);
  for (int e = threadIdx.x; e < 64 * nt; e += kJdThreads) jd_convert_quad(im, my, mx0, nt, e, t);
  __syncthreads();
  const QuantSet &qs = quants[im.quant_set];
  const int j = threadIdx.x;
  if (j < 6 * nt) jd_block(im, qs, my, mx0, j, 0, t, coef, dc);
  __syncthreads();
  if (j < 6 * nt) jd_block(im, qs, my, mx0, j, 1, t, coef, dc);
}

}  // namespace dalib200

using namespace dalib200;  // NOLINT

struct dalib200JpegDistortPlan {
  int max_batch = 0, n = 0;
  std::vector<JdImage> jd;
  std::vector<JpegImage> images;
  std::vector<QuantSet> quants;
  std::vector<int64_t> first_strip, first_work, first_fused, first_quad, first_item;
  ReconTotals totals;
  int64_t total_strips = 0, total_blocks = 0, plane_bytes = 0;
  int16_t *d_coef = nullptr; size_t d_coef_cap = 0;
  int16_t *d_dc = nullptr; size_t d_dc_cap = 0;
  uint8_t *d_planes = nullptr; size_t d_planes_cap = 0;
  DescArena arena;                           // [JdImage | JpegImage | QuantSet | five prefixes], one H2D copy per launch
  cudaEvent_t uploaded = nullptr;
  bool pending = false;
};

namespace {

template <typename T>
int Grow(T *&ptr, size_t &cap, size_t need) {
  if (need <= cap) return DALIB200_SUCCESS;
  const size_t ncap = std::max(need + need / 4, (size_t)4096);
  if (ptr) cudaFree(ptr);
  ptr = nullptr; cap = 0;
  DB_CUDA(cudaMalloc(reinterpret_cast<void **>(&ptr), ncap * sizeof(T)));
  cap = ncap;
  return DALIB200_SUCCESS;
}

inline size_t Align16(size_t v) { return (v + 15) / 16 * 16; }

}  // namespace

extern "C" {

int dalib200JpegDistortPlanCreate(dalib200JpegDistortPlan **plan, int max_batch) try {
  DB_CHECK_ARG(plan && max_batch > 0, "JpegDistortPlanCreate: bad arguments");
  auto *p = new dalib200JpegDistortPlan();
  p->max_batch = max_batch;
  if (cudaEventCreateWithFlags(&p->uploaded, cudaEventDisableTiming) != cudaSuccess) {
    SetLastError("JpegDistortPlanCreate: cudaEventCreate failed"); delete p; return DALIB200_ERROR_CUDA;
  }
  *plan = p;
  return DALIB200_SUCCESS;
} DB_API_CATCH

int dalib200JpegDistortPlanDestroy(dalib200JpegDistortPlan *p) try {
  if (!p) return DALIB200_SUCCESS;
  if (p->uploaded) { cudaEventSynchronize(p->uploaded); cudaEventDestroy(p->uploaded); }
  p->arena.Free();
  for (void *b : { (void *)p->d_coef, (void *)p->d_dc, (void *)p->d_planes }) if (b) cudaFree(b);
  delete p;
  return DALIB200_SUCCESS;
} DB_API_CATCH

int dalib200JpegDistortPlanSetup(dalib200JpegDistortPlan *p, int n, const dalib200JpegDistortSample *samples) try {
  DB_CHECK_ARG(p && n >= 0 && n <= p->max_batch && (n == 0 || samples), "JpegDistortPlanSetup: bad arguments (n = %d, max_batch = %d)", n,
               p ? p->max_batch : 0);
  p->n = 0;
  char msg[256];
  for (int i = 0; i < n; i++) {
    const int rc = JdCheckSample(i, samples[i].height, samples[i].width, samples[i].quality, msg, sizeof(msg));
    if (rc) { SetLastError("%s", msg); return rc; }
  }
  p->jd.resize(n); p->images.resize(n); p->quants.clear();
  p->first_strip.resize(n); p->first_work.resize(n); p->first_fused.resize(n); p->first_quad.resize(n); p->first_item.resize(n);
  std::map<int, int> quant_of;
  ReconTotals t;
  int64_t strips = 0, blocks = 0, planes = 0;
  for (int i = 0; i < n; i++) {
    const int q = samples[i].quality;
    auto it = quant_of.find(q);
    if (it == quant_of.end()) {
      QuantSet qs;
      JdQuantTables(q, qs);
      p->quants.push_back(qs);
      it = quant_of.emplace(q, (int)p->quants.size() - 1).first;
    }
    JdImage &d = p->jd[i];
    JpegImage &im = p->images[i];
    JdPlanImage(samples[i].height, samples[i].width, it->second, blocks, d, im);
    p->first_strip[i] = strips;
    strips += (int64_t)d.mcuy * d.strips_x;
    blocks += JdBlocks(d.height, d.width);
    ReconAddImage(im, true, false, t, &p->first_work[i], &p->first_fused[i], &p->first_quad[i], &p->first_item[i]);
    if (im.fast_color != 2)                  // the two-kernel path goes through the component planes
      for (int c = 0; c < 3; c++) {
        im.plane_w[c] = (int)Align16((size_t)im.mcux * im.hs[c] * 8); im.plane_h[c] = im.mcuy * im.vs[c] * 8;
        im.plane_off[c] = planes;
        planes += Align16((size_t)im.plane_w[c] * im.plane_h[c]);
      }
  }
  DB_CHECK_ARG(strips < (1ll << 31), "JpegDistortPlanSetup: batch of %lld MCU strips exceeds the grid limit", (long long)strips);
  p->totals = t; p->total_strips = strips; p->total_blocks = blocks; p->plane_bytes = planes;
  p->n = n;
  return DALIB200_SUCCESS;
} DB_API_CATCH

int dalib200JpegDistortLaunch(dalib200JpegDistortPlan *p, const void *const *in_ptrs, void *const *out_ptrs, dalib200Stream_t stream) try {
  DB_CHECK_ARG(p && (p->n == 0 || (in_ptrs && out_ptrs)), "JpegDistortLaunch: bad arguments");
  const int n = p->n;
  if (n == 0) return DALIB200_SUCCESS;
  int rc;
  if ((rc = Grow(p->d_coef, p->d_coef_cap, (size_t)p->total_blocks * 64))) return rc;
  if ((rc = Grow(p->d_dc, p->d_dc_cap, (size_t)p->total_blocks))) return rc;
  if (p->plane_bytes > 0 && (rc = Grow(p->d_planes, p->d_planes_cap, (size_t)p->plane_bytes + 64))) return rc;
  const size_t nq = p->quants.size();
  const size_t o_img = Align16(sizeof(JdImage) * n), o_q = o_img + Align16(sizeof(JpegImage) * n), o_pre = o_q + sizeof(QuantSet) * nq;
  const size_t pre = Align16(sizeof(int64_t) * n), bytes = o_pre + 5 * pre;
  // the previous batch's descriptors may still be on their way to the device from the pinned buffer
  if (p->pending) { DB_CUDA(cudaEventSynchronize(p->uploaded)); p->pending = false; }
  if ((rc = p->arena.Reserve(bytes))) return rc;
  uint8_t *h = p->arena.host;
  JdImage *hj = reinterpret_cast<JdImage *>(h);
  JpegImage *hi = reinterpret_cast<JpegImage *>(h + o_img);
  for (int i = 0; i < n; i++) {
    hj[i] = p->jd[i]; hj[i].in = static_cast<const uint8_t *>(in_ptrs[i]);
    hi[i] = p->images[i]; hi[i].out = static_cast<uint8_t *>(out_ptrs[i]);
  }
  memcpy(h + o_q, p->quants.data(), sizeof(QuantSet) * nq);
  const std::vector<int64_t> *pres[5] = { &p->first_strip, &p->first_work, &p->first_fused, &p->first_quad, &p->first_item };
  for (int k = 0; k < 5; k++) memcpy(h + o_pre + k * pre, pres[k]->data(), sizeof(int64_t) * n);
  cudaStream_t s = stream;
  if ((rc = p->arena.Upload(bytes, s))) return rc;
  DB_CUDA(cudaEventRecord(p->uploaded, s));
  p->pending = true;
  const uint8_t *dv = p->arena.dev;
  const auto *d_quants = reinterpret_cast<const QuantSet *>(dv + o_q);
  {
    ProfScope ps_("jpeg_distort_fdct", s);
    jpeg_distort_fdct_kernel<<<(unsigned)p->total_strips, kJdThreads, 0, s>>>(reinterpret_cast<const JdImage *>(dv),
                                                                             reinterpret_cast<const int64_t *>(dv + o_pre), n, d_quants,
                                                                             p->d_coef, p->d_dc);
  }
  CountLaunch();
  ReconLaunch ra;
  ra.d_images = reinterpret_cast<const JpegImage *>(dv + o_img); ra.nimages = n;
  ra.totals = p->totals;
  ra.d_first_work = reinterpret_cast<const int64_t *>(dv + o_pre + pre);
  ra.d_first_fused = reinterpret_cast<const int64_t *>(dv + o_pre + 2 * pre);
  ra.d_first_quad = reinterpret_cast<const int64_t *>(dv + o_pre + 3 * pre);
  ra.d_first_item = reinterpret_cast<const int64_t *>(dv + o_pre + 4 * pre);
  ra.d_coef = p->d_coef; ra.d_dc = p->d_dc; ra.d_quants = d_quants; ra.d_planes = p->d_planes;
  if ((rc = LaunchReconstruct(ra, s))) return rc;
  if (p->totals.work > 0) CountLaunch();     // idct_kernel (LaunchReconstruct counts the colour launches)
  DB_CUDA(cudaGetLastError());
  return DALIB200_SUCCESS;
} DB_API_CATCH

// test accessor: quantised coefficients of one sample as the forward kernel wrote them (MCU order, natural order in each block, DC
// absolute).  Synchronises the device.
int dalib200JpegDistortDebugGetCoefficients(dalib200JpegDistortPlan *p, int sample, int16_t *out, size_t count) try {
  DB_CHECK_ARG(p && out && sample >= 0 && sample < p->n && p->d_coef, "JpegDistortDebugGetCoefficients: bad arguments");
  const JdImage &d = p->jd[sample];
  const size_t have = (size_t)JdBlocks(d.height, d.width) * 64;
  DB_CHECK_ARG(count <= have, "JpegDistortDebugGetCoefficients: sample has %zu coefficients", have);
  DB_CUDA(cudaDeviceSynchronize());
  DB_CUDA(cudaMemcpy(out, p->d_coef + d.blk0 * 64, count * sizeof(int16_t), cudaMemcpyDeviceToHost));
  std::vector<int16_t> dcs((count + 63) / 64);
  DB_CUDA(cudaMemcpy(dcs.data(), p->d_dc + d.blk0, dcs.size() * sizeof(int16_t), cudaMemcpyDeviceToHost));
  for (size_t b = 0; b * 64 < count; b++) out[b * 64] = dcs[b];
  return DALIB200_SUCCESS;
} DB_API_CATCH

}  // extern "C"
