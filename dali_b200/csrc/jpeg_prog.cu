// dali_b200/csrc/jpeg_prog.cu -- entropy stage of PROGRESSIVE (SOF2) JPEG streams inside decoders.image.
//
// The reference's mixed decoder accepts progressive streams (nvimgcodec falls back to libjpeg-turbo for them); real datasets contain
// them.  A progressive scan cannot be entered in the middle (a refinement pass is decoded relative to the coefficients already there),
// so the baseline path's self-synchronising subsequence decode does not apply.  What is parallel: the images of a batch, and the scans
// of one image that touch different components or different coefficient bands -- the planner (jpeg_prog_plan.h) sorts them into
// dependency waves (the usual 10-scan script of libjpeg runs in 3).  One launch per wave, one warp per scan with one working lane:
// the decode is a chain of dependent operations, 32 lanes in different scans would only serialise.  Everything behind the entropy stage
// (DC prefix sum, IDCT, upsampling, colour, post pass) is the baseline path's: the scans write the same coefficient arena.
// This is a correctness path, not a fast one: ~0.1 us per symbol on the critical path (a 500 kB stream: tens of ms).
#include "common.cuh"
#include "jpeg_prog.h"
#include <algorithm>

namespace dalib200 {

__global__ void __launch_bounds__(32) prog_scan_kernel(const ProgScan *__restrict__ scans, int first, const ProgImage *__restrict__ images,
                                                       const ProgHuff *__restrict__ huff, const uint8_t *__restrict__ raw, int16_t *coef,
                                                       int32_t *status) {
  if (threadIdx.x != 0) return;
  const ProgScan s = scans[first + blockIdx.x];
  const ProgImage im = images[s.image];
  if (prog_decode_scan(s, im, huff, raw, coef)) status[im.sample] = 1;
}

__global__ void __launch_bounds__(256) prog_dc_kernel(const ProgImage *__restrict__ images, const int64_t *__restrict__ first_blk, int nimages,
                                                      int64_t total, const int16_t *__restrict__ coef, int16_t *__restrict__ dc,
                                                      int32_t *status) {
  const int64_t step = (int64_t)gridDim.x * blockDim.x;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += step) {
    const int i = last_at_most(first_blk, 0, nimages - 1, e);
    prog_dc_difference(images[i], coef, dc, e - first_blk[i]);
    if (e == first_blk[i] && images[i].incomplete) status[images[i].sample] = 1;
  }
}

int LaunchProgressive(const ProgLaunch &a, cudaStream_t s) {
  if (a.nimages == 0) return DALIB200_SUCCESS;
  for (const ProgImage &im : *a.h_images)
    DB_CUDA(cudaMemsetAsync(a.d_coef + im.coef_off, 0, sizeof(int16_t) * 64 * (size_t)im.mcux * im.mcuy * im.bpm, s));
  const std::vector<int> &wb = *a.wave_begin;
  for (size_t w = 0; w + 1 < wb.size(); w++) {
    const int cnt = wb[w + 1] - wb[w];
    if (cnt <= 0) continue;
    ProfScope ps_("jpeg_prog_scan", s);
    prog_scan_kernel<<<cnt, 32, 0, s>>>(a.d_scans, wb[w], a.d_images, a.d_huff, a.d_raw, a.d_coef, a.d_status);
    CountLaunch();
  }
  if (a.total_blocks > 0) {
    const int grid = (int)std::min<int64_t>((a.total_blocks + 255) / 256, (int64_t)NumSMs() * 8);
    ProfScope ps_("jpeg_prog_dc", s);
    prog_dc_kernel<<<grid, 256, 0, s>>>(a.d_images, a.d_first_blk, a.nimages, a.total_blocks, a.d_coef, a.d_dc, a.d_status);
    CountLaunch();
  }
  DB_CUDA(cudaGetLastError());
  return DALIB200_SUCCESS;
}

}  // namespace dalib200
