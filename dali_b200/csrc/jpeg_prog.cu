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
#include "jpeg_prog_plan.h"
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

void ProgStage::Clear() {
  images.clear(); scans.clear(); huff.clear(); wave_begin.clear(); first_blk.clear(); table_cache.clear();
  total_blocks = 0;
}

int ProgStage::Plan(const uint8_t *d, size_t len, size_t sb, size_t se, int sample, int64_t raw_off, int64_t coef_off, const JpegImage &im,
                    uint16_t quant[4][64], std::string *err) {
  ProgImage pim;
  memset(&pim, 0, sizeof(pim));
  const size_t first_new = scans.size();
  if (int rc = PlanProgressive(d, len, sb, (int)images.size(), &pim, scans, huff, table_cache, quant, err)) return rc;
  for (size_t k = first_new; k < scans.size(); k++)
    if ((size_t)scans[k].data_off + scans[k].data_len > se - sb) {
      // a scan that runs into the trimmed end-of-image marker ends in front of it
      auto &sc = scans[k];
      sc.data_len = sc.data_off >= se - sb ? 0 : (uint32_t)(se - sb - sc.data_off);
    }
  if (pim.ncomp != im.ncomp || pim.mcux != im.mcux || pim.mcuy != im.mcuy || pim.bpm != im.bpm) {
    *err = "internal error (progressive frame layout)";
    return DALIB200_ERROR_INTERNAL;
  }
  pim.sample = sample;
  pim.raw_off = raw_off;
  pim.coef_off = coef_off;
  first_blk.push_back(total_blocks);
  total_blocks += (int64_t)im.mcux * im.mcuy * im.bpm;
  images.push_back(pim);
  return DALIB200_SUCCESS;
}

void ProgStage::SortWaves() {
  if (scans.empty()) return;
  std::stable_sort(scans.begin(), scans.end(), [](const ProgScan &a, const ProgScan &b) { return a.wave < b.wave; });
  const int nw = scans.back().wave + 1;
  wave_begin.assign(nw + 1, 0);
  for (const auto &sc : scans) wave_begin[sc.wave + 1]++;
  for (int w = 0; w < nw; w++) wave_begin[w + 1] += wave_begin[w];
}

int ProgStage::Enqueue(const StageInputs &in, cudaStream_t s) {
  const ProgImage *d_images; const ProgScan *d_scans; const ProgHuff *d_huff; const int64_t *d_first_blk;
  if (int rc = arena.Pack(s, std::tie(d_images, d_scans, d_huff, d_first_blk), images, scans, huff, first_blk)) return rc;
  for (const ProgImage &im : images)
    DB_CUDA(cudaMemsetAsync(in.d_coef + im.coef_off, 0, sizeof(int16_t) * 64 * (size_t)im.mcux * im.mcuy * im.bpm, s));
  for (size_t w = 0; w + 1 < wave_begin.size(); w++) {
    const int cnt = wave_begin[w + 1] - wave_begin[w];
    if (cnt <= 0) continue;
    Launch("jpeg_prog_scan", prog_scan_kernel, cnt, 32, 0, s, d_scans, wave_begin[w], d_images, d_huff, in.d_raw, in.d_coef, in.d_status);
  }
  if (total_blocks > 0) {
    const int grid = (int)std::min<int64_t>((total_blocks + 255) / 256, (int64_t)NumSMs() * 8);
    Launch("jpeg_prog_dc", prog_dc_kernel, grid, 256, 0, s, d_images, d_first_blk, (int)images.size(), total_blocks, in.d_coef, in.d_dc, in.d_status);
  }
  DB_CUDA(cudaGetLastError());
  return DALIB200_SUCCESS;
}

}  // namespace dalib200
