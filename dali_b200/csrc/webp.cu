// dali_b200/csrc/webp.cu -- lossy WebP decoding inside decoders.image: entropy decode, reconstruction, loop filter, colour conversion.
//
// The planner (webp_plan.h) parses the RIFF chunks and the frame and partition-0 headers on the host; the macroblock data is only
// touched here (bodies in webp_core.h):
//   webp_entropy  one working lane per image walks the macroblock rows in order: segment, skip flag and intra modes from partition 0,
//                 tokens from partition (row mod P).  Token contexts need the row above, so the partitions of one image do not run
//                 independently.  Writes a record per macroblock and its 384 dequantised coefficients (the Y2 WHT folded in).
//   webp_recon    one CTA per image walks the wavefront d = x + 2y, one thread per macroblock on the diagonal: (x, y) needs (x - 1, y),
//                 (x, y - 1) and (x + 1, y - 1), all on earlier diagonals.  Intra prediction plus inverse DCT into padded, unfiltered
//                 Y / U / V planes in plan scratch.
//   webp_filter   the loop filter in place on the same wavefront: the top edge of (x, y) reads pixels the left edge of (x + 1, y - 1)
//                 wrote, and two macroblocks on one diagonal touch disjoint pixels.
//   webp_color    one thread per output pixel: fancy upsampling and YUV -> RGB / BGR, or cv2's GRAY rule, into the decode window.
// Orientation, region of interest, YCbCr and float output are the JPEG path's post pass over that window (jpeg.cu jpeg_post_kernel).
// Every macroblock row is decoded whatever the window, so that a sample's status is cv2's whatever crop is asked for.
#include "common.cuh"
#include "webp.h"
#include <algorithm>

namespace dalib200 {

constexpr int kWebpWaveThreads = 128;

__global__ void __launch_bounds__(32) webp_entropy_kernel(const WebpImage *__restrict__ images, int nimages, int lanes,
                                                          const uint8_t *__restrict__ raw, uint8_t *scratch, int32_t *status) {
  if ((int)threadIdx.x >= lanes) return;
  for (int k = blockIdx.x * lanes + threadIdx.x; k < nimages; k += gridDim.x * lanes) {
    const WebpImage &im = images[k];
    if (webp_entropy(im, raw, reinterpret_cast<WebpMb *>(scratch + im.mb_off), reinterpret_cast<int16_t *>(scratch + im.coef_off),
                     reinterpret_cast<uint32_t *>(scratch + im.ctx_off)))
      status[im.sample] = 1;
  }
}

// the macroblocks of diagonal d = x + 2y, spread over the CTA's threads; a barrier between diagonals
template <bool kFilter>
__global__ void __launch_bounds__(kWebpWaveThreads) webp_wave_kernel(const WebpImage *__restrict__ images, uint8_t *scratch,
                                                                     const int32_t *status) {
  const WebpImage &im = images[blockIdx.x];
  if (status[im.sample]) return;                              // the entropy decode failed: the records are not complete
  if (kFilter && im.filter_type == 0) return;
  const WebpMb *mbs = reinterpret_cast<const WebpMb *>(scratch + im.mb_off);
  const int16_t *coef = reinterpret_cast<const int16_t *>(scratch + im.coef_off);
  const int ndiag = im.mb_w + 2 * (im.mb_h - 1);
  for (int d = 0; d < ndiag; d++) {
    const int y_lo = max(0, (d - im.mb_w + 2) / 2), y_hi = min(im.mb_h - 1, d / 2);
    for (int y = y_lo + (int)threadIdx.x; y <= y_hi; y += blockDim.x) {
      const int x = d - 2 * y;
      if (kFilter) webp_filter_mb(im, mbs, scratch, x, y);
      else webp_recon_mb(im, mbs, coef, scratch, x, y);
    }
    __syncthreads();
  }
}

__global__ void __launch_bounds__(256) webp_color_kernel(const WebpImage *__restrict__ images, int nimages, int64_t total, uint8_t *scratch) {
  const int64_t step = (int64_t)gridDim.x * blockDim.x;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += step) {
    const WebpImage &im = images[last_at_most(images, 0, nimages - 1, e, [](const WebpImage &m) { return m.first_px; })];
    const int64_t lp = e - im.first_px;
    const int ly = (int)(lp / im.win_w), lx = (int)(lp - (int64_t)ly * im.win_w);
    webp_pixel(im, scratch, lx, ly);
  }
}

int WebpStage::Plan(const uint8_t *data, size_t len, int sample, int64_t raw_off, StreamInfo *info, std::string *err) {
  WebpImage im;
  int64_t bytes = 0;
  if (int rc = PlanWebp(data, len, (int)images.size(), &im, scratch_bytes, &bytes, info, err)) return rc;
  scratch_bytes += bytes;
  im.sample = sample; im.raw_off = raw_off;
  images.push_back(im);
  return DALIB200_SUCCESS;
}

int WebpStage::Enqueue(const StageInputs &in, cudaStream_t s) {
  const int64_t total_px = FillWindows(images, in.images);
  const WebpImage *d_images;
  if (int rc = arena.Pack(s, std::tie(d_images), images)) return rc;
  const int nimages = (int)images.size();
  const SerialLanes g = SerialLaneGeometry(nimages, 1 << 30);
  Launch("webp_entropy", webp_entropy_kernel, g.warps, 32, 0, s, d_images, nimages, g.lanes, in.d_raw, d_scratch, in.d_status);
  Launch("webp_recon", webp_wave_kernel<false>, nimages, kWebpWaveThreads, 0, s, d_images, d_scratch, in.d_status);
  Launch("webp_filter", webp_wave_kernel<true>, nimages, kWebpWaveThreads, 0, s, d_images, d_scratch, in.d_status);
  if (total_px > 0) {
    const int grid = (int)std::min<int64_t>((total_px + 255) / 256, (int64_t)NumSMs() * 16);
    Launch("webp_color", webp_color_kernel, grid, 256, 0, s, d_images, nimages, total_px, d_scratch);
  }
  DB_CUDA(cudaGetLastError());
  return DALIB200_SUCCESS;
}

}  // namespace dalib200
