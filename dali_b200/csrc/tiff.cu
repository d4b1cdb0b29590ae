// dali_b200/csrc/tiff.cu -- TIFF decoding inside decoders.image: segment decode, colour conversion.
//
// The planner (tiff_plan.h) walks the IFD on the host and builds the segment table; the image data itself is only touched here:
//   tiff_segment  one lane per segment (strip or tile of one plane): LZW / Deflate / PackBits / raw copy into plan scratch, then the
//                 horizontal predictor undone row by row (tiff_decode_segment, tiff_core.h).  Each thread owns a kTiffSlotBytes slot of
//                 plan-owned global memory for the LZW string starts or the inflate tables, so that the kernel keeps no stack frame.
//   tiff_color    one thread per output pixel: gathers the samples from their segments and planes and applies libtiff's RGBA rules
//                 and cv2's GRAY rule, into the decode window
// Orientation, region of interest, YCbCr and float output are the JPEG path's post pass over that window (jpeg.cu jpeg_post_kernel).
#include "common.cuh"
#include "tiff.h"
#include <algorithm>

namespace dalib200 {

// tiff_segment: one working lane per segment (SerialLaneGeometry); each lane owns a 16 KB slot, so the lanes are capped at 33 792
// (540 MB of slots at most)
constexpr int kTiffMaxWorkers = 33792;

__global__ void __launch_bounds__(32) tiff_segment_kernel(const TiffImage *__restrict__ images, const TiffSeg *__restrict__ segs,
                                                          int nsegs, int lanes, const uint8_t *__restrict__ raw, uint8_t *dec,
                                                          uint8_t *slots, int32_t *status) {
  if ((int)threadIdx.x >= lanes) return;
  const int w = blockIdx.x * lanes + threadIdx.x;             // working lane, and its slot
  void *slot = slots + (size_t)w * kTiffSlotBytes;
  for (int k = w; k < nsegs; k += gridDim.x * lanes) {
    const TiffSeg &s = segs[k];
    const TiffImage &im = images[s.image];
    if (*(volatile int32_t *)&status[im.sample]) continue;   // another segment of the image failed: the image is not decoded
    if (tiff_decode_segment(im, s, raw, dec + s.dec_off, slot)) status[im.sample] = 1;
  }
}

__global__ void __launch_bounds__(256) tiff_color_kernel(const TiffImage *__restrict__ images, int nimages, int64_t total,
                                                         const TiffSeg *__restrict__ segs, const uint8_t *__restrict__ dec) {
  const int64_t step = (int64_t)gridDim.x * blockDim.x;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += step) {
    const TiffImage &im = images[last_at_most(images, 0, nimages - 1, e, [](const TiffImage &m) { return m.first_px; })];
    const int64_t lp = e - im.first_px;
    const int ly = (int)(lp / im.win_w), lx = (int)(lp - (int64_t)ly * im.win_w);
    tiff_pixel(im, segs, dec, lx, ly);
  }
}

int TiffStage::Plan(const uint8_t *data, size_t len, int sample, int64_t raw_off, StreamInfo *info, std::string *err) {
  TiffImage im;
  int64_t bytes = 0;
  if (int rc = PlanTiff(data, len, (int)images.size(), &im, segs, dec_bytes, &bytes, info, err)) return rc;
  dec_bytes += bytes;
  im.sample = sample; im.raw_off = raw_off;
  images.push_back(im);
  return DALIB200_SUCCESS;
}

int TiffStage::Reserve() {
  const SerialLanes g = SerialLaneGeometry((int)segs.size(), kTiffMaxWorkers);     // a slot per tiff_segment thread
  int rc;
  if ((rc = GrowDevice(d_dec, d_dec_cap, (size_t)dec_bytes + 16))) return rc;
  return GrowDevice(d_slots, d_slots_cap, (size_t)(g.warps * g.lanes) * kTiffSlotBytes);
}

int TiffStage::Enqueue(const StageInputs &in, cudaStream_t s) {
  const int64_t total_px = FillWindows(images, in.images);
  const TiffImage *d_images; const TiffSeg *d_segs;
  if (int rc = arena.Pack(s, std::tie(d_images, d_segs), images, segs)) return rc;
  const int nsegs = (int)segs.size();
  if (nsegs > 0) {
    const SerialLanes g = SerialLaneGeometry(nsegs, kTiffMaxWorkers);
    Launch("tiff_segment", tiff_segment_kernel, g.warps, 32, 0, s, d_images, d_segs, nsegs, g.lanes, in.d_raw, d_dec, d_slots, in.d_status);
  }
  if (total_px > 0) {
    const int grid = (int)std::min<int64_t>((total_px + 255) / 256, (int64_t)NumSMs() * 16);
    Launch("tiff_color", tiff_color_kernel, grid, 256, 0, s, d_images, (int)images.size(), total_px, d_segs, d_dec);
  }
  DB_CUDA(cudaGetLastError());
  return DALIB200_SUCCESS;
}

}  // namespace dalib200
