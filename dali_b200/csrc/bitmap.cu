// dali_b200/csrc/bitmap.cu -- BMP and PNM decoding inside decoders.image: serial unpack of RLE / ASCII images, colour conversion.
//
// The planner (bitmap_plan.h) parses the headers on the host; the pixel data itself is only touched here:
//   bitmap_unpack  one lane per RLE4 / RLE8 BMP or ASCII PNM image (SerialLaneGeometry): expands it into an 8-bit plane of plan scratch
//                  (bitmap_unpack, bitmap_core.h).  Not launched for a batch whose images are all uncompressed.
//   bitmap_color   16 window pixels per thread, read from the staged raster (uncompressed images: no scratch, no copy) or from the plane,
//                  converted to RGB / BGR / GRAY and written with 16-byte stores into the decode window
// Orientation, region of interest, YCbCr and float output are the JPEG path's post pass over that window (jpeg.cu jpeg_post_kernel).
#include "common.cuh"
#include "bitmap.h"
#include <algorithm>

namespace dalib200 {

__global__ void __launch_bounds__(32) bitmap_unpack_kernel(const BitmapImage *__restrict__ images, const int32_t *__restrict__ list,
                                                           int nlist, int lanes, const uint8_t *__restrict__ raw, uint8_t *scratch,
                                                           int32_t *status) {
  if ((int)threadIdx.x >= lanes) return;
  for (int k = blockIdx.x * lanes + threadIdx.x; k < nlist; k += gridDim.x * lanes) {
    const BitmapImage &im = images[list[k]];
    if (bitmap_unpack(im, raw + im.raw_off, scratch + im.plane_off)) status[im.sample] = 1;
  }
}

__global__ void __launch_bounds__(256) bitmap_color_kernel(const BitmapImage *__restrict__ images, int nimages, int64_t total,
                                                           const uint8_t *__restrict__ raw, const uint8_t *__restrict__ scratch) {
  const int64_t step = (int64_t)gridDim.x * blockDim.x;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += step) {
    const BitmapImage &im = images[last_at_most(images, 0, nimages - 1, e, [](const BitmapImage &m) { return m.first_grp; })];
    bitmap_group(im, im.unpack == kBitmapDirect ? raw + im.raw_off : scratch + im.plane_off, e - im.first_grp);
  }
}

int BitmapStage::Plan(const uint8_t *data, size_t len, int sample, int64_t raw_off, StreamInfo *info, std::string *err) {
  BitmapImage im;
  int64_t bytes = 0;
  if (int rc = PlanBitmap(data, len, &im, scratch_bytes, &bytes, info, err)) return rc;
  scratch_bytes += bytes;
  if (im.unpack != kBitmapDirect) unpack.push_back((int32_t)images.size());
  im.sample = sample; im.raw_off = raw_off;
  images.push_back(im);
  return DALIB200_SUCCESS;
}

int BitmapStage::Enqueue(const StageInputs &in, cudaStream_t s) {
  FillWindows(images, in.images);
  int64_t groups = 0;                        // each image's first_grp: the prefix of the 16-pixel groups of the windows
  for (BitmapImage &d : images) {
    d.first_grp = groups;
    groups += ((int64_t)d.win_w * d.win_h + kBitmapGroup - 1) / kBitmapGroup;
  }
  const BitmapImage *d_images; const int32_t *d_unpack;
  if (int rc = arena.Pack(s, std::tie(d_images, d_unpack), images, unpack)) return rc;
  const int nunpack = (int)unpack.size();
  if (nunpack > 0) {
    const SerialLanes g = SerialLaneGeometry(nunpack, 1 << 30);
    Launch("bitmap_unpack", bitmap_unpack_kernel, g.warps, 32, 0, s, d_images, d_unpack, nunpack, g.lanes, in.d_raw, d_scratch, in.d_status);
  }
  if (groups > 0) {
    const int grid = (int)std::min<int64_t>((groups + 255) / 256, (int64_t)NumSMs() * 16);
    Launch("bitmap_color", bitmap_color_kernel, grid, 256, 0, s, d_images, (int)images.size(), groups, in.d_raw, d_scratch);
  }
  DB_CUDA(cudaGetLastError());
  return DALIB200_SUCCESS;
}

}  // namespace dalib200
