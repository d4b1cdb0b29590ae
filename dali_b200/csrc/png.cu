// dali_b200/csrc/png.cu -- PNG decoding inside decoders.image: CRC check of the IDAT chunks, inflate + unfilter, colour conversion.
//
// The planner (png_plan.h) walks the chunk headers on the host; the image data itself is only touched here:
//   png_crc      one thread per IDAT chunk: CRC-32 over type and data against the stored value (the chunks of a large image run in
//                parallel)
//   png_inflate  one working thread per image: the zlib stream -> filtered scanlines in plan scratch -> unfiltered in place
//                (png_inflate_unfilter, png_core.h).  Deflate is a serial chain; this is a correctness path, not a fast one.
//   png_color    one thread per output pixel: unpack / palette / 16 -> 8 bits / alpha dropped / GRAY rule, into the decode window
// Orientation, region of interest, YCbCr and float output are the JPEG path's post pass over that window (jpeg.cu jpeg_post_kernel).
#include "common.cuh"
#include "png.h"
#include <algorithm>

namespace dalib200 {

__global__ void __launch_bounds__(128) png_crc_kernel(const PngChunk *__restrict__ chunks, int nchunks, const PngImage *__restrict__ images,
                                                      const uint8_t *__restrict__ raw, int32_t *status) {
  __shared__ uint32_t table[256];
  for (int i = threadIdx.x; i < 256; i += blockDim.x) table[i] = png_crc_table_entry(i);
  __syncthreads();
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= nchunks) return;
  const PngChunk ch = chunks[k];
  const PngImage &im = images[ch.image];
  if (!png_chunk_crc_ok(raw + im.raw_off + ch.off - 4, ch.len, table)) status[im.sample] = 1;
}

__global__ void __launch_bounds__(32) png_inflate_kernel(const PngImage *__restrict__ images, const PngChunk *__restrict__ chunks,
                                                         const uint8_t *__restrict__ raw, uint8_t *scan, int32_t *status) {
  if (threadIdx.x != 0) return;
  const PngImage &im = images[blockIdx.x];
  if (status[im.sample]) return;                              // a CRC error: the data is not decoded
  InflateWork w;
  if (png_inflate_unfilter(im, chunks, raw, scan + im.scan_off, w)) status[im.sample] = 1;
}

__global__ void __launch_bounds__(256) png_color_kernel(const PngImage *__restrict__ images, int nimages, int64_t total,
                                                        const uint8_t *__restrict__ scan) {
  const int64_t step = (int64_t)gridDim.x * blockDim.x;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += step) {
    const PngImage &im = images[last_at_most(images, 0, nimages - 1, e, [](const PngImage &m) { return m.first_px; })];
    const int64_t lp = e - im.first_px;
    const int ly = (int)(lp / im.win_w), lx = (int)(lp - (int64_t)ly * im.win_w);
    png_pixel(im, scan + im.scan_off, lx, ly);
  }
}

int PngStage::Plan(const uint8_t *data, size_t len, int sample, int64_t raw_off, StreamInfo *info, std::string *err) {
  PngImage im;
  if (int rc = PlanPng(data, len, (int)images.size(), &im, chunks, info, err)) return rc;
  im.scan_off = scan_bytes;
  scan_bytes += (int64_t)Align((size_t)im.scan_bytes, 16);
  im.sample = sample; im.raw_off = raw_off;
  images.push_back(im);
  return DALIB200_SUCCESS;
}

int PngStage::Enqueue(const StageInputs &in, cudaStream_t s) {
  const int64_t total_px = FillWindows(images, in.images);
  const PngImage *d_images; const PngChunk *d_chunks;
  if (int rc = arena.Pack(s, std::tie(d_images, d_chunks), images, chunks)) return rc;
  const int nimages = (int)images.size(), nchunks = (int)chunks.size();
  if (nchunks > 0) Launch("png_crc", png_crc_kernel, (nchunks + 127) / 128, 128, 0, s, d_chunks, nchunks, d_images, in.d_raw, in.d_status);
  Launch("png_inflate", png_inflate_kernel, nimages, 32, 0, s, d_images, d_chunks, in.d_raw, d_scan, in.d_status);
  if (total_px > 0) {
    const int grid = (int)std::min<int64_t>((total_px + 255) / 256, (int64_t)NumSMs() * 16);
    Launch("png_color", png_color_kernel, grid, 256, 0, s, d_images, nimages, total_px, d_scan);
  }
  DB_CUDA(cudaGetLastError());
  return DALIB200_SUCCESS;
}

}  // namespace dalib200
