// dali_b200/csrc/jpeg_recon.h -- the JPEG reconstruct stage (dequantisation, islow IDCT, chroma upsampling, colour conversion) as
// the decoder (jpeg.cu) and fn.jpeg_compression_distortion (jpeg_distort.cu) share it: the per-image descriptor the kernels read, the
// host-side choice of kernel per image with its work-list prefix, and the launch of idct_kernel / idct_color_420 / color_fast_kernel /
// color_kernel.  The kernels read quantised coefficients from an int16 arena (MCU order, natural order in each block) and the absolute
// DC of every block from a compact int16 array.
#ifndef DALI_B200_CSRC_JPEG_RECON_H_
#define DALI_B200_CSRC_JPEG_RECON_H_
#include <stdint.h>
#include "../../include/dali_b200.h"
#include "host_device.h"

#if defined(__CUDACC__)
#include <cuda_runtime.h>
#endif

namespace dalib200 {

constexpr int kMaxBlocksPerMcu = 10;

struct QuantSet { uint16_t q[4][64]; };       // natural order

// GRAY of an RGB-coded JPEG pixel (libjpeg-turbo rgb_gray_convert): the baseline path's Adobe-0 / R-G-B images and lossless RGB.
DB_HD int RgbJpegGray(int r, int g, int b) { return (r * 19595 + g * 38470 + b * 7471 + 32768) >> 16; }

// Colour space of the decoded components (libjpeg default_decompress_parms).  Decided once per image by the plan; the kernels read
// nothing else to pick the conversion.
enum JpegColor : int32_t {
  kColorGray = 0,     // 1 component
  kColorYCbCr = 1,    // 3 components
  kColorRGB = 2,      // 3 components: Adobe transform 0, or R/G/B component ids without JFIF / Adobe markers
  kColorCMYK = 3,     // 4 components: Adobe transform 0, or no Adobe marker
  kColorYCCK = 4,     // 4 components: any other Adobe transform (components 0..2 are the YCbCr of 255 - C, 255 - M, 255 - Y)
};

struct JpegImage {
  uint8_t *out;               // HWC u8
  int32_t width, height, ncomp;
  int32_t hs[4], vs[4], hmax, vmax;
  int32_t mcux, mcuy, bpm;    // MCUs per row / column, blocks per MCU
  int32_t blk_comp[kMaxBlocksPerMcu];      // component of each block in the MCU
  int32_t blk_dc[kMaxBlocksPerMcu], blk_ac[kMaxBlocksPerMcu];   // table index (0..3) into TableSet
  int32_t blk_x[kMaxBlocksPerMcu], blk_y[kMaxBlocksPerMcu];     // block offset inside the MCU (in blocks)
  int32_t tq[4];
  int32_t restart_interval;
  int32_t table_set, quant_set;
  int32_t unit_begin, unit_end;            // segments (restart intervals or the whole scan)
  int32_t subseq_begin;                    // first global subsequence
  int32_t nsub;                            // upper bound of subsequences (from raw length)
  int32_t block_begin;                     // first sync block
  int32_t wblock_begin;                    // first block of the write pass (kWriteThreads subsequences each)
  int64_t coef_off;                        // int16 offset into the coefficient arena
  int64_t plane_off[4];                    // byte offsets into the plane arena
  int32_t plane_w[4], plane_h[4];          // padded plane sizes (multiples of the MCU)
  int32_t out_type, fancy;
  int32_t color;                           // JpegColor
  int32_t fast_color;                      // 1: color_fast_kernel, 2: idct_color_420 (4:2:0 fancy -> RGB / BGR), 0: color_kernel
  // decode window: the pixels [win_x0, win_x0 + win_w) x [win_y0, win_y0 + win_h) of the (un-oriented) image are produced, `out`
  // is a tight win_h x win_w x C buffer (the caller's sample, or plan scratch when a post pass follows).  win_x0 % 8 == 0.
  int32_t win_x0, win_y0, win_w, win_h;
  int32_t mcu_x0, mcu_y0, mcu_nx, mcu_ny;  // MCUs whose blocks the IDCT transforms (window + chroma upsampling halo)
};

// An entropy-coded unit (a restart interval, or a whole scan) as U1 - U3 (jpeg.cu) un-stuff it: a baseline segment, or a restart
// interval of a lossless sample (ljpeg.cu), which has no subsequences or slots of the baseline path.
struct JpegUnit {
  uint32_t raw_off, raw_len;               // in the staged byte buffer
  uint32_t clean_off;                      // in the clean buffer (bytes, 16-aligned)
  uint32_t first_chunk;                    // global chunk index
  int32_t image;
  int32_t first_subseq;                    // image-local
  int32_t nsub_max;
  int64_t slot_base;                       // first coefficient slot of this unit (image-local)
  int64_t nslots;                          // expected number of slots (= MCUs * bpm * 64)
};
constexpr int kChunkBytes = 4096;            // un-stuffing chunk
constexpr uint32_t kCleanPad = 32;           // zero bytes behind the clean stream of every unit (at least: units are 16-byte aligned)

// idct_color_420 (jpeg.cu): work item = a strip of kFusedMcus MCU columns of one image's window, walked down one MCU row ("band") at a
// time over a segment of at most kFusedMaxBands bands.
constexpr int kFusedMcus = 16;                     // 256 luma columns per strip
constexpr int kFusedMaxBands = 24;
constexpr int kFusedThreads = 128;                 // >= 6 * kFusedMcus + 4 blocks: one IDCT per thread and band
constexpr int kFusedCPitch = 8 * kFusedMcus + 16;  // chroma tile: byte 8 + (i - 8 * first MCU column) holds chroma column i

struct FusedGeo { int mx0, mx_end, nstrips, m0, nbands, nseg, seg_len; };
DB_HD FusedGeo fused_geo(const JpegImage &im) {
  FusedGeo g;
  const int wx1 = im.win_x0 + im.win_w, wy1 = im.win_y0 + im.win_h, last = im.mcuy - 1;
  g.mx0 = im.win_x0 >> 4; g.mx_end = ((wx1 - 1) >> 4) + 1;                  // MCU columns that hold window pixels
  g.nstrips = (g.mx_end - g.mx0 + kFusedMcus - 1) / kFusedMcus;
  g.m0 = (im.win_y0 + 1) >> 4; if (g.m0 > last) g.m0 = last;                // band of row win_y0: min((y + 1) >> 4, last)
  const int m1 = wy1 >> 4;
  g.nbands = (m1 < last ? m1 : last) - g.m0 + 1;
  g.nseg = (g.nbands + kFusedMaxBands - 1) / kFusedMaxBands;
  g.seg_len = (g.nbands + g.nseg - 1) / g.nseg;
  return g;
}

// Running totals of the reconstruct work lists: IDCT blocks (idct_kernel), fused strips (idct_color_420), colour quads (color_kernel)
// and colour items (color_fast_kernel).
struct ReconTotals { int64_t work = 0, fused = 0, quads = 0, items = 0; };

#if defined(__CUDACC__)
// Chooses the reconstruct path of a JPEG image (im.fast_color) from its colour space, sampling, output type and width, stores the
// image's first entry of each work list (the totals so far) and adds its work.  planes_only: IDCT into the planes, no colour work.
void ReconAddImage(JpegImage &im, bool fancy, bool planes_only, ReconTotals &t, int64_t *first_work, int64_t *first_fused,
                   int64_t *first_quad, int64_t *first_item);

struct ReconLaunch {
  const JpegImage *d_images; int nimages;
  ReconTotals totals;
  const int64_t *d_first_work, *d_first_fused, *d_first_quad, *d_first_item;   // device copies of the prefixes, nimages entries each
  const int16_t *d_coef, *d_dc;
  const QuantSet *d_quants;
  uint8_t *d_planes;                         // component planes of the images that do not take idct_color_420 (JpegImage::plane_off)
};
// Enqueues the reconstruct kernels of the images' windows into JpegImage::out.  Returns a DALIB200 status.
int LaunchReconstruct(const ReconLaunch &a, cudaStream_t s);
#endif

}  // namespace dalib200
#endif  // DALI_B200_CSRC_JPEG_RECON_H_
