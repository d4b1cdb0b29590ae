// dali_b200/csrc/jpeg_prog.h -- the progressive-JPEG entropy stage of decoders.image (jpeg_prog.cu), planned and run by the image decoder
// plan (jpeg.cu).
#ifndef DALI_B200_CSRC_JPEG_PROG_H_
#define DALI_B200_CSRC_JPEG_PROG_H_
#include <map>
#include <string>
#include <vector>
#include "decode_stage.h"
#include "jpeg_prog_core.h"

namespace dalib200 {

// Progressive and multi-scan samples: the scans run wave by wave into the plan's coefficient arena and leave the DC as differences for
// dc_scan; everything behind that is the baseline path's.  A scan is a serial chain on ONE warp (milliseconds for a large image) that
// leaves the GPU empty: the stage runs beside the baseline samples' entropy kernels.
struct ProgStage : SideStage {
  bool Empty() const override { return images.empty(); }
  void Clear() override;
  // Plans the scans of sample `sample` of stream d[0, len), whose first scan's data starts at `sb` and whose last ends at `se`; `im` is
  // the frame layout the baseline plan derived, the coefficients start at `coef_off`, the staged bytes at `raw_off`.  quant[c]: the
  // quantisation table component c latched at its first scan (PlanProgressive).  Returns a DALIB200 status; *err says why on failure.
  int Plan(const uint8_t *d, size_t len, size_t sb, size_t se, int sample, int64_t raw_off, int64_t coef_off, const JpegImage &im,
           uint16_t quant[4][64], std::string *err);
  void SortWaves();                          // after the batch's last sample

  std::vector<ProgImage> images;
  std::vector<ProgScan> scans;               // sorted by wave
  std::vector<ProgHuff> huff;
  std::vector<int> wave_begin;               // scans [wave_begin[w], wave_begin[w + 1]) run in launch w
  std::vector<int64_t> first_blk;            // prefix sum of the blocks of the images
  int64_t total_blocks = 0;
  std::map<std::string, int> table_cache;    // Huffman tables of the batch, deduplicated by content

 protected:
  // clears the coefficient blocks of the images, runs the scans wave by wave and writes the DC differences the shared dc_scan stage
  // expects
  int Enqueue(const StageInputs &in, cudaStream_t s) override;
};

}  // namespace dalib200
#endif  // DALI_B200_CSRC_JPEG_PROG_H_
