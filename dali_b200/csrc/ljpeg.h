// dali_b200/csrc/ljpeg.h -- the lossless JPEG stage of decoders.image (ljpeg.cu), planned and run by the image decoder plan (jpeg.cu)
// once U1 - U3 have un-stuffed its units.
#ifndef DALI_B200_CSRC_LJPEG_H_
#define DALI_B200_CSRC_LJPEG_H_
#include <string>
#include <vector>
#include "decode_stage.h"
#include "ljpeg_plan.h"

namespace dalib200 {

struct LjpegStage : SideStage {
  bool Empty() const override { return images.empty(); }
  void Clear() override { images.clear(); units.clear(); tables.clear(); bands.clear(); total_sub = 0; diff_elems = 0; }
  void Destroy() override { SideStage::Destroy(); cudaFree(d_diff); cudaFree(d_rec); cudaFree(d_first); }
  // Checks the frame `f` of sample `sample`, appends its image record, tables and reconstruction bands, and one JpegUnit (to `junits`)
  // + LjpegUnit per restart interval of its scan d[sb, len), whose bytes sit at `raw` + their offset behind sb in the raw staging area;
  // `clean` and `chunks` advance as for a baseline unit.  *scan_end receives the end of the scan data.  Returns a DALIB200 status; *err
  // says why on failure.
  int Plan(const LjpegFrame &f, int sample, const uint8_t *d, size_t len, size_t sb, size_t raw, std::vector<JpegUnit> &junits,
           size_t &clean, uint32_t &chunks, size_t *scan_end, std::string *err);

  std::vector<LjpegImage> images;
  std::vector<LjpegUnit> units;
  std::vector<LjpegTable> tables;
  std::vector<LjpegBand> bands;
  int64_t total_sub = 0, diff_elems = 0;
  int16_t *d_diff = nullptr; size_t d_diff_cap = 0;     // differences, reconstructed in place (grow only)
  uint64_t *d_rec = nullptr; size_t d_rec_cap = 0;      // subsequence records (grow only)
  uint32_t *d_first = nullptr; size_t d_first_cap = 0;  // first symbol of each subsequence (grow only)

 protected:
  int Reserve() override;
  // L1 - L5 on the clean streams of the stage's units
  int Enqueue(const StageInputs &in, cudaStream_t s) override;
};

}  // namespace dalib200
#endif  // DALI_B200_CSRC_LJPEG_H_
