// dali_b200/csrc/tiff.h -- the TIFF stage of decoders.image (tiff.cu), planned and run by the image decoder plan (jpeg.cu).
#ifndef DALI_B200_CSRC_TIFF_H_
#define DALI_B200_CSRC_TIFF_H_
#include <vector>
#include "decode_stage.h"
#include "tiff_plan.h"

namespace dalib200 {

struct TiffStage : StreamStage {
  bool Empty() const override { return images.empty(); }
  void Clear() override { images.clear(); segs.clear(); dec_bytes = 0; }
  void Destroy() override { SideStage::Destroy(); cudaFree(d_dec); cudaFree(d_slots); }
  int Plan(const uint8_t *data, size_t len, int sample, int64_t raw_off, StreamInfo *info, std::string *err) override;

  std::vector<TiffImage> images;
  std::vector<TiffSeg> segs;
  int64_t dec_bytes = 0;
  uint8_t *d_dec = nullptr; size_t d_dec_cap = 0;       // decoded segments (TiffSeg::dec_off; grow only)
  uint8_t *d_slots = nullptr; size_t d_slots_cap = 0;   // segment working memory, kTiffSlotBytes per tiff_segment thread (grow only)

 protected:
  int Reserve() override;
  // segment decode (one lane per segment), conversion of the decode windows
  int Enqueue(const StageInputs &in, cudaStream_t s) override;
};

}  // namespace dalib200
#endif  // DALI_B200_CSRC_TIFF_H_
