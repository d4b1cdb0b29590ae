// dali_b200/csrc/bitmap.h -- the BMP / PNM stage of decoders.image (bitmap.cu), planned and run by the image decoder plan (jpeg.cu).
#ifndef DALI_B200_CSRC_BITMAP_H_
#define DALI_B200_CSRC_BITMAP_H_
#include <vector>
#include "decode_stage.h"
#include "bitmap_plan.h"

namespace dalib200 {

struct BitmapStage : StreamStage {
  bool Empty() const override { return images.empty(); }
  void Clear() override { images.clear(); unpack.clear(); scratch_bytes = 0; }
  void Destroy() override { SideStage::Destroy(); cudaFree(d_scratch); }
  int Plan(const uint8_t *data, size_t len, int sample, int64_t raw_off, StreamInfo *info, std::string *err) override;

  std::vector<BitmapImage> images;
  std::vector<int32_t> unpack;               // the RLE / ASCII images among them (indices into images)
  int64_t scratch_bytes = 0;
  uint8_t *d_scratch = nullptr; size_t d_scratch_cap = 0;   // unpacked planes (BitmapImage::plane_off; grow only)

 protected:
  int Reserve() override { return GrowDevice(d_scratch, d_scratch_cap, (size_t)scratch_bytes + 16); }
  // RLE / ASCII unpack (one lane per image, only when some image needs it), conversion of the decode windows
  int Enqueue(const StageInputs &in, cudaStream_t s) override;
};

}  // namespace dalib200
#endif  // DALI_B200_CSRC_BITMAP_H_
