// dali_b200/csrc/webp.h -- the WebP stage of decoders.image (webp.cu), planned and run by the image decoder plan (jpeg.cu).
#ifndef DALI_B200_CSRC_WEBP_H_
#define DALI_B200_CSRC_WEBP_H_
#include <vector>
#include "decode_stage.h"
#include "webp_plan.h"

namespace dalib200 {

struct WebpStage : StreamStage {
  bool Empty() const override { return images.empty(); }
  void Clear() override { images.clear(); scratch_bytes = 0; }
  void Destroy() override { SideStage::Destroy(); cudaFree(d_scratch); }
  int Plan(const uint8_t *data, size_t len, int sample, int64_t raw_off, StreamInfo *info, std::string *err) override;

  std::vector<WebpImage> images;
  int64_t scratch_bytes = 0;
  uint8_t *d_scratch = nullptr; size_t d_scratch_cap = 0;   // coefficients, macroblock records, planes, column contexts (grow only)

 protected:
  int Reserve() override { return GrowDevice(d_scratch, d_scratch_cap, (size_t)scratch_bytes + 16); }
  // entropy decode (one lane per image), reconstruction and loop filter (one CTA per image, macroblock wavefront), conversion of the
  // decode windows
  int Enqueue(const StageInputs &in, cudaStream_t s) override;
};

}  // namespace dalib200
#endif  // DALI_B200_CSRC_WEBP_H_
