// dali_b200/csrc/png.h -- the PNG stage of decoders.image (png.cu), planned and run by the image decoder plan (jpeg.cu).
#ifndef DALI_B200_CSRC_PNG_H_
#define DALI_B200_CSRC_PNG_H_
#include <vector>
#include "decode_stage.h"
#include "png_plan.h"

namespace dalib200 {

struct PngStage : StreamStage {
  bool Empty() const override { return images.empty(); }
  void Clear() override { images.clear(); chunks.clear(); scan_bytes = 0; }
  void Destroy() override { SideStage::Destroy(); cudaFree(d_scan); }
  int Plan(const uint8_t *data, size_t len, int sample, int64_t raw_off, StreamInfo *info, std::string *err) override;

  std::vector<PngImage> images;
  std::vector<PngChunk> chunks;
  int64_t scan_bytes = 0;
  uint8_t *d_scan = nullptr; size_t d_scan_cap = 0;   // filtered scanlines (PngImage::scan_off; grow only)

 protected:
  int Reserve() override { return GrowDevice(d_scan, d_scan_cap, (size_t)scan_bytes + 16); }
  // IDAT CRCs, inflate + unfilter (one thread per image), conversion of the decode windows
  int Enqueue(const StageInputs &in, cudaStream_t s) override;
};

}  // namespace dalib200
#endif  // DALI_B200_CSRC_PNG_H_
