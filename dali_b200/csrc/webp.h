// dali_b200/csrc/webp.h -- launch interface of the WebP stage (webp.cu), called by dalib200JpegLaunch for the WebP samples of a batch.
#ifndef DALI_B200_CSRC_WEBP_H_
#define DALI_B200_CSRC_WEBP_H_
#include <cuda_runtime.h>
#include "webp_core.h"

namespace dalib200 {

struct WebpLaunch {
  const WebpImage *d_images; int nimages;
  int64_t total_px;                          // window pixels of all WebP images (WebpImage::first_px is their prefix)
  const uint8_t *d_raw;                      // the plan's staged bytes
  uint8_t *d_scratch;                        // coefficients, macroblock records, planes, column contexts (WebpImage::*_off)
  int32_t *d_status;
};
// entropy decode (one lane per image), reconstruction and loop filter (one CTA per image, macroblock wavefront), conversion of the
// decode windows.  Returns a DALIB200 status.
int LaunchWebp(const WebpLaunch &a, cudaStream_t s);

}  // namespace dalib200
#endif  // DALI_B200_CSRC_WEBP_H_
