// dali_b200/csrc/png.h -- launch interface of the PNG stage (png.cu), called by dalib200JpegLaunch for the PNG samples of a batch.
#ifndef DALI_B200_CSRC_PNG_H_
#define DALI_B200_CSRC_PNG_H_
#include <cuda_runtime.h>
#include "png_core.h"

namespace dalib200 {

struct PngLaunch {
  const PngImage *d_images; int nimages;
  const PngChunk *d_chunks; int nchunks;
  int64_t total_px;                          // window pixels of all PNG images (PngImage::first_px is their prefix)
  const uint8_t *d_raw;                      // the plan's staged bytes
  uint8_t *d_scan;                           // scratch for the filtered scanlines (PngImage::scan_off)
  int32_t *d_status;
};
// IDAT CRCs, inflate + unfilter (one thread per image), conversion of the decode windows.  Returns a DALIB200 status.
int LaunchPng(const PngLaunch &a, cudaStream_t s);

}  // namespace dalib200
#endif  // DALI_B200_CSRC_PNG_H_
