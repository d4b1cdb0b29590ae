// dali_b200/csrc/tiff.h -- launch interface of the TIFF stage (tiff.cu), called by dalib200JpegLaunch for the TIFF samples of a batch.
#ifndef DALI_B200_CSRC_TIFF_H_
#define DALI_B200_CSRC_TIFF_H_
#include <cuda_runtime.h>
#include "tiff_core.h"

namespace dalib200 {

struct TiffLaunch {
  const TiffImage *d_images; int nimages;
  const TiffSeg *d_segs; int nsegs;
  int64_t total_px;                          // window pixels of all TIFF images (TiffImage::first_px is their prefix)
  const uint8_t *d_raw;                      // the plan's staged bytes
  uint8_t *d_dec;                            // scratch for the decoded segments (TiffSeg::dec_off)
  uint8_t *d_slots;                          // TiffSlotCount(nsegs) x kTiffSlotBytes of segment working memory
  int32_t *d_status;
};
// threads of tiff_segment, and so working-memory slots, for `nsegs` segments
int TiffSlotCount(int nsegs);
// segment decode (one lane per segment), conversion of the decode windows.  Returns a DALIB200 status.
int LaunchTiff(const TiffLaunch &a, cudaStream_t s);

}  // namespace dalib200
#endif  // DALI_B200_CSRC_TIFF_H_
