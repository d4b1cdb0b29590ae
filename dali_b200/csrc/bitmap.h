// dali_b200/csrc/bitmap.h -- launch interface of the BMP / PNM stage (bitmap.cu), called by dalib200JpegLaunch for the BMP and PNM
// samples of a batch.
#ifndef DALI_B200_CSRC_BITMAP_H_
#define DALI_B200_CSRC_BITMAP_H_
#include <cuda_runtime.h>
#include <vector>
#include "bitmap_core.h"

namespace dalib200 {

struct BitmapLaunch {
  const BitmapImage *d_images; int nimages;
  const int32_t *d_unpack; int nunpack;      // the images (indices into d_images) that bitmap_unpack expands first
  int64_t total_groups;                      // pixel groups of all windows (BitmapImage::first_grp is their prefix)
  const uint8_t *d_raw;                      // the plan's staged bytes
  uint8_t *d_scratch;                        // the unpacked planes (BitmapImage::plane_off)
  int32_t *d_status;
};
// Sets each image's first_grp from its window (after FillWindows) and returns the group total.
int64_t BitmapGroups(std::vector<BitmapImage> &images);
// RLE / ASCII unpack (one lane per image, only when nunpack > 0), conversion of the decode windows.  Returns a DALIB200 status.
int LaunchBitmap(const BitmapLaunch &a, cudaStream_t s);

}  // namespace dalib200
#endif  // DALI_B200_CSRC_BITMAP_H_
