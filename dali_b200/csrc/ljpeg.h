// dali_b200/csrc/ljpeg.h -- launch interface of the lossless JPEG stage (ljpeg.cu), called by dalib200JpegLaunch for the lossless
// samples of a batch once U1 - U3 have un-stuffed their units.
#ifndef DALI_B200_CSRC_LJPEG_H_
#define DALI_B200_CSRC_LJPEG_H_
#include <cuda_runtime.h>
#include "ljpeg_core.h"

namespace dalib200 {

// Enqueues L1 - L5 on `s`.  Returns a DALIB200 status.
int LaunchLjpeg(const LjpegLaunch &a, cudaStream_t s);

}  // namespace dalib200
#endif  // DALI_B200_CSRC_LJPEG_H_
