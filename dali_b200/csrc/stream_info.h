// dali_b200/csrc/stream_info.h -- what the PNG, TIFF and WebP planners (png_plan.h, tiff_plan.h, webp_plan.h) report of a stream to the
// image decoder plan besides the device descriptors: the fields JpegGetInfo returns and the byte range the plan stages for the device.
// Plain C++.
#ifndef DALI_B200_CSRC_STREAM_INFO_H_
#define DALI_B200_CSRC_STREAM_INFO_H_
#include <stddef.h>

namespace dalib200 {

struct StreamInfo {
  int width = 0, height = 0, components = 0, orientation = 1;
  size_t stage_begin = 0, stage_end = 0;   // the bytes the device reads (each planner says which)
};

}  // namespace dalib200
#endif  // DALI_B200_CSRC_STREAM_INFO_H_
