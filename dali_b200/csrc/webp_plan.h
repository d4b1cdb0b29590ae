// dali_b200/csrc/webp_plan.h -- host-side planning of a lossy WebP stream inside the image decoder plan: the walk of the RIFF chunks
// (simple format, or VP8X with ICCP / ALPH / EXIF / XMP chunks around one VP8 chunk), the VP8 frame header, and the first partition's
// header fields up to the first macroblock -- segment header, filter header, partition table, quantizer indices, token probability
// updates, skip probability -- turned into the WebpImage record the device stages read (webp_core.h).  No per-macroblock work.  Plain
// C++ (no CUDA types): jpeg.cu calls it from JpegGetInfo / JpegPlanSetup, tools/emul/webp_emul.cc from the CPU tests.
//
// The checks restate libwebp's (src/dec/webp_dec.c ParseHeadersInternal, vp8_dec.c VP8GetHeaders): a bad RIFF or chunk size, a chunk
// overrunning the RIFF, a VP8X canvas that differs from the frame, a bad start code, an inter frame, profile > 3, a hidden frame or a
// first partition that does not fit are DALIB200_ERROR_BAD_DATA; lossless (VP8L) and animated streams are DALIB200_ERROR_UNSUPPORTED.
// An ALPH chunk is skipped: the colour decode of cv2 does not depend on it (DESIGN.md section 2).
#ifndef DALI_B200_CSRC_WEBP_PLAN_H_
#define DALI_B200_CSRC_WEBP_PLAN_H_
#include <cstring>
#include <string>
#include "../../include/dali_b200.h"
#include "exif.h"
#include "stream_info.h"
#include "webp_core.h"

namespace dalib200 {

inline bool IsWebpStream(const uint8_t *p, size_t n) { return n >= 12 && !memcmp(p, "RIFF", 4) && !memcmp(p + 8, "WEBP", 4); }

// RFC 6386 section 14.1 (libwebp kDcTable / kAcTable)
static const uint8_t kWebpDcTable[128] = {
    4,   5,   6,   7,   8,   9,  10,  10,  11,  12,  13,  14,  15,  16,  17,  17,
   18,  19,  20,  20,  21,  21,  22,  22,  23,  23,  24,  25,  25,  26,  27,  28,
   29,  30,  31,  32,  33,  34,  35,  36,  37,  37,  38,  39,  40,  41,  42,  43,
   44,  45,  46,  46,  47,  48,  49,  50,  51,  52,  53,  54,  55,  56,  57,  58,
   59,  60,  61,  62,  63,  64,  65,  66,  67,  68,  69,  70,  71,  72,  73,  74,
   75,  76,  76,  77,  78,  79,  80,  81,  82,  83,  84,  85,  86,  87,  88,  89,
   91,  93,  95,  96,  98, 100, 101, 102, 104, 106, 108, 110, 112, 114, 116, 118,
  122, 124, 126, 128, 130, 132, 134, 136, 138, 140, 143, 145, 148, 151, 154, 157
};
static const uint16_t kWebpAcTable[128] = {
    4,   5,   6,   7,   8,   9,  10,  11,  12,  13,  14,  15,  16,  17,  18,  19,
   20,  21,  22,  23,  24,  25,  26,  27,  28,  29,  30,  31,  32,  33,  34,  35,
   36,  37,  38,  39,  40,  41,  42,  43,  44,  45,  46,  47,  48,  49,  50,  51,
   52,  53,  54,  55,  56,  57,  58,  60,  62,  64,  66,  68,  70,  72,  74,  76,
   78,  80,  82,  84,  86,  88,  90,  92,  94,  96,  98, 100, 102, 104, 106, 108,
  110, 112, 114, 116, 119, 122, 125, 128, 131, 134, 137, 140, 143, 146, 149, 152,
  155, 158, 161, 164, 167, 170, 173, 177, 181, 185, 189, 193, 197, 201, 205, 209,
  213, 217, 221, 225, 229, 234, 239, 245, 249, 254, 259, 264, 269, 274, 279, 284
};
// RFC 6386 section 13.5 (default token probabilities) and 13.4 (probabilities of their updates), [type][band][ctx][node]
static const uint8_t kWebpCoeffsProba0[4][8][3][11] = {
  {
    { { 128, 128, 128, 128, 128, 128, 128, 128, 128, 128, 128 },
      { 128, 128, 128, 128, 128, 128, 128, 128, 128, 128, 128 },
      { 128, 128, 128, 128, 128, 128, 128, 128, 128, 128, 128 } },
    { { 253, 136, 254, 255, 228, 219, 128, 128, 128, 128, 128 },
      { 189, 129, 242, 255, 227, 213, 255, 219, 128, 128, 128 },
      { 106, 126, 227, 252, 214, 209, 255, 255, 128, 128, 128 } },
    { {   1,  98, 248, 255, 236, 226, 255, 255, 128, 128, 128 },
      { 181, 133, 238, 254, 221, 234, 255, 154, 128, 128, 128 },
      {  78, 134, 202, 247, 198, 180, 255, 219, 128, 128, 128 } },
    { {   1, 185, 249, 255, 243, 255, 128, 128, 128, 128, 128 },
      { 184, 150, 247, 255, 236, 224, 128, 128, 128, 128, 128 },
      {  77, 110, 216, 255, 236, 230, 128, 128, 128, 128, 128 } },
    { {   1, 101, 251, 255, 241, 255, 128, 128, 128, 128, 128 },
      { 170, 139, 241, 252, 236, 209, 255, 255, 128, 128, 128 },
      {  37, 116, 196, 243, 228, 255, 255, 255, 128, 128, 128 } },
    { {   1, 204, 254, 255, 245, 255, 128, 128, 128, 128, 128 },
      { 207, 160, 250, 255, 238, 128, 128, 128, 128, 128, 128 },
      { 102, 103, 231, 255, 211, 171, 128, 128, 128, 128, 128 } },
    { {   1, 152, 252, 255, 240, 255, 128, 128, 128, 128, 128 },
      { 177, 135, 243, 255, 234, 225, 128, 128, 128, 128, 128 },
      {  80, 129, 211, 255, 194, 224, 128, 128, 128, 128, 128 } },
    { {   1,   1, 255, 128, 128, 128, 128, 128, 128, 128, 128 },
      { 246,   1, 255, 128, 128, 128, 128, 128, 128, 128, 128 },
      { 255, 128, 128, 128, 128, 128, 128, 128, 128, 128, 128 } }
  },
  {
    { { 198,  35, 237, 223, 193, 187, 162, 160, 145, 155,  62 },
      { 131,  45, 198, 221, 172, 176, 220, 157, 252, 221,   1 },
      {  68,  47, 146, 208, 149, 167, 221, 162, 255, 223, 128 } },
    { {   1, 149, 241, 255, 221, 224, 255, 255, 128, 128, 128 },
      { 184, 141, 234, 253, 222, 220, 255, 199, 128, 128, 128 },
      {  81,  99, 181, 242, 176, 190, 249, 202, 255, 255, 128 } },
    { {   1, 129, 232, 253, 214, 197, 242, 196, 255, 255, 128 },
      {  99, 121, 210, 250, 201, 198, 255, 202, 128, 128, 128 },
      {  23,  91, 163, 242, 170, 187, 247, 210, 255, 255, 128 } },
    { {   1, 200, 246, 255, 234, 255, 128, 128, 128, 128, 128 },
      { 109, 178, 241, 255, 231, 245, 255, 255, 128, 128, 128 },
      {  44, 130, 201, 253, 205, 192, 255, 255, 128, 128, 128 } },
    { {   1, 132, 239, 251, 219, 209, 255, 165, 128, 128, 128 },
      {  94, 136, 225, 251, 218, 190, 255, 255, 128, 128, 128 },
      {  22, 100, 174, 245, 186, 161, 255, 199, 128, 128, 128 } },
    { {   1, 182, 249, 255, 232, 235, 128, 128, 128, 128, 128 },
      { 124, 143, 241, 255, 227, 234, 128, 128, 128, 128, 128 },
      {  35,  77, 181, 251, 193, 211, 255, 205, 128, 128, 128 } },
    { {   1, 157, 247, 255, 236, 231, 255, 255, 128, 128, 128 },
      { 121, 141, 235, 255, 225, 227, 255, 255, 128, 128, 128 },
      {  45,  99, 188, 251, 195, 217, 255, 224, 128, 128, 128 } },
    { {   1,   1, 251, 255, 213, 255, 128, 128, 128, 128, 128 },
      { 203,   1, 248, 255, 255, 128, 128, 128, 128, 128, 128 },
      { 137,   1, 177, 255, 224, 255, 128, 128, 128, 128, 128 } }
  },
  {
    { { 253,   9, 248, 251, 207, 208, 255, 192, 128, 128, 128 },
      { 175,  13, 224, 243, 193, 185, 249, 198, 255, 255, 128 },
      {  73,  17, 171, 221, 161, 179, 236, 167, 255, 234, 128 } },
    { {   1,  95, 247, 253, 212, 183, 255, 255, 128, 128, 128 },
      { 239,  90, 244, 250, 211, 209, 255, 255, 128, 128, 128 },
      { 155,  77, 195, 248, 188, 195, 255, 255, 128, 128, 128 } },
    { {   1,  24, 239, 251, 218, 219, 255, 205, 128, 128, 128 },
      { 201,  51, 219, 255, 196, 186, 128, 128, 128, 128, 128 },
      {  69,  46, 190, 239, 201, 218, 255, 228, 128, 128, 128 } },
    { {   1, 191, 251, 255, 255, 128, 128, 128, 128, 128, 128 },
      { 223, 165, 249, 255, 213, 255, 128, 128, 128, 128, 128 },
      { 141, 124, 248, 255, 255, 128, 128, 128, 128, 128, 128 } },
    { {   1,  16, 248, 255, 255, 128, 128, 128, 128, 128, 128 },
      { 190,  36, 230, 255, 236, 255, 128, 128, 128, 128, 128 },
      { 149,   1, 255, 128, 128, 128, 128, 128, 128, 128, 128 } },
    { {   1, 226, 255, 128, 128, 128, 128, 128, 128, 128, 128 },
      { 247, 192, 255, 128, 128, 128, 128, 128, 128, 128, 128 },
      { 240, 128, 255, 128, 128, 128, 128, 128, 128, 128, 128 } },
    { {   1, 134, 252, 255, 255, 128, 128, 128, 128, 128, 128 },
      { 213,  62, 250, 255, 255, 128, 128, 128, 128, 128, 128 },
      {  55,  93, 255, 128, 128, 128, 128, 128, 128, 128, 128 } },
    { { 128, 128, 128, 128, 128, 128, 128, 128, 128, 128, 128 },
      { 128, 128, 128, 128, 128, 128, 128, 128, 128, 128, 128 },
      { 128, 128, 128, 128, 128, 128, 128, 128, 128, 128, 128 } }
  },
  {
    { { 202,  24, 213, 235, 186, 191, 220, 160, 240, 175, 255 },
      { 126,  38, 182, 232, 169, 184, 228, 174, 255, 187, 128 },
      {  61,  46, 138, 219, 151, 178, 240, 170, 255, 216, 128 } },
    { {   1, 112, 230, 250, 199, 191, 247, 159, 255, 255, 128 },
      { 166, 109, 228, 252, 211, 215, 255, 174, 128, 128, 128 },
      {  39,  77, 162, 232, 172, 180, 245, 178, 255, 255, 128 } },
    { {   1,  52, 220, 246, 198, 199, 249, 220, 255, 255, 128 },
      { 124,  74, 191, 243, 183, 193, 250, 221, 255, 255, 128 },
      {  24,  71, 130, 219, 154, 170, 243, 182, 255, 255, 128 } },
    { {   1, 182, 225, 249, 219, 240, 255, 224, 128, 128, 128 },
      { 149, 150, 226, 252, 216, 205, 255, 171, 128, 128, 128 },
      {  28, 108, 170, 242, 183, 194, 254, 223, 255, 255, 128 } },
    { {   1,  81, 230, 252, 204, 203, 255, 192, 128, 128, 128 },
      { 123, 102, 209, 247, 188, 196, 255, 233, 128, 128, 128 },
      {  20,  95, 153, 243, 164, 173, 255, 203, 128, 128, 128 } },
    { {   1, 222, 248, 255, 216, 213, 128, 128, 128, 128, 128 },
      { 168, 175, 246, 252, 235, 205, 255, 255, 128, 128, 128 },
      {  47, 116, 215, 255, 211, 212, 255, 255, 128, 128, 128 } },
    { {   1, 121, 236, 253, 212, 214, 255, 255, 128, 128, 128 },
      { 141,  84, 213, 252, 201, 202, 255, 219, 128, 128, 128 },
      {  42,  80, 160, 240, 162, 185, 255, 205, 128, 128, 128 } },
    { {   1,   1, 255, 128, 128, 128, 128, 128, 128, 128, 128 },
      { 244,   1, 255, 128, 128, 128, 128, 128, 128, 128, 128 },
      { 238,   1, 255, 128, 128, 128, 128, 128, 128, 128, 128 } }
  }
};
static const uint8_t kWebpCoeffsUpdateProba[4][8][3][11] = {
  {
    { { 255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255 },
      { 255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255 },
      { 255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255 } },
    { { 176, 246, 255, 255, 255, 255, 255, 255, 255, 255, 255 },
      { 223, 241, 252, 255, 255, 255, 255, 255, 255, 255, 255 },
      { 249, 253, 253, 255, 255, 255, 255, 255, 255, 255, 255 } },
    { { 255, 244, 252, 255, 255, 255, 255, 255, 255, 255, 255 },
      { 234, 254, 254, 255, 255, 255, 255, 255, 255, 255, 255 },
      { 253, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255 } },
    { { 255, 246, 254, 255, 255, 255, 255, 255, 255, 255, 255 },
      { 239, 253, 254, 255, 255, 255, 255, 255, 255, 255, 255 },
      { 254, 255, 254, 255, 255, 255, 255, 255, 255, 255, 255 } },
    { { 255, 248, 254, 255, 255, 255, 255, 255, 255, 255, 255 },
      { 251, 255, 254, 255, 255, 255, 255, 255, 255, 255, 255 },
      { 255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255 } },
    { { 255, 253, 254, 255, 255, 255, 255, 255, 255, 255, 255 },
      { 251, 254, 254, 255, 255, 255, 255, 255, 255, 255, 255 },
      { 254, 255, 254, 255, 255, 255, 255, 255, 255, 255, 255 } },
    { { 255, 254, 253, 255, 254, 255, 255, 255, 255, 255, 255 },
      { 250, 255, 254, 255, 254, 255, 255, 255, 255, 255, 255 },
      { 254, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255 } },
    { { 255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255 },
      { 255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255 },
      { 255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255 } }
  },
  {
    { { 217, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255 },
      { 225, 252, 241, 253, 255, 255, 254, 255, 255, 255, 255 },
      { 234, 250, 241, 250, 253, 255, 253, 254, 255, 255, 255 } },
    { { 255, 254, 255, 255, 255, 255, 255, 255, 255, 255, 255 },
      { 223, 254, 254, 255, 255, 255, 255, 255, 255, 255, 255 },
      { 238, 253, 254, 254, 255, 255, 255, 255, 255, 255, 255 } },
    { { 255, 248, 254, 255, 255, 255, 255, 255, 255, 255, 255 },
      { 249, 254, 255, 255, 255, 255, 255, 255, 255, 255, 255 },
      { 255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255 } },
    { { 255, 253, 255, 255, 255, 255, 255, 255, 255, 255, 255 },
      { 247, 254, 255, 255, 255, 255, 255, 255, 255, 255, 255 },
      { 255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255 } },
    { { 255, 253, 254, 255, 255, 255, 255, 255, 255, 255, 255 },
      { 252, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255 },
      { 255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255 } },
    { { 255, 254, 254, 255, 255, 255, 255, 255, 255, 255, 255 },
      { 253, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255 },
      { 255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255 } },
    { { 255, 254, 253, 255, 255, 255, 255, 255, 255, 255, 255 },
      { 250, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255 },
      { 254, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255 } },
    { { 255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255 },
      { 255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255 },
      { 255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255 } }
  },
  {
    { { 186, 251, 250, 255, 255, 255, 255, 255, 255, 255, 255 },
      { 234, 251, 244, 254, 255, 255, 255, 255, 255, 255, 255 },
      { 251, 251, 243, 253, 254, 255, 254, 255, 255, 255, 255 } },
    { { 255, 253, 254, 255, 255, 255, 255, 255, 255, 255, 255 },
      { 236, 253, 254, 255, 255, 255, 255, 255, 255, 255, 255 },
      { 251, 253, 253, 254, 254, 255, 255, 255, 255, 255, 255 } },
    { { 255, 254, 254, 255, 255, 255, 255, 255, 255, 255, 255 },
      { 254, 254, 254, 255, 255, 255, 255, 255, 255, 255, 255 },
      { 255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255 } },
    { { 255, 254, 255, 255, 255, 255, 255, 255, 255, 255, 255 },
      { 254, 254, 255, 255, 255, 255, 255, 255, 255, 255, 255 },
      { 254, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255 } },
    { { 255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255 },
      { 254, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255 },
      { 255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255 } },
    { { 255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255 },
      { 255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255 },
      { 255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255 } },
    { { 255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255 },
      { 255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255 },
      { 255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255 } },
    { { 255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255 },
      { 255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255 },
      { 255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255 } }
  },
  {
    { { 248, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255 },
      { 250, 254, 252, 254, 255, 255, 255, 255, 255, 255, 255 },
      { 248, 254, 249, 253, 255, 255, 255, 255, 255, 255, 255 } },
    { { 255, 253, 253, 255, 255, 255, 255, 255, 255, 255, 255 },
      { 246, 253, 253, 255, 255, 255, 255, 255, 255, 255, 255 },
      { 252, 254, 251, 254, 254, 255, 255, 255, 255, 255, 255 } },
    { { 255, 254, 252, 255, 255, 255, 255, 255, 255, 255, 255 },
      { 248, 254, 253, 255, 255, 255, 255, 255, 255, 255, 255 },
      { 253, 255, 254, 254, 255, 255, 255, 255, 255, 255, 255 } },
    { { 255, 251, 254, 255, 255, 255, 255, 255, 255, 255, 255 },
      { 245, 251, 254, 255, 255, 255, 255, 255, 255, 255, 255 },
      { 253, 253, 254, 255, 255, 255, 255, 255, 255, 255, 255 } },
    { { 255, 251, 253, 255, 255, 255, 255, 255, 255, 255, 255 },
      { 252, 253, 254, 255, 255, 255, 255, 255, 255, 255, 255 },
      { 255, 254, 255, 255, 255, 255, 255, 255, 255, 255, 255 } },
    { { 255, 252, 255, 255, 255, 255, 255, 255, 255, 255, 255 },
      { 249, 255, 254, 255, 255, 255, 255, 255, 255, 255, 255 },
      { 255, 255, 254, 255, 255, 255, 255, 255, 255, 255, 255 } },
    { { 255, 255, 253, 255, 255, 255, 255, 255, 255, 255, 255 },
      { 250, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255 },
      { 255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255 } },
    { { 255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255 },
      { 254, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255 },
      { 255, 255, 255, 255, 255, 255, 255, 255, 255, 255, 255 } }
  }
};

// Scratch of one image: coefficients, macroblock records, padded planes, column context (16-byte aligned each)
inline int64_t WebpScratchBytes(int mb_w, int mb_h) {
  const int64_t nmb = (int64_t)mb_w * mb_h;
  auto al = [](int64_t v) { return (v + 15) & ~(int64_t)15; };
  return al(nmb * 768) + al(nmb * (int64_t)sizeof(WebpMb)) + al(nmb * 384) + al((int64_t)mb_w * 4);
}

// Plans image `image`: its scratch ranges start at `scratch_base` (*scratch_bytes receives their size), its staged bytes are given by
// info->stage_begin / stage_end, from behind the frame header to the end of the input (partition offsets are relative to stage_begin).
// Returns a DALIB200 status.
inline int PlanWebp(const uint8_t *p, size_t n, int image, WebpImage *im, int64_t scratch_base, int64_t *scratch_bytes, StreamInfo *info,
                    std::string *err) {
  (void)image;
  auto fail = [&](int rc, const std::string &m) { if (err) *err = "WebP: " + m; return rc; };
  auto bad = [&](const std::string &m) { return fail(DALIB200_ERROR_BAD_DATA, m); };
  auto unsupported = [&](const std::string &m) { return fail(DALIB200_ERROR_UNSUPPORTED, m); };
  auto le32 = [&](size_t o) { return (uint32_t)p[o] | ((uint32_t)p[o + 1] << 8) | ((uint32_t)p[o + 2] << 16) | ((uint32_t)p[o + 3] << 24); };
  auto le24 = [&](size_t o) { return (uint32_t)p[o] | ((uint32_t)p[o + 1] << 8) | ((uint32_t)p[o + 2] << 16); };
  auto tag = [&](size_t o, const char *t) { return !memcmp(p + o, t, 4); };
  memset(im, 0, sizeof(*im));
  *info = StreamInfo();
  if (!IsWebpStream(p, n)) return bad("missing RIFF / WEBP header");
  // ---- RIFF (libwebp ParseRIFF): at least one chunk header, inside the data.  Bytes behind the RIFF are still data to the VP8
  // decoder: libwebp hands it everything from the frame header to the end of the input (see the partitions below).
  const uint32_t riff = le32(4);
  constexpr uint32_t kMaxChunkPayload = ~0u - 8 - 1;
  if (riff < 12) return bad("RIFF size too small");
  if (riff > kMaxChunkPayload) return bad("RIFF size too large");
  if (riff > n - 8) return bad("truncated stream (RIFF size " + std::to_string(riff) + ", " + std::to_string(n) + " bytes)");
  const size_t riff_end = (size_t)riff + 8;
  size_t pos = 12;
  // ---- VP8X and the chunks in front of the frame (libwebp ParseVP8X / ParseOptionalChunks)
  bool vp8x = false;
  uint32_t flags = 0, cw = 0, ch = 0;
  if (n - pos >= 8 && tag(pos, "VP8X")) {
    if (le32(pos + 4) != 10) return bad("VP8X chunk of size " + std::to_string(le32(pos + 4)) + " (10 expected)");
    if (n - pos < 18) return bad("truncated VP8X chunk");
    flags = le32(pos + 8); cw = 1 + le24(pos + 12); ch = 1 + le24(pos + 15);
    if ((uint64_t)cw * ch >= (1ull << 32)) return bad("VP8X canvas too large");
    if (flags & 0x02) return unsupported("animated WebP is not supported");
    vp8x = true;
    pos += 18;
    // every chunk up to and including the frame chunk, padded to an even size, must lie inside the RIFF (an odd-sized frame chunk
    // ending at the RIFF's end without its padding byte is refused); the frame chunk's data may run past the input's end here, the
    // frame checks below catch that
    uint64_t total = 12 + 18;                               // bytes of the RIFF so far, its 8-byte header included
    for (;;) {
      if (n - pos < 8) return bad("truncated stream: no VP8 chunk");
      const uint32_t cs = le32(pos + 4);
      if (cs > kMaxChunkPayload) return bad("chunk size too large");
      const uint64_t disk = (8ull + cs + 1) & ~1ull;
      total += disk;
      if (total > (uint64_t)riff_end) return bad("a chunk overruns the RIFF");
      if (tag(pos, "VP8 ") || tag(pos, "VP8L")) break;
      if (disk > n - pos) return bad("truncated chunk");
      if (tag(pos, "ANIM") || tag(pos, "ANMF")) return unsupported("animated WebP is not supported");
      pos += (size_t)disk;
    }
  }
  // ---- the frame chunk (libwebp ParseVP8Header)
  if (n - pos < 8) return bad("truncated stream: no VP8 chunk");
  if (tag(pos, "VP8L")) return unsupported("lossless WebP (VP8L) is not supported");
  if (tag(pos, "ANIM") || tag(pos, "ANMF")) return unsupported("animated WebP is not supported");
  if (!tag(pos, "VP8 ")) return bad("no VP8 chunk");
  const uint32_t csize = le32(pos + 4);
  if (csize > riff - 12) return bad("the VP8 chunk overruns the RIFF");
  if (csize > n - pos - 8) return bad("truncated VP8 chunk");
  const uint8_t *f = p + pos + 8;
  // ---- the EXIF orientation, as cv2 reads it (libwebp's demuxer): from the first EXIF chunk, when VP8X flags EXIF and every chunk
  // from VP8X to the RIFF's end is complete (padded size inside the RIFF, no partial chunk header).  Otherwise cv2 reads no EXIF and
  // applies none; the image itself still decodes, so a damaged chunk behind the frame is not an error here either.
  int orientation = 1;
  if (vp8x && (flags & 0x08)) {
    int first = 0;
    size_t q = 12;
    while (q < riff_end) {
      if (riff_end - q < 8) { first = 0; break; }
      const uint64_t disk = (8ull + le32(q + 4) + 1) & ~1ull;
      if (disk > riff_end - q) { first = 0; break; }
      if (!first && tag(q, "EXIF")) {
        const uint8_t *e = p + q + 8;
        const int el = (int)le32(q + 4);
        first = el >= 6 && !memcmp(e, "Exif\0\0", 6) ? ParseExifOrientation(e + 6, el - 6) : ParseExifOrientation(e, el);
      }
      q += (size_t)disk;
    }
    orientation = first ? first : 1;
  }
  // ---- frame header (libwebp VP8GetInfo / VP8GetHeaders).  The VP8 decoder reads from the frame header to the END OF THE INPUT,
  // not of the chunk (libwebp DecodeInto): partition 0 and the partition table are bounded by that, the token partitions are clamped
  // to it, and the last one runs up to it.  Only VP8GetInfo compares the first partition with the chunk size.
  if (n - pos - 8 < 10) return bad("truncated VP8 frame header");
  if (n - (pos + 8) - 10 > 0xFFFFFFFFull) return unsupported("streams of 4 GiB or more are not supported");
  const uint32_t bits = f[0] | (f[1] << 8) | (f[2] << 16);
  const uint32_t p0len = bits >> 5;
  if (bits & 1) return bad("not a key frame");
  if (((bits >> 1) & 7) > 3) return bad("profile " + std::to_string((bits >> 1) & 7) + " (at most 3)");
  if (!((bits >> 4) & 1)) return bad("frame not displayable");
  if (p0len >= csize) return bad("first partition larger than the frame");
  if (f[3] != 0x9d || f[4] != 0x01 || f[5] != 0x2a) return bad("bad start code");
  const int W = (f[6] | (f[7] << 8)) & 0x3fff, H = (f[8] | (f[9] << 8)) & 0x3fff;
  if (W == 0 || H == 0) return bad("zero image size");
  if (vp8x && ((uint32_t)W != cw || (uint32_t)H != ch)) return bad("VP8X canvas differs from the frame size");
  const uint32_t rest = (uint32_t)(n - (pos + 8) - 10);     // partition 0, the partition sizes, the token partitions
  if (p0len > rest) return bad("bad partition length");
  const uint8_t *base = f + 10;
  WebpBits br;
  webp_bits_init(br, base, p0len);
  webp_bit(br, 0x80); webp_bit(br, 0x80);                  // colour space, clamping type: not used by the decoder
  // segment header (libwebp ParseSegmentHeader)
  int use_segment = webp_bit(br, 0x80), absolute_delta = 1;
  int quantizer[4] = {0, 0, 0, 0}, filter_strength[4] = {0, 0, 0, 0};
  uint8_t seg_p[3] = {255, 255, 255};
  int update_map = 0;
  if (use_segment) {
    update_map = webp_bit(br, 0x80);
    if (webp_bit(br, 0x80)) {
      absolute_delta = webp_bit(br, 0x80);
      for (int s = 0; s < 4; s++) quantizer[s] = webp_bit(br, 0x80) ? webp_signed_value(br, 7) : 0;
      for (int s = 0; s < 4; s++) filter_strength[s] = webp_bit(br, 0x80) ? webp_signed_value(br, 6) : 0;
    }
    if (update_map)
      for (int s = 0; s < 3; s++) seg_p[s] = webp_bit(br, 0x80) ? (uint8_t)webp_value(br, 8) : 255;
  }
  if (br.eof) return bad("cannot parse the segment header");
  // filter header (libwebp ParseFilterHeader)
  const int simple = webp_bit(br, 0x80);
  const int level = (int)webp_value(br, 6), sharpness = (int)webp_value(br, 3);
  const int use_lf_delta = webp_bit(br, 0x80);
  int ref_lf_delta0 = 0, mode_lf_delta0 = 0;
  if (use_lf_delta && webp_bit(br, 0x80)) {
    for (int i = 0; i < 4; i++) if (webp_bit(br, 0x80)) { const int d = webp_signed_value(br, 6); if (i == 0) ref_lf_delta0 = d; }
    for (int i = 0; i < 4; i++) if (webp_bit(br, 0x80)) { const int d = webp_signed_value(br, 6); if (i == 0) mode_lf_delta0 = d; }
  }
  if (br.eof) return bad("cannot parse the filter header");
  // partitions (libwebp ParsePartitions): a size past the data is clamped; the last partition must not be empty
  const int nparts = 1 << webp_value(br, 2);
  const uint32_t after = rest - p0len;
  if (after < 3u * (nparts - 1)) return bad("cannot read the partition sizes");
  uint32_t part_start = p0len + 3 * (nparts - 1), left = after - 3 * (nparts - 1);
  for (int k = 0; k < nparts - 1; k++) {
    const uint8_t *sz = base + p0len + 3 * k;
    uint32_t ps = sz[0] | (sz[1] << 8) | (sz[2] << 16);
    if (ps > left) ps = left;
    im->part_off[k] = part_start; im->part_len[k] = ps;
    part_start += ps; left -= ps;
  }
  im->part_off[nparts - 1] = part_start; im->part_len[nparts - 1] = left;
  if (left == 0) return bad("the last partition is empty");
  im->nparts = nparts;
  // quantizers (libwebp VP8ParseQuant)
  const int base_q0 = (int)webp_value(br, 7);
  int dq[5];
  for (int k = 0; k < 5; k++) dq[k] = webp_bit(br, 0x80) ? webp_signed_value(br, 4) : 0;
  const int dqy1_dc = dq[0], dqy2_dc = dq[1], dqy2_ac = dq[2], dquv_dc = dq[3], dquv_ac = dq[4];
  auto clip = [](int v, int m) { return v < 0 ? 0 : v > m ? m : v; };
  for (int s = 0; s < 4; s++) {
    int q = base_q0;
    if (use_segment) { q = quantizer[s]; if (!absolute_delta) q += base_q0; }
    else if (s > 0) { memcpy(im->dq[s], im->dq[0], sizeof(im->dq[0])); continue; }
    int16_t *m = im->dq[s];
    m[0] = kWebpDcTable[clip(q + dqy1_dc, 127)];
    m[1] = (int16_t)kWebpAcTable[clip(q, 127)];
    m[2] = (int16_t)(kWebpDcTable[clip(q + dqy2_dc, 127)] * 2);
    int y2ac = (kWebpAcTable[clip(q + dqy2_ac, 127)] * 101581) >> 16;   // x * 155 / 100
    m[3] = (int16_t)(y2ac < 8 ? 8 : y2ac);
    m[4] = kWebpDcTable[clip(q + dquv_dc, 117)];
    m[5] = (int16_t)kWebpAcTable[clip(q + dquv_ac, 127)];
  }
  webp_bit(br, 0x80);                                       // refresh_entropy_probs: a single frame, not used
  // token probabilities (libwebp VP8ParseProba) and the skip probability
  for (int t = 0; t < 4; t++)
    for (int b = 0; b < 8; b++)
      for (int c = 0; c < 3; c++)
        for (int k = 0; k < 11; k++)
          im->proba[t][b][c][k] = webp_bit(br, kWebpCoeffsUpdateProba[t][b][c][k]) ? (uint8_t)webp_value(br, 8) : kWebpCoeffsProba0[t][b][c][k];
  im->use_skip = webp_bit(br, 0x80);
  im->skip_p = im->use_skip ? (uint8_t)webp_value(br, 8) : 0;
  // partition 0 at the first macroblock (a read past its end is found by the device stage, as libwebp finds it in the row loop)
  im->br0.pos = (uint32_t)(br.buf - base); im->br0.end = p0len;
  im->br0.value = br.value; im->br0.range = br.range; im->br0.bits = br.bits; im->br0.eof = br.eof;
  im->update_map = update_map;
  memcpy(im->seg_p, seg_p, 3);
  // filter strengths (libwebp PrecomputeFilterStrengths); no filtering at all when the frame's level is 0
  im->filter_type = level == 0 ? 0 : simple ? 1 : 2;
  if (im->filter_type)
    for (int s = 0; s < 4; s++) {
      int base_level = level;
      if (use_segment) { base_level = filter_strength[s]; if (!absolute_delta) base_level += level; }
      for (int i4 = 0; i4 <= 1; i4++) {
        int lv = base_level;
        if (use_lf_delta) { lv += ref_lf_delta0; if (i4) lv += mode_lf_delta0; }
        lv = lv < 0 ? 0 : lv > 63 ? 63 : lv;
        if (lv > 0) {
          int ilevel = lv;
          if (sharpness > 0) {
            ilevel >>= sharpness > 4 ? 2 : 1;
            if (ilevel > 9 - sharpness) ilevel = 9 - sharpness;
          }
          if (ilevel < 1) ilevel = 1;
          im->f_ilevel[s][i4] = (uint8_t)ilevel;
          im->f_limit[s][i4] = (uint8_t)(2 * lv + ilevel);
          im->f_hev[s][i4] = (uint8_t)(lv >= 40 ? 2 : lv >= 15 ? 1 : 0);
        }
      }
    }
  im->width = W; im->height = H;
  im->mb_w = (W + 15) >> 4; im->mb_h = (H + 15) >> 4;
  const int64_t nmb = (int64_t)im->mb_w * im->mb_h;
  auto al = [](int64_t v) { return (v + 15) & ~(int64_t)15; };
  im->coef_off = scratch_base;
  im->mb_off = im->coef_off + al(nmb * 768);
  im->plane_off = im->mb_off + al(nmb * (int64_t)sizeof(WebpMb));
  im->ctx_off = im->plane_off + al(nmb * 384);
  *scratch_bytes = WebpScratchBytes(im->mb_w, im->mb_h);
  info->width = W; info->height = H;
  info->components = vp8x && (flags & 0x10) ? 4 : 3;
  info->orientation = vp8x ? orientation : 1;
  info->stage_begin = (size_t)(base - p); info->stage_end = (size_t)(base - p) + rest;
  return DALIB200_SUCCESS;
}

}  // namespace dalib200
#endif  // DALI_B200_CSRC_WEBP_PLAN_H_
