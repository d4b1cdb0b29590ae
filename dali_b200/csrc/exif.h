// dali_b200/csrc/exif.h -- the orientation tag of an EXIF (TIFF) block, shared by the JPEG (APP1) and PNG (eXIf) planners.
#ifndef DALI_B200_CSRC_EXIF_H_
#define DALI_B200_CSRC_EXIF_H_
#include <stdint.h>

namespace dalib200 {

// EXIF orientation 1..8 of the TIFF structure at p[0, len) ("II" / "MM" byte order), 1 when absent or malformed
inline int ParseExifOrientation(const uint8_t *p, int len) {
  if (len < 8) return 1;
  bool le;
  if (p[0] == 'I' && p[1] == 'I') le = true; else if (p[0] == 'M' && p[1] == 'M') le = false; else return 1;
  auto r16 = [&](unsigned o) { return le ? (p[o] | (p[o + 1] << 8)) : ((p[o] << 8) | p[o + 1]); };
  auto r32 = [&](unsigned o) { return le ? (unsigned)(p[o] | (p[o + 1] << 8) | (p[o + 2] << 16) | ((unsigned)p[o + 3] << 24))
                                         : (((unsigned)p[o] << 24) | (p[o + 1] << 16) | (p[o + 2] << 8) | p[o + 3]); };
  const uint64_t ulen = (uint64_t)len;                      // 64-bit offsets: a crafted IFD offset must not wrap the bound checks
  const uint64_t ifd = r32(4);
  if (ifd + 2 > ulen) return 1;
  int n = r16((unsigned)ifd);
  for (int i = 0; i < n; i++) {
    const uint64_t e64 = ifd + 2 + 12ull * (uint64_t)i;
    if (e64 + 12 > ulen) return 1;
    const unsigned e = (unsigned)e64;
    if (r16(e) == 0x0112) { int v = r16(e + 8); return (v >= 1 && v <= 8) ? v : 1; }
  }
  return 1;
}

}  // namespace dalib200
#endif  // DALI_B200_CSRC_EXIF_H_
