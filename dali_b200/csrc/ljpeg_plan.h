// dali_b200/csrc/ljpeg_plan.h -- plan set-up of a lossless JPEG (SOF3) sample: the checks of what the decoder takes, the device tables,
// the split of the scan into restart intervals, the LjpegImage record.  Plain C++: no per-sample work beyond the marker walk (jpeg.cu
// ParseHeaders) and the search for the restart markers.
#ifndef DALI_B200_CSRC_LJPEG_PLAN_H_
#define DALI_B200_CSRC_LJPEG_PLAN_H_
#include <stddef.h>
#include <string.h>
#include <string>
#include <vector>
#include "../../include/dali_b200.h"
#include "ljpeg_core.h"

namespace dalib200 {

// What the plan needs of the frame and its scan; filled from the parsed headers.
struct LjpegFrame {
  int width = 0, height = 0, ncomp = 0, precision = 0;
  int hs[4] = {0}, vs[4] = {0};
  int scan_ncomp = 0, td[4] = {0};              // td: the DC table of each scan component, in frame order
  bool scan_in_frame_order = false;             // the scan lists each frame component once, in frame order (T.81 B.2.3)
  int pred = 0, se = 0, ah = 0, pt = 0;         // Ss (predictor), Se, Ah, Al (point transform)
  int restart_interval = 0;
  bool jfif = false;
  int adobe_transform = -1;
  const uint8_t *bits[4] = {nullptr}, *vals[4] = {nullptr};   // DHT class 0 tables by id (bits[1..16]); null: not defined
};

// Builds the device table of a DHT table.  Returns false for a table libjpeg-turbo refuses (jpeg_make_d_derived_tbl: more than 256
// values, a code that does not fit its length, the all-ones code, or a value above 16).  The baseline path's tables (jpeg.cu
// BuildDeviceTable) cannot serve here: their entries keep the magnitude category in 4 bits, which folds category 16 onto 0.
inline bool BuildLjpegTable(const uint8_t *bits, const uint8_t *vals, LjpegTable &t) {
  memset(&t, 0, sizeof(t));
  int n = 0;
  for (int l = 1; l <= 16; l++) n += bits[l];
  if (n > 256) return false;
  for (int k = 0; k < n; k++) if (vals[k] > 16) return false;
  memcpy(t.vals, vals, n);
  int code = 0, k = 0;
  for (int l = 1; l <= 16; l++) {
    if (code + bits[l] > 1 << l) return false;  // the codes of length l would overflow it: checked before any LUT entry is written
    t.valoff[l] = k - code;
    for (int i = 0; i < bits[l]; i++, k++, code++)
      if (l <= kLjpegLutBits)
        for (int e = 0; e < 1 << (kLjpegLutBits - l); e++) t.lut[(code << (kLjpegLutBits - l)) + e] = (uint16_t)(l | (vals[k] << 8));
    if (code >= 1 << l) return false;           // the codes of length l overflow it (the all-ones code among them)
    t.maxcode[l] = code << (16 - l);
    code <<= 1;
  }
  return true;
}

// Checks a lossless frame and builds its image record (without the arena offsets and the window) and tables.  Returns a DALIB200
// status; `err` says why a stream is refused.
inline int PlanLjpegFrame(const LjpegFrame &f, LjpegImage *im, std::vector<LjpegTable> &tables, std::string *err) {
  auto fail = [&](int rc, const char *what) { *err = std::string("lossless JPEG: ") + what; return rc; };
  if (f.precision < 2 || f.precision > 16) return fail(DALIB200_ERROR_BAD_DATA, "sample precision outside 2..16");
  if (f.precision > 8) return fail(DALIB200_ERROR_UNSUPPORTED, "sample precision above 8 bits is not supported (no 16-bit output)");
  if (f.ncomp != 1 && f.ncomp != 3) return fail(DALIB200_ERROR_UNSUPPORTED, "only 1- or 3-component lossless JPEG is supported");
  for (int c = 0; c < f.ncomp; c++)
    if (f.hs[c] != 1 || f.vs[c] != 1) return fail(DALIB200_ERROR_UNSUPPORTED, "sampling factors other than 1x1 are not supported");
  if (f.scan_ncomp != f.ncomp) return fail(DALIB200_ERROR_UNSUPPORTED, "a lossless frame coded in more than one scan is not supported");
  if (!f.scan_in_frame_order) return fail(DALIB200_ERROR_BAD_DATA, "scan components out of frame order or repeated");
  if (f.pred < 1 || f.pred > 7 || f.se != 0 || f.ah != 0) return fail(DALIB200_ERROR_BAD_DATA, "bad predictor or scan parameters");
  if (f.pt >= f.precision) return fail(DALIB200_ERROR_BAD_DATA, "point transform not below the sample precision");
  if (f.ncomp == 3 && (f.jfif || f.adobe_transform > 0))
    return fail(DALIB200_ERROR_UNSUPPORTED, "colour-transformed (JFIF or Adobe YCbCr) lossless JPEG is not supported");
  if (f.restart_interval % f.width)
    return fail(DALIB200_ERROR_UNSUPPORTED, "a restart interval that is not a whole number of lines");
  memset(im, 0, sizeof(*im));
  im->width = f.width; im->height = f.height; im->ncomp = f.ncomp;
  im->precision = f.precision; im->pt = f.pt; im->pred = f.pred;
  for (int c = 0; c < f.ncomp; c++) {
    const int id = f.td[c];
    if (id > 3 || !f.bits[id]) return fail(DALIB200_ERROR_BAD_DATA, "missing Huffman table");
    LjpegTable t;
    if (!BuildLjpegTable(f.bits[id], f.vals[id], t)) return fail(DALIB200_ERROR_BAD_DATA, "bad Huffman table");
    im->table[c] = (int32_t)tables.size();
    tables.push_back(t);
  }
  return DALIB200_SUCCESS;
}

// Largest entropy-coded unit: the subsequence records hold 32-bit bit positions and symbol prefixes, and a chain walks at most
// kLjpegMaxChain subsequences.  A larger restart interval (or scan without restarts) is refused at plan set-up.
constexpr size_t kLjpegMaxUnitBytes = (size_t)kLjpegMaxChain << (kLjpegLog2Sub - 3);

// Splits the entropy-coded data [b, e) of a scan into its `nunits` restart intervals at the RSTn markers: exactly nunits byte ranges
// (an interval whose marker is missing is empty).  Returns true when the markers are out of sequence, missing or in excess.
inline bool SplitLjpegUnits(const uint8_t *d, size_t b, size_t e, int64_t nunits, std::vector<std::pair<size_t, size_t>> &out) {
  out.clear();
  bool bad = false;
  size_t begin = b;
  const uint8_t *q = d + b, *end = d + e;
  int next = 0;
  while (true) {
    const uint8_t *f = q < end ? static_cast<const uint8_t *>(memchr(q, 0xFF, end - q)) : nullptr;
    if (!f || f + 1 >= end) break;
    if (f[1] >= 0xD0 && f[1] <= 0xD7) {
      if ((int64_t)out.size() + 1 < nunits) out.emplace_back(begin, (size_t)(f - d));
      else bad = true;
      bad |= f[1] - 0xD0 != next;
      next = (next + 1) & 7;
      begin = (size_t)(f - d) + 2; q = f + 2;
    } else {
      q = f + 1;
    }
  }
  out.emplace_back(begin, e);
  if ((int64_t)out.size() < nunits) bad = true;
  while ((int64_t)out.size() < nunits) out.emplace_back(e, e);
  return bad;
}

}  // namespace dalib200
#endif  // DALI_B200_CSRC_LJPEG_PLAN_H_
