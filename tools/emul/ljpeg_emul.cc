// tools/emul/ljpeg_emul.cc -- TEST INFRASTRUCTURE.  Runs the lossless JPEG decode of the product on the host.
//
// The planner (dali_b200/csrc/ljpeg_plan.h) is plain C++ and the kernels of ljpeg.cu are thin wrappers around the host/device bodies of
// ljpeg_core.h.  This file compiles them with the host compiler and runs them the way a launch does, so that tests/test_ljpeg_cpu.py can
// compare the decode with the encoder's samples and cv2.imdecode on a machine without a GPU, and run mutated streams under ASan +
// UBSan.  The marker walk below stands in for jpeg.cu ParseHeaders (which the host fuzzer covers through the library); the un-stuffing
// stands in for U1 - U3 and writes each unit's clean stream, word-swapped, into a heap buffer of exactly the size and zero pad the plan
// gives it on the device: any read past it is a sanitizer report.  The chains of ljpeg_sync run in REVERSE subsequence order, so that a
// result that depended on the order in which the device's threads run would show up here.
//   g++ -std=c++17 -O2 -ffp-contract=off -shared -fPIC -I/usr/local/cuda/include tools/emul/ljpeg_emul.cc
#include <algorithm>
#include <cstdlib>
#include <string>
#include <vector>
#include "../../dali_b200/csrc/jpeg_recon.h"
#include "../../dali_b200/csrc/ljpeg_plan.h"

using namespace dalib200;

namespace {
constexpr uint32_t kPad = 32;                      // jpeg_recon.h kCleanPad: zero bytes behind every clean stream
inline int rd16(const uint8_t *p) { return (p[0] << 8) | p[1]; }

// the marker walk of ParseHeaders, reduced to what a lossless frame needs.  Returns a DALIB200 status.
int Walk(const uint8_t *p, size_t n, LjpegFrame &f, size_t &scan_begin, int &ncomp_sof) {
  if (n < 4 || p[0] != 0xFF || p[1] != 0xD8) return DALIB200_ERROR_BAD_DATA;
  int cid[4] = {0};
  bool sof = false;
  for (size_t pos = 2; pos + 4 <= n;) {
    if (p[pos] != 0xFF) return DALIB200_ERROR_BAD_DATA;
    while (pos < n && p[pos] == 0xFF) pos++;
    if (pos >= n) break;
    const int m = p[pos++];
    if (m == 0xD8 || (m >= 0xD0 && m <= 0xD7) || m == 0x01) continue;
    if (m == 0xD9 || pos + 2 > n) break;
    const int L = rd16(p + pos);
    if (L < 2 || pos + L > n) return DALIB200_ERROR_BAD_DATA;
    const uint8_t *s = p + pos + 2;
    const int sl = L - 2;
    if (m == 0xC4) {
      for (int o = 0; o < sl;) {
        if (o + 17 > sl) return DALIB200_ERROR_BAD_DATA;
        const int tc = s[o] >> 4, th = s[o] & 15;
        if (th > 3 || tc > 1) return DALIB200_ERROR_BAD_DATA;
        int cnt = 0;
        for (int i = 1; i <= 16; i++) cnt += s[o + i];
        if (cnt > 256 || o + 17 + cnt > sl) return DALIB200_ERROR_BAD_DATA;
        if (tc == 0) { f.bits[th] = s + o; f.vals[th] = s + o + 17; }    // the counts are bits[1..16], as HostHuff keeps them
        o += 17 + cnt;
      }
    } else if (m == 0xC3) {
      if (sl < 6) return DALIB200_ERROR_BAD_DATA;
      f.precision = s[0]; f.height = rd16(s + 1); f.width = rd16(s + 3); f.ncomp = ncomp_sof = s[5];
      if (f.ncomp < 1 || f.ncomp > 4 || sl < 6 + 3 * f.ncomp) return DALIB200_ERROR_BAD_DATA;
      for (int c = 0; c < f.ncomp; c++) {
        cid[c] = s[6 + 3 * c]; f.hs[c] = s[7 + 3 * c] >> 4; f.vs[c] = s[7 + 3 * c] & 15;
        if (f.hs[c] < 1 || f.hs[c] > 4 || f.vs[c] < 1 || f.vs[c] > 4) return DALIB200_ERROR_BAD_DATA;
      }
      sof = true;
    } else if ((m >= 0xC0 && m <= 0xCF) && m != 0xC4 && m != 0xC8 && m != 0xCC) {
      return DALIB200_ERROR_UNSUPPORTED;         // another coding process: not this decoder's business here
    } else if (m == 0xDD) {
      if (sl >= 2) f.restart_interval = rd16(s);
    } else if (m == 0xE0) {
      if (sl >= 5 && !memcmp(s, "JFIF\0", 5)) f.jfif = true;
    } else if (m == 0xEE) {
      if (sl >= 12 && !memcmp(s, "Adobe", 5)) f.adobe_transform = s[11];
    } else if (m == 0xDA) {
      if (!sof || sl < 1) return DALIB200_ERROR_BAD_DATA;
      f.scan_ncomp = s[0];
      if (f.scan_ncomp < 1 || f.scan_ncomp > 4 || sl < 1 + 2 * f.scan_ncomp) return DALIB200_ERROR_BAD_DATA;
      f.scan_in_frame_order = true;
      for (int i = 0; i < f.scan_ncomp; i++) {
        int ci = -1;
        for (int c = 0; c < f.ncomp; c++) if (cid[c] == s[1 + 2 * i]) ci = c;
        if (ci < 0) return DALIB200_ERROR_BAD_DATA;
        f.td[ci] = s[2 + 2 * i] >> 4;
        f.scan_in_frame_order &= ci == i;
      }
      if (sl >= 4 + 2 * f.scan_ncomp) {
        const uint8_t *t = s + 1 + 2 * f.scan_ncomp;
        f.pred = t[0]; f.se = t[1]; f.ah = t[2] >> 4; f.pt = t[2] & 15;
      } else {
        f.se = 63;
      }
      scan_begin = pos + L;
      break;
    }
    pos += L;
  }
  if (!sof || f.width == 0 || f.height == 0 || !scan_begin) return DALIB200_ERROR_BAD_DATA;
  return DALIB200_SUCCESS;
}
}  // namespace

// info: { width, height, components, units }.  out (width * height * C, C = 1 for out_type GRAY, else 3) may be NULL: plan only.
// Returns the planner's DALIB200 status (non-zero: rejected at plan set-up), or -1 when the device stage sets the sample's status.
extern "C" int emul_ljpeg_decode(const uint8_t *data, size_t len, int out_type, uint8_t *out, int *info) {
  LjpegFrame f;
  size_t sb = 0;
  int nc = 0;
  int rc = Walk(data, len, f, sb, nc);
  if (rc) return rc;
  LjpegImage im;
  std::vector<LjpegTable> tables;
  std::string err;
  if ((rc = PlanLjpegFrame(f, &im, tables, &err))) return rc;
  if ((int64_t)f.width * f.height >= (1ll << 31)) return DALIB200_ERROR_UNSUPPORTED;
  size_t se = len;
  if (se >= sb + 2 && data[se - 2] == 0xFF && data[se - 1] == 0xD9) se -= 2;
  const int W = f.width, H = f.height, C = f.ncomp;
  const int lines = f.restart_interval ? f.restart_interval / W : H;
  const int nunits = (H + lines - 1) / lines;
  std::vector<std::pair<size_t, size_t>> segs;
  im.bad_rst = SplitLjpegUnits(data, sb, se, nunits, segs);
  for (const auto &sg : segs) if (sg.second - sg.first > kLjpegMaxUnitBytes) return DALIB200_ERROR_UNSUPPORTED;
  info[0] = W; info[1] = H; info[2] = C; info[3] = nunits;
  if (!out) return 0;
  // U1 - U3: one clean stream per unit, FF 00 -> FF, word-swapped, zero-padded; each in a buffer of its own
  std::vector<uint8_t *> clean(nunits);
  std::vector<uint32_t> clean_len(nunits);
  std::vector<LjpegUnit> units(nunits);
  int64_t sub = 0;
  for (int k = 0; k < nunits; k++) {
    const size_t b = segs[k].first, e = segs[k].second, raw_len = e - b;
    const size_t alloc = (raw_len + kPad + 15) & ~(size_t)15;
    clean[k] = static_cast<uint8_t *>(calloc(alloc, 1));
    uint32_t q = 0;
    for (size_t i = b; i < e; i++) {
      if (i > b && data[i] == 0 && data[i - 1] == 0xFF) continue;
      clean[k][q ^ 3u] = data[i];
      q++;
    }
    clean_len[k] = q;
    LjpegUnit &u = units[k];
    u.junit = k; u.image = 0; u.first_sub = sub; u.clean_off = 0;
    u.nsub = (int32_t)((raw_len + (1u << (kLjpegLog2Sub - 3)) - 1) >> (kLjpegLog2Sub - 3));
    const int y0 = k * lines, y1 = std::min(H, y0 + lines);
    u.nsym = (int64_t)(y1 - y0) * W * C;
    u.sym_off = (int64_t)y0 * W * C;
    sub += u.nsub;
  }
  std::vector<uint64_t> rec(sub + 1, 0);
  std::vector<uint32_t> first(sub + 1, 0);
  int16_t *diff = static_cast<int16_t *>(malloc(sizeof(int16_t) * (size_t)W * H * C));
  int status = im.bad_rst ? -1 : 0;
  auto amax = [](uint64_t *p, uint64_t v) { const uint64_t o = *p; if (v > o) *p = v; return o; };
  // ljpeg_sync: every subsequence, last first
  for (int64_t g = sub - 1; g >= 0; g--) {
    int k = nunits - 1;
    while (units[k].first_sub > g) k--;
    ljpeg_walk(im, units[k], g, clean[k], clean_len.data(), tables.data(), rec.data(), amax);
  }
  // ljpeg_scan
  for (int k = 0; k < nunits; k++) {
    const LjpegUnit &u = units[k];
    const uint32_t nsub = (clean_len[k] * 8u + (1u << kLjpegLog2Sub) - 1) >> kLjpegLog2Sub;
    uint32_t run = 0;
    for (uint32_t i = 0; i < nsub; i++) { first[u.first_sub + i] = run; run += ljpeg_count(rec[u.first_sub + i]); }
    if ((int64_t)run < u.nsym) status = -1;
    for (int64_t s = run; s < u.nsym; s++) diff[u.sym_off + s] = 0;
  }
  // ljpeg_write, in reverse order too
  for (int64_t g = sub - 1; g >= 0; g--) {
    int k = nunits - 1;
    while (units[k].first_sub > g) k--;
    if (ljpeg_write(im, units[k], g, clean[k], clean_len.data(), tables.data(), rec.data(), first[g], diff)) status = -1;
  }
  // ljpeg_recon: the wavefront's dependencies hold in raster order; each band of each component from its first line
  const int32_t init = 1 << (im.precision - im.pt - 1);
  for (int k = 0; k < nunits; k++)
    for (int c = 0; c < C; c++) {
      const int y0 = k * lines, y1 = std::min(H, y0 + lines);
      for (int y = y0; y < y1; y++)
        for (int x = 0; x < W; x++) {
          auto at = [&](int yy, int xx) -> int16_t & { return diff[((int64_t)yy * W + xx) * C + c]; };
          const bool fl = y == y0;
          const int32_t Ra = x ? (uint16_t)at(y, x - 1) : 0, Rb = fl ? 0 : (uint16_t)at(y - 1, x), Rc = fl || !x ? 0 : (uint16_t)at(y - 1, x - 1);
          at(y, x) = (int16_t)((at(y, x) + ljpeg_predict(im.pred, fl, x, init, Ra, Rb, Rc)) & 0xFFFF);
        }
    }
  // ljpeg_color
  im.out = out; im.out_type = out_type; im.win_x0 = 0; im.win_y0 = 0; im.win_w = W; im.win_h = H; im.diff_off = 0;
  for (int64_t e = 0; e < (int64_t)W * H; e++)
    ljpeg_pixel(im, diff, e, [](int r, int g, int b) { return RgbJpegGray(r, g, b); });
  free(diff);
  for (uint8_t *c : clean) free(c);
  return status;
}
