// dali_b200/csrc/jpeg_prog_plan.h -- host-side planning of a multi-scan JPEG -- PROGRESSIVE (SOF2), or a sequential frame (SOF0 / SOF1)
// whose components are coded in separate scans: the marker walk over the whole stream (the
// Huffman tables may be redefined between scans), one ProgScan per SOS with the table snapshot it decodes with, the extent of its
// entropy-coded bytes, and the dependency wave it runs in.  Plain C++ (no CUDA types): jpeg.cu calls it from JpegPlanSetup,
// tools/emul/jpeg_prog_emul.cc from the CPU emulation test.
//
// T.81 Annex B (markers), G.1 (progression rules); table derivation after libjpeg jdhuff.c jpeg_make_d_derived_tbl.
#ifndef DALI_B200_CSRC_JPEG_PROG_PLAN_H_
#define DALI_B200_CSRC_JPEG_PROG_PLAN_H_
#include <algorithm>
#include <cstring>
#include <map>
#include <string>
#include <vector>
#include "jpeg_prog_core.h"

namespace dalib200 {

namespace progdetail {
struct RawHuff { uint8_t bits[17]; uint8_t vals[256]; bool present = false; };

inline bool DeriveTable(const RawHuff &r, ProgHuff *t) {
  memset(t, 0, sizeof(*t));
  int size[257], code_of[257], n = 0;
  for (int l = 1; l <= 16; l++) for (int i = 0; i < r.bits[l]; i++) { if (n >= 256) return false; size[n++] = l; }
  int code = 0, si = n ? size[0] : 0, p = 0;
  while (p < n) {
    while (p < n && size[p] == si) code_of[p++] = code++;
    if (code > (1 << si)) return false;           // codes of this length exhausted: not a prefix code
    code <<= 1; si++;
  }
  p = 0;
  for (int l = 1; l <= 16; l++) {
    if (r.bits[l]) { t->valoffset[l] = p - code_of[p]; p += r.bits[l]; t->maxcode[l] = code_of[p - 1]; }
    else t->maxcode[l] = -1;
  }
  t->maxcode[0] = -1;
  t->maxcode[17] = 0xFFFFF;
  p = 0;
  for (int l = 1; l <= 8; l++)
    for (int i = 0; i < r.bits[l]; i++, p++) {
      const int first = code_of[p] << (8 - l);
      for (int k = 0; k < (1 << (8 - l)); k++) t->look[first + k] = (uint16_t)((l << 8) | r.vals[p]);
    }
  memcpy(t->vals, r.vals, 256);
  return true;
}
inline int Rd16(const uint8_t *p) { return (p[0] << 8) | p[1]; }
}  // namespace progdetail

// Walks stream[0, n).  `base`: file offset the scans' data_off are relative to (the first scan's data = what the decoder stages).
// Fills im's geometry (not coef_off / raw_off / sample), appends the scans (image index = `image`) and the derived tables (deduplicated
// through `table_cache`).  Returns 0, or DALIB200_ERROR_BAD_DATA / _UNSUPPORTED with *err.
inline int PlanProgressive(const uint8_t *d, size_t n, size_t base, int image, ProgImage *im, std::vector<ProgScan> &scans,
                           std::vector<ProgHuff> &huff, std::map<std::string, int> &table_cache, std::string *err) {
  using namespace progdetail;
  auto bad = [&](const char *m) { if (err) *err = m; return DALIB200_ERROR_BAD_DATA; };
  auto unsup = [&](const char *m) { if (err) *err = m; return DALIB200_ERROR_UNSUPPORTED; };
  if (n < 4 || d[0] != 0xFF || d[1] != 0xD8) return bad("not a JPEG stream (missing SOI)");
  RawHuff dc[4], ac[4];
  int width = 0, height = 0, ncomp = 0, cid[4] = { 0 }, hs[4] = { 0 }, vs[4] = { 0 }, hmax = 1, vmax = 1;
  bool got_sof = false, sequential = false;
  int dri = 0;
  const size_t first_scan = scans.size();
  int coef_bits[4][64];                              // libjpeg's coef_bits: the Al each coefficient has reached, -1 = never sent
  for (auto &cb : coef_bits) for (int &v : cb) v = -1;
  size_t pos = 2;
  auto table_index = [&](const RawHuff &r, int *idx) {
    if (!r.present) return false;
    std::string key(reinterpret_cast<const char *>(r.bits), 17);
    key.append(reinterpret_cast<const char *>(r.vals), 256);
    auto it = table_cache.find(key);
    if (it == table_cache.end()) {
      ProgHuff t;
      if (!DeriveTable(r, &t)) return false;
      huff.push_back(t);
      it = table_cache.emplace(key, (int)huff.size() - 1).first;
    }
    *idx = it->second;
    return true;
  };
  while (pos + 4 <= n) {
    if (d[pos] != 0xFF) return bad("JPEG: marker expected");
    while (pos < n && d[pos] == 0xFF) pos++;
    if (pos >= n) break;
    const int m = d[pos++];
    if (m == 0xD8 || (m >= 0xD0 && m <= 0xD7) || m == 0x01 || m == 0x00) continue;
    if (m == 0xD9) break;
    if (pos + 2 > n) break;
    const int L = Rd16(d + pos);
    if (L < 2 || pos + L > n) {
      if (scans.size() > first_scan) break;        // cut off between two scans: decode what is there, reported as incomplete below
      return bad("JPEG: truncated segment");
    }
    const uint8_t *s = d + pos + 2;
    const int sl = L - 2;
    if (m == 0xC4) {
      int o = 0;
      while (o < sl) {
        if (o + 17 > sl) return bad("JPEG: bad DHT");
        const int tc = s[o] >> 4, th = s[o] & 15; o++;
        if (th > 3 || tc > 1) return bad("JPEG: bad DHT id");
        RawHuff &h = tc ? ac[th] : dc[th];
        int cnt = 0; h.bits[0] = 0;
        for (int i = 1; i <= 16; i++) { h.bits[i] = s[o++]; cnt += h.bits[i]; }
        if (cnt > 256 || o + cnt > sl) return bad("JPEG: bad DHT counts");
        memset(h.vals, 0, sizeof(h.vals));
        memcpy(h.vals, s + o, cnt); o += cnt;
        h.present = true;
      }
    } else if (m == 0xC2 || m == 0xC0 || m == 0xC1) {
      if (got_sof) return bad("JPEG: two frame headers");
      sequential = m != 0xC2;                          // a sequential frame coded in several scans (one per component)
      if (sl < 6) return bad("JPEG: bad SOF");
      height = Rd16(s + 1); width = Rd16(s + 3); ncomp = s[5];
      if (s[0] != 8) return unsup("only 8-bit JPEG is supported");
      if ((ncomp != 1 && ncomp != 3 && ncomp != 4) || sl < 6 + 3 * ncomp) return unsup("only 1-, 3- or 4-component JPEG is supported");
      for (int c = 0; c < ncomp; c++) {
        cid[c] = s[6 + 3 * c]; hs[c] = s[7 + 3 * c] >> 4; vs[c] = s[7 + 3 * c] & 15;
        if (hs[c] < 1 || hs[c] > 4 || vs[c] < 1 || vs[c] > 4) return bad("JPEG: bad sampling factors");
      }
      if (ncomp == 1) hs[0] = vs[0] = 1;                     // a single component is never interleaved
      for (int c = 0; c < ncomp; c++) { hmax = std::max(hmax, hs[c]); vmax = std::max(vmax, vs[c]); }
      if (width == 0 || height == 0) return bad("JPEG: zero image size");
      got_sof = true;
    } else if (m == 0xDD) {
      if (sl >= 2) dri = Rd16(s);
    } else if (m == 0xDA) {
      if (!got_sof) return bad("JPEG: SOS before SOF");
      if (sl < 1) return bad("JPEG: bad SOS");
      ProgScan sc;
      memset(&sc, 0, sizeof(sc));
      sc.ncomp = s[0];
      if (sc.ncomp < 1 || sc.ncomp > 4 || sl < 4 + 2 * sc.ncomp) return bad("JPEG: bad SOS");
      int td[4], ta[4];
      for (int i = 0; i < sc.ncomp; i++) {
        int ci = -1;
        for (int c = 0; c < ncomp; c++) if (cid[c] == s[1 + 2 * i]) ci = c;
        if (ci < 0) return bad("JPEG: SOS references an unknown component");
        for (int k = 0; k < i; k++) if (sc.comp[k] == ci) return bad("JPEG: SOS names a component twice");
        sc.comp[i] = ci; td[i] = s[2 + 2 * i] >> 4; ta[i] = s[2 + 2 * i] & 15;
        if (td[i] > 3 || ta[i] > 3) return bad("JPEG: bad Huffman table id");
      }
      const uint8_t *t = s + 1 + 2 * sc.ncomp;
      sc.ss = t[0]; sc.se = t[1]; sc.ah = t[2] >> 4; sc.al = t[2] & 15;
      // G.1.1.1: DC scans carry Ss = Se = 0 and may interleave components; AC scans one component, 1 <= Ss <= Se <= 63; a refinement
      // scan sends exactly the next lower bit
      if (sequential) {
        if (sc.ss != 0 || sc.se != 63 || sc.ah != 0 || sc.al != 0) return bad("JPEG: bad scan parameters in a sequential frame");
        sc.seq = 1;
      } else {
        if (sc.ss > sc.se || sc.se > 63 || sc.al > 13 || sc.ah > 13) return bad("JPEG: bad progression parameters");
        if (sc.ss == 0 ? sc.se != 0 : sc.ncomp != 1) return bad("JPEG: bad progression parameters");
        if (sc.ah != 0 && sc.ah != sc.al + 1) return bad("JPEG: bad successive approximation");
      }
      if (sc.ncomp != 1 && sc.ncomp != ncomp) return unsup("scans that interleave a subset of the components are not supported");
      for (int i = 0; i < sc.ncomp; i++) {
        if (sc.seq) { if (!table_index(dc[td[i]], &sc.dc_tbl[i]) || !table_index(ac[ta[i]], &sc.seq_ac_tbl[i])) return bad("JPEG: missing or invalid Huffman table"); }
        else if (sc.ss == 0) { if (sc.ah == 0 && !table_index(dc[td[i]], &sc.dc_tbl[i])) return bad("JPEG: missing or invalid Huffman table"); }
        else if (!table_index(ac[ta[i]], &sc.ac_tbl)) return bad("JPEG: missing or invalid Huffman table");
      }
      for (int i = 0; i < sc.ncomp; i++) for (int k = sc.ss; k <= sc.se; k++) coef_bits[sc.comp[i]][k] = sc.al;
      sc.image = image;
      sc.restart_interval = dri;
      // entropy-coded bytes: up to the first FF that is followed by neither 00 nor RSTn
      size_t b = pos + L, e = b;
      for (;;) {
        const uint8_t *f = e < n ? static_cast<const uint8_t *>(memchr(d + e, 0xFF, n - e)) : nullptr;
        if (!f) { e = n; break; }
        e = f - d;
        if (e + 1 >= n) { e = n; break; }
        if (d[e + 1] == 0 || (d[e + 1] >= 0xD0 && d[e + 1] <= 0xD7)) { e += 2; continue; }
        break;
      }
      if (b < base) return bad("JPEG: internal scan offset");
      if (e - b >= (1ull << 32) || b - base >= (1ull << 32)) return unsup("scans of 4 GiB or more are not supported");
      sc.data_off = (uint32_t)(b - base); sc.data_len = (uint32_t)(e - b);
      if (scans.size() - first_scan >= 1024) return unsup("more than 1024 scans");
      scans.push_back(sc);
      pos = e;
      continue;
    } else if (m >= 0xC0 && m <= 0xCF && m != 0xC4 && m != 0xC8 && m != 0xCC) {
      return unsup("not a Huffman-coded DCT JPEG (lossless / arithmetic / hierarchical)");
    }
    pos += L;
  }
  if (!got_sof) return bad("JPEG: no frame header found");
  if (scans.size() == first_scan) return bad("JPEG: no scan found");
  // waves: a scan waits for every earlier scan that shares a component AND a coefficient with it
  for (size_t i = first_scan; i < scans.size(); i++) {
    int w = 0;
    for (size_t k = first_scan; k < i; k++) {
      const ProgScan &a = scans[k], &b = scans[i];
      if (a.se < b.ss || b.se < a.ss) continue;
      bool share = false;
      for (int x = 0; x < a.ncomp; x++) for (int y = 0; y < b.ncomp; y++) share |= a.comp[x] == b.comp[y];
      if (share) w = std::max(w, a.wave + 1);
    }
    scans[i].wave = w;
  }
  // geometry
  im->ncomp = ncomp;
  im->mcux = (width + 8 * hmax - 1) / (8 * hmax);
  im->mcuy = (height + 8 * vmax - 1) / (8 * vmax);
  int bpm = 0;
  for (int c = 0; c < 4; c++) { im->hs[c] = im->vs[c] = 1; im->blk0[c] = 0; im->wblk[c] = im->hblk[c] = 0; }
  for (int c = 0; c < ncomp; c++) {
    im->hs[c] = hs[c]; im->vs[c] = vs[c];
    im->blk0[c] = bpm;
    bpm += hs[c] * vs[c];
    const int cw = (width * hs[c] + hmax - 1) / hmax, ch = (height * vs[c] + vmax - 1) / vmax;
    im->wblk[c] = (cw + 7) / 8; im->hblk[c] = (ch + 7) / 8;
  }
  im->bpm = bpm;
  im->incomplete = 0;                                // a stream that stops before every coefficient has its last bit decodes, with a status
  for (int c = 0; c < ncomp; c++) for (int k = 0; k < 64; k++) im->incomplete |= coef_bits[c][k] != 0;
  return DALIB200_SUCCESS;
}

}  // namespace dalib200
#endif  // DALI_B200_CSRC_JPEG_PROG_PLAN_H_
