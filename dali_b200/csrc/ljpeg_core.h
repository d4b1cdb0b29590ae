// dali_b200/csrc/ljpeg_core.h -- lossless JPEG (SOF3, ITU-T T.81 Annex H) decoding written once for device and host: the descriptors
// the kernels of ljpeg.cu read, the Huffman symbol reader over the un-stuffed stream, and the per-thread bodies of the passes.
//
// The entropy-coded data of a lossless scan is a run of (category, extra bits) symbols, one per sample, the components interleaved
// (every Hi = Vi = 1).  The decode follows the baseline path's self-synchronising scheme (jpeg.cu, Weissenberger & Schmidt): every
// 2^kLjpegLog2Sub-bit subsequence of a unit (a restart interval, or the whole scan) is decoded speculatively from its first bit in
// component phase 0, and chains carry exit states to the right until they agree with what is already recorded.  The decoder state is
// only (bit position, component phase): a symbol never spans a block structure.
#ifndef DALI_B200_CSRC_LJPEG_CORE_H_
#define DALI_B200_CSRC_LJPEG_CORE_H_
#include <stdint.h>
#include "host_device.h"

namespace dalib200 {

constexpr int kLjpegLog2Sub = 10;              // subsequence: 1024 bits = 128 bytes of the clean stream
constexpr int kLjpegLutBits = 9;               // first-level lookup of the Huffman codes

// One DHT table as the device reads it.  lut[i] = code length | category << 8 for the codes of at most kLjpegLutBits bits that the
// left-aligned index i starts with, 0 for a longer code; maxcode[l] = (last code of length l + 1) << (16 - l), the exclusive bound of
// the left-aligned 16-bit codes of length l (T.81 F.2.2.3); valoff[l] = index of the first value of length l - its code.
struct LjpegTable {
  uint16_t lut[1 << kLjpegLutBits];
  int32_t maxcode[17], valoff[17];
  uint8_t vals[256];
};

struct LjpegImage {
  int32_t sample;                // batch index (status word)
  int32_t width, height, ncomp;  // ncomp: 1 or 3
  int32_t precision, pt, pred;   // P, point transform, predictor 1..7
  int32_t table[3];              // index into the table array, per component
  int32_t bad_rst;               // the restart markers are out of sequence, missing or in excess: the sample's status is set
  int64_t diff_off;              // int16 offset of the image's samples (H x W x ncomp, interleaved) in the difference arena
  // output, filled at launch: the window [win_x0, win_x0 + win_w) x [win_y0, win_y0 + win_h) goes to `out` as a tight win_h x win_w x C
  // buffer, C = 1 for GRAY, 3 for RGB / BGR
  uint8_t *out;
  int32_t win_x0, win_y0, win_w, win_h, out_type;
  int64_t first_px;              // prefix of window pixels over the lossless images
};

// One entropy-coded unit: a restart interval of whole lines, or the whole scan.  Its bytes are un-stuffed by the JPEG path's U1 - U3
// together with every other unit of the batch (JpegUnit `junit`).
struct LjpegUnit {
  int32_t junit;                 // index of the JpegUnit: clean stream offset and length
  int32_t image;                 // LjpegImage index
  int64_t first_sub;             // first global lossless subsequence
  int32_t nsub;                  // subsequences reserved (from the raw length; the clean stream may need fewer)
  uint32_t clean_off;            // byte offset of the clean stream (= the JpegUnit's)
  int64_t nsym;                  // symbols (samples) the unit must hold
  int64_t sym_off;               // int16 offset of its first sample in the difference arena
};

// Reconstruction work: the samples of one component of the lines [y0, y1) of an image (a restart band, or the whole image).
struct LjpegBand { int32_t image, comp, y0, y1; };

// What the kernels of ljpeg.cu read (LjpegStage::Enqueue, ljpeg.h).
struct LjpegLaunch {
  const LjpegImage *d_images; int nimages;
  const LjpegUnit *d_units; int nunits;
  const LjpegTable *d_tables;
  const LjpegBand *d_bands; int nbands;
  int64_t total_sub;                 // subsequences of all units (LjpegUnit::first_sub is their prefix)
  int64_t total_px;                  // window pixels of all images (LjpegImage::first_px is their prefix)
  const uint8_t *d_clean;            // the batch's clean streams and their lengths (per JpegUnit)
  const uint32_t *d_unit_clean_len;
  uint64_t *d_rec;                   // total_sub records
  uint32_t *d_first;                 // total_sub first-symbol indices
  int16_t *d_diff;                   // the difference arena, reconstructed in place
  int32_t *d_status;
};

// ---- the subsequence record: [31:0] exit bit position, [33:32] component phase, [44:34] symbols that start in the subsequence,
// [63:45] priority = distance of the chain that wrote it from the chain's origin (see ljpeg_walk)
constexpr uint64_t kLjpegStateMask = (1ull << 34) - 1;
constexpr uint32_t kLjpegMaxChain = (1u << 19) - 1;
DB_HD uint64_t ljpeg_pack(uint32_t pos, int phase, uint32_t cnt, uint32_t prio) {
  return (uint64_t)pos | ((uint64_t)(uint32_t)phase << 32) | ((uint64_t)(cnt & 2047u) << 34) | ((uint64_t)prio << 45);
}
DB_HD uint32_t ljpeg_count(uint64_t r) { return (uint32_t)(r >> 34) & 2047u; }

// 32 bits of the clean stream at bit `pos`.  The clean stream is word-swapped (jpeg.cu unstuff_scatter): a 32-bit load is big-endian.
DB_HD uint32_t ljpeg_peek(const uint32_t *w, uint32_t pos) {
  const uint32_t i = pos >> 5, s = pos & 31u;
  const uint64_t v = ((uint64_t)w[i] << 32) | w[i + 1];
  return (uint32_t)((v << s) >> 32);
}

// Decodes the symbol at the top of `hi`: returns the bits it takes (code + extra bits) and its difference in `diff`.  A code that no
// table entry matches takes 16 bits with difference 0 and sets `bad` (a speculative decode meets those all the time; only the write
// pass reports them).  Category 16 is 32768 with no extra bits (T.81 H.1.2.2), stored as the int16 -32768 (the same modulo 2^16).
DB_HD uint32_t ljpeg_symbol(const LjpegTable &t, uint32_t hi, int32_t &diff, bool &bad) {
  uint32_t e = t.lut[hi >> (32 - kLjpegLutBits)];
  if (e == 0) {
    const int32_t code16 = (int32_t)(hi >> 16);
    int l = kLjpegLutBits + 1;
    while (l <= 16 && code16 >= t.maxcode[l]) l++;
    if (l > 16) { diff = 0; bad = true; return 16; }
    e = (uint32_t)l | ((uint32_t)t.vals[(t.valoff[l] + (code16 >> (16 - l))) & 0xFF] << 8);
  }
  const uint32_t len = e & 0xFFu, cat = e >> 8;
  if (cat == 0) { diff = 0; return len; }
  if (cat >= 16) { diff = -32768; return len; }
  const uint32_t bits = (hi << len) >> (32u - cat);               // len + cat <= 31
  diff = bits >> (cat - 1) ? (int32_t)bits : (int32_t)bits - (int32_t)((1u << cat) - 1u);
  return len + cat;
}

// Decodes the symbols that START before bit `end` from (pos, phase): advances them and counts the symbols.  No output: the
// synchronisation passes only need the state.
DB_HD void ljpeg_span(const uint32_t *w, const LjpegTable *const *tab, int ncomp, uint32_t &pos, int &phase, uint32_t end,
                         uint32_t &cnt) {
  bool bad = false;
  while (pos < end) {
    int32_t d;
    pos += ljpeg_symbol(*tab[phase], ljpeg_peek(w, pos), d, bad);
    phase = phase + 1 == ncomp ? 0 : phase + 1;
    cnt++;
  }
}

// Geometry of one subsequence.
struct LjpegSub { const uint32_t *w; uint32_t jl, nsub_eff, clean_bits; };
DB_HD LjpegSub ljpeg_sub(const LjpegUnit &u, int64_t g, const uint8_t *clean, const uint32_t *unit_clean_len) {
  LjpegSub s;
  s.w = reinterpret_cast<const uint32_t *>(clean + u.clean_off);
  s.jl = (uint32_t)(g - u.first_sub);
  s.clean_bits = unit_clean_len[u.junit] * 8u;
  s.nsub_eff = (s.clean_bits + (1u << kLjpegLog2Sub) - 1) >> kLjpegLog2Sub;
  return s;
}

// L1 + L2a, one thread per subsequence g of unit u: the speculative decode of g from its first bit in phase 0, then the chain that
// carries its exit state to the right.  Every visit publishes (state, symbol count) with a max on the record, priority in the top bits,
// BEFORE comparing with the record it replaced:
//   * the old record has a higher priority: a chain that started further left has been here; this one stops;
//   * the old state equals the new one: synchronised, everything to the right was decoded from this state; the chain stops;
//   * otherwise the chain moves on to the next subsequence with priority + 1.
// The chain of the unit's first subsequence starts from the true state and has the highest priority everywhere, so every record ends up
// written by a chain that entered the subsequence in its true state, whatever the order in which the threads run.  `atomic_max`
// returns the old value.
template <class AtomicMax>
DB_HD void ljpeg_walk(const LjpegImage &im, const LjpegUnit &u, int64_t g, const uint8_t *clean, const uint32_t *unit_clean_len,
                         const LjpegTable *tables, uint64_t *rec, AtomicMax atomic_max) {
  const LjpegSub s = ljpeg_sub(u, g, clean, unit_clean_len);
  if (s.jl >= s.nsub_eff) return;
  const LjpegTable *tab[3] = { tables + im.table[0], tables + im.table[im.ncomp > 1 ? 1 : 0], tables + im.table[im.ncomp > 2 ? 2 : 0] };
  uint32_t pos = s.jl << kLjpegLog2Sub, jl = s.jl;
  int phase = 0;
  for (uint32_t prio = 0;; prio++) {
    uint32_t cnt = 0;
    const uint32_t end = (jl + 1) << kLjpegLog2Sub;
    ljpeg_span(s.w, tab, im.ncomp, pos, phase, end < s.clean_bits ? end : s.clean_bits, cnt);
    const uint64_t nr = ljpeg_pack(pos, phase, cnt, prio);
    const uint64_t old = atomic_max(rec + u.first_sub + jl, nr);
    if (prio > 0 && (uint32_t)(old >> 45) >= prio) break;
    if (prio > 0 && ((old ^ nr) & kLjpegStateMask) == 0) break;
    if (jl + 1 >= s.nsub_eff || prio >= kLjpegMaxChain) break;
    jl++;
  }
}

// L3, one thread per subsequence: decodes it from its true entry state and writes the differences of its symbols (first symbol index
// `first`, the exclusive scan of the counts) into the arena.  Symbols at or past the unit's sample count are the pad bits behind the
// data.  Returns true when a code of the unit's data matches no table entry.
DB_HD bool ljpeg_write(const LjpegImage &im, const LjpegUnit &u, int64_t g, const uint8_t *clean, const uint32_t *unit_clean_len,
                          const LjpegTable *tables, const uint64_t *rec, uint32_t first, int16_t *diff) {
  const LjpegSub s = ljpeg_sub(u, g, clean, unit_clean_len);
  if (s.jl >= s.nsub_eff) return false;
  const LjpegTable *tab[3] = { tables + im.table[0], tables + im.table[im.ncomp > 1 ? 1 : 0], tables + im.table[im.ncomp > 2 ? 2 : 0] };
  uint32_t pos = 0;
  int phase = 0;
  if (s.jl > 0) { const uint64_t r = rec[g - 1]; pos = (uint32_t)r; phase = (int)((r >> 32) & 3u); }
  uint32_t end = (s.jl + 1) << kLjpegLog2Sub;
  if (end > s.clean_bits) end = s.clean_bits;
  bool bad = false;
  int16_t *out = diff + u.sym_off;
  for (int64_t k = first; pos < end && k < u.nsym; k++) {
    int32_t d;
    bool b = false;
    pos += ljpeg_symbol(*tab[phase], ljpeg_peek(s.w, pos), d, b);
    bad |= b;
    phase = phase + 1 == im.ncomp ? 0 : phase + 1;
    out[k] = (int16_t)d;
  }
  return bad;
}

// L4 step: the prediction of sample (x, y) of a component (T.81 H.1.2.1; libjpeg-turbo jdpred.c).  The first line of the scan and of
// every restart band is predicted by 2^(P - Pt - 1) at x = 0 and by Ra behind it; the first column of every other line by Rb.  Ra, Rb
// and Rc are reconstructed values in [0, 65535]; the caller adds the difference modulo 2^16.
DB_HD int32_t ljpeg_predict(int pred, bool first_line, int x, int32_t init, int32_t Ra, int32_t Rb, int32_t Rc) {
  if (first_line) return x == 0 ? init : Ra;
  if (x == 0) return Rb;
  switch (pred) {
    case 1: return Ra;
    case 2: return Rb;
    case 3: return Rc;
    case 4: return Ra + Rb - Rc;
    case 5: return Ra + ((Rb - Rc) >> 1);
    case 6: return Rb + ((Ra - Rc) >> 1);
    default: return (Ra + Rb) >> 1;
  }
}

// L5: one pixel of the window: the reconstructed samples << Pt, kept to 8 bits as libjpeg-turbo's JSAMPLE cast keeps them.  One
// component: GRAY, or the sample replicated for RGB / BGR.  Three components: R, G, B as stored; GRAY by `gray` (the baseline path's
// rule for an RGB JPEG).
template <class Gray>
DB_HD void ljpeg_pixel(const LjpegImage &im, const int16_t *diff, int64_t e, Gray gray) {
  const int lx = (int)(e % im.win_w), ly = (int)(e / im.win_w);
  const int64_t s = ((int64_t)(im.win_y0 + ly) * im.width + im.win_x0 + lx) * im.ncomp;
  const int sh = im.pt;
  const int r = ((uint16_t)diff[im.diff_off + s] << sh) & 0xFF;
  const int g = im.ncomp == 3 ? ((uint16_t)diff[im.diff_off + s + 1] << sh) & 0xFF : r;
  const int b = im.ncomp == 3 ? ((uint16_t)diff[im.diff_off + s + 2] << sh) & 0xFF : r;
  if (im.out_type == 2 /* DALIB200_GRAY */) { im.out[e] = (uint8_t)(im.ncomp == 3 ? gray(r, g, b) : r); return; }
  uint8_t *o = im.out + 3 * e;
  const bool bgr = im.out_type == 1 /* DALIB200_BGR */;
  o[0] = (uint8_t)(bgr ? b : r); o[1] = (uint8_t)g; o[2] = (uint8_t)(bgr ? r : b);
}

}  // namespace dalib200
#endif  // DALI_B200_CSRC_LJPEG_CORE_H_
