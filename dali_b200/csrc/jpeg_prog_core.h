// dali_b200/csrc/jpeg_prog_core.h -- entropy decoding of PROGRESSIVE (SOF2) JPEG scans, written once for device and host.
//
// A progressive stream is a sequence of scans, each a Huffman-coded pass over one band [Ss, Se] of the coefficients of one component
// (AC) or over the DC coefficients of several (T.81 Annex G): first passes send the bits above Al, refinement passes one more bit.  A
// refinement pass is decoded relative to the coefficients already there, so a scan cannot be entered in the middle the way the
// baseline decoder's self-synchronising subsequences are; what IS independent are scans that touch different components or different
// bands.  The planner (jpeg_prog_plan.h) sorts the scans of every image into dependency waves; the device runs one wave per launch, one
// warp (one working lane) per scan: prog_decode_scan() below.  The same function compiled by a host compiler is what
// tools/emul/jpeg_prog_emul.cc runs to pin it against libjpeg-turbo's output without a GPU (tests/test_jpeg_prog_cpu.py).
//
// Follows libjpeg's jdphuff.c (decode_mcu_DC_first / AC_first / DC_refine / AC_refine, process_restart), the decoder behind the
// reference's nvimgcodec CPU backend; bit reader and table layout after jdhuff.c (jpeg_make_d_derived_tbl, 8-bit look-ahead).
#ifndef DALI_B200_CSRC_JPEG_PROG_CORE_H_
#define DALI_B200_CSRC_JPEG_PROG_CORE_H_
#include <stdint.h>
#include "host_device.h"

namespace dalib200 {

struct ProgHuff {              // one Huffman table
  uint16_t look[256];          // (length << 8) | symbol for codes of at most 8 bits, 0 = longer
  int32_t maxcode[18];         // largest code of each length (-1: none); [17] = sentinel above every 16-bit code
  int32_t valoffset[17];       // symbol index = code + valoffset[length]
  uint8_t vals[256];
};

struct ProgScan {
  uint32_t data_off, data_len; // entropy-coded bytes of the scan, relative to the image's staged bytes (up to the next non-RST marker)
  int32_t image;               // index into the ProgImage array
  int32_t ncomp, comp[4];      // components of the scan (frame component indices)
  int32_t dc_tbl[4], ac_tbl;   // indices into the ProgHuff array (DC scans: per component; AC scans: ac_tbl)
  int32_t seq_ac_tbl[4];       // sequential scans (below): the AC table of each component
  int32_t seq;                 // 1: a scan of a SEQUENTIAL (SOF0 / SOF1) frame that is coded in several scans: whole blocks, DC + AC
  int32_t ss, se, ah, al;
  int32_t restart_interval;    // MCUs of THIS scan between restart markers, 0 = none
  int32_t wave;
};

struct ProgImage {
  int64_t coef_off;            // int16 offset of the image's coefficients: block b at coef_off + 64 b, blocks in MCU order
  int64_t raw_off;             // byte offset of the image's staged bytes
  int32_t sample;              // batch index (status word)
  int32_t incomplete;          // the stream ends before the progression is complete (scans missing): reported like a truncation
  int32_t ncomp, mcux, mcuy, bpm;
  int32_t hs[4], vs[4];
  int32_t blk0[4];             // first block of the component inside an MCU (blocks of a component: v-major, h fastest)
  int32_t wblk[4], hblk[4];    // blocks per row / column of the component in a single-component scan: ceil(component extent / 8)
};

#if defined(__CUDACC__)
__device__ const uint8_t d_prog_natural[64] = {
   0,  1,  8, 16,  9,  2,  3, 10, 17, 24, 32, 25, 18, 11,  4,  5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13,  6,  7, 14, 21, 28,
  35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63 };
#endif
static const uint8_t h_prog_natural[64] = {
   0,  1,  8, 16,  9,  2,  3, 10, 17, 24, 32, 25, 18, 11,  4,  5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13,  6,  7, 14, 21, 28,
  35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63 };
// zig-zag index -> natural index; a run past 63 (corrupt data) lands on 63, as on the guard entries of libjpeg's jpeg_natural_order
DB_HD int prog_natural(int k) {
  if (k > 63) k = 63;
#if defined(__CUDA_ARCH__)
  return d_prog_natural[k];
#else
  return h_prog_natural[k];
#endif
}

// Bit reader over the stuffed bytes of one scan (jdhuff.c jpeg_fill_bit_buffer): FF 00 is a data byte FF; any other FF xx is a marker --
// the reader stops there and supplies zero bits, remembering that it ran dry (libjpeg: insufficient_data).
struct ProgBits {
  const uint8_t *p, *end;
  uint32_t acc;                // the window: `nbits` bits at the top, the last `pad` of them zero padding supplied in place of data
  int nbits, pad;
  bool dry;                    // padding has been CONSUMED (the window is filled ahead of use: merely touching the end is not an error)
};
DB_HD void pb_fill(ProgBits &b) {
  while (b.nbits <= 24) {
    uint32_t v = 0;
    bool real = false;
    if (b.p < b.end) {
      v = *b.p;
      if (v != 0xFF) { b.p++; real = true; }
      else if (b.p + 1 < b.end && b.p[1] == 0) { b.p += 2; real = true; }
      else v = 0;                                           // marker (or a lone FF at the end): stay in front of it
    }
    if (!real) b.pad += 8;
    b.acc |= v << (24 - b.nbits);
    b.nbits += 8;
  }
}
DB_HD void pb_drop(ProgBits &b, int n) {
  b.acc <<= n; b.nbits -= n;
  if (b.nbits < b.pad) { b.dry = true; b.pad = b.nbits > 0 ? b.nbits : 0; }
}
DB_HD int pb_get(ProgBits &b, int n) {                      // 0 <= n <= 16
  if (n == 0) return 0;
  if (b.nbits < n) pb_fill(b);
  const int v = (int)(b.acc >> (32 - n));
  pb_drop(b, n);
  return v;
}
DB_HD int pb_huff(ProgBits &b, const ProgHuff &h) {         // jdhuff.c HUFF_DECODE + jpeg_huff_decode
  if (b.nbits < 17) pb_fill(b);
  const uint32_t e = h.look[b.acc >> 24];
  if (e) { pb_drop(b, (int)(e >> 8)); return (int)(e & 255u); }
  int l = 9;
  int32_t code = (int32_t)(b.acc >> 23);
  while (code > h.maxcode[l]) { l++; code = (int32_t)(b.acc >> (32 - l)); }
  pb_drop(b, l);
  if (l > 16) return 0;                                     // garbage: libjpeg warns and uses symbol 0
  return h.vals[(code + h.valoffset[l]) & 255];
}
DB_HD int pb_extend(int v, int s) { return v < (1 << (s - 1)) ? v - (1 << s) + 1 : v; }      // HUFF_EXTEND, s >= 1

// jdphuff.c process_restart: drop the partial byte, step over the RSTn marker, reset the predictors
DB_HD void pb_restart(ProgBits &b) {
  b.acc = 0; b.nbits = 0; b.pad = 0; b.dry = false;
  while (b.p + 1 < b.end) {
    if (b.p[0] == 0xFF && b.p[1] >= 0xD0 && b.p[1] <= 0xD7) { b.p += 2; return; }
    b.p++;
  }
  b.p = b.end;
}

// arena block of block (bx, by) of component c in a single-component scan / of block k of MCU m in an interleaved scan
DB_HD int64_t prog_block_single(const ProgImage &im, int c, int bx, int by) {
  const int mx = bx / im.hs[c], my = by / im.vs[c];
  return ((int64_t)my * im.mcux + mx) * im.bpm + im.blk0[c] + (by % im.vs[c]) * im.hs[c] + (bx % im.hs[c]);
}

// Decodes one scan into the image's coefficient blocks (natural order inside a block; slot 0 holds the ABSOLUTE DC value while the
// scans run).  Returns 0, or 1 when the data ran out before the scan was complete (the remaining blocks keep what they had).
DB_HD int prog_decode_scan(const ProgScan &s, const ProgImage &im, const ProgHuff *huff, const uint8_t *raw, int16_t *coef_arena) {
  ProgBits b;
  b.p = raw + im.raw_off + s.data_off; b.end = b.p + s.data_len; b.acc = 0; b.nbits = 0; b.pad = 0; b.dry = false;
  int16_t *coef = coef_arena + im.coef_off;
  const bool single = s.ncomp == 1;
  const int c0 = s.comp[0];
  const int mcus_x = single ? im.wblk[c0] : im.mcux, mcus_y = single ? im.hblk[c0] : im.mcuy;
  const int64_t nmcu = (int64_t)mcus_x * mcus_y;
  int last_dc[4] = { 0, 0, 0, 0 };
  uint32_t eobrun = 0;
  int to_restart = s.restart_interval;
  bool insufficient = false;
  int truncated = 0;
  const int p1 = 1 << s.al, m1 = -(1 << s.al);
  int mx = 0, my = 0;
  for (int64_t m = 0; m < nmcu; m++) {
    if (s.restart_interval) {
      if (to_restart == 0) {
        pb_restart(b);
        last_dc[0] = last_dc[1] = last_dc[2] = last_dc[3] = 0;
        eobrun = 0; insufficient = false;
        to_restart = s.restart_interval;
      }
      to_restart--;
    }
    if (!insufficient) {
      if (s.seq) {                                           // ---- sequential scan (jdhuff.c decode_mcu): whole blocks
        for (int ci = 0; ci < s.ncomp; ci++) {
          const int c = s.comp[ci];
          const int nb = single ? 1 : im.hs[c] * im.vs[c];
          const ProgHuff &hd = huff[s.dc_tbl[ci]], &ha = huff[s.seq_ac_tbl[ci]];
          for (int k = 0; k < nb; k++) {
            const int64_t blk = single ? prog_block_single(im, c, mx, my) : m * im.bpm + im.blk0[c] + k;
            int16_t *q = coef + blk * 64;
            int t = pb_huff(b, hd) & 15;
            if (t) t = pb_extend(pb_get(b, t), t);
            last_dc[ci] += t;
            q[0] = (int16_t)last_dc[ci];
            for (int z = 1; z < 64; z++) {
              int rs = pb_huff(b, ha);
              const int r = rs >> 4;
              rs &= 15;
              if (rs) {
                z += r;
                q[prog_natural(z)] = (int16_t)pb_extend(pb_get(b, rs), rs);
              } else if (r == 15) {
                z += 15;
              } else {
                break;
              }
            }
          }
        }
      } else if (s.ss == 0) {                                // ---- DC scans: every block of the MCU
        for (int ci = 0; ci < s.ncomp; ci++) {
          const int c = s.comp[ci];
          const int nb = single ? 1 : im.hs[c] * im.vs[c];
          for (int k = 0; k < nb; k++) {
            const int64_t blk = single ? prog_block_single(im, c, mx, my) : m * im.bpm + im.blk0[c] + k;
            int16_t *q = coef + blk * 64;
            if (s.ah == 0) {                                 // decode_mcu_DC_first
              int t = pb_huff(b, huff[s.dc_tbl[ci]]) & 15;  // a DC symbol is a size category
              if (t) t = pb_extend(pb_get(b, t), t);
              last_dc[ci] += t;
              q[0] = (int16_t)((uint32_t)last_dc[ci] << s.al);
            } else if (pb_get(b, 1)) {                       // decode_mcu_DC_refine
              q[0] = (int16_t)(q[0] | p1);
            }
          }
        }
      } else {                                               // ---- AC scans: one block
        int16_t *q = coef + prog_block_single(im, c0, mx, my) * 64;
        const ProgHuff &h = huff[s.ac_tbl];
        if (s.ah == 0) {                                     // decode_mcu_AC_first
          if (eobrun > 0) eobrun--;
          else {
            for (int k = s.ss; k <= s.se; k++) {
              int t = pb_huff(b, h);
              const int r = t >> 4;
              t &= 15;
              if (t) {
                k += r;
                const int v = pb_extend(pb_get(b, t), t);
                q[prog_natural(k)] = (int16_t)((uint32_t)v << s.al);
              } else if (r == 15) {
                k += 15;
              } else {
                eobrun = 1u << r;
                if (r) eobrun += (uint32_t)pb_get(b, r);
                eobrun--;
                break;
              }
            }
          }
        } else {                                             // decode_mcu_AC_refine
          int k = s.ss;
          if (eobrun == 0) {
            for (; k <= s.se; k++) {
              int t = pb_huff(b, h);
              int r = t >> 4;
              t &= 15;
              if (t) {
                t = pb_get(b, 1) ? p1 : m1;                  // the size must be 1: a newly nonzero coefficient is +-1 << Al
              } else if (r != 15) {
                eobrun = 1u << r;
                if (r) eobrun += (uint32_t)pb_get(b, r);
                break;                                       // the rest of the block is handled by the EOB logic below
              }
              // step over already-nonzero coefficients (each takes a correction bit) and r still-zero ones
              do {
                int16_t *tc = q + prog_natural(k);
                if (*tc != 0) {
                  if (pb_get(b, 1) && (*tc & p1) == 0) *tc = (int16_t)(*tc >= 0 ? *tc + p1 : *tc + m1);
                } else if (--r < 0) {
                  break;
                }
                k++;
              } while (k <= s.se);
              if (t) q[prog_natural(k)] = (int16_t)t;
            }
          }
          if (eobrun > 0) {
            for (; k <= s.se; k++) {
              int16_t *tc = q + prog_natural(k);
              if (*tc != 0 && pb_get(b, 1) && (*tc & p1) == 0) *tc = (int16_t)(*tc >= 0 ? *tc + p1 : *tc + m1);
            }
            eobrun--;
          }
        }
      }
      if (b.dry) { insufficient = true; truncated = 1; }    // zero bits were supplied: the following MCUs are skipped (jdphuff.c)
    }
    if (++mx == mcus_x) { mx = 0; my++; }
  }
  return truncated;
}

// After the last wave: slot 0 of every block holds the absolute DC.  The IDCT stage takes the DC from the decoder's compact per-block
// array, in which dc_scan_kernel (jpeg.cu) accumulates differences component by component in MCU order; this writes the difference
// of block `blk` (index inside the image) to its predecessor in exactly that order, so that the shared stage can stay as it is.
DB_HD void prog_dc_difference(const ProgImage &im, const int16_t *coef_arena, int16_t *dc_arena, int64_t blk) {
  const int64_t m = blk / im.bpm;
  const int b = (int)(blk - m * im.bpm);
  int c = 0;
  while (c + 1 < im.ncomp && b >= im.blk0[c + 1]) c++;
  const int nb = im.hs[c] * im.vs[c], j = b - im.blk0[c];
  int prev = 0;
  if (j > 0) prev = coef_arena[im.coef_off + (blk - 1) * 64];
  else if (m > 0) prev = coef_arena[im.coef_off + ((m - 1) * im.bpm + im.blk0[c] + nb - 1) * 64];
  dc_arena[im.coef_off / 64 + blk] = (int16_t)(coef_arena[im.coef_off + blk * 64] - prev);
}

}  // namespace dalib200
#endif  // DALI_B200_CSRC_JPEG_PROG_CORE_H_
