// dali_b200/csrc/equalize_core.h -- the per-thread bodies of fn.experimental.equalize (csrc/equalize.cu), written as host/device
// functions so that tools/emul/equalize_emul.cc and tools/emul/cuda_emul_stub.cc run the very code the device runs.
//
// A sample is F frames of frame_bytes = H * W * C bytes; a plane is the H * W pixels of one (frame, channel).  Byte f of a frame belongs
// to channel (f / stride) % C, with stride 1 for channel-last layouts and H * W for CHW.  Each frame is cut into work items of
// kEqChunk bytes; an item never crosses a frame.  Two kernels:
//   HIST   counts the item's bytes into private bins in shared memory (one set of C x 256 bins per group of warps, `nsub` sets), then
//          adds the non-zero bins to the frame's u32 histogram in global memory with integer atomics.  Each thread keeps up to four
//          runs of equal bins in registers (one per channel modulo 4) and adds a run when it ends, so a flat image costs one shared
//          atomic per run instead of one per byte, and the lanes of a warp do not all queue on one address.
//   APPLY  builds the look-up tables of the item's frame in shared memory straight from the global histogram (one warp per channel:
//          a lane scans 8 bins), then maps the item's bytes through them.
// Both read the item with 16-byte vector loads between a scalar head and tail, so any byte offset of the input and output works.
// The histogram is integer, so the output is exact and the same alone or in any batch, whatever order the atomics land in.
#ifndef DALI_B200_CSRC_EQUALIZE_CORE_H_
#define DALI_B200_CSRC_EQUALIZE_CORE_H_

#include <stdint.h>
#include <string.h>
#include <math.h>
#include "host_device.h"

namespace dalib200 {

constexpr int kEqThreads = 256;
constexpr int64_t kEqChunk = 32768;           // bytes of one work item
constexpr int kEqMaxChannels = 16;            // planner limit on C (DESIGN.md section 2)
constexpr int kEqSmemWords = 8192;            // private bins of the histogram kernel: 32 KiB
constexpr int kEqMaxSub = kEqThreads / 32;    // at most one set of private bins per warp

struct EqSample {
  const uint8_t *in; uint8_t *out;            // bound at launch
  int64_t frame_bytes;                        // H * W * C
  int64_t first_item, items, ipf;             // items = frames * ipf (items per frame)
  int64_t hist_off;                           // u32 index of the sample's first bin in the batch histogram (frame-major, C x 256 per frame)
  uint32_t plane;                             // H * W, pixels of one plane (< 2^31)
  uint32_t stride;                            // 1 (channel-last) or H * W (CHW)
  int32_t C, nsub;                            // channels; sets of private bins of the histogram kernel (warp w uses set w % nsub)
  uint32_t skip_cb;                           // (kEqSkip % C) * 256: the channel step of eq_skip when stride is 1
};

// The bytes [b0, b0 + len) of frame `frame` that work item `local` of the sample covers.
struct EqItem { int64_t frame, b0; uint32_t len; };

DB_HD EqItem eq_item(const EqSample &d, int64_t local) {
  EqItem it;
  it.frame = local / d.ipf;
  it.b0 = (local - it.frame * d.ipf) * kEqChunk;
  const int64_t rest = d.frame_bytes - it.b0;
  it.len = (uint32_t)(rest < kEqChunk ? rest : kEqChunk);
  return it;
}

// The channel of a byte as `cb` = channel * 256 and its position `r` inside the current run of `stride` bytes of that channel.
struct EqCursor { uint32_t cb, r; };

DB_HD EqCursor eq_cursor(const EqSample &d, int64_t f) {   // byte f of a frame; 32-bit division where it fits
  uint64_t q;
  EqCursor u;
  if (((uint64_t)f >> 32) == 0) {
    q = (uint32_t)f / d.stride;
    u.r = (uint32_t)f - (uint32_t)q * d.stride;
  } else {
    q = (uint64_t)f / d.stride;
    u.r = (uint32_t)((uint64_t)f - q * d.stride);
  }
  u.cb = (uint32_t)((q >> 32) == 0 ? (uint32_t)q % (uint32_t)d.C : q % (uint32_t)d.C) << 8;
  return u;
}
DB_HD void eq_advance(const EqSample &d, EqCursor &u) {
  if (++u.r == d.stride) {
    u.r = 0;
    u.cb += 256;
    if (u.cb == (uint32_t)d.C << 8) u.cb = 0;
  }
}
// From the byte after one thread's vector to the start of its next one, kEqSkip bytes on: no division.
constexpr uint32_t kEqSkip = kEqThreads * 16 - 16;
DB_HD void eq_skip(const EqSample &d, EqCursor &u) {
  const uint32_t cend = (uint32_t)d.C << 8;
  if (d.stride == 1) {
    u.cb += d.skip_cb;
    if (u.cb >= cend) u.cb -= cend;
    return;
  }
  u.r += kEqSkip;
  while (u.r >= d.stride) {
    u.r -= d.stride;
    u.cb += 256;
    if (u.cb == cend) u.cb = 0;
  }
}

DB_HD void eq_add(uint32_t *h, uint32_t k, uint32_t v) {
#ifdef __CUDA_ARCH__
  atomicAdd(h + k, v);
#else
  h[k] += v;
#endif
}

// Up to four open runs of one thread: run s holds bin key[s] (channel * 256 + value) of a channel c with c % 4 == s.
struct EqRuns { uint32_t key[4], cnt[4]; };

DB_HD void eq_runs_init(EqRuns &s) {
  for (int k = 0; k < 4; k++) { s.key[k] = 0xFFFFFFFFu; s.cnt[k] = 0; }
}
DB_HD void eq_runs_count(EqRuns &s, uint32_t *h, uint32_t bin) {
  const uint32_t slot = (bin >> 8) & 3;
#ifdef __CUDA_ARCH__
#pragma unroll
#endif
  for (uint32_t k = 0; k < 4; k++) {      // constant indices once unrolled: the runs stay in registers
    if (k != slot) continue;
    if (s.key[k] == bin) { s.cnt[k]++; continue; }
    if (s.cnt[k]) eq_add(h, s.key[k], s.cnt[k]);
    s.key[k] = bin;
    s.cnt[k] = 1;
  }
}
DB_HD void eq_runs_flush(EqRuns &s, uint32_t *h) {
  for (int k = 0; k < 4; k++)
    if (s.cnt[k]) eq_add(h, s.key[k], s.cnt[k]);
}

DB_HD void eq_count_word(const EqSample &d, EqCursor &u, EqRuns &s, uint32_t *h, uint32_t w) {
  for (int b = 0; b < 4; b++) {
    eq_runs_count(s, h, u.cb + ((w >> (8 * b)) & 255u));
    eq_advance(d, u);
  }
}

// 16 bytes at a 16-byte aligned address, as four little-endian words
DB_HD void eq_load16(const uint8_t *p, uint32_t w[4]) {
#ifdef __CUDA_ARCH__
  const uint4 x = __ldg(reinterpret_cast<const uint4 *>(p));
  w[0] = x.x; w[1] = x.y; w[2] = x.z; w[3] = x.w;
#else
  memcpy(w, p, 16);
#endif
}
DB_HD void eq_store16(uint8_t *q, const uint32_t y[4]) {
#ifdef __CUDA_ARCH__
  *reinterpret_cast<uint4 *>(q) = make_uint4(y[0], y[1], y[2], y[3]);
#else
  memcpy(q, y, 16);
#endif
}

// The bytes of `len` at address p before its first 16-byte boundary.
DB_HD uint32_t eq_head(const void *p, uint32_t len) {
  const uint32_t h = (uint32_t)((16 - ((uintptr_t)p & 15)) & 15);
  return h < len ? h : len;
}

// HIST, thread `tid` of the item: counts its bytes into `h`, the C x 256 private bins of the thread's set.
DB_HD void eq_hist_thread(const EqSample &d, int64_t local, uint32_t *h, int tid) {
  const EqItem it = eq_item(d, local);
  const uint8_t *p = d.in + it.frame * d.frame_bytes + it.b0;
  const uint32_t head = eq_head(p, it.len), nvec = (it.len - head) / 16, tail = head + nvec * 16;
  EqRuns s;
  eq_runs_init(s);
  if ((uint32_t)tid < head) eq_runs_count(s, h, eq_cursor(d, it.b0 + tid).cb + p[tid]);
  if (tail + tid < it.len) eq_runs_count(s, h, eq_cursor(d, it.b0 + tail + tid).cb + p[tail + tid]);
  EqCursor u = eq_cursor(d, it.b0 + head + 16 * (int64_t)tid);
  for (uint32_t v = tid; v < nvec; v += kEqThreads) {
    uint32_t w[4];
    eq_load16(p + head + 16 * v, w);
    for (int k = 0; k < 4; k++) eq_count_word(d, u, s, h, w[k]);
    eq_skip(d, u);
  }
  eq_runs_flush(s, h);
}

// HIST, after the item: thread `tid` adds bins tid, tid + kEqThreads, ... of the `nsub` private sets to the frame's histogram.
DB_HD void eq_hist_flush(const EqSample &d, int64_t local, const uint32_t *sh, uint32_t *hist, int tid) {
  const uint32_t nb = (uint32_t)d.C * 256;
  uint32_t *g = hist + d.hist_off + eq_item(d, local).frame * nb;
  for (uint32_t b = tid; b < nb; b += kEqThreads) {
    uint32_t v = 0;
    for (int k = 0; k < d.nsub; k++) v += sh[k * nb + b];
    if (v) eq_add(g, b, v);
  }
}

// ---- the look-up table of one plane: cv2.equalizeHist's, exactly.  i = the first non-zero bin; if hist[i] == total the plane is
// flat and maps to itself; else lut[i] = 0 and lut[k > i] = sat_u8(rint_even((float)sum_k * (255.f / (float)(total - hist[i])))), with
// sum_k = hist[i + 1] + ... + hist[k], every operation correctly rounded fp32.
DB_HD float eq_scale(uint32_t total, uint32_t hfirst) {
#ifdef __CUDA_ARCH__
  return __fdiv_rn(255.0f, __int2float_rn((int)(total - hfirst)));
#else
  return 255.0f / (float)(int)(total - hfirst);
#endif
}
DB_HD uint8_t eq_lut_value(uint32_t sum, float scale) {
#ifdef __CUDA_ARCH__
  const int q = __float2int_rn(__fmul_rn(__int2float_rn((int)sum), scale));
#else
  const int q = (int)nearbyintf((float)(int)sum * scale);   // the default rounding mode: to nearest, ties to even
#endif
  return (uint8_t)(q < 0 ? 0 : q > 255 ? 255 : q);
}

// Lane `lane` (0-31) of the warp that builds a plane's table writes entries 8 lane ... 8 lane + 7.  h: the plane's 256 bins; first,
// hfirst: the first non-zero bin and its count; cum: the sum of the bins before 8 lane.
DB_HD void eq_lut_lane(const uint32_t *h, int lane, uint32_t first, uint32_t hfirst, uint32_t total, uint32_t cum, uint8_t *lut) {
  const bool flat = hfirst == total;
  const float scale = flat ? 0.0f : eq_scale(total, hfirst);
  for (uint32_t k = 8 * lane; k < 8 * (uint32_t)lane + 8; k++) {
    cum += h[k];
    lut[k] = flat ? (uint8_t)k : k <= first ? 0 : eq_lut_value(cum - hfirst, scale);
  }
}

// The first non-zero bin among the 8 of a lane, or 8.
DB_HD uint32_t eq_first_in_lane(const uint32_t *h, int lane) {
  uint32_t k = 0;
  while (k < 8 && h[8 * lane + k] == 0) k++;
  return k;
}

// The warp's scan run lane by lane: the table of one plane of `total` (> 0) pixels.
DB_HD void eq_lut_plane(const uint32_t *h, uint32_t total, uint8_t *lut) {
  uint32_t first = 0;
  while (h[first] == 0) first++;
  uint32_t cum = 0;
  for (int lane = 0; lane < 32; lane++) {
    eq_lut_lane(h, lane, first, h[first], total, cum, lut);
    for (int k = 0; k < 8; k++) cum += h[8 * lane + k];
  }
}

// ---- APPLY, thread `tid` of the item: maps its bytes through `lut` (C x 256 entries).  The 16-byte vectors follow the output's
// alignment; they are loaded as vectors too when the input shares it, else byte by byte.
DB_HD void eq_apply_thread(const EqSample &d, int64_t local, const uint8_t *lut, int tid) {
  const EqItem it = eq_item(d, local);
  const int64_t off = it.frame * d.frame_bytes + it.b0;
  const uint8_t *p = d.in + off;
  uint8_t *q = d.out + off;
  const uint32_t head = eq_head(q, it.len), nvec = (it.len - head) / 16, tail = head + nvec * 16;
  if ((uint32_t)tid < head) q[tid] = lut[eq_cursor(d, it.b0 + tid).cb + p[tid]];
  if (tail + tid < it.len) q[tail + tid] = lut[eq_cursor(d, it.b0 + tail + tid).cb + p[tail + tid]];
  const bool vec_in = (((uintptr_t)p ^ (uintptr_t)q) & 15) == 0;
  EqCursor u = eq_cursor(d, it.b0 + head + 16 * (int64_t)tid);
  for (uint32_t v = tid; v < nvec; v += kEqThreads) {
    const uint32_t o = head + 16 * v;
    uint32_t w[4];
    if (vec_in) {
      eq_load16(p + o, w);
    } else {
      for (int k = 0; k < 4; k++)
        w[k] = (uint32_t)p[o + 4 * k] | (uint32_t)p[o + 4 * k + 1] << 8 | (uint32_t)p[o + 4 * k + 2] << 16 | (uint32_t)p[o + 4 * k + 3] << 24;
    }
    uint32_t y[4];
    for (int k = 0; k < 4; k++) {
      y[k] = 0;
      for (int b = 0; b < 4; b++) {
        y[k] |= (uint32_t)lut[u.cb + ((w[k] >> (8 * b)) & 255u)] << (8 * b);
        eq_advance(d, u);
      }
    }
    eq_store16(q + o, y);
    eq_skip(d, u);
  }
}

}  // namespace dalib200

#endif  // DALI_B200_CSRC_EQUALIZE_CORE_H_
