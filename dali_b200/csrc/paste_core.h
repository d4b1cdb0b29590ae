// dali_b200/csrc/paste_core.h -- the per-thread bodies of fn.multi_paste and fn.paste (csrc/paste.cu), written as host/device
// functions so that tools/emul/paste_emul.cc and tools/emul/cuda_emul_stub.cc run the very code the device runs.
//
// The planner (csrc/paste_plan.h) sees each output as rows of W * C elements.  It cuts the rows into bands at the regions' y-edges; in
// a band every row is made of the same segments: sorted, disjoint and covering the row, each either a fill or a copy from one source
// sample.  A copy segment's source element at output row y and column col is base + y * pitch + col, so one segment serves every row
// of its band.  A row finds its band by a binary search over the output's bands and, inside the band, the segment at a column by a
// binary search over the band's segments: the device work per row does not depend on the number of regions beyond those two searches.
//
// The output of a sample is cut into 16-byte slots at 16-byte boundaries of the output address (a partial slot at each end).  A work
// item is kPsSlotsPerItem consecutive slots of one output; thread t takes slots t + k kPsThreads.  A full slot inside one row and one
// segment is a fill (one 16-byte store of a pre-rotated pattern, the table of csrc/erase_plan.h) or a copy: a same-type copy is one
// 16-byte store fed by one aligned 16-byte load, by two aligned loads and funnel shifts when both lie inside the segment's source run,
// and by element loads otherwise; a converting copy goes element by element through arith_core.h's ConvertSat.  A slot cut by a
// segment edge is assembled element by element in registers.  Partial slots and slots that cross a row end go element by element.
// Only the visible part of each region is read; every output element belongs to exactly one slot, so it is written once, and nothing
// depends on the rest of the batch.
#ifndef DALI_B200_CSRC_PASTE_CORE_H_
#define DALI_B200_CSRC_PASTE_CORE_H_

#include <stdint.h>
#include <string.h>
#include "host_device.h"
#include "arith_core.h"
#include "erase_core.h"

namespace dalib200 {

constexpr int kPsThreads = 256;
constexpr int kPsSlotsPerThread = 4;
constexpr int kPsSlotsPerItem = kPsThreads * kPsSlotsPerThread;   // 16 KiB of output per work item
constexpr int kPsMaxInputs = 64;

struct PsBand { int64_t row, off, cnt; };     // rows [row, next band's row); segments [off, off + cnt) of the output's list
// Elements [lo, next segment's lo) of a row y.  src < 0: the fill; else element base + y * pitch + col of source src (an index into
// the launch's table of input pointers).
struct PsSeg { int64_t lo, base, pitch; int32_t src, pad; };

struct PsSample {
  void *out;                                   // bound at launch
  const PsBand *bands; const PsSeg *segs;      // bound at launch: the output's bands and segments in the uploaded copy
  int64_t first_item, items;
  int64_t n, run;                              // elements, elements of a row (W * C)
  int32_t nbands, pad;
};

// What a launch shares: the input pointers, the fill table (erase_plan.h's ErFillTable, in the output type) and the types.
struct PsBatch {
  const void *const *srcs;
  const uint8_t *fill;
  int32_t nfill, in_type, out_type, pad;
};

// The segment of [j, e) that holds column col: the last one whose lo is at most col (segment j starts at or before col).
DB_HD int64_t ps_seg_at(const PsSeg *s, int64_t j, int64_t e, int64_t col) {
  e--;
  while (j < e) {
    const int64_t mid = (j + e + 1) >> 1;
    if (s[mid].lo <= col) j = mid; else e = mid - 1;
  }
  return j;
}

// The segments [*j, *e) of a row.
DB_HD void ps_row_segs(const PsSample &d, uint64_t row, int64_t *j, int64_t *e) {
  const PsBand &b = d.bands[last_at_most(d.bands, 0, d.nbands - 1, (int64_t)row, [](const PsBand &x) { return x.row; })];
  *j = b.off;
  *e = b.off + b.cnt;
}

// The fill of output element e: channel e mod C, since a row holds whole pixels.
template <int OSZ> DB_HD uint64_t ps_fill_elem(const PsBatch &B, int64_t e) {
  typedef typename ErElem<OSZ>::T T;
  T x;
  memcpy(&x, B.fill + (B.nfill == 1 ? 0 : (int64_t)((uint64_t)e % (uint64_t)B.nfill)) * OSZ, OSZ);
  return x;
}

// One output element's bits: the fill of its channel, or the source element (converted when CVT).
template <int OSZ, bool CVT> DB_HD uint64_t ps_elem(const PsBatch &B, const PsSeg &s, uint64_t row, int64_t col, int64_t e) {
  if (s.src < 0) return ps_fill_elem<OSZ>(B, e);
  const int64_t k = s.base + (int64_t)row * s.pitch + col;
  if (CVT) return arith_to_bits(arith_cast(arith_load(B.srcs[s.src], k, B.in_type), B.in_type, B.out_type), B.out_type);
  typedef typename ErElem<OSZ>::T T;
  return static_cast<const T *>(B.srcs[s.src])[k];
}

// Elements [lo, hi) of the output, one by one (partial slots and slots that cross a row end).
template <int OSZ, bool CVT> DB_HD void ps_elements(const PsSample &d, const PsBatch &B, int64_t lo, int64_t hi) {
  typedef typename ErElem<OSZ>::T T;
  uint64_t row = er_div((uint64_t)lo, (uint64_t)d.run);
  int64_t col = lo - (int64_t)row * d.run, j, je;
  ps_row_segs(d, row, &j, &je);
  j = ps_seg_at(d.segs, j, je, col);
  for (int64_t e = lo; e < hi; e++, col++) {
    if (col == d.run) {
      row++;
      col = 0;
      ps_row_segs(d, row, &j, &je);
    }
    while (j + 1 < je && d.segs[j + 1].lo <= col) j++;
    static_cast<T *>(d.out)[e] = (T)ps_elem<OSZ, CVT>(B, d.segs[j], row, col, e);
  }
}

// 16 source bytes at p, which is not 16-byte aligned, from the two aligned 16-byte words around them (device only).
#if defined(__CUDA_ARCH__)
__device__ __forceinline__ ErVec ps_load16_shifted(const uint8_t *p) {
  const uintptr_t a = (uintptr_t)p;
  const uint4 *q = reinterpret_cast<const uint4 *>(a & ~(uintptr_t)15);
  const uint4 v0 = __ldg(q), v1 = __ldg(q + 1);
  uint32_t w[8] = { v0.x, v0.y, v0.z, v0.w, v1.x, v1.y, v1.z, v1.w };
  const uint32_t sh = (uint32_t)(a & 15u), b = (sh & 3u) * 8u;
  if (sh & 8u) {
#pragma unroll
    for (int t = 0; t < 6; t++) w[t] = w[t + 2];
  }
  if (sh & 4u) {
#pragma unroll
    for (int t = 0; t < 5; t++) w[t] = w[t + 1];
  }
  ErVec r;
  r.w[0] = (uint64_t)__funnelshift_r(w[0], w[1], b) | (uint64_t)__funnelshift_r(w[1], w[2], b) << 32;
  r.w[1] = (uint64_t)__funnelshift_r(w[2], w[3], b) | (uint64_t)__funnelshift_r(w[3], w[4], b) << 32;
  return r;
}
#endif

// One 16-byte slot of the output.
template <int OSZ, bool CVT> DB_HD void ps_slot(const PsSample &d, const PsBatch &B, int64_t slot) {
  constexpr int V = 16 / OSZ;
  const int shift = (int)(((uintptr_t)d.out & 15) / OSZ);
  const int64_t e0 = slot * V - shift;
  if (e0 >= d.n) return;
  if (e0 < 0 || e0 + V > d.n) {
    ps_elements<OSZ, CVT>(d, B, e0 < 0 ? 0 : e0, e0 + V < d.n ? e0 + V : d.n);
    return;
  }
  const uint64_t row = er_div((uint64_t)e0, (uint64_t)d.run);
  const int64_t c0 = e0 - (int64_t)row * d.run;
  if (c0 + V > d.run) {
    ps_elements<OSZ, CVT>(d, B, e0, e0 + V);
    return;
  }
  int64_t j, je;
  ps_row_segs(d, row, &j, &je);
  j = ps_seg_at(d.segs, j, je, c0);
  uint8_t *const out = static_cast<uint8_t *>(d.out) + e0 * OSZ;
  const PsSeg &s = d.segs[j];
  const int64_t next = j + 1 < je ? d.segs[j + 1].lo : d.run;
  if (next >= c0 + V) {                                                   // one segment
    if (s.src < 0) {
      const uint8_t *const pat = B.fill + er_rot_off(B.nfill, OSZ);
      er_store16(out, er_load16(B.nfill == 1 ? pat : pat + (e0 % B.nfill) * 16));
      return;
    }
    if (!CVT) {
      const int64_t k0 = s.base + (int64_t)row * s.pitch;               // the source element of column 0
      const uint8_t *const sp = static_cast<const uint8_t *>(B.srcs[s.src]);
      const uint8_t *const in = sp + (k0 + c0) * OSZ;
      if ((((uintptr_t)in) & 15) == 0) {
        er_store16(out, er_load16(in));
        return;
      }
#if defined(__CUDA_ARCH__)
      // both aligned words inside the segment's source run [k0 + s.lo, k0 + next): no byte outside the visible region is read
      const uintptr_t w0 = (uintptr_t)in & ~(uintptr_t)15;
      if (w0 >= (uintptr_t)(sp + (k0 + s.lo) * OSZ) && w0 + 32 <= (uintptr_t)(sp + (k0 + next) * OSZ)) {
        er_store16(out, ps_load16_shifted(in));
        return;
      }
#else
      ErVec v;
      memcpy(&v, in, 16);
      er_store16(out, v);
      return;
#endif
    }
    ErVec v = {};
ER_PRAGMA(unroll)
    for (int k = 0; k < V; k++) er_put<OSZ>(v, k, ps_elem<OSZ, CVT>(B, s, row, c0 + k, e0 + k));
    er_store16(out, v);
    return;
  }
  ErVec v = {};                                                          // a segment edge inside the slot
ER_PRAGMA(unroll)
  for (int k = 0; k < V; k++) {
    while (j + 1 < je && d.segs[j + 1].lo <= c0 + k) j++;
    er_put<OSZ>(v, k, ps_elem<OSZ, CVT>(B, d.segs[j], row, c0 + k, e0 + k));
  }
  er_store16(out, v);
}

// Work item `local` of an output, as thread tid runs it.
template <int OSZ, bool CVT> DB_HD void ps_item(const PsSample &d, const PsBatch &B, int64_t local, int tid) {
ER_PRAGMA(unroll 1)
  for (int k = 0; k < kPsSlotsPerThread; k++) ps_slot<OSZ, CVT>(d, B, local * kPsSlotsPerItem + k * kPsThreads + tid);
}

}  // namespace dalib200

#endif  // DALI_B200_CSRC_PASTE_CORE_H_
