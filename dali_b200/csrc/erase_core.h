// dali_b200/csrc/erase_core.h -- the per-thread bodies of fn.erase (csrc/erase.cu), written as host/device functions so that
// tools/emul/erase_emul.cc and tools/emul/cuda_emul_stub.cc run the very code the device runs.
//
// The planner (csrc/erase_plan.h) reduces a sample to rows x an inner run: the run is the innermost erased axis merged with every
// axis after it, the rows are the axes before it.  Whether a row is covered by a region depends only on the row's coordinates on the
// erased outer axes; their row-major index is the row's key.  The planner cuts the key space into bands in which the covered
// intervals of the run do not change, and gives each band its sorted, disjoint interval list.  A row finds its band by a binary
// search over the sample's bands and, inside the band, the interval at a column by a binary search over the band's intervals: the
// device work per row does not depend on the number of regions beyond those two searches.
//
// The output of a sample is cut into 16-byte slots at 16-byte boundaries of the output address (a partial slot at each end).  A
// work item is kErSlotsPerItem consecutive slots of one sample; thread t takes slots t + k kErThreads.  A full slot inside one row
// is copied (one 16-byte load and store when input and output are aligned alike, else element loads and one 16-byte store), filled
// (one 16-byte store of a pre-built pattern) or, where an interval edge falls inside it, assembled element by element; input
// elements inside the erased union are never read.  Partial slots and slots that cross a row end go element by element.  Every
// output element belongs to exactly one slot, so it is written once, and nothing depends on the rest of the batch.
#ifndef DALI_B200_CSRC_ERASE_CORE_H_
#define DALI_B200_CSRC_ERASE_CORE_H_

#include <stdint.h>
#include <string.h>
#include "host_device.h"

namespace dalib200 {

constexpr int kErThreads = 256;
constexpr int kErSlotsPerThread = 4;
constexpr int kErSlotsPerItem = kErThreads * kErSlotsPerThread;   // 16 KiB of output per work item
constexpr int kErMaxDim = 6;

struct ErBand { int64_t key, off, cnt; };  // keys [key, next band's key); intervals [off, off + cnt) of the sample's list
struct ErIval { int64_t lo, hi; };         // elements [lo, hi) of the inner run

struct ErSample {
  const void *in; void *out;                 // bound at launch
  const ErBand *bands; const ErIval *ivals;  // bound at launch: the sample's bands and intervals in the uploaded copy
  int64_t first_item, items;
  int64_t n, run;                            // elements, elements of the inner run
  int64_t cstride;                           // elements between two channels of a per-channel fill (1 otherwise)
  int64_t ext[kErMaxDim], kst[kErMaxDim];    // the groups of outer axes: extent and stride in the key space (0: not erased)
  int32_t ngroups, gfirst;                   // gfirst: the outermost erased group, -1 when no outer axis is erased
  int32_t nbands, esz;
};

struct alignas(16) ErVec { uint64_t w[2]; };

#if defined(__CUDACC__)
#define ER_PRAGMA(x) _Pragma(#x)
#else
#define ER_PRAGMA(x)
#endif

// a / b and a % b, in 32 bits when both fit
DB_HD uint64_t er_div(uint64_t a, uint64_t b) {
  if (((a | b) >> 32) == 0) return (uint32_t)a / (uint32_t)b;
  return a / b;
}

DB_HD ErVec er_load16(const void *p) {
#if defined(__CUDA_ARCH__)
  const uint4 v = __ldg(static_cast<const uint4 *>(p));
  ErVec r;
  r.w[0] = (uint64_t)v.x | (uint64_t)v.y << 32;
  r.w[1] = (uint64_t)v.z | (uint64_t)v.w << 32;
  return r;
#else
  ErVec r;
  memcpy(&r, p, 16);
  return r;
#endif
}

DB_HD void er_store16(void *p, const ErVec &v) {
#if defined(__CUDA_ARCH__)
  *static_cast<uint4 *>(p) = make_uint4((uint32_t)v.w[0], (uint32_t)(v.w[0] >> 32), (uint32_t)v.w[1], (uint32_t)(v.w[1] >> 32));
#else
  memcpy(p, &v, 16);
#endif
}

template <int ESZ> struct ErElem;
template <> struct ErElem<1> { typedef uint8_t T; };
template <> struct ErElem<2> { typedef uint16_t T; };
template <> struct ErElem<4> { typedef uint32_t T; };
template <> struct ErElem<8> { typedef uint64_t T; };

// element k (< 16 / ESZ) of a vector, statically indexed once unrolled
template <int ESZ> DB_HD void er_put(ErVec &v, int k, uint64_t x) {
  constexpr int per = 8 / ESZ;
  const int w = k / per, sh = (k % per) * ESZ * 8;
  const uint64_t mask = ESZ == 8 ? ~uint64_t{0} : ((uint64_t{1} << (ESZ * 8)) - 1);
  v.w[w] = (v.w[w] & ~(mask << sh)) | ((x & mask) << sh);
}

// The row's key: its row-major index over the erased outer axes.
DB_HD int64_t er_key(const ErSample &d, uint64_t row) {
  if (d.gfirst < 0) return 0;
  int64_t key = 0;
  for (int g = d.ngroups - 1; g > d.gfirst; g--) {
    const uint64_t q = er_div(row, (uint64_t)d.ext[g]);
    key += (int64_t)(row - q * (uint64_t)d.ext[g]) * d.kst[g];
    row = q;
  }
  if (d.gfirst > 0) row -= er_div(row, (uint64_t)d.ext[d.gfirst]) * (uint64_t)d.ext[d.gfirst];
  return key + (int64_t)row * d.kst[d.gfirst];
}

// The interval list [*b, *e) of a row.
DB_HD void er_row_ivals(const ErSample &d, uint64_t row, int64_t *b, int64_t *e) {
  const int64_t key = er_key(d, row);
  const ErBand &band = d.bands[last_at_most(d.bands, 0, d.nbands - 1, key, [](const ErBand &x) { return x.key; })];
  *b = band.off;
  *e = band.off + band.cnt;
}

// The first interval of [j, e) whose end is past col (e when there is none).
DB_HD int64_t er_first_after(const ErIval *iv, int64_t j, int64_t e, int64_t col) {
  while (j < e) {
    const int64_t mid = (j + e) >> 1;
    if (iv[mid].hi > col) e = mid; else j = mid + 1;
  }
  return j;
}

// The fill table of a batch (csrc/erase_plan.h, ErFillTable): nfill elements, then at the next 16-byte boundary nfill rotated
// patterns (pattern p: the elements of channels p, p + 1, ... mod nfill) and nfill broadcasts (broadcast c: channel c repeated).
DB_HD int64_t er_rot_off(int nfill, int esz) { return ((int64_t)nfill * esz + 15) / 16 * 16; }

template <int ESZ> DB_HD uint64_t er_fill_elem(const ErSample &d, const uint8_t *fill, int nfill, int64_t e) {
  typedef typename ErElem<ESZ>::T T;
  const int64_t c = nfill == 1 ? 0 : (int64_t)(er_div((uint64_t)e, (uint64_t)d.cstride) % (uint64_t)nfill);
  T x;
  memcpy(&x, fill + c * ESZ, ESZ);
  return x;
}

template <int ESZ> DB_HD uint64_t er_in_elem(const ErSample &d, int64_t e) {
  typedef typename ErElem<ESZ>::T T;
  return static_cast<const T *>(d.in)[e];
}

// Elements [lo, hi) of the sample, one by one (partial slots and slots that cross a row end).
template <int ESZ> DB_HD void er_elements(const ErSample &d, const uint8_t *fill, int nfill, int64_t lo, int64_t hi) {
  typedef typename ErElem<ESZ>::T T;
  uint64_t row = er_div((uint64_t)lo, (uint64_t)d.run);
  int64_t col = lo - (int64_t)row * d.run, j, je;
  er_row_ivals(d, row, &j, &je);
  j = er_first_after(d.ivals, j, je, col);
  for (int64_t e = lo; e < hi; e++, col++) {
    if (col == d.run) {
      row++;
      col = 0;
      er_row_ivals(d, row, &j, &je);
    }
    while (j < je && d.ivals[j].hi <= col) j++;
    const bool filled = j < je && d.ivals[j].lo <= col;
    static_cast<T *>(d.out)[e] = (T)(filled ? er_fill_elem<ESZ>(d, fill, nfill, e) : er_in_elem<ESZ>(d, e));
  }
}

// One 16-byte slot of the output.
template <int ESZ> DB_HD void er_slot(const ErSample &d, const uint8_t *fill, int nfill, int64_t slot) {
  constexpr int V = 16 / ESZ;
  const int shift = (int)(((uintptr_t)d.out & 15) / ESZ);
  const int64_t e0 = slot * V - shift;
  if (e0 >= d.n) return;
  if (e0 < 0 || e0 + V > d.n) {
    er_elements<ESZ>(d, fill, nfill, e0 < 0 ? 0 : e0, e0 + V < d.n ? e0 + V : d.n);
    return;
  }
  const uint64_t row = er_div((uint64_t)e0, (uint64_t)d.run);
  const int64_t c0 = e0 - (int64_t)row * d.run;
  if (c0 + V > d.run) {
    er_elements<ESZ>(d, fill, nfill, e0, e0 + V);
    return;
  }
  int64_t j, je;
  er_row_ivals(d, row, &j, &je);
  j = er_first_after(d.ivals, j, je, c0);
  uint8_t *const out = static_cast<uint8_t *>(d.out) + e0 * ESZ;
  const uint8_t *const in = static_cast<const uint8_t *>(d.in) + e0 * ESZ;
  const bool in_aligned = (((uintptr_t)in) & 15) == 0;
  if (j == je || d.ivals[j].lo >= c0 + V) {                              // no erased element: a copy
    if (in_aligned) {
      er_store16(out, er_load16(in));
    } else {
      ErVec v = {};
ER_PRAGMA(unroll)
      for (int k = 0; k < V; k++) er_put<ESZ>(v, k, er_in_elem<ESZ>(d, e0 + k));
      er_store16(out, v);
    }
    return;
  }
  const uint8_t *const pat = fill + er_rot_off(nfill, ESZ);
  if (d.ivals[j].lo <= c0 && d.ivals[j].hi >= c0 + V) {                  // every element erased
    if (nfill == 1) {
      er_store16(out, er_load16(pat));
      return;
    }
    if (d.cstride == 1) {
      er_store16(out, er_load16(pat + (e0 % nfill) * 16));
      return;
    }
    const uint64_t ch = er_div((uint64_t)e0, (uint64_t)d.cstride);
    if (ch == er_div((uint64_t)(e0 + V - 1), (uint64_t)d.cstride)) {
      er_store16(out, er_load16(pat + ((int64_t)nfill + (int64_t)(ch % (uint64_t)nfill)) * 16));
      return;
    }
  }
  ErVec v = {};                                                         // an interval edge inside the slot
ER_PRAGMA(unroll)
  for (int k = 0; k < V; k++) {
    while (j < je && d.ivals[j].hi <= c0 + k) j++;
    const bool filled = j < je && d.ivals[j].lo <= c0 + k;
    er_put<ESZ>(v, k, filled ? er_fill_elem<ESZ>(d, fill, nfill, e0 + k) : er_in_elem<ESZ>(d, e0 + k));
  }
  er_store16(out, v);
}

// Work item `local` of a sample, as thread tid runs it.
template <int ESZ> DB_HD void er_item(const ErSample &d, const uint8_t *fill, int nfill, int64_t local, int tid) {
ER_PRAGMA(unroll 1)
  for (int k = 0; k < kErSlotsPerThread; k++) er_slot<ESZ>(d, fill, nfill, local * kErSlotsPerItem + k * kErThreads + tid);
}

}  // namespace dalib200

#endif  // DALI_B200_CSRC_ERASE_CORE_H_
