// dali_b200/csrc/filter_core.h -- the per-thread bodies of fn.experimental.filter (csrc/filter.cu), written as host/device functions
// so that tools/emul/filter_emul.cc and tools/emul/cuda_emul_stub.cc run the very code the device runs.
//
// A frame is a plane of H rows of W * C elements; channels are filtered independently, so in the flattened row the taps of one filter
// row are C elements apart and one code path serves every channel count.  The output plane (Ho x Wo * C) is cut into strips of
// kFltRows rows x kFltSpan flattened elements; a strip is one work item.  A CTA streams the kFltRows + fh - 1 input rows its strip
// needs through shared memory in chunks of rows (all of them at once for small filters), every load of a chunk in flight before the
// first store: the rows are converted to float32 (exactly) and their border resolved while they are loaded (flt_load_groups,
// flt_load_edges), so the accumulation (flt_accum_row) has no edge cases.  Thread t accumulates the outputs at columns t + k kFltThreads
// (k < kFltElems) of every row of the strip: one shared-memory load of an input element feeds up to kFltRows fmaf, one load of a tap
// kFltElems.  Every output is one fmaf chain in a fixed order -- filter rows outer, columns inner -- so it is bit-identical alone or in
// any batch, at any position and under any tiling.  The host build uses the same fmaf, and is compiled with -ffp-contract=off.
#ifndef DALI_B200_CSRC_FILTER_CORE_H_
#define DALI_B200_CSRC_FILTER_CORE_H_

#include <stdint.h>
#include <string.h>
#include <math.h>
#include "host_device.h"
#include "arith_core.h"

namespace dalib200 {

constexpr int kFltThreads = 256;
constexpr int kFltRows = 8;                                  // output rows of a strip: accumulators per thread and column
constexpr int kFltElems = 4;                                 // output columns per thread, kFltThreads apart
constexpr int kFltSpan = kFltThreads * kFltElems;            // flattened output elements of a strip
constexpr int kFltMaxExtent = 255;                           // planner limits (DESIGN.md section 2)
constexpr int kFltMaxChannels = 64;
constexpr int kFltSmemTaps = 4096;                           // filters of at most this many taps are read from shared memory
constexpr int kFltMaxChunk = 64;                             // window rows loaded between two barriers, at most
constexpr int kFltChunkFloats = 24576;                       // and at most this many floats of them (96 KiB: two CTAs per SM)

enum : int { kFltReflect101 = 0, kFltReflect1001 = 1, kFltWrap = 2, kFltClamp = 3, kFltConstant = 4 };

struct FltSample {
  const void *in; void *out;                 // bound at launch
  const float *filter;                       // fh x fw taps, row-major (device: the caller's GPU filter or the arena's copy)
  const void *fill;                          // nullptr: 0; else fill_n values of the input type (1, or one per frame)
  int64_t first_item, items;                 // items = frames * ipf
  int64_t in_frame, out_frame;               // elements of one input / output frame
  int32_t H, W, C, Ho, Wo;
  int32_t fh, fw, ar, ac;                    // filter extents and anchor (row, column); 0, 0 in valid mode
  int32_t sx, ipf;                           // strips across an output row, items per frame
  int32_t border, fill_n;
  int32_t in_type, out_type;                 // DALIDataType of the data and of the output (the kernel's template arguments)
};

// The in-range index of i on an axis of n (>= 1) elements, or -1 for the fill value; any distance from the edge.
DB_HD int64_t flt_border(int64_t i, int64_t n, int border) {
  if (i >= 0 && i < n) return i;
  switch (border) {
    case kFltReflect101: {                   // dcb|abcd|cba
      if (n == 1) return 0;
      const int64_t p = 2 * (n - 1);
      int64_t m = i % p;
      if (m < 0) m += p;
      return m < n ? m : p - m;
    }
    case kFltReflect1001: {                  // cba|abcd|dcb
      const int64_t p = 2 * n;
      int64_t m = i % p;
      if (m < 0) m += p;
      return m < n ? m : p - 1 - m;
    }
    case kFltWrap: {
      int64_t m = i % n;
      return m < 0 ? m + n : m;
    }
    case kFltClamp: return i < 0 ? 0 : n - 1;
    default: return -1;
  }
}

// Exact conversions of the input types to float32.
DB_HD float flt_to_float(uint8_t v) {
  uint32_t b = 0x4B000000u | v;              // the float 2^23 + v: an FMA-pipe conversion on the device
  float f;
  memcpy(&f, &b, 4);
  return f - 8388608.0f;
}
DB_HD float flt_to_float(int8_t v) { return (float)v; }
DB_HD float flt_to_float(uint16_t v) { return (float)v; }
DB_HD float flt_to_float(int16_t v) { return (float)v; }
DB_HD float flt_to_float(float v) { return v; }

// binary16 is carried as its bits
struct FltHalf { uint16_t bits; };
DB_HD float flt_to_float(FltHalf v) { return arith_f(arith_from_bits(v.bits, kAF16)); }

// ConvertSat of the float32 sum to the output type, as the arithmetic kernel applies it (arith_cast)
template <typename TO> DB_HD TO flt_from_float(float x);
template <> DB_HD float flt_from_float<float>(float x) { return x; }
template <> DB_HD FltHalf flt_from_float<FltHalf>(float x) {
  FltHalf h;
  h.bits = (uint16_t)arith_to_bits(arith_cast(arith_uf(x), kAF32, kAF16), kAF16);
  return h;
}
template <typename TO> DB_HD TO flt_sat_int(float x, float lo, float hi) {   // half away from zero, saturated, NaN -> 0
  if (x != x) return 0;
  const float r = roundf(x);
  return (TO)(r <= lo ? lo : r >= hi ? hi : r);
}
template <> DB_HD uint8_t flt_from_float<uint8_t>(float x) { return flt_sat_int<uint8_t>(x, 0.0f, 255.0f); }
template <> DB_HD int8_t flt_from_float<int8_t>(float x) { return flt_sat_int<int8_t>(x, -128.0f, 127.0f); }
template <> DB_HD uint16_t flt_from_float<uint16_t>(float x) { return flt_sat_int<uint16_t>(x, 0.0f, 65535.0f); }
template <> DB_HD int16_t flt_from_float<int16_t>(float x) { return flt_sat_int<int16_t>(x, -32768.0f, 32767.0f); }

// The strip of work item `local` of a sample: frame, first output row, first flattened output element.
struct FltStrip { int64_t frame; int32_t y0, x0; };

DB_HD FltStrip flt_strip(const FltSample &d, int64_t local) {
  FltStrip s;
  s.frame = local / d.ipf;
  const int32_t rest = (int32_t)(local - s.frame * d.ipf);
  s.y0 = rest / d.sx * kFltRows;
  s.x0 = rest % d.sx * kFltSpan;
  return s;
}

// Floats of one streamed row in shared memory: the strip's span, the (fw - 1) C elements its taps reach beyond it, and up to 3 in front
// so that the row's aligned 4-element groups sit at 16-byte boundaries in shared memory too; a multiple of 4.
DB_HD int flt_row_floats(int fw, int C) { return (kFltSpan + (fw - 1) * C + 3 + 3) & ~3; }

template <typename TI>
DB_HD float flt_fill(const FltSample &d, const FltStrip &s) {
  if (!d.fill) return 0.0f;
  return flt_to_float(static_cast<const TI *>(d.fill)[d.fill_n > 1 ? s.frame : 0]);
}

// The positions of the strip's window row that its stored outputs reach: up to kFltSpan outputs (fewer at the end of the output row)
// and the (fw - 1) C elements the taps reach beyond them.
DB_HD int flt_span(const FltSample &d, const FltStrip &s) {
  const int64_t rest = (int64_t)d.Wo * d.C - s.x0;
  return (int)(rest < kFltSpan ? rest : kFltSpan) + (d.fw - 1) * d.C;
}

// Where window row j (input row y0 - ar + j) comes from and how it lies in shared memory.  Element e0 + p of the input row (e0 = x0 -
// ac C, p < span) goes to buf[sh + p]: sh puts the row's aligned 4-element groups at 16-byte boundaries in shared memory too.  Groups
// ga ... gb - 1 (in units of 4 floats) lie wholly inside the input row and are read with one load each; the other positions go one by
// one through the border map.  A row outside the frame under the constant border is a fill row.
struct FltRowMap { int64_t off; int32_t sh, ga, gb, fill; };     // off: the row's first element in the sample

template <typename TI>
DB_HD FltRowMap flt_row_map(const FltSample &d, const FltStrip &s, int j) {
  FltRowMap m;
  const int span = flt_span(d, s);
  const int64_t e0 = (int64_t)s.x0 - (int64_t)d.ac * d.C, rowlen = (int64_t)d.W * d.C;
  const int64_t ry = flt_border((int64_t)s.y0 - d.ar + j, d.H, d.border);
  m.fill = ry < 0;
  m.off = m.fill ? 0 : s.frame * d.in_frame + ry * rowlen;
  m.sh = m.fill ? 0 : (int)(((uintptr_t)d.in / sizeof(TI) + (uint64_t)(m.off + e0)) & 3);
  const int64_t pa64 = e0 < 0 ? -e0 : 0, pb64 = rowlen - e0 < span ? rowlen - e0 : span;
  const int pa = (int)(pa64 < span ? pa64 : span), pb = (int)(pb64 > pa ? pb64 : pa);
  m.ga = m.fill ? 0 : (m.sh + pa + 3) >> 2;
  m.gb = m.fill ? 0 : (m.sh + pb) >> 2;
  if (m.gb < m.ga) m.gb = m.ga;
  return m;
}

// Groups of loads a thread keeps in flight before its first store: 64 bytes
template <typename TI> struct FltBatch { static constexpr int value = 16 / (int)sizeof(TI); };

// Thread `tid`'s share of the aligned groups of window rows j0 ... j0 + kn - 1 (maps[q]: row j0 + q, at rows + q row_floats): a flat
// list over the rows, FltBatch loads issued before their conversions and 16-byte stores.
template <typename TI>
DB_HD void flt_load_groups(const FltSample &d, const FltStrip &s, const FltRowMap *maps, int kn, float *rows, int row_floats, int tid) {
  constexpr int U = FltBatch<TI>::value;
  const int ngr = row_floats / 4;                                     // group slots of a row
  const int64_t e0 = (int64_t)s.x0 - (int64_t)d.ac * d.C;
  const TI *in = static_cast<const TI *>(d.in);
  for (int base = tid; base < kn * ngr; base += U * kFltThreads) {
    TI v[U][4];
    int dst[U];
#ifdef __CUDA_ARCH__
#pragma unroll
#endif
    for (int u = 0; u < U; u++) {
      const int idx = base + u * kFltThreads, q = idx / ngr;
      dst[u] = -1;
      if (idx >= kn * ngr) continue;
      const FltRowMap m = maps[q];
      const int g = m.ga + (idx - q * ngr);
      if (g >= m.gb) continue;
      const TI *src = in + m.off + e0 - m.sh + 4 * g;
#ifdef __CUDA_ARCH__
      if constexpr (sizeof(TI) == 1) {
        const uint32_t x = __ldg(reinterpret_cast<const uint32_t *>(src));
        memcpy(v[u], &x, 4);
      } else if constexpr (sizeof(TI) == 2) {
        const uint2 x = __ldg(reinterpret_cast<const uint2 *>(src));
        memcpy(v[u], &x, 8);
      } else {
        const uint4 x = __ldg(reinterpret_cast<const uint4 *>(src));
        memcpy(v[u], &x, 16);
      }
#else
      memcpy(v[u], src, sizeof(v[u]));
#endif
      dst[u] = q * row_floats + 4 * g;
    }
#ifdef __CUDA_ARCH__
#pragma unroll
#endif
    for (int u = 0; u < U; u++) {
      if (dst[u] < 0) continue;
#ifdef __CUDA_ARCH__
      *reinterpret_cast<float4 *>(rows + dst[u]) = make_float4(flt_to_float(v[u][0]), flt_to_float(v[u][1]), flt_to_float(v[u][2]),
                                                               flt_to_float(v[u][3]));
#else
      for (int k = 0; k < 4; k++) rows[dst[u] + k] = flt_to_float(v[u][k]);
#endif
    }
  }
}

// Thread `tid`'s share of the other positions of the same rows, one by one: the border on either side, the partial groups at the ends
// of the in-range part, and whole fill rows.  Each row has 32 lanes (row q: slots 32 q ... 32 q + 31 of the flat thread range), so the
// few loads of every row are in flight at once instead of row after row.
template <typename TI>
DB_HD void flt_load_edges(const FltSample &d, const FltStrip &s, const FltRowMap *maps, int kn, float *rows, int row_floats, int tid) {
  const int span = flt_span(d, s);
  const int64_t e0 = (int64_t)s.x0 - (int64_t)d.ac * d.C, rowlen = (int64_t)d.W * d.C;
  const TI *in = static_cast<const TI *>(d.in);
  for (int slot = tid; slot < 32 * kn; slot += kFltThreads) {
    const FltRowMap m = maps[slot >> 5];
    float *buf = rows + (slot >> 5) * row_floats + m.sh;
    const int lo_end = 4 * m.ga - m.sh, hi_start = 4 * m.gb - m.sh;
    const int nlo = lo_end, nhi = span - hi_start;
    for (int k = slot & 31; k < nlo + nhi; k += 32) {
      const int p = k < nlo ? k : hi_start + (k - nlo);
      const int64_t e = e0 + p;
      float v;
      if (m.fill) {
        v = flt_fill<TI>(d, s);
      } else if (e >= 0 && e < rowlen) {
        v = flt_to_float(in[m.off + e]);
      } else {
        const int64_t col = e >= 0 ? e / d.C : -((-e + d.C - 1) / d.C);
        const int64_t rc = flt_border(col, d.W, d.border);
        v = rc < 0 ? flt_fill<TI>(d, s) : flt_to_float(in[m.off + rc * d.C + (e - col * d.C)]);
      }
      buf[p] = v;
    }
  }
}

// Thread `tid` adds window row j (buf + sh: the row's element e0 first) to the output rows t of its strip with 0 <= j - t < fh, tap
// row j - t: acc[t][k] = fmaf(f[j - t][s], x[tid + k kFltThreads + s C], acc[t][k]) for s = 0 ... fw - 1.
DB_HD void flt_accum_row(const FltSample &d, const float *taps, int j, const float *row, float (&acc)[kFltRows][kFltElems], int tid) {
  const int tlo = j - d.fh + 1 > 0 ? j - d.fh + 1 : 0, thi = j < kFltRows - 1 ? j : kFltRows - 1;
  const float *x = row + tid;
  for (int s = 0; s < d.fw; s++, x += d.C) {
    float v[kFltElems];
#ifdef __CUDA_ARCH__
#pragma unroll
#endif
    for (int k = 0; k < kFltElems; k++) v[k] = x[k * kFltThreads];
#ifdef __CUDA_ARCH__
#pragma unroll
#endif
    for (int t = 0; t < kFltRows; t++) {
      if (t < tlo || t > thi) continue;
      const float f = taps[(j - t) * d.fw + s];
#ifdef __CUDA_ARCH__
#pragma unroll
#endif
      for (int k = 0; k < kFltElems; k++) acc[t][k] = fmaf(f, v[k], acc[t][k]);
    }
  }
}

// Thread `tid` writes its outputs of the strip.
template <typename TO>
DB_HD void flt_store(const FltSample &d, const FltStrip &s, const float (&acc)[kFltRows][kFltElems], int tid) {
  const int64_t rowlen = (int64_t)d.Wo * d.C;
  TO *out = static_cast<TO *>(d.out) + s.frame * d.out_frame;
#ifdef __CUDA_ARCH__
#pragma unroll
#endif
  for (int t = 0; t < kFltRows; t++) {
    if (s.y0 + t >= d.Ho) break;
#ifdef __CUDA_ARCH__
#pragma unroll
#endif
    for (int k = 0; k < kFltElems; k++) {
      const int64_t x = (int64_t)s.x0 + tid + k * kFltThreads;
      if (x < rowlen) out[(int64_t)(s.y0 + t) * rowlen + x] = flt_from_float<TO>(acc[t][k]);
    }
  }
}

// The (input, output) element types of a DALIDataType pair: f(TI(), TO()).  Returns false for a pair the kernel does not take.
template <typename F>
DB_HD bool flt_dispatch(int in_type, int out_type, F &&f) {
  switch (in_type * 16 + (out_type == kAF32 ? 1 : 0) * (in_type != kAF32)) {
    case kAU8 * 16: f(uint8_t(), uint8_t()); return true;
    case kAU8 * 16 + 1: f(uint8_t(), float()); return true;
    case kAI8 * 16: f(int8_t(), int8_t()); return true;
    case kAI8 * 16 + 1: f(int8_t(), float()); return true;
    case kAU16 * 16: f(uint16_t(), uint16_t()); return true;
    case kAU16 * 16 + 1: f(uint16_t(), float()); return true;
    case kAI16 * 16: f(int16_t(), int16_t()); return true;
    case kAI16 * 16 + 1: f(int16_t(), float()); return true;
    case kAF16 * 16: f(FltHalf(), FltHalf()); return true;
    case kAF16 * 16 + 1: f(FltHalf(), float()); return true;
    case kAF32 * 16: f(float(), float()); return true;
    default: return false;
  }
}

}  // namespace dalib200

#endif  // DALI_B200_CSRC_FILTER_CORE_H_
