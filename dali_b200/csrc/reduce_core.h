// dali_b200/csrc/reduce_core.h -- the per-thread bodies of the batched axis reduction behind fn.reductions.* (csrc/reduce.cu),
// written as host/device functions so that tools/emul/reduce_emul.cc and tools/emul/cuda_emul_stub.cc run the very code the device
// runs.
//
// A pass (RedPass, built by csrc/reduce_plan.h) reduces one group of neighbouring axes of one sample: the data is [O, R, I], element
// (o, r, i) at (o * R + r) * I + i, and the pass writes [O, I].  R is cut into chunks of `rc` rows; a sample with more than one chunk
// writes one partial per chunk and a combine launch folds them in chunk order.  Two bodies read a chunk:
//   COLUMNS  one thread per output (o, i), looping over the chunk's rows: coalesced when I is wide, and the whole reduction when R
//            is short.
//   INNER    one block per (o, chunk) over the contiguous run of rows * I elements, read with 16-byte vector loads.  The first
//            `active` threads (a multiple of I) each keep V = 16 / sizeof(T) accumulators; since active * V is a multiple of I, the
//            accumulator j of thread t always meets the same i.  Those active * V partials go to shared memory, are folded per i in
//            slices, and the slices of each i are folded by one warp in a fixed butterfly.
// Every order of accumulation is fixed by the sample's shape alone, so a result does not depend on the batch, the grid or the device.
// Floating-point partial sums are never combined with atomics.  Offsets are 64-bit; there is no division per element.
#ifndef DALI_B200_CSRC_REDUCE_CORE_H_
#define DALI_B200_CSRC_REDUCE_CORE_H_

#include <stdint.h>
#include <string.h>
#include <math.h>
#include "host_device.h"

namespace dalib200 {

constexpr int kRedMaxDim = 6;
constexpr int kRedMaxPasses = 3;
constexpr int kRedThreads = 256;
constexpr int kRedSmemBytes = kRedThreads * 16 * 8 + kRedThreads * 8;   // active * V partials and the per-i slices, 8-byte accumulators
// the eight operators (DALIB200_REDUCE_* of include/dali_b200.h)
enum : int32_t { kRedMin = 0, kRedMax, kRedSum, kRedMean, kRedMeanSquare, kRedRms, kRedStdDev, kRedVariance };
// what a pass does with each element: kept as is (combined by min / max / +), squared, or squared after the mean is subtracted
enum : int { kElemMin = 0, kElemMax, kElemSum, kElemSq, kElemSqDev };
enum : int32_t { kAccI64 = 0, kAccU64, kAccF32, kAccF64 };
enum : int32_t { kRedPathColumns = 0, kRedPathInner = 1 };
// DALIDataType codes of the numeric types
enum : int32_t { kRedU8 = 0, kRedU16, kRedU32, kRedU64, kRedI8, kRedI16, kRedI32, kRedI64, kRedF16, kRedF32, kRedF64 };

struct RedHalf { uint16_t bits; };

struct RedPass {
  const uint8_t *in; uint8_t *out, *part; const float *mean;   // bound at launch
  int64_t O, R, I;
  int64_t rc, nchunks;                 // rows per chunk, chunks
  int64_t first_item, items;           // the pass launch: COLUMNS items are 256 outputs x chunks, INNER items (o, chunk)
  int64_t cfirst, citems;              // the combine launch (nchunks > 1): 256 outputs per item
  int64_t count;                       // elements reduced into one output of the sample (divisor of the mean)
  int64_t in_off, out_off, part_off;   // byte offsets in the plan's scratch (in_off: passes after the first)
  int64_t gext[kRedMaxDim], gstr[kRedMaxDim];   // first pass of std_dev / variance: outer groups innermost first and their stride
                                                // in the mean (0 for reduced groups); mean index = sum c_g * gstr[g] + i
  int32_t path, last, ngroups, active; // last: the sample's final pass, which writes the output type
};

struct RedFinal { int32_t op, out_type, ddof, pad; };

// ---- conversions
DB_HD float red_f32_of(uint32_t b) {
#ifdef __CUDA_ARCH__
  return __uint_as_float(b);
#else
  float f; memcpy(&f, &b, 4); return f;
#endif
}
DB_HD double red_f64_of(uint64_t b) {
#ifdef __CUDA_ARCH__
  return __longlong_as_double((long long)b);
#else
  double f; memcpy(&f, &b, 8); return f;
#endif
}
DB_HD uint64_t red_bits_f64(double x) {
#ifdef __CUDA_ARCH__
  return (uint64_t)__double_as_longlong(x);
#else
  uint64_t b; memcpy(&b, &x, 8); return b;
#endif
}
DB_HD float red_h2f(uint16_t h) {
  const uint32_t s = (uint32_t)(h & 0x8000u) << 16, e = (h >> 10) & 31u, m = h & 1023u;
  if (e == 0) { const float f = (float)m * 5.9604644775390625e-8f; return s ? -f : f; }   // zero and subnormals: m * 2^-24
  return red_f32_of(s | (e == 31 ? 0x7F800000u | (m << 13) : ((e + 112u) << 23) | (m << 13)));
}
// double -> half, round to nearest even (numpy's astype(float16)); a float converts through it exactly
DB_HD uint16_t red_d2h(double x) {
  const uint64_t b = red_bits_f64(x), a = b & 0x7FFFFFFFFFFFFFFFull;
  const uint16_t s = (uint16_t)((b >> 48) & 0x8000u);
  if (a > 0x7FF0000000000000ull) return s | 0x7E00u;
  if (a == 0) return s;
  const int e = (int)(a >> 52) - 1023;
  if (e >= 16) return s | 0x7C00u;
  const uint64_t m = (a & ((1ull << 52) - 1)) | (1ull << 52);
  const int shift = e >= -14 ? 42 : 28 - e;
  if (shift > 63) return s;
  uint64_t q = m >> shift;
  const uint64_t rem = m & ((1ull << shift) - 1), half = 1ull << (shift - 1);
  if (rem > half || (rem == half && (q & 1))) q++;
  return e >= -14 ? (uint16_t)(s | (((uint32_t)(e + 14) << 10) + (uint32_t)q)) : (uint16_t)(s | (uint32_t)q);
}

template <typename T> struct RedVal { typedef T type; DB_HD static T get(T v) { return v; } };
template <> struct RedVal<RedHalf> { typedef float type; DB_HD static float get(RedHalf v) { return red_h2f(v.bits); } };

template <typename A> DB_HD A red_inf();
template <> DB_HD float red_inf<float>() { return red_f32_of(0x7F800000u); }
template <> DB_HD double red_inf<double>() { return red_f64_of(0x7FF0000000000000ull); }
template <> DB_HD int64_t red_inf<int64_t>() { return INT64_MAX; }
template <> DB_HD uint64_t red_inf<uint64_t>() { return UINT64_MAX; }
template <typename A> DB_HD A red_ninf();
template <> DB_HD float red_ninf<float>() { return red_f32_of(0xFF800000u); }
template <> DB_HD double red_ninf<double>() { return red_f64_of(0xFFF0000000000000ull); }
template <> DB_HD int64_t red_ninf<int64_t>() { return INT64_MIN; }
template <> DB_HD uint64_t red_ninf<uint64_t>() { return 0; }

template <int E, typename A> DB_HD A red_ident() { return E == kElemMin ? red_inf<A>() : E == kElemMax ? red_ninf<A>() : (A)0; }
// min / max propagate a NaN as np.min / np.max do; sums wrap for integers
template <int E, typename A> DB_HD A red_comb(A a, A x) {
  if (E == kElemMin) return (x < a || x != x) ? x : a;
  if (E == kElemMax) return (x > a || x != x) ? x : a;
  if ((A)0.5 == (A)0) return (A)((uint64_t)a + (uint64_t)x);    // integers wrap modulo 2^64
  return a + x;
}
template <int E, typename A, typename T> DB_HD A red_elem(T v, A m) {
  const A x = (A)RedVal<T>::get(v);
  if (E == kElemSq) return x * x;
  if (E == kElemSqDev) { const A d = x - m; return d * d; }
  return x;
}

// ---- the final value of one output, stored in the output type
template <typename V> DB_HD void red_put(uint8_t *out, int32_t type, int64_t q, V v) {
  switch (type) {
    case kRedU8: reinterpret_cast<uint8_t *>(out)[q] = (uint8_t)v; break;
    case kRedU16: reinterpret_cast<uint16_t *>(out)[q] = (uint16_t)v; break;
    case kRedU32: reinterpret_cast<uint32_t *>(out)[q] = (uint32_t)v; break;
    case kRedU64: reinterpret_cast<uint64_t *>(out)[q] = (uint64_t)v; break;
    case kRedI8: reinterpret_cast<int8_t *>(out)[q] = (int8_t)(uint8_t)v; break;
    case kRedI16: reinterpret_cast<int16_t *>(out)[q] = (int16_t)(uint16_t)v; break;
    case kRedI32: reinterpret_cast<int32_t *>(out)[q] = (int32_t)(uint32_t)v; break;
    case kRedI64: reinterpret_cast<int64_t *>(out)[q] = (int64_t)v; break;
    case kRedF16: reinterpret_cast<uint16_t *>(out)[q] = red_d2h((double)v); break;
    case kRedF32: reinterpret_cast<float *>(out)[q] = (float)v; break;
    default: reinterpret_cast<double *>(out)[q] = (double)v; break;
  }
}
// integer accumulators hold exact sums: the mean family divides them in double, one rounding to the output type follows
template <typename A> DB_HD void red_final(const RedFinal &f, int64_t count, uint8_t *out, int64_t q, A acc) {
  const bool integral = (A)0.5 == (A)0;
  switch (f.op) {
    case kRedMin: case kRedMax: case kRedSum: red_put(out, f.out_type, q, acc); return;
    case kRedMean: case kRedMeanSquare: case kRedRms:
      if (integral || sizeof(A) == 8) {
        double v = (double)acc / (double)count;
        if (f.op == kRedRms) v = sqrt(v);
        red_put(out, f.out_type, q, v);
      } else {
        float v = (float)acc / (float)count;
        if (f.op == kRedRms) v = sqrtf(v);
        red_put(out, f.out_type, q, v);
      }
      return;
    default: {
      const int64_t dv = count - f.ddof > 1 ? count - f.ddof : 1;
      float v = count == 0 ? red_f32_of(0x7FC00000u) : (float)acc / (float)dv;
      if (f.op == kRedStdDev) v = sqrtf(v);
      red_put(out, f.out_type, q, v);
    }
  }
}
// output q of pass d holds acc: a partial of chunk ch, an intermediate of the next pass, or the sample's result
template <typename A> DB_HD void red_store(const RedPass &d, const RedFinal &f, int64_t ch, int64_t q, A acc) {
  if (d.nchunks > 1) { reinterpret_cast<A *>(d.part)[ch * d.O * d.I + q] = acc; return; }
  if (!d.last) { reinterpret_cast<A *>(d.out)[q] = acc; return; }
  red_final(f, d.count, d.out, q, acc);
}

// the mean of output (o, i) (first pass of std_dev / variance)
DB_HD int64_t red_mean_index(const RedPass &d, int64_t o, int64_t i) {
  int64_t idx = i;
  for (int g = 0; g < d.ngroups; g++) {
    const int64_t nx = o / d.gext[g];
    idx += (o - nx * d.gext[g]) * d.gstr[g];
    o = nx;
  }
  return idx;
}

// ---- COLUMNS: thread tid of item `local` folds the rows of one chunk for one output
template <typename T, typename A, int E>
DB_HD void red_columns(const RedPass &d, const RedFinal &f, int64_t local, int tid) {
  const int64_t tile = local / d.nchunks, ch = local - tile * d.nchunks, q = tile * kRedThreads + tid;
  if (q >= d.O * d.I) return;
  const int64_t o = q / d.I, i = q - o * d.I, r0 = ch * d.rc, r1 = r0 + d.rc < d.R ? r0 + d.rc : d.R;
  const A m = E == kElemSqDev ? (A)d.mean[red_mean_index(d, o, i)] : (A)0;
  const T *p = reinterpret_cast<const T *>(d.in) + (o * d.R + r0) * d.I + i;
  A acc = red_ident<E, A>();
  for (int64_t r = r0; r < r1; r++, p += d.I) acc = red_comb<E, A>(acc, red_elem<E, A>(*p, m));
  red_store(d, f, ch, q, acc);
}

// ---- INNER
struct RedRun { int64_t o, ch, len, head; const uint8_t *base; };   // base: 16-byte aligned, `head` elements before the run
template <typename T> DB_HD RedRun red_run(const RedPass &d, int64_t local) {
  RedRun u;
  u.o = local / d.nchunks; u.ch = local - u.o * d.nchunks;
  const int64_t r0 = u.ch * d.rc, r1 = r0 + d.rc < d.R ? r0 + d.rc : d.R;
  u.len = (r1 - r0) * d.I;
  const uint8_t *p = d.in + (u.o * d.R + r0) * d.I * (int64_t)sizeof(T);
  u.head = (int64_t)(((uintptr_t)p & 15u) / sizeof(T));
  u.base = p - u.head * (int64_t)sizeof(T);
  return u;
}
// phase 1: thread tid < d.active folds 16-byte words tid, tid + active, ...; its V partials go to sm[tid * V + j]
template <typename T, typename A, int E>
DB_HD void red_inner_fold(const RedPass &d, const RedRun &u, A *sm, int tid) {
  constexpr int V = 16 / (int)sizeof(T);
  if (tid >= d.active) return;
  A acc[V], m[V];
  for (int j = 0; j < V; j++) {
    acc[j] = red_ident<E, A>();
    m[j] = (A)0;
    if (E == kElemSqDev) {
      int64_t i = ((int64_t)tid * V + j - u.head) % d.I;
      if (i < 0) i += d.I;
      m[j] = (A)d.mean[red_mean_index(d, u.o, i)];
    }
  }
  const int64_t end = u.head + u.len, nvec = (end + V - 1) / V;
  for (int64_t c = tid; c < nvec; c += d.active) {
    const int64_t p0 = c * V;
    if (p0 >= u.head && p0 + V <= end) {
      union { T t[V]; uint64_t w[2]; } w;
#ifdef __CUDA_ARCH__
      const uint4 v = *reinterpret_cast<const uint4 *>(u.base + p0 * (int64_t)sizeof(T));
      w.w[0] = (uint64_t)v.x | ((uint64_t)v.y << 32); w.w[1] = (uint64_t)v.z | ((uint64_t)v.w << 32);
#else
      memcpy(w.w, u.base + p0 * (int64_t)sizeof(T), 16);
#endif
      for (int j = 0; j < V; j++) acc[j] = red_comb<E, A>(acc[j], red_elem<E, A>(w.t[j], m[j]));
    } else {
      for (int j = 0; j < V; j++)
        if (p0 + j >= u.head && p0 + j < end)
          acc[j] = red_comb<E, A>(acc[j], red_elem<E, A>(*reinterpret_cast<const T *>(u.base + (p0 + j) * (int64_t)sizeof(T)), m[j]));
    }
  }
  for (int j = 0; j < V; j++) sm[(int64_t)tid * V + j] = acc[j];
}
// phase 2: thread q < I * S (S = 256 / I slices per i) folds the partials of i = q / S at slice s = q % S into sm2[q]
template <typename T, typename A, int E>
DB_HD void red_inner_slices(const RedPass &d, const RedRun &u, const A *sm, A *sm2, int q) {
  constexpr int V = 16 / (int)sizeof(T);
  const int I = (int)d.I, S = kRedThreads / I;
  if (q >= I * S) return;
  const int i = q / S, s = q - i * S, M = d.active * V / I, p0 = (int)((i + u.head) % I);
  A acc = red_ident<E, A>();
  for (int k = s; k < M; k += S) acc = red_comb<E, A>(acc, sm[p0 + k * I]);
  sm2[q] = acc;
}
// phase 3, lane `lane` of the warp that finishes i: its share of the slices of i (a butterfly over the 32 lanes follows)
template <typename A, int E> DB_HD A red_inner_lane(const RedPass &d, const A *sm2, int i, int lane) {
  const int S = kRedThreads / (int)d.I;
  A acc = red_ident<E, A>();
  for (int s = lane; s < S; s += 32) acc = red_comb<E, A>(acc, sm2[i * S + s]);
  return acc;
}
// the butterfly stated on 32 values (the device runs it with shuffles: v[l] += v[l + off] for off = 16, 8, 4, 2, 1); v[0] is the result
template <typename A, int E> DB_HD A red_tree32(A *v) {
  for (int off = 16; off > 0; off >>= 1)
    for (int l = 0; l < off; l++) v[l] = red_comb<E, A>(v[l], v[l + off]);
  return v[0];
}

// ---- the combine launch: the chunk partials of one output, in chunk order
template <typename A, int E> DB_HD void red_combine(const RedPass &d, const RedFinal &f, int64_t local, int tid) {
  const int64_t oi = d.O * d.I, q = local * kRedThreads + tid;
  if (q >= oi) return;
  const A *p = reinterpret_cast<const A *>(d.part) + q;
  A acc = red_ident<E, A>();
  for (int64_t c = 0; c < d.nchunks; c++, p += oi) acc = red_comb<E, A>(acc, *p);
  if (!d.last) { reinterpret_cast<A *>(d.out)[q] = acc; return; }
  red_final(f, d.count, d.out, q, acc);
}

// ---- the instantiations: every (input type, accumulator, element operation) the planner can produce.  fn(T(), A(), RedElemTag<E>())
template <int E> struct RedElemTag { static constexpr int value = E; };
// the accumulator that keeps the input's kind (min / max, and integer sums): int64, uint64, float (for float16 too) or double
template <typename T> struct RedNatural { typedef typename RedVal<T>::type V; typedef V type; };
template <> struct RedNatural<uint8_t> { typedef uint64_t type; };
template <> struct RedNatural<uint16_t> { typedef uint64_t type; };
template <> struct RedNatural<uint32_t> { typedef uint64_t type; };
template <> struct RedNatural<uint64_t> { typedef uint64_t type; };
template <> struct RedNatural<int8_t> { typedef int64_t type; };
template <> struct RedNatural<int16_t> { typedef int64_t type; };
template <> struct RedNatural<int32_t> { typedef int64_t type; };
template <> struct RedNatural<int64_t> { typedef int64_t type; };
template <typename T, typename Fn> bool red_dispatch_elem(int32_t acc, int elem, Fn &&fn) {
  typedef typename RedNatural<T>::type N;
  constexpr bool integral = (N)0.5 == (N)0;
  switch (elem) {
    case kElemMin: fn(T(), N(), RedElemTag<kElemMin>()); return true;
    case kElemMax: fn(T(), N(), RedElemTag<kElemMax>()); return true;
    case kElemSum: case kElemSq: {
      auto go = [&](auto a) { if (elem == kElemSum) fn(T(), a, RedElemTag<kElemSum>()); else fn(T(), a, RedElemTag<kElemSq>()); return true; };
      if (acc == kAccF32) return go(float());
      if (acc == kAccF64) return go(double());
      if constexpr (integral) return go(N());
      return false;
    }
    default: fn(T(), float(), RedElemTag<kElemSqDev>()); return true;
  }
}
template <typename Fn> bool red_dispatch(int32_t type, int32_t acc, int elem, Fn &&fn) {
  switch (type) {
    case kRedU8: return red_dispatch_elem<uint8_t>(acc, elem, fn);
    case kRedU16: return red_dispatch_elem<uint16_t>(acc, elem, fn);
    case kRedU32: return red_dispatch_elem<uint32_t>(acc, elem, fn);
    case kRedU64: return red_dispatch_elem<uint64_t>(acc, elem, fn);
    case kRedI8: return red_dispatch_elem<int8_t>(acc, elem, fn);
    case kRedI16: return red_dispatch_elem<int16_t>(acc, elem, fn);
    case kRedI32: return red_dispatch_elem<int32_t>(acc, elem, fn);
    case kRedI64: return red_dispatch_elem<int64_t>(acc, elem, fn);
    case kRedF16: return red_dispatch_elem<RedHalf>(acc, elem, fn);
    case kRedF32: return red_dispatch_elem<float>(acc, elem, fn);
    case kRedF64: return red_dispatch_elem<double>(acc, elem, fn);
    default: return false;
  }
}
// the type that holds accumulator kind `acc` (passes after the first read it from scratch)
template <typename Fn> void red_dispatch_acc(int32_t acc, int elem, Fn &&fn) {
  red_dispatch(acc == kAccI64 ? kRedI64 : acc == kAccU64 ? kRedU64 : acc == kAccF32 ? kRedF32 : kRedF64, acc, elem, fn);
}

}  // namespace dalib200

#endif  // DALI_B200_CSRC_REDUCE_CORE_H_
