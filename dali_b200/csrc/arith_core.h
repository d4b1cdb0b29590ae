// dali_b200/csrc/arith_core.h -- the per-element bodies of the arithmetic-expression kernel (csrc/arith.cu), written as host/device
// functions so that tools/emul/arith_emul.cc and tools/emul/cuda_emul_stub.cc run the very code the device runs.
//
// An expression is a short program (built by csrc/arith_plan.h): LOAD / SCALAR instructions bring a tensor operand element or a
// per-sample scalar into a register, every other instruction applies one operator to registers.  A register holds one value in its
// storage form:
//   integers and BOOL   the value as a 64-bit integer (sign-extended for signed types, zero-extended for unsigned ones, BOOL 0 / 1)
//   FLOAT16, FLOAT      the float32 bits in the low word (a FLOAT16 value is a float32 that is exactly a binary16 value)
//   FLOAT64             the double bits
// Operands of an instruction are already in its compute type `ct` (the planner inserts CVT instructions); the result is in `rt`, which
// equals ct except for comparisons (BOOL).  Integer results wrap to their width; a BOOL result is "value != 0".  FLOAT16 nodes are
// computed in float32 and rounded to binary16 (to nearest, ties to even) after every operator.  No product is contracted into a sum:
// the device code is compiled with -fmad=false, the host code with -ffp-contract=off.
#ifndef DALI_B200_CSRC_ARITH_CORE_H_
#define DALI_B200_CSRC_ARITH_CORE_H_

#include <stdint.h>
#include <string.h>
#include <math.h>
#include <type_traits>
#include "host_device.h"

namespace dalib200 {

// type ids: DALIDataType
enum : int { kAU8 = 0, kAU16 = 1, kAU32 = 2, kAU64 = 3, kAI8 = 4, kAI16 = 5, kAI32 = 6, kAI64 = 7, kAF16 = 8, kAF32 = 9, kAF64 = 10,
             kABool = 11, kANumTypes = 12 };

enum ArithOp : uint8_t {
  kOpLoad, kOpScalar, kOpCvt, kOpCast,
  kOpPlus, kOpMinus, kOpAbs, kOpFabs, kOpFloor, kOpCeil, kOpSqrt, kOpRsqrt, kOpCbrt, kOpExp, kOpLog, kOpLog2, kOpLog10,
  kOpSin, kOpCos, kOpTan, kOpAsin, kOpAcos, kOpAtan, kOpSinh, kOpCosh, kOpTanh, kOpAsinh, kOpAcosh, kOpAtanh,
  kOpAdd, kOpSub, kOpMul, kOpFdiv, kOpDiv, kOpPow, kOpFpow, kOpMin, kOpMax, kOpAtan2,
  kOpEq, kOpNeq, kOpLt, kOpLeq, kOpGt, kOpGeq, kOpBitAnd, kOpBitOr, kOpBitXor,
  kOpClamp, kOpCount
};

constexpr int kArithMaxInputs = 16;      // tensor operands and per-sample scalars together
constexpr int kArithMaxScalars = 16;     // constants and per-sample scalars
constexpr int kArithMaxInstr = 64;
constexpr int kArithMaxRegs = 8;       // live values of a program (arith_get / arith_set name each one)
constexpr int kArithMaxDim = 6;
constexpr int kArithEpt = 4;             // elements per thread and instruction

struct ArithInstr {
  uint8_t op, dst, a, b, c, ct, rt, pad;   // LOAD: a = tensor operand; SCALAR: a = scalar slot; CVT / CAST: from ct to rt
};

struct ArithProgram {
  int32_t ninstr, nin, out_type, out_reg;
  int32_t wide;                                     // some value is 64 bits wide (INT64, UINT64, FLOAT64)
  int32_t in_type[kArithMaxInputs];
  ArithInstr ins[kArithMaxInstr];
};

struct ArithSample {
  const void *in[kArithMaxInputs];
  void *out;
  int64_t n, first_item;
  int64_t shape[kArithMaxDim];                      // output extents, innermost last; ndim entries used
  int64_t stride[kArithMaxInputs][kArithMaxDim];    // element strides of each operand over the output's axes (0 on broadcast axes)
  uint64_t scal[kArithMaxScalars];                  // constants and per-sample scalars, in storage form
  uint32_t linear;                                  // bit j: operand j has the output's shape (element index = output index)
  int32_t ndim;
};

DB_HD bool arith_is_float(int t) { return t == kAF16 || t == kAF32 || t == kAF64; }
DB_HD bool arith_is_signed(int t) { return t >= kAI8 && t <= kAI64; }
DB_HD int arith_bits(int t) {
  switch (t) {
    case kAU8: case kAI8: return 8;
    case kAU16: case kAI16: case kAF16: return 16;
    case kAU32: case kAI32: case kAF32: return 32;
    case kABool: return 1;
    default: return 64;
  }
}
DB_HD int arith_size(int t) { return t == kABool ? 1 : arith_bits(t) / 8; }

DB_HD float arith_f(uint64_t v) { float f; uint32_t b = (uint32_t)v; memcpy(&f, &b, 4); return f; }
DB_HD uint64_t arith_uf(float f) { uint32_t b; memcpy(&b, &f, 4); return b; }
DB_HD double arith_d(uint64_t v) { double d; memcpy(&d, &v, 8); return d; }
DB_HD uint64_t arith_ud(double d) { uint64_t b; memcpy(&b, &d, 8); return b; }

#ifdef __CUDA_ARCH__
DB_HD float arith_fadd(float a, float b) { return __fadd_rn(a, b); }
DB_HD float arith_fmul(float a, float b) { return __fmul_rn(a, b); }
#else
DB_HD float arith_fadd(float a, float b) { return a + b; }
DB_HD float arith_fmul(float a, float b) { return a * b; }
#endif

// float32 -> the nearest binary16 value (ties to even, overflow to infinity), as a float32
DB_HD float arith_half_rne(float f) {
  uint32_t b = (uint32_t)arith_uf(f);
  const uint32_t s = b & 0x80000000u, a = b & 0x7FFFFFFFu;
  if (a >= 0x7F800000u) return f;                                   // inf, NaN
  if (a >= 0x477FF000u) return arith_f(s | 0x7F800000u);           // >= 65520 rounds to infinity
  if (a < 0x38800000u) {                                            // below 2^-14: multiples of 2^-24
    const float x = arith_f(a) * 16777216.0f;                       // exact: < 1024
    const float r = arith_fadd(arith_fadd(x, 12582912.0f), -12582912.0f);   // round to an integer, ties to even
    return arith_f(s | (uint32_t)arith_uf(r * 5.9604644775390625e-08f));
  }
  const uint32_t lsb = (a >> 13) & 1u;
  return arith_f(s | ((a + 0xFFFu + lsb) & ~0x1FFFu));
}

// float32 -> binary16 as the CPU backend converts (ConvertSat<float16>): clamped to +-65504, then to nearest, ties away from zero
DB_HD float arith_half_sat(float f) {
  if (f != f) return f;
  f = f > 65504.0f ? 65504.0f : f < -65504.0f ? -65504.0f : f;
  const uint32_t b = (uint32_t)arith_uf(f), s = b & 0x80000000u, a = b & 0x7FFFFFFFu;
  if (a < 0x38800000u) {
    const float r = floorf(arith_fadd(arith_f(a) * 16777216.0f, 0.5f));   // both steps exact
    return arith_f(s | (uint32_t)arith_uf(r * 5.9604644775390625e-08f));
  }
  return arith_f(s | ((a + 0x1000u) & ~0x1FFFu));
}

// an integer of type t from its 64-bit two's complement bits: truncated to the width and re-extended
DB_HD uint64_t arith_wrap(uint64_t x, int t) {
  switch (t) {
    case kAU8: return (uint8_t)x;
    case kAU16: return (uint16_t)x;
    case kAU32: return (uint32_t)x;
    case kAI8: return (uint64_t)(int64_t)(int8_t)x;
    case kAI16: return (uint64_t)(int64_t)(int16_t)x;
    case kAI32: return (uint64_t)(int64_t)(int32_t)x;
    case kABool: return x != 0;
    default: return x;
  }
}

DB_HD double arith_int_to_d(uint64_t v, int t) { return arith_is_signed(t) ? (double)(int64_t)v : (double)v; }
DB_HD float arith_int_to_f(uint64_t v, int t) { return arith_is_signed(t) ? (float)(int64_t)v : (float)v; }

// value conversion of a type promotion (integer widening or re-interpretation, integer -> float, float -> wider float)
DB_HD uint64_t arith_cvt(uint64_t v, int from, int to) {
  if (!arith_is_float(to)) return arith_wrap(v, to);
  if (to == kAF64) return arith_ud(arith_is_float(from) ? (from == kAF64 ? arith_d(v) : (double)arith_f(v)) : arith_int_to_d(v, from));
  if (arith_is_float(from)) return from == kAF64 ? arith_uf((float)arith_d(v)) : v;
  const float f = arith_int_to_f(v, from);
  return arith_uf(to == kAF16 ? arith_half_rne(f) : f);
}

// ConvertSat<to>(from): floats round half away from zero and saturate (NaN -> 0); integers saturate; BOOL is "!= 0";
// -> FLOAT16 goes through float32 and is clamped to +-65504 (ties away); FLOAT64 -> FLOAT rounds to nearest
DB_HD uint64_t arith_cast(uint64_t v, int from, int to) {
  if (to == kABool) return arith_is_float(from) ? (from == kAF64 ? arith_d(v) != 0 : arith_f(v) != 0) : v != 0;
  if (arith_is_float(to)) {
    if (to == kAF64) return arith_cvt(v, from, to);
    float f = arith_is_float(from) ? (from == kAF64 ? (float)arith_d(v) : arith_f(v)) : arith_int_to_f(v, from);
    return arith_uf(to == kAF16 ? arith_half_sat(f) : f);
  }
  const bool sgn = arith_is_signed(to);
  const int w = arith_bits(to);
  const double hi = sgn ? (w == 64 ? 9223372036854775808.0 : (double)((int64_t{1} << (w - 1)) - 1))
                        : (w == 64 ? 18446744073709551616.0 : (double)((uint64_t{1} << w) - 1));
  const double lo = sgn ? -(double)(uint64_t{1} << (w - 1)) : 0.0;
  const uint64_t maxv = sgn ? (uint64_t{1} << (w - 1)) - 1 : (w == 64 ? ~uint64_t{0} : (uint64_t{1} << w) - 1);
  const uint64_t minv = sgn ? (uint64_t)(-(int64_t)((uint64_t{1} << (w - 1)) - 1) - 1) : 0;
  if (arith_is_float(from)) {
    const double x = from == kAF64 ? arith_d(v) : (double)arith_f(v);
    if (x != x) return 0;
    const double r = round(x);
    if (r >= hi) return maxv;
    if (r <= lo) return minv;
    return sgn ? (uint64_t)(int64_t)r : (uint64_t)r;
  }
  if (arith_is_signed(from)) {
    const int64_t s = (int64_t)v;
    if (s > 0 && (uint64_t)s > maxv) return maxv;
    if (s < 0 && (!sgn || s < (int64_t)minv)) return minv;
    return (uint64_t)s;
  }
  return v > maxv ? maxv : v;                                       // unsigned or BOOL source
}

template <typename F>
DB_HD F arith_fop(int op, F a, F b, F c) {
  switch (op) {
    case kOpPlus: return a;
    case kOpMinus: return -a;
    case kOpAbs: case kOpFabs: return fabs(a);
    case kOpFloor: return floor(a);
    case kOpCeil: return ceil(a);
    case kOpSqrt: return sqrt(a);
    case kOpRsqrt: return F(1) / sqrt(a);
    case kOpCbrt: return cbrt(a);
    case kOpExp: return exp(a);
    case kOpLog: return log(a);
    case kOpLog2: return log2(a);
    case kOpLog10: return log10(a);
    case kOpSin: return sin(a);
    case kOpCos: return cos(a);
    case kOpTan: return tan(a);
    case kOpAsin: return asin(a);
    case kOpAcos: return acos(a);
    case kOpAtan: return atan(a);
    case kOpSinh: return sinh(a);
    case kOpCosh: return cosh(a);
    case kOpTanh: return tanh(a);
    case kOpAsinh: return asinh(a);
    case kOpAcosh: return acosh(a);
    case kOpAtanh: return atanh(a);
    case kOpAdd: return a + b;
    case kOpSub: return a - b;
    case kOpMul: return a * b;
    case kOpFdiv: return a / b;
    case kOpPow: case kOpFpow: return pow(a, b);
    case kOpAtan2: return atan2(a, b);
    case kOpMin: return b < a ? b : a;
    case kOpMax: return a < b ? b : a;
    case kOpClamp: return a < b ? b : (c < a ? c : a);
    default: return a;
  }
}

// float32: the float math library functions (no promotion to double); + - * through the non-contracting intrinsics
template <>
DB_HD float arith_fop<float>(int op, float a, float b, float c) {
  switch (op) {
    case kOpPlus: return a;
    case kOpMinus: return -a;
    case kOpAbs: case kOpFabs: return fabsf(a);
    case kOpFloor: return floorf(a);
    case kOpCeil: return ceilf(a);
    case kOpSqrt: return sqrtf(a);
    case kOpRsqrt: return 1.0f / sqrtf(a);
    case kOpCbrt: return cbrtf(a);
    case kOpExp: return expf(a);
    case kOpLog: return logf(a);
    case kOpLog2: return log2f(a);
    case kOpLog10: return log10f(a);
    case kOpSin: return sinf(a);
    case kOpCos: return cosf(a);
    case kOpTan: return tanf(a);
    case kOpAsin: return asinf(a);
    case kOpAcos: return acosf(a);
    case kOpAtan: return atanf(a);
    case kOpSinh: return sinhf(a);
    case kOpCosh: return coshf(a);
    case kOpTanh: return tanhf(a);
    case kOpAsinh: return asinhf(a);
    case kOpAcosh: return acoshf(a);
    case kOpAtanh: return atanhf(a);
    case kOpAdd: return arith_fadd(a, b);
    case kOpSub: return arith_fadd(a, -b);
    case kOpMul: return arith_fmul(a, b);
    case kOpFdiv: return a / b;
    case kOpPow: case kOpFpow: return powf(a, b);
    case kOpAtan2: return atan2f(a, b);
    case kOpMin: return b < a ? b : a;
    case kOpMax: return a < b ? b : a;
    case kOpClamp: return a < b ? b : (c < a ? c : a);
    default: return a;
  }
}

template <typename F>
DB_HD bool arith_fcmp(int op, F a, F b) {
  switch (op) {
    case kOpEq: return a == b;
    case kOpNeq: return a != b;
    case kOpLt: return a < b;
    case kOpLeq: return a <= b;
    case kOpGt: return a > b;
    default: return a >= b;
  }
}

template <typename U>
DB_HD U arith_upow(U b, U e, bool sgn) {
  typedef typename std::make_signed<U>::type S;
  if (sgn && (S)e < 0) {
    if ((S)b == 1) return 1;
    if ((S)b == -1) return (e & 1) ? (U)~U(0) : U(1);
    return 0;
  }
  U r = 1;
  while (e) { if (e & 1) r *= b; b *= b; e >>= 1; }
  return r;
}

// an integer / BOOL operator in I (int64_t / uint64_t, or int32_t / uint32_t when no operand is wider than 32 bits: the result
// wraps to the same value); the result's bits are zero-extended, arith_wrap gives them their type
template <typename I>
DB_HD uint64_t arith_iop(int op, I a, I b, I c) {
  typedef typename std::make_unsigned<I>::type U;
  const bool sgn = I(-1) < I(0);
  const U ua = (U)a, ub = (U)b;
  switch (op) {
    case kOpPlus: return ua;
    case kOpMinus: return (U)(U(0) - ua);
    case kOpAbs: return (U)(sgn && (ua >> (sizeof(U) * 8 - 1)) ? U(0) - ua : ua);
    case kOpAdd: return (U)(ua + ub);
    case kOpSub: return (U)(ua - ub);
    case kOpMul: return (U)(ua * ub);
    case kOpDiv: return b == 0 ? 0 : (sgn && b == I(-1)) ? (U)(U(0) - ua) : (U)(a / b);
    case kOpPow: return arith_upow<U>(ua, ub, sgn);
    case kOpMin: return (U)(b < a ? b : a);
    case kOpMax: return (U)(a < b ? b : a);
    case kOpClamp: return (U)(a < b ? b : (c < a ? c : a));
    case kOpBitAnd: return (U)(ua & ub);
    case kOpBitOr: return (U)(ua | ub);
    case kOpBitXor: return (U)(ua ^ ub);
    case kOpEq: return a == b;
    case kOpNeq: return a != b;
    case kOpLt: return a < b;
    case kOpLeq: return a <= b;
    case kOpGt: return a > b;
    case kOpGeq: return a >= b;
    default: return ua;
  }
}

DB_HD bool arith_is_cmp(int op) { return op >= kOpEq && op <= kOpGeq; }

// one operator instruction (not LOAD / SCALAR) on register values.  kWide = false: the program holds no 64-bit value (ArithProgram::
// wide), so integers are computed in 32 bits and the FLOAT64 code is left out.
template <bool kWide>
DB_HD uint64_t arith_apply(const ArithInstr &I, uint64_t a, uint64_t b, uint64_t c) {
  const int ct = I.ct, rt = I.rt;
  if (I.op == kOpCvt) return arith_cvt(a, ct, rt);
  if (I.op == kOpCast) return arith_cast(a, ct, rt);
  if (kWide && ct == kAF64) {
    if (arith_is_cmp(I.op)) return arith_fcmp<double>(I.op, arith_d(a), arith_d(b));
    return arith_ud(arith_fop<double>(I.op, arith_d(a), arith_d(b), arith_d(c)));
  }
  if (ct == kAF32 || ct == kAF16) {
    if (arith_is_cmp(I.op)) return arith_fcmp<float>(I.op, arith_f(a), arith_f(b));
    const float r = arith_fop<float>(I.op, arith_f(a), arith_f(b), arith_f(c));
    return arith_uf(ct == kAF16 ? arith_half_rne(r) : r);
  }
  uint64_t r;
  if (kWide) r = arith_is_signed(ct) ? arith_iop<int64_t>(I.op, (int64_t)a, (int64_t)b, (int64_t)c) : arith_iop<uint64_t>(I.op, a, b, c);
  else r = arith_is_signed(ct) ? arith_iop<int32_t>(I.op, (int32_t)a, (int32_t)b, (int32_t)c)
                               : arith_iop<uint32_t>(I.op, (uint32_t)a, (uint32_t)b, (uint32_t)c);
  return arith_is_cmp(I.op) ? r : arith_wrap(r, rt);
}

// the storage form of one element of type t from its raw bits (the low arith_size(t) bytes of raw)
DB_HD uint64_t arith_from_bits(uint64_t raw, int t) {
  switch (t) {
    case kAU8: case kABool: return (uint8_t)raw;
    case kAU16: return (uint16_t)raw;
    case kAU32: case kAF32: return (uint32_t)raw;
    case kAI8: return (uint64_t)(int64_t)(int8_t)raw;
    case kAI16: return (uint64_t)(int64_t)(int16_t)raw;
    case kAI32: return (uint64_t)(int64_t)(int32_t)raw;
    case kAF16: {                                                     // binary16 -> float32, exact
      const uint32_t h = (uint16_t)raw;
      const uint32_t s = (h & 0x8000u) << 16, e = (h >> 10) & 0x1Fu, m = h & 0x3FFu;
      if (e == 0x1Fu) return s | 0x7F800000u | (m << 13);
      if (e) return s | ((e + 112u) << 23) | (m << 13);
      return arith_uf(arith_f(s | 0x3F800000u) * ((float)m * 5.9604644775390625e-08f));
    }
    default: return raw;
  }
}

// the raw bits of a storage value of type t (a FLOAT16 value is a float32 that is exactly a binary16 value)
DB_HD uint64_t arith_to_bits(uint64_t v, int t) {
  if (t != kAF16) return v;
  const uint32_t b = (uint32_t)v, s = (b >> 16) & 0x8000u, a = b & 0x7FFFFFFFu;
  if (a >= 0x7F800000u) return s | 0x7C00u | (a > 0x7F800000u ? 0x200u | ((a >> 13) & 0x3FFu) : 0u);
  if (a >= 0x38800000u) return s | ((a - (112u << 23)) >> 13);
  return s | (uint32_t)(arith_f(a) * 16777216.0f);
}

DB_HD uint64_t arith_load(const void *p, int64_t k, int t) {
  const uint8_t *q = static_cast<const uint8_t *>(p) + k * arith_size(t);
  switch (arith_size(t)) {
    case 1: return arith_from_bits(*q, t);
    case 2: return arith_from_bits(*reinterpret_cast<const uint16_t *>(q), t);
    case 4: return arith_from_bits(*reinterpret_cast<const uint32_t *>(q), t);
    default: return arith_from_bits(*reinterpret_cast<const uint64_t *>(q), t);
  }
}

DB_HD void arith_store(void *p, int64_t k, int t, uint64_t v) {
  uint8_t *q = static_cast<uint8_t *>(p) + k * arith_size(t);
  const uint64_t b = arith_to_bits(v, t);
  switch (arith_size(t)) {
    case 1: *q = (uint8_t)b; break;
    case 2: *reinterpret_cast<uint16_t *>(q) = (uint16_t)b; break;
    case 4: *reinterpret_cast<uint32_t *>(q) = (uint32_t)b; break;
    default: *reinterpret_cast<uint64_t *>(q) = b; break;
  }
}

// element index inside operand j of output element e
DB_HD int64_t arith_index(const ArithSample &d, int j, int64_t e) {
  if ((d.linear >> j) & 1u) return e;
  int64_t idx = 0;
  for (int a = d.ndim - 1; a >= 0; a--) {
    const int64_t q = e / d.shape[a];
    idx += (e - q * d.shape[a]) * d.stride[j][a];
    e = q;
  }
  return idx;
}

#ifdef __CUDA_ARCH__
#define ARITH_UNROLL _Pragma("unroll")
#else
#define ARITH_UNROLL
#endif

// kArithEpt consecutive elements of type t starting at element e of p: one access of kArithEpt * size bytes (16 bytes for 4-byte
// types, two of 16 for 8-byte ones) when p + e is aligned to it, else element by element
struct alignas(16) ArithVec { uint64_t w[kArithEpt * 8 / 8]; };   // kArithEpt * 8 bytes: room for kArithEpt 8-byte elements
DB_HD bool arith_vec_ok(const void *p, int64_t e, int sz) {
  return ((uintptr_t)(static_cast<const uint8_t *>(p) + e * sz) & (uintptr_t)(kArithEpt * sz - 1)) == 0;
}
DB_HD void arith_load_run(const void *p, int64_t e, int t, uint64_t (&v)[kArithEpt]) {
  const int sz = arith_size(t);
  const uint8_t *q = static_cast<const uint8_t *>(p) + e * sz;
  ArithVec u;
  switch (sz) {
    case 1: u.w[0] = *reinterpret_cast<const uint32_t *>(q); break;
    case 2: u.w[0] = *reinterpret_cast<const uint64_t *>(q); break;
    case 4: { const ArithVec &a = *reinterpret_cast<const ArithVec *>(q); u.w[0] = a.w[0]; u.w[1] = a.w[1]; break; }
    default: {
      const ArithVec &a = *reinterpret_cast<const ArithVec *>(q);
      const ArithVec &b = *reinterpret_cast<const ArithVec *>(q + 16);
      u.w[0] = a.w[0]; u.w[1] = a.w[1]; u.w[2] = b.w[0]; u.w[3] = b.w[1];
      break;
    }
  }
  ARITH_UNROLL
  for (int k = 0; k < kArithEpt; k++) {
    const int bit = k * sz * 8;
    const uint64_t raw = sz == 8 ? u.w[k] : u.w[bit >> 6] >> (bit & 63);
    v[k] = arith_from_bits(raw, t);
  }
}
DB_HD void arith_store_run(void *p, int64_t e, int t, const uint64_t (&v)[kArithEpt]) {
  const int sz = arith_size(t);
  uint8_t *q = static_cast<uint8_t *>(p) + e * sz;
  ArithVec u;
  ARITH_UNROLL
  for (int k = 0; k < kArithEpt; k++) u.w[k] = 0;
  ARITH_UNROLL
  for (int k = 0; k < kArithEpt; k++) {
    const uint64_t b = arith_to_bits(v[k], t);
    const int bit = k * sz * 8;
    if (sz == 8) u.w[k] = b;
    else u.w[bit >> 6] |= (b & ((uint64_t{1} << (sz * 8)) - 1)) << (bit & 63);
  }
  switch (sz) {
    case 1: *reinterpret_cast<uint32_t *>(q) = (uint32_t)u.w[0]; break;
    case 2: *reinterpret_cast<uint64_t *>(q) = u.w[0]; break;
    case 4: { ArithVec &a = *reinterpret_cast<ArithVec *>(q); a.w[0] = u.w[0]; a.w[1] = u.w[1]; break; }
    default: {
      ArithVec &a = *reinterpret_cast<ArithVec *>(q);
      ArithVec &b = *reinterpret_cast<ArithVec *>(q + 16);
      a.w[0] = u.w[0]; a.w[1] = u.w[1]; b.w[0] = u.w[2]; b.w[1] = u.w[3];
      break;
    }
  }
}

// The value file of a thread: register j of the program holds r[j][0 .. kArithEpt).  It is only ever indexed with constants (the
// switches below dispatch on the instruction's register field, which is uniform across the block), so it stays in registers.
#define ARITH_REGS(X) X(0) X(1) X(2) X(3) X(4) X(5) X(6) X(7)
template <typename R>
DB_HD void arith_get(const R (&r)[kArithMaxRegs][kArithEpt], int j, R (&v)[kArithEpt]) {
  switch (j) {
#define ARITH_GET(J) case J: ARITH_UNROLL for (int k = 0; k < kArithEpt; k++) v[k] = r[J][k]; break;
    ARITH_REGS(ARITH_GET)
#undef ARITH_GET
    default: break;
  }
}
template <typename R>
DB_HD void arith_set(R (&r)[kArithMaxRegs][kArithEpt], int j, const R (&v)[kArithEpt]) {
  switch (j) {
#define ARITH_SET(J) case J: ARITH_UNROLL for (int k = 0; k < kArithEpt; k++) r[J][k] = v[k]; break;
    ARITH_REGS(ARITH_SET)
#undef ARITH_SET
    default: break;
  }
}
#undef ARITH_REGS

// a register value of type t held in R (uint32_t: the low word of the storage form) -> the storage form
template <typename R>
DB_HD uint64_t arith_widen(R x, int t) {
  return sizeof(R) == 8 || !arith_is_signed(t) ? (uint64_t)x : (uint64_t)(int64_t)(int32_t)(uint32_t)x;
}

// The common FLOAT operators and integer -> FLOAT conversions over a thread's kArithEpt values, dispatched once for all of them; the
// same arithmetic as arith_apply.  Returns false for every other instruction.
template <typename R>
DB_HD bool arith_apply_f32(const ArithInstr &I, const R (&a)[kArithEpt], const R (&b)[kArithEpt], const R (&c)[kArithEpt],
                              R (&v)[kArithEpt]) {
  if (I.rt != kAF32) return false;
  if (I.op == kOpCvt || I.op == kOpCast) {
    if (arith_is_float(I.ct) || arith_bits(I.ct) == 64) return false;
    const bool sgn = arith_is_signed(I.ct);
    ARITH_UNROLL
    for (int k = 0; k < kArithEpt; k++) v[k] = (R)arith_uf(sgn ? (float)(int32_t)(uint32_t)a[k] : (float)(uint32_t)a[k]);
    return true;
  }
  if (I.ct != kAF32) return false;
  float x[kArithEpt], y[kArithEpt], z[kArithEpt];
  ARITH_UNROLL
  for (int k = 0; k < kArithEpt; k++) { x[k] = arith_f(a[k]); y[k] = arith_f(b[k]); z[k] = arith_f(c[k]); }
  switch (I.op) {
#define ARITH_F32_CASE(OP, EXPR) case OP: { ARITH_UNROLL for (int k = 0; k < kArithEpt; k++) v[k] = (R)arith_uf(EXPR); return true; }
    ARITH_F32_CASE(kOpAdd, arith_fadd(x[k], y[k]))
    ARITH_F32_CASE(kOpSub, arith_fadd(x[k], -y[k]))
    ARITH_F32_CASE(kOpMul, arith_fmul(x[k], y[k]))
    ARITH_F32_CASE(kOpFdiv, x[k] / y[k])
    ARITH_F32_CASE(kOpMin, y[k] < x[k] ? y[k] : x[k])
    ARITH_F32_CASE(kOpMax, x[k] < y[k] ? y[k] : x[k])
    ARITH_F32_CASE(kOpClamp, x[k] < y[k] ? y[k] : (z[k] < x[k] ? z[k] : x[k]))
#undef ARITH_F32_CASE
    default: return false;
  }
}

// Elements base + tid * kArithEpt + k (k < kArithEpt, below end) of sample d: a thread takes kArithEpt consecutive elements, so that
// operands with the output's shape are read and the output written with one vector access per thread and instruction, and every
// instruction is decoded once per kArithEpt elements.  kWide must be p.wide: without 64-bit values the value file is 32 bits wide.
template <bool kWide>
DB_HD void arith_elements(const ArithProgram &p, const ArithSample &d, int64_t base, int64_t end, int tid) {
  typedef typename std::conditional<kWide, uint64_t, uint32_t>::type R;
  const int64_t e0 = base + (int64_t)tid * kArithEpt;
  if (e0 >= end) return;
  const bool full = e0 + kArithEpt <= end;
  R r[kArithMaxRegs][kArithEpt] = {};
  for (int i = 0; i < p.ninstr; i++) {
    const ArithInstr I = p.ins[i];
    R v[kArithEpt];
    if (I.op == kOpLoad) {
      const void *src = d.in[I.a];
      uint64_t w[kArithEpt];
      if (full && ((d.linear >> I.a) & 1u) && arith_vec_ok(src, e0, arith_size(I.ct))) {
        arith_load_run(src, e0, I.ct, w);
      } else {
        ARITH_UNROLL
        for (int k = 0; k < kArithEpt; k++) w[k] = e0 + k < end ? arith_load(src, arith_index(d, I.a, e0 + k), I.ct) : 0;
      }
      ARITH_UNROLL
      for (int k = 0; k < kArithEpt; k++) v[k] = (R)w[k];
    } else if (I.op == kOpScalar) {
      const R s = (R)d.scal[I.a];
      ARITH_UNROLL
      for (int k = 0; k < kArithEpt; k++) v[k] = s;
    } else {
      R a[kArithEpt], b[kArithEpt], c[kArithEpt];
      arith_get(r, I.a, a);
      arith_get(r, I.b, b);
      arith_get(r, I.c, c);
      if (!arith_apply_f32(I, a, b, c, v)) {
        ARITH_UNROLL
        for (int k = 0; k < kArithEpt; k++)
          v[k] = (R)arith_apply<kWide>(I, arith_widen(a[k], I.ct), arith_widen(b[k], I.ct), arith_widen(c[k], I.ct));
      }
    }
    arith_set(r, I.dst, v);
  }
  R o[kArithEpt];
  arith_get(r, p.out_reg, o);
  uint64_t v[kArithEpt];
  ARITH_UNROLL
  for (int k = 0; k < kArithEpt; k++) v[k] = arith_widen(o[k], p.out_type);
  if (full && arith_vec_ok(d.out, e0, arith_size(p.out_type))) {
    arith_store_run(d.out, e0, p.out_type, v);
  } else {
    for (int k = 0; k < kArithEpt && e0 + k < end; k++) arith_store(d.out, e0 + k, p.out_type, v[k]);
  }
}

}  // namespace dalib200

#endif  // DALI_B200_CSRC_ARITH_CORE_H_
