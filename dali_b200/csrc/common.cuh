// dali_b200/csrc/common.cuh -- shared host/device helpers for the sm_90a kernels.
#ifndef DALI_B200_CSRC_COMMON_CUH_
#define DALI_B200_CSRC_COMMON_CUH_

#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <atomic>
#include <cstdio>
#include <cstdarg>
#include <string>
#include <utility>
#include <vector>
#include "../../include/dali_b200.h"
#include "host_device.h"

namespace dalib200 {

// ---------------------------------------------------------------------------------------------
// error plumbing (thread-local message, as the reference C API does: dali/c_api_2/error_handling.cc)
void SetLastError(const char *fmt, ...);
extern std::atomic<uint64_t> g_launch_count;   // dalib200GetLaunchCount

#define DB_CHECK_ARG(cond, ...)                                   \
  do { if (!(cond)) { ::dalib200::SetLastError(__VA_ARGS__); return DALIB200_ERROR_INVALID_ARGUMENT; } } while (0)

#define DB_CUDA(call)                                                                           \
  do { cudaError_t e__ = (call); if (e__ != cudaSuccess) {                                      \
    ::dalib200::SetLastError("CUDA error %s at %s:%d (%s)", cudaGetErrorName(e__), __FILE__, __LINE__, \
                             cudaGetErrorString(e__));                                          \
    return DALIB200_ERROR_CUDA; } } while (0)

int NumSMs();

// Launch shape of a kernel whose working lanes each run one serial chain (tiff_segment, webp_entropy): one warp per CTA and `lanes`
// working lanes in each warp (the others return).  Serial chains diverge from each other at once, so lanes of one warp share its issue
// slots: with few chains every chain gets a warp of its own, spread over all SMs; with more chains than resident warps, the warps fill
// up to 32 lanes.  At most `max_workers` lanes in all.
struct SerialLanes { int warps, lanes; };
SerialLanes SerialLaneGeometry(int nchains, int max_workers);

// Optional per-launch timing (CUDA events on the launching stream), switched on by dalib200ProfilingEnable.
// bench.py uses it to time the dominant kernel live inside the timed region.  Launch (below) brackets every launch with them.
void ProfBegin(const char *name, cudaStream_t s);
void ProfEnd(cudaStream_t s);

// ---------------------------------------------------------------------------------------------
// numerics shared by the kernels -- these restate the reference HOST (CPU backend) conventions,
// which are the parity target (SURVEY.md Appendix C).
#ifdef __CUDACC__

// include/dali/core/convert.h:306-324: host ConvertSat<uint8_t>(float) = clamp(std::round(x)) -- half AWAY.
__device__ __forceinline__ uint8_t sat_u8_half_away(float x) {
  // All on the FMA / ALU pipes (FRND and F2I run on the quarter-rate conversion pipe): x + 1.5 * 2^23 rounds x to the nearest
  // integer, ties to EVEN, in the low mantissa bits; the exact remainder d = x - rne(x) tells a tie that went down (d == 0.5),
  // which round-half-AWAY sends up instead.  Ties of negative x only matter below the clamp (result 0 either way).
  x = fminf(fmaxf(x, -1.0f), 256.0f);
  const float y = __fadd_rn(x, 12582912.0f);
  const float d = __fsub_rn(x, __fsub_rn(y, 12582912.0f));
  int i = __float_as_int(y) - 0x4B400000 + (d == 0.5f ? 1 : 0);
  return (uint8_t)min(max(i, 0), 255);
}
// The same conversion for values already known to lie in (-0.5, 255.5) (e.g. bilinear blends of bytes): setting the lowest mantissa
// bit moves exactly the ties (x.5, whose lowest bit is clear) just above the midpoint, so one round-to-nearest-EVEN addition of
// 1.5 * 2^23 leaves round-half-AWAY(x) in the low byte of the sum.  2 instructions; checked against sat_u8_half_away over the whole
// range by dalib200DebugCheckHalfConversion.  Returns the sum's bits: the caller takes byte 0 (e.g. with a PRMT while packing).
__device__ __forceinline__ uint32_t round_u8_bits(float x) {
  return __float_as_uint(__fadd_rn(__uint_as_float(__float_as_uint(x) | 1u), 12582912.0f));
}
// dali/kernels/common/simd.h:233-263: the SSE2 store path rounds half to EVEN (cvtps2dq) then saturates.
__device__ __forceinline__ uint8_t sat_u8_half_even(float x) {
  x = fminf(fmaxf(x, 0.0f), 255.0f);
  return (uint8_t)__float2int_rn(x);
}

// include/dali/util/half.hpp:464-540 (HALF_ROUND_STYLE=1, HALF_ROUND_TIES_TO_EVEN=0 at :233,:242):
// float -> half, round to nearest, ties AWAY from zero; after the +-65504 clamp of
// include/dali/core/convert.h:168-176.
// This is the integer restatement; the kernels use float2half_ties_away below (one hardware conversion), which
// dalib200DebugCheckHalfConversion proves identical for all 2^32 inputs.
__device__ __forceinline__ uint16_t float2half_ties_away_ref(float f) {
  f = fminf(fmaxf(f, -65504.0f), 65504.0f);     // NaN propagates through fminf/fmaxf as the other operand: documented deviation
  const uint32_t bits = __float_as_uint(f);
  const uint32_t sign = (bits >> 16) & 0x8000u, abits = bits & 0x7FFFFFFFu;
  if (abits >= (113u << 23)) {
    // normal half: rebias the exponent and add half an ulp of the half format (bit 12) before truncating -- the carry runs
    // into the exponent exactly like the generic formula below (base + (mant >> 13) + ((mant >> 12) & 1))
    return (uint16_t)(sign | ((abits - (112u << 23) + 0x1000u) >> 13));
  }
  const uint32_t e = abits >> 23, mant = abits & 0x7FFFFFu;
  uint32_t base, shift;
  if (e < 103u)       { base = 0u; shift = 24u; }
  else                { base = 1u << (e - 103u); shift = 126u - e; }     // 103 <= e < 113: subnormal half
  const uint32_t h = sign + base + (mant >> shift);
  const uint32_t rnd = ((mant >> (shift - 1u)) | (uint32_t)(e == 102u)) & 1u;
  return (uint16_t)(h + rnd);
}

// Ties-away through the hardware's round-to-nearest-EVEN conversion: a tie has at least its lowest mantissa bit clear (13+ dropped
// bits of the form 10...0), so setting bit 0 moves exactly the ties just above the midpoint and leaves every other value on its side
// of every midpoint.  3 instructions instead of ~15.
__device__ __forceinline__ uint16_t float2half_ties_away(float f) {
  f = fminf(fmaxf(f, -65504.0f), 65504.0f);
  const float g = __uint_as_float(__float_as_uint(f) | 1u);
  unsigned short h;
  asm("cvt.rn.f16.f32 %0, %1;" : "=h"(h) : "f"(g));
  return h;
}

// exact u8 -> f32 on the ALU/FMA pipes (no I2F): 0x4B000000 | b is the float 2^23 + b
__device__ __forceinline__ float u8_to_float(uint32_t b) { return __uint_as_float(0x4B000000u | b) - 8388608.0f; }

template <typename T> struct OutConv;
template <> struct OutConv<float> {
  __device__ __forceinline__ static float cvt(float v) { return v; }
};
template <> struct OutConv<uint16_t> {   // float16 bits
  __device__ __forceinline__ static uint16_t cvt(float v) { return float2half_ties_away(v); }
};

// mul and add that the compiler may NOT contract into an FMA: the reference CPU binary targets
// baseline x86-64 (no FMA), so a*b+c is rounded twice there.
__device__ __forceinline__ float mul_rn(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ float add_rn(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ float sub_rn(float a, float b) { return __fsub_rn(a, b); }

// Pre-emphasised sample i of a signal of `len` (>= 1) samples: x[i] - c * x[i - 1] with x[-1] = 0 / x[0] / x[1] for the
// DALIB200_BORDER_ZERO / CLAMP / REFLECT rule (x[0] when len == 1), rounded twice; c == 0 copies.  The stand-alone
// PreemphasisFilter kernel and the spectrogram's fused framing both evaluate it, so the two paths agree bit for bit.
template <typename T>
__device__ __forceinline__ float preemph_at(const T *__restrict__ x, int64_t i, int64_t len, float c, int border) {
  const float v = (float)__ldg(x + i);
  if (c == 0.0f) return v;
  float p;
  if (i > 0) p = (float)__ldg(x + i - 1);
  else p = border == DALIB200_BORDER_ZERO ? 0.0f : (border == DALIB200_BORDER_CLAMP || len < 2) ? v : (float)__ldg(x + 1);
  return __fsub_rn(v, __fmul_rn(c, p));
}

__device__ __forceinline__ uint32_t ld_nc_u32(const uint32_t *p) {
  uint32_t v;
  asm volatile("ld.global.nc.u32 %0, [%1];" : "=r"(v) : "l"(p));
  return v;
}

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
// ---- shared-memory accesses through 32-bit shared-window addresses.  Hot loops that reach shared memory through generic
// pointers make the compiler re-derive the shared window base (S2R SR_CgaCtaId / MOV / LEA) next to every access; a plain
// integer address costs nothing.  The asm is volatile: it must stay behind the barrier that published the data.
__device__ __forceinline__ uint32_t lds_u32(uint32_t a) { uint32_t v; asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(a)); return v; }
__device__ __forceinline__ uint32_t lds_u16(uint32_t a) { unsigned short v; asm volatile("ld.shared.u16 %0, [%1];" : "=h"(v) : "r"(a)); return v; }
__device__ __forceinline__ uint32_t lds_u8(uint32_t a) { uint32_t v; asm volatile("ld.shared.u8 %0, [%1];" : "=r"(v) : "r"(a)); return v; }
__device__ __forceinline__ void sts_u32(uint32_t a, uint32_t v) { asm volatile("st.shared.u32 [%0], %1;" :: "r"(a), "r"(v) : "memory"); }
__device__ __forceinline__ void sts_u16(uint32_t a, uint32_t v) { asm volatile("st.shared.u16 [%0], %1;" :: "r"(a), "h"((unsigned short)v) : "memory"); }

// ---- mbarrier + TMA bulk copy (cp.async.bulk, sm_90+ PTX): shared by the resample ring and the warp source tiles
__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t *bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" :: "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity) {
  asm volatile("{\n\t.reg .pred p;\n\tWAIT_%=:\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t@p bra DONE_%=;\n\tbra WAIT_%=;\n\tDONE_%=:\n\t}"
               :: "r"(smem_u32(bar)), "r"(parity) : "memory");
}
// the same wait for a lone producer lane: it backs off between polls -- a spinning try_wait loop of one lane takes issue slots
// of resample_stream_kernel on the scheduler it shares with two consumer warps
__device__ __forceinline__ void mbar_wait_backoff(uint64_t *bar, uint32_t parity) {
  uint32_t done = 0;
  for (;;) {
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                 : "=r"(done) : "r"(smem_u32(bar)), "r"(parity) : "memory");
    if (done) break;
    __nanosleep(200);
  }
}
__device__ __forceinline__ void bulk_g2s(void *dst, const void *src, uint32_t bytes, uint64_t *bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               :: "r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}

// TMA tiled load through a tensor map (cuTensorMapEncodeTiled): a boxDim[0] x boxDim[1] x 1 tile of a rank-3 tensor at element
// coordinates (c0, c1, c2) into shared memory; out-of-range parts of the box are zero filled by the unit.  SASS: UTMALDG.3D.
__device__ __forceinline__ void tma_load_3d(void *dst, const void *tmap, int c0, int c1, int c2, uint64_t *bar) {
  asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];"
               :: "r"(smem_u32(dst)), "l"(tmap), "r"(c0), "r"(c1), "r"(c2), "r"(smem_u32(bar)) : "memory");
}

// Every kernel launch of the library goes through here: an NVTX range and, with profiling on, one timing record under `name`
// around the launch, and one count in dalib200GetLaunchCount.  So the count and the records are the launches, one each.
template <typename... P, typename... A>
inline void Launch(const char *name, void (*kernel)(P...), dim3 grid, dim3 block, size_t smem, cudaStream_t s, A &&...args) {
  ProfBegin(name, s);
  kernel<<<grid, block, smem, s>>>(std::forward<A>(args)...);
  ProfEnd(s);
  g_launch_count.fetch_add(1, std::memory_order_relaxed);
}

#endif  // __CUDACC__

}  // namespace dalib200

// Host-only declarations: kept at the end of the header so that the line tables of the device code above do not move.
#include <algorithm>
#include <cstring>
#include <exception>
#include <new>
#include <tuple>
namespace dalib200 {
inline size_t Align(size_t v, size_t a) { return (v + a - 1) / a * a; }

// Grow-only pinned host memory that per-batch data is staged in for asynchronous copies to the device.  It keeps the one rule that
// makes reusing it safe: the host side is not rewritten while a copy may still be reading it.  Stage() hands the host side out only
// after the copies covered by the last Record() have finished.  The event behind that is created at the first Record().
class PinnedStage {
 public:
  // Waits for the last recorded copies, grows the buffer to at least `bytes` (doubling from 4 KiB; a grown buffer does not keep its
  // contents) and sets *host to its host side.
  template <typename T> int Stage(size_t bytes, T **host) {
    const int rc = Grow(bytes, nullptr);
    *host = reinterpret_cast<T *>(host_);
    return rc;
  }
  int Record(cudaStream_t s);   // after the caller's copies out of the buffer are enqueued on s
  void Free();                  // waits for the last recorded copies, then frees the buffer and the event

 protected:
  int Grow(size_t bytes, uint8_t **dev);   // Stage's wait and growth; grows *dev to the same capacity when dev is given
  uint8_t *host_ = nullptr;
  size_t cap_ = 0;

 private:
  cudaEvent_t uploaded_ = nullptr;
  bool pending_ = false;
};

// A pinned stage with a device copy of the same capacity, for per-batch descriptors: one H2D copy per launch.
class DescArena : public PinnedStage {
 public:
  uint8_t *dev = nullptr;
  int Reserve(size_t bytes) { return Grow(bytes, &dev); }    // Stage without the host pointer (e.g. max_batch at plan creation)
  template <typename T> int Stage(size_t bytes, T **host) {
    const int rc = Reserve(bytes);
    *host = reinterpret_cast<T *>(host_);
    return rc;
  }
  int Upload(size_t bytes, cudaStream_t s);   // async H2D of the first `bytes`, then Record(s)
  void Free();
  // Stages the vectors back to back, each at a 16-byte boundary, uploads them on s and points each of `dev` at its vector's copy:
  //   arena.Pack(s, std::tie(d_images, d_chunks), images, chunks)
  template <typename... T> int Pack(cudaStream_t s, std::tuple<const T *&...> out, const std::vector<T> &...v) {
    size_t off[sizeof...(T)], bytes = 0, k = 0;
    ((off[k++] = bytes, bytes = Align(bytes + sizeof(T) * v.size(), 16)), ...);
    uint8_t *h;
    if (int rc = Stage(bytes, &h)) return rc;
    k = 0;
    (memcpy(h + off[k++], v.data(), sizeof(T) * v.size()), ...);
    if (int rc = Upload(bytes, s)) return rc;
    k = 0;
    std::apply([&](auto &...d) { ((d = reinterpret_cast<std::remove_reference_t<decltype(d)>>(dev + off[k++])), ...); }, out);
    return DALIB200_SUCCESS;
  }
};

// A grow-only device buffer of `cap` elements: when `need` exceeds it, it is replaced (contents not kept) by one of need + need / 4,
// at least 4096, elements.  cudaFree waits for the device, so launches still reading the old buffer finish first.
template <typename T>
int GrowDevice(T *&ptr, size_t &cap, size_t need) {
  if (need <= cap) return DALIB200_SUCCESS;
  const size_t ncap = std::max(need + need / 4, (size_t)4096);
  if (ptr) cudaFree(ptr);
  ptr = nullptr; cap = 0;
  DB_CUDA(cudaMalloc(reinterpret_cast<void **>(&ptr), ncap * sizeof(T)));
  cap = ncap;
  return DALIB200_SUCCESS;
}

// a * b * c < 2^31 for non-negative extents, without overflowing on the way (the kernels index a sample with 32-bit arithmetic)
inline bool ElementsFit31(int64_t a, int64_t b, int64_t c) {
  const int64_t lim = (int64_t{1} << 31) - 1;
  if (a < 0 || b < 0 || c < 0) return false;
  if (a == 0 || b == 0 || c == 0) return true;
  if (a > lim / b) return false;
  return a * b <= lim / c;
}
}  // namespace dalib200
// The C-ABI never lets a C++ exception escape (std::bad_alloc / std::length_error from a host-side table of absurd size would otherwise
// terminate the caller's process): every entry point is a function-try-block closed by this handler.
#define DB_API_CATCH                                                                                                       \
  catch (const std::bad_alloc &) { ::dalib200::SetLastError("out of host memory"); return DALIB200_ERROR_INTERNAL; }      \
  catch (const std::exception &e__) { ::dalib200::SetLastError("unexpected C++ exception: %s", e__.what()); return DALIB200_ERROR_INTERNAL; } \
  catch (...) { ::dalib200::SetLastError("unexpected C++ exception"); return DALIB200_ERROR_INTERNAL; }

#endif  // DALI_B200_CSRC_COMMON_CUH_
