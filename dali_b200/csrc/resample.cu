// dali_b200/csrc/resample.cu -- fused two-pass separable resampling for sm_90a.
//
// Parity target: the reference CPU kernel SeparableResampleCPU (dali/kernels/imgproc/resample/
// separable_cpu.h:149-249) driven by SeparableResamplingSetup<2>::SetupSample (resampling_setup.cc:271-337):
//   * per-axis filter choice / radius / LUT rescale            (resampling_setup.cc:27-76, params.h:40-56,
//                                                                resampling_filters.cu:66-142)
//   * pass order from the cost model                            (resampling_setup.cc:131-192)
//   * coefficient tables: idx = ceil(x*scale + s0), c_k = f((idx - sx + k)*fscale), normalised BEFORE
//     accumulation                                              (resampling_impl_cpu.cc:22-47)
//   * acc = sum_k c_k * src[clamp(idx+k)]   k ascending, mul and add rounded separately (SSE2, no FMA)
//   * fp32 intermediate between the passes; final u8 store rounds half-to-even where the reference runs
//     its SSE path and half-away in its scalar tails            (simd.h:233-263, convert.h:306-324,
//                                                                resampling_impl_cpu.h:95-124,126-222,245-336)
// The reference GPU kernel (resampling_impl.cuh) normalises after accumulation with FMAs and writes
// the fp32 intermediate to HBM; here BOTH passes of an output tile run in one CTA with the
// intermediate held in shared memory, so HBM sees the input once and the output once.
//
// Algorithmic bytes per unit (SURVEY.md 8d): in_h*in_w*C*sizeof(In) + out_h*out_w*C*sizeof(Out).
// The per-axis host setup (filters, pass order, tables) is resample_axis.h, shared with the 3-D resampler.
#include "common.cuh"
#include "resample_axis.h"
#include <algorithm>
#include <cmath>
#include <cstring>
#include <map>
#include <tuple>

namespace dalib200 {

constexpr int kTmpFloats = 24 * 1024;     // 96 KB of fp32 intermediate per CTA -> 2 CTAs / SM
constexpr int kMaxTileH = 16;             // output rows per tile in the vertical-first order
constexpr int kMaxSupportSmem = 64;       // vertical taps whose coefficients are staged in smem
constexpr int kTileTableBytes = kMaxTileH * kMaxSupportSmem * 8;   // offsets (in 4-byte words) into the table arena
constexpr int kWalkMax = 96;              // steps (source rows incl. border repeats) of one tile's row walk
constexpr int kWalkSlots = 4;             // output rows that may be "open" at the same source row
constexpr int kWalkWords = 3;             // 32-bit word columns per thread
static_assert(kWalkMax * kWalkSlots * 16 + kWalkMax * 8 <= kTileTableBytes, "walk tables must fit the tile table area");

struct RsDesc {
  const void *in;
  void *out;
  int32_t in_h, in_w, C, out_h, out_w;
  int32_t vfirst;
  int32_t idx_off[2], coef_off[2], support[2], base[2], extent[2];   // [0] = x, [1] = y
  int32_t flags_off;         // per-output-column rounding flags (horizontal last pass, u8 out) or -1
  int32_t simd_flat_end;     // vertical last pass, u8 out: flat x*C+c < this -> half-to-even
  int32_t tile_h, tile_w, tiles_x, tiles_y;
  int32_t aligned4;          // input base and row pitch are multiples of 4 bytes (filled at launch)
  float neg_zero;            // -0.0f, read at run time: an addend ptxas cannot fold (see stage B of resample_stream_kernel)
  int32_t use_stream;        // this sample is processed by resample_stream_kernel (decided at launch)
  int32_t tile_walk;         // the tile kernel may use the row walk (tile step count fits)
  int32_t walk_slots;        // > 0: vertical pass by the row walk with this many accumulator slots (see walk_vertical_u8)
  int32_t walk_off;          // streamed samples: per-chunk offsets of the walk records in the table arena (see BuildWalkRecords)
  int64_t first_tile;
  // planar 4:2:0 YCbCr source (decoder planes, see resample_planar_kernel): the sample is the window [crop_y, +in_h) x [crop_x, +in_w)
  // of an img_h x img_w image
  const uint8_t *pl[3];
  int32_t pitch_y, pitch_c, img_w, img_h, crop_x, crop_y;
};

// ---------------------------------------------------------------------------------------------
// device

template <typename T> __device__ __forceinline__ float ld_as_float(const T *p);
template <> __device__ __forceinline__ float ld_as_float<uint8_t>(const uint8_t *p) { return (float)__ldg(p); }
template <> __device__ __forceinline__ float ld_as_float<float>(const float *p) { return __ldg(p); }

template <typename Out> __device__ __forceinline__ Out rs_store_cvt(float v, bool half_even);
template <> __device__ __forceinline__ float rs_store_cvt<float>(float v, bool) { return v; }
template <> __device__ __forceinline__ uint8_t rs_store_cvt<uint8_t>(float v, bool half_even) {
  return half_even ? sat_u8_half_even(v) : sat_u8_half_away(v);
}


// ---- fp32 pairs: two independent IEEE mul / add / fma, each rounded once, never contracted (sm_90a has no packed f32x2
// instructions, so each pair is two scalar instructions)
__device__ __forceinline__ float2 mul2_rn(float2 a, float2 b) {
  return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y));
}
__device__ __forceinline__ float2 add2_rn(float2 a, float2 b) {
  return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y));
}
// exact u8 -> f32 without the (slow) I2F pipe: 0x4B000000 | b is the float 2^23 + b; subtracting 2^23 is exact
__device__ __forceinline__ float2 bytes01_to_float(uint32_t w) {
  const float2 m = make_float2(__uint_as_float(__byte_perm(w, 0x4B000000u, 0x7440)), __uint_as_float(__byte_perm(w, 0x4B000000u, 0x7441)));
  return add2_rn(m, make_float2(-8388608.0f, -8388608.0f));
}
__device__ __forceinline__ float2 bytes23_to_float(uint32_t w) {
  const float2 m = make_float2(__uint_as_float(__byte_perm(w, 0x4B000000u, 0x7442)), __uint_as_float(__byte_perm(w, 0x4B000000u, 0x7443)));
  return add2_rn(m, make_float2(-8388608.0f, -8388608.0f));
}

__device__ __forceinline__ float2 fma2_rn(float2 a, float2 b, float2 c) {
  return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y));
}

// ---------------------------------------------------------------------------------------------
// Vertical pass of a tile as a ROW WALK (u8 input, 32-bit aligned rows).
//
// The tile's output rows t = 0..th-1 read the (unclamped) source rows u in [idx[t], idx[t] + Sy).  Instead of gathering the
// Sy taps of every output row (each source row is then fetched and converted ~Sy/scale times), the walk visits the source
// rows umin..umax ONCE, in ascending order, and adds each of them into the output rows that are open at that row: output
// row t lives in accumulator slot t % W, where W (host-checked) guarantees that rows t and t + W are never open together.
// Ascending u is ascending k for every t, so the accumulation order of the reference (k = 0..Sy-1) is kept; clamped border
// rows are simply visited once per unclamped u.
//
// The product is formed WITHOUT converting the byte: m = 2^23 + b (a PRMT), then fma(m, c, -2^23 c) = RN(b * c) exactly
// (the FMA is exact before its single rounding and 2^23 c is a power-of-two multiple of c), i.e. the reference's separately
// rounded mul; the sum is a separate add.rn -- two roundings, like SSE2 mulps + addps.  (fma followed by add cannot be
// contracted.)
struct WalkTables {
  float4 ent[kWalkMax][kWalkSlots];     // (c, c, -2^23 c, -2^23 c) of the tap that slot s takes from step j, or zeros
  int32_t row[kWalkMax];                // absolute clamped source row of step j
  uint32_t fin[kWalkMax];               // byte s = output row (tile-local) that slot s completes at step j, 0xFF = none
};

__device__ __forceinline__ void walk_vertical_u8(const uint8_t *__restrict__ in8, int64_t pitch, int words, int row_elems,
                                                 int th, int Sy, int W, const int32_t *__restrict__ idx_y,
                                                 const float *__restrict__ coef_y, int oy0, int by, int ey,
                                                 float *__restrict__ tmp, WalkTables *__restrict__ wt) {
  const int ia = idx_y[oy0], ib = idx_y[oy0 + th - 1];
  const int umin = min(ia, ib), J = max(ia, ib) + Sy - umin;
  for (int e = threadIdx.x; e < J * kWalkSlots; e += blockDim.x) (&wt->ent[0][0])[e] = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int j = threadIdx.x; j < J; j += blockDim.x) { wt->row[j] = by + min(max(umin + j, 0), ey - 1); wt->fin[j] = 0xFFFFFFFFu; }
  __syncthreads();
  for (int e = threadIdx.x; e < th * Sy; e += blockDim.x) {
    const int t = e / Sy, k = e - t * Sy;
    const int j = idx_y[oy0 + t] + k - umin, s = t % W;
    const float c = coef_y[(int64_t)(oy0 + t) * Sy + k];
    const float d = mul_rn(c, -8388608.0f);
    wt->ent[j][s] = make_float4(c, c, d, d);
    if (k == Sy - 1) reinterpret_cast<uint8_t *>(&wt->fin[j])[s] = (uint8_t)t;
  }
  __syncthreads();
  constexpr int G = 4, NW = kWalkWords;
  for (int jw0 = threadIdx.x; jw0 < words; jw0 += blockDim.x * NW) {
    const uint8_t *colp[NW];
    bool okw[NW];
#pragma unroll
    for (int q = 0; q < NW; q++) { okw[q] = jw0 + q * (int)blockDim.x < words; colp[q] = in8 + 4 * (jw0 + (okw[q] ? q * (int)blockDim.x : 0)); }
    float2 acc[kWalkSlots][NW][2];
#pragma unroll
    for (int s = 0; s < kWalkSlots; s++)
#pragma unroll
      for (int q = 0; q < NW; q++) acc[s][q][0] = acc[s][q][1] = make_float2(0.f, 0.f);
    uint32_t wa[G][NW], wb[G][NW];
    auto load = [&](uint32_t (&w)[G][NW], int j0) {
#pragma unroll
      for (int g = 0; g < G; g++) {
        if (j0 + g < J) {
          const int64_t ro = (int64_t)wt->row[j0 + g] * pitch;
#pragma unroll
          for (int q = 0; q < NW; q++) w[g][q] = ld_nc_u32(reinterpret_cast<const uint32_t *>(colp[q] + ro));
        }
      }
    };
    auto process = [&](const uint32_t (&w)[G][NW], int j0) {
#pragma unroll
      for (int g = 0; g < G; g++) {
        const int j = j0 + g;
        if (j < J) {
          float2 m[NW][2];
#pragma unroll
          for (int q = 0; q < NW; q++) {
            m[q][0] = make_float2(__uint_as_float(__byte_perm(w[g][q], 0x4B000000u, 0x7440)), __uint_as_float(__byte_perm(w[g][q], 0x4B000000u, 0x7441)));
            m[q][1] = make_float2(__uint_as_float(__byte_perm(w[g][q], 0x4B000000u, 0x7442)), __uint_as_float(__byte_perm(w[g][q], 0x4B000000u, 0x7443)));
          }
#pragma unroll
          for (int s = 0; s < kWalkSlots; s++) {
            if (s < W) {
              const float4 e = wt->ent[j][s];
              if (e.x != 0.0f) {
                const float2 c2 = make_float2(e.x, e.y), d2 = make_float2(e.z, e.w);
#pragma unroll
                for (int q = 0; q < NW; q++) {
                  acc[s][q][0] = add2_rn(acc[s][q][0], fma2_rn(m[q][0], c2, d2));
                  acc[s][q][1] = add2_rn(acc[s][q][1], fma2_rn(m[q][1], c2, d2));
                }
              }
            }
          }
          const uint32_t f = wt->fin[j];
          if (f != 0xFFFFFFFFu) {
#pragma unroll
            for (int s = 0; s < kWalkSlots; s++) {
              const uint32_t t = (f >> (8 * s)) & 0xFFu;
              if (t != 0xFFu) {
#pragma unroll
                for (int q = 0; q < NW; q++) {
                  if (okw[q])
                    *reinterpret_cast<float4 *>(tmp + t * row_elems + 4 * (jw0 + q * (int)blockDim.x)) =
                        make_float4(acc[s][q][0].x, acc[s][q][0].y, acc[s][q][1].x, acc[s][q][1].y);
                  acc[s][q][0] = acc[s][q][1] = make_float2(0.f, 0.f);
                }
              }
            }
          }
        }
      }
    };
    load(wa, 0);
    for (int j0 = 0; j0 < J; j0 += 2 * G) {
      load(wb, j0 + G);
      process(wa, j0);
      load(wa, j0 + 2 * G);
      process(wb, j0 + G);
    }
  }
}

// One CTA = one output tile of one sample.  smem: fp32 intermediate of the tile.
template <typename In, typename Out>
__global__ void __launch_bounds__(256) resample_fused_kernel(const RsDesc *__restrict__ descs, const int32_t *__restrict__ tab,
                                                             int n, int64_t total_tiles) {
  extern __shared__ __align__(16) float tmp[];
  for (int64_t tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
    const int s = last_at_most(descs, 0, n - 1, tile, [](const RsDesc &d) { return d.first_tile; });
    const RsDesc &d = descs[s];
    if (d.use_stream) continue;
    const int64_t tl = tile - d.first_tile;
    const int ty = (int)((uint32_t)tl / (uint32_t)d.tiles_x), tx = (int)((uint32_t)tl - (uint32_t)ty * (uint32_t)d.tiles_x);
    const int oy0 = ty * d.tile_h, ox0 = tx * d.tile_w;
    const int th = min(d.tile_h, d.out_h - oy0), tw = min(d.tile_w, d.out_w - ox0);
    const int C = d.C;
    const int Sx = d.support[0], Sy = d.support[1];
    const int32_t *idx_x = tab + d.idx_off[0], *idx_y = tab + d.idx_off[1];
    const float *coef_x = reinterpret_cast<const float *>(tab + d.coef_off[0]);
    const float *coef_y = reinterpret_cast<const float *>(tab + d.coef_off[1]);
    const int bx = d.base[0], ex = d.extent[0], by = d.base[1], ey = d.extent[1];
    const In *in = static_cast<const In *>(d.in);
    Out *out = static_cast<Out *>(d.out);
    const int64_t pitch = (int64_t)d.in_w * C;
    const uint8_t *flags = d.flags_off >= 0 ? reinterpret_cast<const uint8_t *>(tab + d.flags_off) : nullptr;

    if (d.vfirst) {
      // absolute column span needed by this tile (indices are monotonic in x)
      const int ia = idx_x[ox0], ib = idx_x[ox0 + tw - 1];
      const int cmin = bx + min(max(min(ia, ib), 0), ex - 1);
      const int cmax = bx + min(max(max(ia, ib) + Sx - 1, 0), ex - 1);
      // byte span of a row, widened to whole 32-bit words (stays inside the row: pitch % 4 == 0 on the fast path)
      const bool fast = sizeof(In) == 1 && d.aligned4;
      const int e0 = fast ? ((cmin * C) & ~3) : cmin * C;
      const int e1 = fast ? (((cmax + 1) * C + 3) & ~3) : (cmax + 1) * C;
      const int row_elems = e1 - e0;
      // ---- per-tile tables in smem: vertical coefficients and clamped source rows of the th output rows
      float *s_cy = tmp + kTmpFloats;
      int *s_row = reinterpret_cast<int *>(s_cy + kMaxTileH * kMaxSupportSmem);
      const bool tables = Sy <= kMaxSupportSmem;
      const bool walk = fast && d.tile_walk;
      if (walk) {
        walk_vertical_u8(reinterpret_cast<const uint8_t *>(in) + e0, pitch, row_elems >> 2, row_elems, th, Sy, d.walk_slots, idx_y, coef_y,
                         oy0, by, ey, tmp, reinterpret_cast<WalkTables *>(s_cy));
      } else if (tables) {
        for (int e = threadIdx.x; e < th * Sy; e += blockDim.x) {
          const int t = e / Sy, k = e - t * Sy;
          s_cy[e] = coef_y[(int64_t)(oy0 + t) * Sy + k];
          s_row[e] = by + min(max(idx_y[oy0 + t] + k, 0), ey - 1);
        }
        __syncthreads();
      }
      if (walk) {
        // done above
      } else if (fast && tables) {
        // stage A (fast): one thread = one 32-bit word column, all th output rows; u8 -> f32 via byte_perm,
        // separately rounded mul / add (two roundings, exactly like the reference's SSE mul + add)
        const int words = row_elems >> 2;
        const uint8_t *in8 = reinterpret_cast<const uint8_t *>(in) + e0;
        for (int jw = threadIdx.x; jw < words; jw += blockDim.x) {
          const uint8_t *colp = in8 + 4 * jw;
          for (int t = 0; t < th; t++) {
            float2 a01 = make_float2(0.0f, 0.0f), a23 = make_float2(0.0f, 0.0f);
            const float *cy = s_cy + t * Sy;
            const int *rr = s_row + t * Sy;
            // taps in chunks of 8: all loads of a chunk are issued before the first use (memory-level parallelism;
            // with 2 CTAs x 256 threads per SM the kernel is otherwise latency bound), accumulation stays in k order
            for (int k0 = 0; k0 < Sy; k0 += 8) {
              uint32_t wv[8];
#pragma unroll
              for (int j = 0; j < 8; j++)
                wv[j] = k0 + j < Sy ? ld_nc_u32(reinterpret_cast<const uint32_t *>(colp + (int64_t)rr[k0 + j] * pitch)) : 0u;
#pragma unroll
              for (int j = 0; j < 8; j++) {
                if (k0 + j < Sy) {
                  // the products use mul.rn (__fmul_rn, never contracted into an FMA): two roundings, like the reference
                  const float ck = cy[k0 + j];
                  const float2 f01 = bytes01_to_float(wv[j]), f23 = bytes23_to_float(wv[j]);
                  a01 = add2_rn(a01, make_float2(mul_rn(f01.x, ck), mul_rn(f01.y, ck)));
                  a23 = add2_rn(a23, make_float2(mul_rn(f23.x, ck), mul_rn(f23.y, ck)));
                }
              }
            }
            *reinterpret_cast<float4 *>(tmp + t * row_elems + 4 * jw) = make_float4(a01.x, a01.y, a23.x, a23.y);
          }
        }
      } else {
        // stage A (generic): vertical FIR   tmp[t][j] = sum_k cy[t][k] * in[row(t,k)][e0 + j]
        for (int e = threadIdx.x; e < th * row_elems; e += blockDim.x) {
          const int t = e / row_elems, j = e - t * row_elems;
          const int oy = oy0 + t;
          const int i0 = idx_y[oy];
          const float *cy = coef_y + (int64_t)oy * Sy;
          const In *col = in + e0 + j;
          float acc = 0.0f;
          for (int k = 0; k < Sy; k++) {
            const int r = by + min(max(i0 + k, 0), ey - 1);
            acc = add_rn(acc, mul_rn(ld_as_float<In>(col + r * pitch), cy[k]));
          }
          tmp[e] = acc;
        }
      }
      __syncthreads();
      // stage B: horizontal FIR from the smem intermediate; one thread = one (x, c) column of the tile, all th rows,
      // so every coefficient is fetched once and reused th times
      for (int e = threadIdx.x; e < tw * C; e += blockDim.x) {
        const int c = e % C, x = e / C;
        const int ox = ox0 + x;
        const int i0 = idx_x[ox];
        const float *cx = coef_x + (int64_t)ox * Sx;
        const bool he = flags ? flags[ox] != 0 : false;
        float acc[kMaxTileH];
#pragma unroll
        for (int t = 0; t < kMaxTileH; t++) acc[t] = 0.0f;
        for (int k = 0; k < Sx; k++) {
          const int sx = (bx + min(max(i0 + k, 0), ex - 1)) * C + c - e0;
          const float ck = cx[k];
#pragma unroll
          for (int t = 0; t < kMaxTileH; t++)
            if (t < th) acc[t] = add_rn(acc[t], mul_rn(ck, tmp[t * row_elems + sx]));
        }
#pragma unroll
        for (int t = 0; t < kMaxTileH; t++)
          if (t < th) out[((int64_t)(oy0 + t) * d.out_w + ox) * C + c] = rs_store_cvt<Out>(acc[t], he);
      }
    } else {
      const int ia = idx_y[oy0], ib = idx_y[oy0 + th - 1];
      const int rmin = by + min(max(min(ia, ib), 0), ey - 1);
      const int rmax = by + min(max(max(ia, ib) + Sy - 1, 0), ey - 1);
      const int rows = rmax - rmin + 1;
      const int row_elems = tw * C;
      // stage A: horizontal FIR   tmp[r][x*C+c] = sum_k cx[x][k] * in[rmin + r][col(x,k)][c]
      for (int e = threadIdx.x; e < rows * row_elems; e += blockDim.x) {
        const int c = e % C;
        const int x = (e / C) % tw;
        const int r = e / row_elems;
        const int ox = ox0 + x;
        const int i0 = idx_x[ox];
        const float *cx = coef_x + (int64_t)ox * Sx;
        const In *rowp = in + (int64_t)(rmin + r) * pitch + c;
        float acc = 0.0f;
        for (int k = 0; k < Sx; k++) {
          const int sx = bx + min(max(i0 + k, 0), ex - 1);
          acc = add_rn(acc, mul_rn(cx[k], ld_as_float<In>(rowp + (int64_t)sx * C)));
        }
        tmp[e] = acc;
      }
      __syncthreads();
      // stage B: vertical FIR from the smem intermediate
      for (int e = threadIdx.x; e < th * row_elems; e += blockDim.x) {
        const int t = e / row_elems, j = e - t * row_elems;
        const int oy = oy0 + t;
        const int i0 = idx_y[oy];
        const float *cy = coef_y + (int64_t)oy * Sy;
        float acc = 0.0f;
        for (int k = 0; k < Sy; k++) {
          const int r = by + min(max(i0 + k, 0), ey - 1) - rmin;
          acc = add_rn(acc, mul_rn(tmp[r * row_elems + j], cy[k]));
        }
        const int flat = ox0 * C + j;
        out[((int64_t)oy * d.out_w + ox0) * C + j] = rs_store_cvt<Out>(acc, flat < d.simd_flat_end);
      }
    }
    __syncthreads();
  }
}

// =============================================================================================
// STREAMING variant of the vertical-first path (u8 input, rows 16-byte aligned) -- the C2 hot case.
//
// A work item is a column strip x [oy0, oy1) of one sample.  A producer warp streams the strip's source rows, ONCE and in
// order, into a shared-memory ring with TMA bulk copies (cp.async.bulk ... mbarrier::complete_tx); eight consumer warps
// run the row walk (see walk_vertical_u8) over the ring, keep the open output rows in registers ACROSS chunks of 8 output
// rows (so there is no vertical overlap between chunks: every source byte is loaded and converted once per strip), park each
// finished output row in shared memory and, every 8 rows, run the horizontal pass from there.  The producer runs ahead
// across chunk and item boundaries, so HBM latency is hidden by the ring, not by occupancy.  The walk tables of a chunk
// (see BuildWalkRecords) are precomputed in the plan; the producer copies them into one of two record buffers ahead of the
// chunk's rows.
constexpr int kStRowBytes = 2048;         // one source row segment
constexpr int kStSlotRows = 4;            // ring slot = FOUR consecutive source rows of a chunk: one mbarrier wait / proxy fence / arrive
                                          // per slot instead of per row (the per-row synchronisation stalled the walk)
constexpr int kStStages = 5;              // 4 slots (16 rows) in flight while one is read: the most that fits 2 CTAs / SM
constexpr int kStTH = 8;                  // output rows per chunk
constexpr int kStSeg = 7 * kStTH;         // output rows per work item (a multiple of kStTH: chunk c of a sample starts at row c * kStTH)
constexpr int kStConsumers = 256;
constexpr int kStThreads = kStConsumers + 32;
constexpr int kStSlotBytes = kStSlotRows * kStRowBytes;
// walk records of one chunk: ent[kWalkMax][kWalkSlots] float2 (c, RN(-2^23 c)) of the tap that slot s takes from step j, or zeros,
// then fin[kWalkMax] (byte s = chunk-local output row that slot s completes at step j, 0xFF = none)
constexpr int kWalkEntBytes = kWalkMax * kWalkSlots * 8;
constexpr int kWalkRecBytes = kWalkEntBytes + kWalkMax * 4;
constexpr int kStSmemBytes = kStTH * kStRowBytes * 4 + kStStages * kStSlotBytes + 2 * kWalkRecBytes + (2 * kStStages + 4) * 8;
static_assert(2 * (kStSmemBytes + 1024) <= 228 * 1024, "two streaming CTAs must fit one SM");

struct RsItem { int32_t sample, ox0, tw, oy0, oy1; };

__device__ __forceinline__ void consumer_bar() { asm volatile("bar.sync 1, %0;" :: "n"(kStConsumers) : "memory"); }

struct StripGeom { int e0, bytes; };
__device__ __forceinline__ StripGeom strip_geom(const RsDesc &d, const int32_t *idx_x, int ox0, int tw) {
  const int ia = idx_x[ox0], ib = idx_x[ox0 + tw - 1];
  const int bx = d.base[0], ex = d.extent[0], Sx = d.support[0];
  const int cmin = bx + min(max(min(ia, ib), 0), ex - 1);
  const int cmax = bx + min(max(max(ia, ib) + Sx - 1, 0), ex - 1);
  StripGeom g;
  g.e0 = (cmin * d.C) & ~15;
  g.bytes = (((cmax + 1) * d.C + 15) & ~15) - g.e0;
  return g;
}

template <typename Out, int WMAX>
__global__ void __launch_bounds__(kStThreads, 2) resample_stream_kernel(const RsDesc *__restrict__ descs, const int32_t *__restrict__ tab,
                                                                        const RsItem *__restrict__ items, int nitems) {
  extern __shared__ __align__(128) uint8_t st_smem[];
  float *tmp2 = reinterpret_cast<float *>(st_smem);                               // [4 row pairs][RE][2]
  uint8_t *ring = st_smem + kStTH * kStRowBytes * 4;
  uint8_t *recs = ring + kStStages * kStSlotBytes;                                // [2][kWalkRecBytes]
  uint64_t *full = reinterpret_cast<uint64_t *>(recs + 2 * kWalkRecBytes);
  uint64_t *empty = full + kStStages;
  uint64_t *rfull = empty + kStStages, *rempty = rfull + 2;                       // the two record buffers
  const int tid = threadIdx.x;
  if (tid == 0) {
    for (int s = 0; s < kStStages; s++) { mbar_init(&full[s], 1); mbar_init(&empty[s], kStConsumers / 32); }
    for (int s = 0; s < 2; s++) { mbar_init(&rfull[s], 1); mbar_init(&rempty[s], kStConsumers / 32); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  if (tid >= kStConsumers) {
    // ------------------------------------------------------------------ producer warp: one lane issues the bulk copies
    if (tid == kStConsumers) {
      uint32_t stage = 0, par = 1, rb = 0, rpar = 1;
      for (int item = blockIdx.x; item < nitems; item += gridDim.x) {
        const RsItem it = items[item];
        const RsDesc &d = descs[it.sample];
        if (!d.use_stream) continue;
        const int32_t *idx_x = tab + d.idx_off[0], *idx_y = tab + d.idx_off[1];
        const int Sy = d.support[1], by = d.base[1], ey = d.extent[1];
        const StripGeom g = strip_geom(d, idx_x, it.ox0, it.tw);
        const int64_t pitch = (int64_t)d.in_w * d.C;
        const uint8_t *src0 = static_cast<const uint8_t *>(d.in) + g.e0;
        const int ustart = idx_y[it.oy0];
        // the same chunking as the consumers: slots group the rows of ONE chunk (a chunk ends with a partial slot)
        for (int cy0 = it.oy0; cy0 < it.oy1; cy0 += kStTH) {
          const int th = min(kStTH, it.oy1 - cy0);
          const int cs = cy0 == it.oy0 ? ustart : idx_y[cy0 - 1] + Sy;
          const int J = idx_y[cy0 + th - 1] + Sy - cs;
          {
            const int32_t *rec = tab + tab[d.walk_off + cy0 / kStTH];
            const uint32_t fin_bytes = (uint32_t)((J + 3) & ~3) * 4u;
            mbar_wait(&rempty[rb], rpar);
            mbar_expect_tx(&rfull[rb], (uint32_t)J * kWalkSlots * 8u + fin_bytes);
            bulk_g2s(recs + rb * kWalkRecBytes, rec, (uint32_t)J * kWalkSlots * 8u, &rfull[rb]);
            bulk_g2s(recs + rb * kWalkRecBytes + kWalkEntBytes, rec + J * kWalkSlots * 2, fin_bytes, &rfull[rb]);
            if (++rb == 2) { rb = 0; rpar ^= 1u; }
          }
          for (int j = 0; j < J; j += kStSlotRows) {
            const int nr = min(kStSlotRows, J - j);
            mbar_wait(&empty[stage], par);
            mbar_expect_tx(&full[stage], (uint32_t)(g.bytes * nr));
            for (int q = 0; q < nr; q++) {
              const int row = by + min(max(cs + j + q, 0), ey - 1);
              bulk_g2s(ring + stage * kStSlotBytes + q * kStRowBytes, src0 + row * pitch, (uint32_t)g.bytes, &full[stage]);
            }
            if (++stage == kStStages) { stage = 0; par ^= 1u; }
          }
        }
      }
    }
    return;
  }
  // -------------------------------------------------------------------- consumers
  constexpr int NW = 2;
  const int lane = tid & 31;
  uint32_t stage = 0, par = 0, rb = 0, rpar = 0;
  for (int item = blockIdx.x; item < nitems; item += gridDim.x) {
    const RsItem it = items[item];
    const RsDesc &d = descs[it.sample];
    if (!d.use_stream) continue;
    const int C = d.C, Sx = d.support[0], Sy = d.support[1];
    const int32_t *idx_x = tab + d.idx_off[0], *idx_y = tab + d.idx_off[1];
    const float *coef_x = reinterpret_cast<const float *>(tab + d.coef_off[0]);
    const int bx = d.base[0], ex = d.extent[0];
    const StripGeom g = strip_geom(d, idx_x, it.ox0, it.tw);
    const int RE = g.bytes, words = g.bytes >> 2;
    const uint8_t *flags = d.flags_off >= 0 ? reinterpret_cast<const uint8_t *>(tab + d.flags_off) : nullptr;
    Out *out = static_cast<Out *>(d.out);
    const int ustart = idx_y[it.oy0];
    bool okw[NW];
#pragma unroll
    for (int q = 0; q < NW; q++) okw[q] = tid + q * kStConsumers < words;
    float2 acc[WMAX][NW][2];
#pragma unroll
    for (int s = 0; s < WMAX; s++)
#pragma unroll
      for (int q = 0; q < NW; q++) acc[s][q][0] = acc[s][q][1] = make_float2(0.f, 0.f);

    for (int cy0 = it.oy0; cy0 < it.oy1; cy0 += kStTH) {
      const int th = min(kStTH, it.oy1 - cy0);
      const int cs = cy0 == it.oy0 ? ustart : idx_y[cy0 - 1] + Sy;
      const int J = idx_y[cy0 + th - 1] + Sy - cs;
      // ---- the chunk's walk records, copied in by the producer
      const float2 (*ent)[kWalkSlots] = reinterpret_cast<const float2 (*)[kWalkSlots]>(recs + rb * kWalkRecBytes);
      const uint32_t *fin = reinterpret_cast<const uint32_t *>(recs + rb * kWalkRecBytes + kWalkEntBytes);
      mbar_wait(&rfull[rb], rpar);
      // ---- stage A: row walk over the ring.  Closed slots (c = d = 0, exact zeros) are skipped by a CTA-uniform branch;
      //      the only other data-dependent branch is the rare "row finished" one.
      for (int j2 = 0; j2 < J; j2 += kStSlotRows) {
        mbar_wait(&full[stage], par);
        const uint32_t *rw = reinterpret_cast<const uint32_t *>(ring + stage * kStSlotBytes);
        uint32_t wr[kStSlotRows][NW];
#pragma unroll
        for (int r2 = 0; r2 < kStSlotRows; r2++)
#pragma unroll
          for (int q = 0; q < NW; q++) wr[r2][q] = rw[r2 * (kStRowBytes / 4) + tid + q * kStConsumers];   // always inside the slot
        // release the slot only once the words have ARRIVED in registers (the asm consumes them): the LDS of a warp completes
        // for all lanes together, and the slot is rewritten by the async proxy as soon as all 8 warps have arrived
#ifndef DALIB200_NO_RING_FENCE
        asm volatile("fence.proxy.async.shared::cta;" :: "r"(wr[0][0]), "r"(wr[0][NW - 1]), "r"(wr[kStSlotRows - 1][0]), "r"(wr[kStSlotRows - 1][NW - 1]) : "memory");
#else
        asm volatile("" :: "r"(wr[0][0]), "r"(wr[kStSlotRows - 1][NW - 1]) : "memory");
#endif
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty[stage]);
        if (++stage == kStStages) { stage = 0; par ^= 1u; }
#pragma unroll
        for (int r2 = 0; r2 < kStSlotRows; r2++) {
        const int j = j2 + r2;
        if (j >= J) continue;
        uint32_t w[NW];
#pragma unroll
        for (int q = 0; q < NW; q++) w[q] = wr[r2][q];
        float2 cd[kWalkSlots];
        {
          const float4 e01 = *reinterpret_cast<const float4 *>(&ent[j][0]);
          cd[0] = make_float2(e01.x, e01.y); cd[1] = make_float2(e01.z, e01.w);
          if (WMAX > 2) {
            const float4 e23 = *reinterpret_cast<const float4 *>(&ent[j][2]);
            cd[2] = make_float2(e23.x, e23.y); cd[3] = make_float2(e23.z, e23.w);
          }
        }
        float2 m[NW][2];
#pragma unroll
        for (int q = 0; q < NW; q++) {
          m[q][0] = make_float2(__uint_as_float(__byte_perm(w[q], 0x4B000000u, 0x7440)), __uint_as_float(__byte_perm(w[q], 0x4B000000u, 0x7441)));
          m[q][1] = make_float2(__uint_as_float(__byte_perm(w[q], 0x4B000000u, 0x7442)), __uint_as_float(__byte_perm(w[q], 0x4B000000u, 0x7443)));
        }
#pragma unroll
        for (int s = 0; s < WMAX; s++) {
          const float2 c2 = make_float2(cd[s].x, cd[s].x), d2 = make_float2(cd[s].y, cd[s].y);
          if (cd[s].x == 0.0f) continue;          // CTA-uniform: a closed slot (or a zero tap) would only add +0
#pragma unroll
          for (int q = 0; q < NW; q++) {
            acc[s][q][0] = add2_rn(acc[s][q][0], fma2_rn(m[q][0], c2, d2));
            acc[s][q][1] = add2_rn(acc[s][q][1], fma2_rn(m[q][1], c2, d2));
          }
        }
        const uint32_t f = fin[j];
        if (f != 0xFFFFFFFFu) {
#pragma unroll
          for (int s = 0; s < WMAX; s++) {
            const uint32_t tl = (f >> (8 * s)) & 0xFFu;
            if (tl != 0xFFu) {
              // parked rows are laid out by BYTE LANE: byte k of source word w of a row pair sits at float2 index k * words + w
              // (x = even row of the pair, y = odd row).  A warp's store of one byte lane then covers 32 consecutive float2 --
              // 2-way bank conflicts instead of the 8-way conflicts of the natural [byte][pair] order
              float *dst = tmp2 + ((size_t)(tl >> 1) * RE) * 2 + (tl & 1u);
#pragma unroll
              for (int q = 0; q < NW; q++) {
                if (okw[q]) {
                  float *p4 = dst + 2 * (tid + q * kStConsumers);
                  p4[0] = acc[s][q][0].x; p4[2 * words] = acc[s][q][0].y; p4[4 * words] = acc[s][q][1].x; p4[6 * words] = acc[s][q][1].y;
                }
                acc[s][q][0] = acc[s][q][1] = make_float2(0.f, 0.f);
              }
            }
          }
        }
        }            // rows of the slot
      }
      // release the record buffer to the producer's next bulk copy (the async proxy), as a ring slot is released
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
      __syncwarp();
      if (lane == 0) mbar_arrive(&rempty[rb]);
      if (++rb == 2) { rb = 0; rpar ^= 1u; }
      consumer_bar();
      // ---- stage B: horizontal pass of the chunk's th rows, two rows per packed operation
      const int npair = (th + 1) >> 1;
      for (int e = tid; e < it.tw * C; e += kStConsumers) {
        const int x = e / C, c = e - x * C;
        const int ox = it.ox0 + x;
        const int i0 = idx_x[ox];
        const float *cx = coef_x + (int64_t)ox * Sx;
        const bool he = flags ? flags[ox] != 0 : false;
        float2 a[kStTH / 2];
#pragma unroll
        for (int p = 0; p < kStTH / 2; p++) a[p] = make_float2(0.f, 0.f);
        // fma(v, c, -0) == RN(v * c), the reference's separately rounded product.  The -0 comes from the descriptor: with a
        // literal, ptxas 12.9 rewrites the fma as a mul and then contracts mul + add into one FFMA2 (a single rounding).
        const float2 nz = make_float2(d.neg_zero, d.neg_zero);
        const bool interior = i0 >= 0 && i0 + Sx <= ex;
        const int col0 = (bx + i0) * C + c - g.e0;
        for (int k = 0; k < Sx; k++) {
          const int col = interior ? col0 + k * C : (bx + min(max(i0 + k, 0), ex - 1)) * C + c - g.e0;
          const float ck = cx[k];
          const float2 c2 = make_float2(ck, ck);
          const float2 *src = reinterpret_cast<const float2 *>(tmp2) + (col & 3) * words + (col >> 2);      // byte-lane layout, see stage A
#pragma unroll
          for (int p = 0; p < kStTH / 2; p++)
            if (p < npair) a[p] = add2_rn(a[p], fma2_rn(src[(size_t)p * RE], c2, nz));
        }
#pragma unroll
        for (int p = 0; p < kStTH / 2; p++) {
          const int t0 = 2 * p;
          if (t0 < th) out[((int64_t)(cy0 + t0) * d.out_w + ox) * C + c] = rs_store_cvt<Out>(a[p].x, he);
          if (t0 + 1 < th) out[((int64_t)(cy0 + t0 + 1) * d.out_w + ox) * C + c] = rs_store_cvt<Out>(a[p].y, he);
        }
      }
      consumer_bar();   // the next chunk's walk overwrites the parked rows
    }
  }
}

// =============================================================================================
// PLANAR variant of the streaming kernel: decode -> resize without the RGB image (SURVEY.md 8f rank 1).
//
// The source is the decoder's planar 4:2:0 output (Y at full, Cb / Cr at half resolution); the strip's rows are streamed through the
// ring as [Y row | Cb near | Cb far | Cr near | Cr far] (five bulk copies per row, near / far = the two chroma rows libjpeg's h2v2
// fancy upsampling blends for that luma row).  A consumer thread owns two neighbouring pixels (one chroma column): it forms the
// vertically blended chroma of its column and the two next to it, the horizontally blended values of its two pixels, converts to RGB
// with libjpeg's fixed-point coefficients (jdcolor.c, SCALEBITS 16), and feeds the six bytes straight into the row walk as
// 2^23 + b floats -- the decoded RGB image (6.2 MB per 1080p sample, written and read back by the two-kernel path) never exists.
// Everything behind that point (slots, parking, horizontal pass, rounding flags) is the streaming kernel's.
// Bit-exact with decode-then-resize: the per-pixel arithmetic is the colour kernel's, the filter arithmetic the streaming kernel's.
constexpr int kPlPx = 512;                 // strip width in pixels (2 per consumer thread)
constexpr int kPlChroma = kPlPx / 2 + 32;  // chroma samples per slot row (16 of halo on each side, 16-byte granules)
constexpr int kPlSlot = kPlPx + 4 * kPlChroma;
constexpr int kPlStages = 16;
constexpr int kPlSmemBytes = kStTH * kPlPx * 3 * 4 + kPlStages * kPlSlot + kWalkMax * kWalkSlots * 16 + kWalkMax * 4 + 2 * kPlStages * 8;

struct PlanarGeom { int px0, npx, c0, e0; };
__device__ __forceinline__ PlanarGeom planar_geom(const RsDesc &d, const int32_t *idx_x, int ox0, int tw) {
  const int ia = idx_x[ox0], ib = idx_x[ox0 + tw - 1];
  const int bx = d.base[0], ex = d.extent[0], Sx = d.support[0];
  const int cmin = d.crop_x + bx + min(max(min(ia, ib), 0), ex - 1);
  const int cmax = d.crop_x + bx + min(max(max(ia, ib) + Sx - 1, 0), ex - 1);
  PlanarGeom g;
  g.px0 = cmin & ~31;
  g.npx = ((cmax + 1 - g.px0) + 31) & ~31;
  g.c0 = max((g.px0 >> 1) - 16, 0);
  g.e0 = (g.px0 - d.crop_x) * 3;
  return g;
}

template <int WMAX>
__global__ void __launch_bounds__(kStThreads, 2) resample_planar_kernel(const RsDesc *__restrict__ descs, const int32_t *__restrict__ tab,
                                                                        const RsItem *__restrict__ items, int nitems) {
  extern __shared__ __align__(128) uint8_t st_smem[];
  float *tmp2 = reinterpret_cast<float *>(st_smem);                               // [4 row pairs][RE][2]
  uint8_t *ring = st_smem + kStTH * kPlPx * 3 * 4;
  float2 (*ent)[kWalkSlots] = reinterpret_cast<float2 (*)[kWalkSlots]>(ring + kPlStages * kPlSlot);
  uint32_t *fin = reinterpret_cast<uint32_t *>(ring + kPlStages * kPlSlot + kWalkMax * kWalkSlots * 16);
  uint64_t *full = reinterpret_cast<uint64_t *>(fin + kWalkMax);
  uint64_t *empty = full + kPlStages;
  const int tid = threadIdx.x;
  if (tid == 0) {
    for (int s = 0; s < kPlStages; s++) { mbar_init(&full[s], 1); mbar_init(&empty[s], kStConsumers / 32); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  if (tid >= kStConsumers) {
    // ------------------------------------------------------------------ producer warp: one lane issues the bulk copies
    if (tid == kStConsumers) {
      uint32_t stage = 0, par = 1;
      for (int item = blockIdx.x; item < nitems; item += gridDim.x) {
        const RsItem it = items[item];
        const RsDesc &d = descs[it.sample];
        const int32_t *idx_x = tab + d.idx_off[0], *idx_y = tab + d.idx_off[1];
        const int Sy = d.support[1], by = d.base[1], ey = d.extent[1];
        const PlanarGeom g = planar_geom(d, idx_x, it.ox0, it.tw);
        const int dh = (d.img_h + 1) >> 1;
        const uint32_t ybytes = (uint32_t)min(g.npx, d.pitch_y - g.px0);
        const uint32_t cbytes = (uint32_t)min(g.npx / 2 + 32, d.pitch_c - g.c0);
        const int ustart = idx_y[it.oy0], uend = idx_y[it.oy1 - 1] + Sy - 1;
        for (int u = ustart; u <= uend; u++) {
          mbar_wait_backoff(&empty[stage], par);
          mbar_expect_tx(&full[stage], ybytes + 4u * cbytes);
          const int fy = d.crop_y + by + min(max(u, 0), ey - 1);
          const int rn = fy >> 1;
          const int rf = min(max((fy & 1) ? rn + 1 : rn - 1, 0), dh - 1);
          uint8_t *slot = ring + stage * kPlSlot;
          bulk_g2s(slot, d.pl[0] + (int64_t)fy * d.pitch_y + g.px0, ybytes, &full[stage]);
          bulk_g2s(slot + kPlPx, d.pl[1] + (int64_t)rn * d.pitch_c + g.c0, cbytes, &full[stage]);
          bulk_g2s(slot + kPlPx + kPlChroma, d.pl[1] + (int64_t)rf * d.pitch_c + g.c0, cbytes, &full[stage]);
          bulk_g2s(slot + kPlPx + 2 * kPlChroma, d.pl[2] + (int64_t)rn * d.pitch_c + g.c0, cbytes, &full[stage]);
          bulk_g2s(slot + kPlPx + 3 * kPlChroma, d.pl[2] + (int64_t)rf * d.pitch_c + g.c0, cbytes, &full[stage]);
          if (++stage == kPlStages) { stage = 0; par ^= 1u; }
        }
      }
    }
    return;
  }
  // -------------------------------------------------------------------- consumers
  const int lane = tid & 31;
  const uint32_t a_ring = smem_u32(ring);
  uint32_t stage = 0, par = 0;
  for (int item = blockIdx.x; item < nitems; item += gridDim.x) {
    const RsItem it = items[item];
    const RsDesc &d = descs[it.sample];
    const int C = 3, Sx = d.support[0], Sy = d.support[1];
    const int32_t *idx_x = tab + d.idx_off[0], *idx_y = tab + d.idx_off[1];
    const float *coef_x = reinterpret_cast<const float *>(tab + d.coef_off[0]);
    const int bx = d.base[0], ex = d.extent[0];
    const PlanarGeom g = planar_geom(d, idx_x, it.ox0, it.tw);
    const int RE = g.npx * 3;
    const uint8_t *flags = d.flags_off >= 0 ? reinterpret_cast<const uint8_t *>(tab + d.flags_off) : nullptr;
    uint8_t *out = static_cast<uint8_t *>(d.out);
    const int ustart = idx_y[it.oy0];
    const bool okw = 2 * tid < g.npx;
    // chroma column of this thread and the edge rules of h2v2 fancy upsampling (jdsample.c)
    const int ci = (g.px0 >> 1) + tid, dw = (d.img_w + 1) >> 1;
    const bool first_col = ci == 0, last_col = ci >= dw - 1;
    const uint32_t coff = (uint32_t)(ci - g.c0);                    // position inside the chroma slot rows
    const uint32_t o_prev = first_col ? coff : coff - 1u, o_next = coff + 1u;
    float2 acc[WMAX][3];
#pragma unroll
    for (int s = 0; s < WMAX; s++)
#pragma unroll
      for (int q = 0; q < 3; q++) acc[s][q] = make_float2(0.f, 0.f);

    for (int cy0 = it.oy0; cy0 < it.oy1; cy0 += kStTH) {
      const int th = min(kStTH, it.oy1 - cy0);
      const int cs = cy0 == it.oy0 ? ustart : idx_y[cy0 - 1] + Sy;
      const int J = idx_y[cy0 + th - 1] + Sy - cs;
      // ---- the chunk's walk records from the plan (see BuildWalkRecords)
      {
        const int32_t *rec = tab + tab[d.walk_off + cy0 / kStTH];
        for (int e = tid; e < J * kWalkSlots * 2; e += kStConsumers) reinterpret_cast<int32_t *>(&ent[0][0])[e] = rec[e];
        for (int j = tid; j < J; j += kStConsumers) fin[j] = (uint32_t)rec[J * kWalkSlots * 2 + j];
      }
      consumer_bar();
      // ---- stage A: row walk over the ring, pixels produced on the fly
      for (int j = 0; j < J; j++) {
        mbar_wait(&full[stage], par);
        const uint32_t a_slot = a_ring + stage * kPlSlot;
        const uint32_t yw = lds_u16(a_slot + 2u * tid);
        uint32_t cbn[3], cbf[3], crn[3], crf[3];
        {
          const uint32_t a_c = a_slot + kPlPx;
          cbn[0] = lds_u8(a_c + o_prev); cbn[1] = lds_u8(a_c + coff); cbn[2] = lds_u8(a_c + o_next);
          cbf[0] = lds_u8(a_c + kPlChroma + o_prev); cbf[1] = lds_u8(a_c + kPlChroma + coff); cbf[2] = lds_u8(a_c + kPlChroma + o_next);
          crn[0] = lds_u8(a_c + 2 * kPlChroma + o_prev); crn[1] = lds_u8(a_c + 2 * kPlChroma + coff); crn[2] = lds_u8(a_c + 2 * kPlChroma + o_next);
          crf[0] = lds_u8(a_c + 3 * kPlChroma + o_prev); crf[1] = lds_u8(a_c + 3 * kPlChroma + coff); crf[2] = lds_u8(a_c + 3 * kPlChroma + o_next);
        }
        // release the slot once the values have ARRIVED in registers (see resample_stream_kernel)
#ifndef DALIB200_NO_RING_FENCE
        asm volatile("fence.proxy.async.shared::cta;" :: "r"(yw), "r"(crf[2]) : "memory");
#else
        asm volatile("" :: "r"(yw), "r"(crf[2]), "r"(cbn[0]), "r"(cbf[1]), "r"(crn[2]) : "memory");
#endif
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty[stage]);
        if (++stage == kPlStages) { stage = 0; par ^= 1u; }
        float2 cd[kWalkSlots];
        {
          const float4 e01 = *reinterpret_cast<const float4 *>(&ent[j][0]);
          cd[0] = make_float2(e01.x, e01.y); cd[1] = make_float2(e01.z, e01.w);
          if (WMAX > 2) {
            const float4 e23 = *reinterpret_cast<const float4 *>(&ent[j][2]);
            cd[2] = make_float2(e23.x, e23.y); cd[3] = make_float2(e23.z, e23.w);
          }
        }
        // chroma: vertical blend 3 * near + far of the three columns, then the horizontal blend of the two pixels
        int cb[2], cr[2];
        {
          const int b0 = 3 * (int)cbn[0] + (int)cbf[0], b1 = 3 * (int)cbn[1] + (int)cbf[1], b2 = 3 * (int)cbn[2] + (int)cbf[2];
          const int r0 = 3 * (int)crn[0] + (int)crf[0], r1 = 3 * (int)crn[1] + (int)crf[1], r2 = 3 * (int)crn[2] + (int)crf[2];
          cb[0] = first_col ? (b1 * 4 + 8) >> 4 : (b1 * 3 + b0 + 8) >> 4;
          cb[1] = last_col ? (b1 * 4 + 7) >> 4 : (b1 * 3 + b2 + 7) >> 4;
          cr[0] = first_col ? (r1 * 4 + 8) >> 4 : (r1 * 3 + r0 + 8) >> 4;
          cr[1] = last_col ? (r1 * 4 + 7) >> 4 : (r1 * 3 + r2 + 7) >> 4;
        }
        uint32_t m[6];
#pragma unroll
        for (int k = 0; k < 2; k++) {
          const int yy = (int)((yw >> (8 * k)) & 0xFFu);
          const int cbm = cb[k] - 128, crm = cr[k] - 128;
          const int r = yy + ((91881 * crm + 32768) >> 16);
          const int gq = yy + ((-22554 * cbm + 32768 - 46802 * crm) >> 16);
          const int b = yy + ((116130 * cbm + 32768) >> 16);
          m[3 * k] = 0x4B000000u | (uint32_t)min(max(r, 0), 255);
          m[3 * k + 1] = 0x4B000000u | (uint32_t)min(max(gq, 0), 255);
          m[3 * k + 2] = 0x4B000000u | (uint32_t)min(max(b, 0), 255);
        }
        const float2 m01 = make_float2(__uint_as_float(m[0]), __uint_as_float(m[1]));
        const float2 m23 = make_float2(__uint_as_float(m[2]), __uint_as_float(m[3]));
        const float2 m45 = make_float2(__uint_as_float(m[4]), __uint_as_float(m[5]));
#pragma unroll
        for (int s = 0; s < WMAX; s++) {
          const float2 c2 = make_float2(cd[s].x, cd[s].x), d2 = make_float2(cd[s].y, cd[s].y);
          acc[s][0] = add2_rn(acc[s][0], fma2_rn(m01, c2, d2));
          acc[s][1] = add2_rn(acc[s][1], fma2_rn(m23, c2, d2));
          acc[s][2] = add2_rn(acc[s][2], fma2_rn(m45, c2, d2));
        }
        const uint32_t f = fin[j];
        if (f != 0xFFFFFFFFu) {
#pragma unroll
          for (int s = 0; s < WMAX; s++) {
            const uint32_t tl = (f >> (8 * s)) & 0xFFu;
            if (tl != 0xFFu) {
              if (okw) {
                float *p6 = tmp2 + ((size_t)(tl >> 1) * RE) * 2 + (tl & 1u) + 12 * tid;
                p6[0] = acc[s][0].x; p6[2] = acc[s][0].y; p6[4] = acc[s][1].x; p6[6] = acc[s][1].y; p6[8] = acc[s][2].x; p6[10] = acc[s][2].y;
              }
              acc[s][0] = acc[s][1] = acc[s][2] = make_float2(0.f, 0.f);
            }
          }
        }
      }
      consumer_bar();
      // ---- stage B: horizontal pass of the chunk's th rows, two rows per packed operation (as in resample_stream_kernel)
      const int npair = (th + 1) >> 1;
      for (int e = tid; e < it.tw * C; e += kStConsumers) {
        const int x = e / C, c = e - x * C;
        const int ox = it.ox0 + x;
        const int i0 = idx_x[ox];
        const float *cx = coef_x + (int64_t)ox * Sx;
        const bool he = flags ? flags[ox] != 0 : false;
        float2 a[kStTH / 2];
#pragma unroll
        for (int p = 0; p < kStTH / 2; p++) a[p] = make_float2(0.f, 0.f);
        const float2 nz = make_float2(d.neg_zero, d.neg_zero);
        const bool interior = i0 >= 0 && i0 + Sx <= ex;
        const int col0 = (bx + i0) * C + c - g.e0;
        for (int k = 0; k < Sx; k++) {
          const int col = interior ? col0 + k * C : (bx + min(max(i0 + k, 0), ex - 1)) * C + c - g.e0;
          const float ck = cx[k];
          const float2 c2 = make_float2(ck, ck);
          const float2 *src = reinterpret_cast<const float2 *>(tmp2) + col;
#pragma unroll
          for (int p = 0; p < kStTH / 2; p++)
            if (p < npair) a[p] = add2_rn(a[p], fma2_rn(src[(size_t)p * RE], c2, nz));
        }
#pragma unroll
        for (int p = 0; p < kStTH / 2; p++) {
          const int t0 = 2 * p;
          if (t0 < th) out[((int64_t)(cy0 + t0) * d.out_w + ox) * C + c] = rs_store_cvt<uint8_t>(a[p].x, he);
          if (t0 + 1 < th) out[((int64_t)(cy0 + t0 + 1) * d.out_w + ox) * C + c] = rs_store_cvt<uint8_t>(a[p].y, he);
        }
      }
    }
  }
}

}  // namespace dalib200

using namespace dalib200;  // NOLINT

namespace {

// (kTmpFloats etc. are defined next to the kernel)

struct TableKey {
  int in_size, out_size, ftype, base, extent;
  uint32_t origin_bits, scale_bits, fscale_bits, fanchor_bits;
  bool operator<(const TableKey &o) const {
    return std::tie(in_size, out_size, ftype, base, extent, origin_bits, scale_bits, fscale_bits, fanchor_bits) <
           std::tie(o.in_size, o.out_size, o.ftype, o.base, o.extent, o.origin_bits, o.scale_bits, o.fscale_bits, o.fanchor_bits);
  }
};
inline uint32_t fbits(float f) { uint32_t u; memcpy(&u, &f, 4); return u; }

}  // namespace

struct dalib200ResamplePlan {
  int max_batch = 0, n = 0;
  int in_dtype = DALIB200_UINT8, out_dtype = DALIB200_UINT8;
  std::vector<RsDesc> descs;
  std::vector<int32_t> tables;                 // host copy of the table arena (idx, coef bits, flags)
  std::vector<int32_t> uploaded_tables;        // what the device arena currently holds
  std::map<TableKey, AxisTableRef> cache;      // dedup of axis tables within a batch
  std::map<int, int> walk_cache;               // vertical axis table offset -> its walk records (BuildWalkRecords)
  std::vector<int> order0;
  int64_t total_tiles = 0;
  DescArena desc_arena, table_arena, item_arena;
  std::vector<RsItem> items;                   // strips of the samples that qualify for the streaming kernel
  std::vector<uint8_t> stream_ok;              // structural eligibility per sample (alignment is checked at launch)
  std::vector<int> path;                       // per sample: 0 = tile kernel, 1 = streaming kernel (last launch)
  bool tables_dirty = true;
  bool smem_opted[13] = { false, false, false, false, false, false, false, false, false, false, false, false, false };
  bool planar_mode = false;                    // strips sized for resample_planar_kernel (set by ...SetupPlanar)
};

namespace {

// The most steps J of the row walk of one chunk, over the chunks of kStTH output rows of every kStSeg-row work item: the chunking of
// BuildWalkRecords and of the kernels.
int MaxChunkSteps(const int32_t *iy, int out_h, int Sy) {
  int m = 0;
  for (int o = 0; o < out_h; o += kStSeg)
    for (int c0 = o, o1 = std::min(o + kStSeg, out_h); c0 < o1; c0 += kStTH) {
      const int cs = c0 == o ? iy[o] : iy[c0 - 1] + Sy;
      m = std::max(m, iy[std::min(c0 + kStTH, o1) - 1] + Sy - cs);
    }
  return m;
}

// Walk records of the streaming kernels for one vertical axis: the tables stage A of resample_stream_kernel and resample_planar_kernel
// walks by.  Chunks of kStTH output rows restart at every kStSeg-row work item, as the kernels' chunks do.  The records of a chunk
// cover the steps j = 0..J-1 of its row walk: ent[j][s] = (c, RN(-2^23 c)) of the tap that accumulator slot s takes at step j, or exact
// zeros for a closed slot (the kernels skip a slot with c == 0), and fin[j], whose byte s is the chunk-local output row that slot s
// completes at step j (0xFF: none).  -2^23 c is a power-of-two scaling of c, so the host product is the device's mul.rn bit for bit.
// Layout: one arena word offset per chunk, then per chunk (16-byte aligned, for the bulk copies) ent[J][kWalkSlots] as float2 and
// fin[J] padded to a multiple of 4 words.  Returns the offset of the per-chunk offsets, or -1 if the arena would exceed its limit.
int BuildWalkRecords(std::vector<int32_t> &arena, int idx_off, int coef_off, int out_h, int Sy, int W) {
  const std::vector<int32_t> iy(arena.begin() + idx_off, arena.begin() + idx_off + out_h);
  const std::vector<int32_t> cw(arena.begin() + coef_off, arena.begin() + coef_off + static_cast<size_t>(out_h) * Sy);
  auto chunk_steps = [&](int o, int c0, int c1, int &cs) {
    cs = c0 == o ? iy[o] : iy[c0 - 1] + Sy;
    return iy[c1 - 1] + Sy - cs;
  };
  const int nchunks = (out_h + kStTH - 1) / kStTH;
  int64_t words = static_cast<int64_t>(arena.size()) + nchunks;
  for (int o = 0; o < out_h; o += kStSeg)
    for (int c0 = o, o1 = std::min(o + kStSeg, out_h), cs; c0 < o1; c0 += kStTH) {
      const int J = chunk_steps(o, c0, std::min(c0 + kStTH, o1), cs);
      words += 3 + static_cast<int64_t>(J) * kWalkSlots * 2 + ((J + 3) & ~3);
    }
  if (words >= kMaxTableWords) return -1;
  const int off = static_cast<int>(arena.size());
  arena.resize(arena.size() + nchunks);
  for (int o = 0; o < out_h; o += kStSeg) {
    const int o1 = std::min(o + kStSeg, out_h);
    for (int c0 = o; c0 < o1; c0 += kStTH) {
      int cs;
      const int J = chunk_steps(o, c0, std::min(c0 + kStTH, o1), cs);
      arena.resize((arena.size() + 3) & ~static_cast<size_t>(3));
      const size_t r = arena.size(), rf = r + static_cast<size_t>(J) * kWalkSlots * 2;
      arena[off + c0 / kStTH] = static_cast<int32_t>(r);
      arena.resize(rf + ((J + 3) & ~3), -1);
      std::fill(arena.begin() + r, arena.begin() + rf, 0);
      uint8_t *fin = reinterpret_cast<uint8_t *>(arena.data() + rf);
      // rows open during the chunk: from its first row up to the first one that opens after the chunk's last step
      for (int t = c0; t < o1 && iy[t] < cs + J; t++) {
        for (int k = 0; k < Sy; k++) {
          const int j = iy[t] + k - cs;
          if (j < 0 || j >= J) continue;
          float c;
          memcpy(&c, &cw[static_cast<size_t>(t) * Sy + k], sizeof(c));
          const float d = c * -8388608.0f;
          memcpy(&arena[r + (static_cast<size_t>(j) * kWalkSlots + t % W) * 2], &c, sizeof(c));
          memcpy(&arena[r + (static_cast<size_t>(j) * kWalkSlots + t % W) * 2 + 1], &d, sizeof(d));
          if (k == Sy - 1) fin[4 * j + t % W] = static_cast<uint8_t>(t - c0);
        }
      }
    }
  }
  return off;
}

// The launch's descriptors, staged in desc_arena by the caller, go to the device, then the tables if they changed since their last
// upload, then the streaming kernels' work items if `items` is set.
int UploadLaunchData(dalib200ResamplePlan *p, bool items, cudaStream_t stream) {
  auto upload = [stream](DescArena &arena, const void *src, size_t bytes) {
    uint8_t *h;
    int rc = arena.Stage(bytes, &h);
    if (rc) return rc;
    memcpy(h, src, bytes);
    return arena.Upload(bytes, stream);
  };
  int rc = p->desc_arena.Upload(sizeof(RsDesc) * p->n, stream);
  if (rc) return rc;
  if (p->tables_dirty) {
    if ((rc = upload(p->table_arena, p->tables.data(), p->tables.size() * sizeof(int32_t)))) return rc;
    p->uploaded_tables = p->tables;
    p->tables_dirty = false;
  }
  return items ? upload(p->item_arena, p->items.data(), p->items.size() * sizeof(RsItem)) : DALIB200_SUCCESS;
}

}  // namespace

extern "C" {

int dalib200ResamplePlanCreate(dalib200ResamplePlan **plan, int max_batch) try {
  DB_CHECK_ARG(plan && max_batch > 0, "ResamplePlanCreate: bad arguments");
  auto *p = new dalib200ResamplePlan();
  p->max_batch = max_batch;
  int rc = p->desc_arena.Reserve(sizeof(RsDesc) * max_batch);
  if (rc) { delete p; return rc; }
  *plan = p;
  return DALIB200_SUCCESS;
} DB_API_CATCH

int dalib200ResamplePlanDestroy(dalib200ResamplePlan *p) try {
  if (!p) return DALIB200_SUCCESS;
  p->desc_arena.Free(); p->table_arena.Free(); p->item_arena.Free();
  delete p;
  return DALIB200_SUCCESS;
} DB_API_CATCH

int dalib200ResamplePlanGetPath(const dalib200ResamplePlan *p, int sample) try {
  if (!p || sample < 0 || sample >= p->n) return -1;
  return p->path[sample];
} DB_API_CATCH

int dalib200ResamplePlanGetStreamInfo(const dalib200ResamplePlan *p, int sample, int32_t info[4]) try {
  DB_CHECK_ARG(p && info && sample >= 0 && sample < p->n && sample < static_cast<int>(p->descs.size()),
               "ResamplePlanGetStreamInfo: bad arguments");
  const RsDesc &d = p->descs[sample];
  info[0] = p->stream_ok[sample];
  info[1] = d.walk_slots;
  info[2] = d.out_h > 0 && d.out_w > 0 ? MaxChunkSteps(p->tables.data() + d.idx_off[1], d.out_h, d.support[1]) : 0;
  info[3] = static_cast<int32_t>(std::count_if(p->items.begin(), p->items.end(), [&](const RsItem &it) { return it.sample == sample; }));
  return DALIB200_SUCCESS;
} DB_API_CATCH

int dalib200ResamplePlanGetOrder(const dalib200ResamplePlan *p, int sample) try {
  if (!p || sample < 0 || sample >= p->n) return -1;
  return p->order0[sample];
} DB_API_CATCH

int dalib200ResamplePlanSetup(dalib200ResamplePlan *p, int n, const dalib200ResampleSample *samples, int in_dtype, int out_dtype) try {
  DB_CHECK_ARG(p && samples && n >= 0, "ResamplePlanSetup: null argument");
  DB_CHECK_ARG(n <= p->max_batch, "ResamplePlanSetup: batch %d exceeds plan capacity %d", n, p->max_batch);
  DB_CHECK_ARG((in_dtype == DALIB200_UINT8 && (out_dtype == DALIB200_UINT8 || out_dtype == DALIB200_FLOAT)) ||
               (in_dtype == DALIB200_FLOAT && out_dtype == DALIB200_FLOAT),
               "Resize: unsupported type combination in=%d out=%d (u8->u8, u8->f32, f32->f32)", in_dtype, out_dtype);
  p->descs.assign(n, RsDesc());
  p->order0.assign(n, 0);
  p->items.clear();
  p->stream_ok.assign(n, 0);
  p->path.assign(n, 0);
  p->tables.clear();
  p->cache.clear();
  p->walk_cache.clear();
  int64_t tiles = 0;
  for (int i = 0; i < n; i++) {
    const auto &s = samples[i];
    DB_CHECK_ARG(s.in_h > 0 && s.in_w > 0 && s.channels >= 1 && s.channels <= 16,
                 "Resize: sample %d has unsupported input shape %dx%dx%d", i, s.in_h, s.in_w, s.channels);
    DB_CHECK_ARG(s.out_h >= 0 && s.out_w >= 0, "Resize: sample %d has negative output size", i);
    DB_CHECK_ARG(ElementsFit31(s.in_h, s.in_w, s.channels) && ElementsFit31(s.out_h, s.out_w, s.channels),
                 "Resize: sample %d: images of 2^31 elements or more are not supported", i);
    for (int a = 0; a < 2; a++) {
      for (const dalib200FilterDesc *f : { &s.min_filter[a], &s.mag_filter[a] })
        DB_CHECK_ARG(FilterDescValid(*f), "Resize: sample %d: invalid filter (type %d, radius %g)", i, f->type, static_cast<double>(f->radius));
      DB_CHECK_ARG(!s.use_roi[a] || RoiFinite(s.roi_start[a], s.roi_end[a]), "Resize: sample %d: the region of interest must be finite", i);
    }
    RsDesc &d = p->descs[i];
    memset(&d, 0, sizeof(d));
    d.in_h = s.in_h; d.in_w = s.in_w; d.C = s.channels; d.out_h = s.out_h; d.out_w = s.out_w;
    d.flags_off = -1; d.simd_flat_end = 0;
    d.first_tile = tiles;
    d.tile_h = d.tile_w = 1; d.tiles_x = d.tiles_y = 0;
    if (s.out_h == 0 || s.out_w == 0) continue;
    AxisSetup ax[2];
    // axis 0 = x <- params index 1 ; axis 1 = y <- params index 0
    SetupAxis(ax[0], s.in_w, s.out_w, s.use_roi[1] != 0, s.roi_start[1], s.roi_end[1], s.min_filter[1], s.mag_filter[1]);
    SetupAxis(ax[1], s.in_h, s.out_h, s.use_roi[0] != 0, s.roi_start[0], s.roi_end[0], s.min_filter[0], s.mag_filter[0]);
    int order[2];
    ProcessingOrder(ax, 2, order);
    const int first = order[0];
    p->order0[i] = first;
    d.vfirst = first == 1;
    for (int a = 0; a < 2; a++) {
      CropAxis(ax[a], a == first);
      DB_CHECK_ARG(ax[a].extent > 0, "Resize: sample %d has an empty region of interest", i);
      TableKey key{ ax[a].in_size, ax[a].out_size, ax[a].ftype * 2 + a, ax[a].base, ax[a].extent, fbits(ax[a].origin),
                    fbits(ax[a].scale), fbits(ax[a].filter.scale), fbits(ax[a].filter.anchor) };
      auto it = p->cache.find(key);
      AxisTableRef ref;
      if (it == p->cache.end()) {
        DB_CHECK_ARG(static_cast<int64_t>(ax[a].out_size) * (static_cast<int64_t>(ax[a].support) + 1) + static_cast<int64_t>(p->tables.size()) <
                         kMaxTableWords,
                     "Resize: sample %d needs %lld filter taps per output along axis %d (%d -> %d): the filter tables would exceed 256 MB", i,
                     static_cast<long long>(ax[a].support), a, ax[a].in_size, ax[a].out_size);
        BuildTable(p->tables, ref, ax[a], a);
        p->cache[key] = ref;
      } else {
        ref = it->second;
      }
      d.idx_off[a] = ref.idx_off; d.coef_off[a] = ref.coef_off; d.support[a] = ref.support;
      d.base[a] = ax[a].base; d.extent[a] = ax[a].extent;
    }
    if (out_dtype == DALIB200_UINT8) {
      if (first == 1) {   // horizontal pass is last
        if (ax[0].ftype != DALIB200_FILTER_NN)
          d.flags_off = BuildHorzFlags(p->tables, d.idx_off[0], s.out_w, ax[0].extent, d.support[0]);
      } else {            // vertical pass is last: SSE over flat_w in groups of 16 (cpu.h:95-124,362-390)
        if (ax[1].ftype != DALIB200_FILTER_NN) d.simd_flat_end = (s.out_w * s.channels / 16) * 16;
      }
    }
    // ---- tiling: the fp32 intermediate of a tile must fit kTmpFloats
    const int C = s.channels;
    const int32_t *ix = p->tables.data() + d.idx_off[0], *iy = p->tables.data() + d.idx_off[1];
    auto span_of = [](const int32_t *idx, int o0, int cnt, int S, int extent) {
      int a = idx[o0], b = idx[o0 + cnt - 1];
      int lo = std::min(std::max(std::min(a, b), 0), extent - 1);
      int hi = std::min(std::max(std::max(a, b) + S - 1, 0), extent - 1);
      return hi - lo + 1;
    };
    auto max_span = [&](const int32_t *idx, int out, int t, int S, int extent) {
      int m = 0;
      for (int o = 0; o < out; o += t) m = std::max(m, span_of(idx, o, std::min(t, out - o), S, extent));
      return m;
    };
    int th, tw;
    bool fits = false;
    if (d.vfirst) {
      tw = s.out_w; th = 0;
      for (;;) {
        int span = max_span(ix, s.out_w, tw, d.support[0], d.extent[0]);
        th = std::min({ kTmpFloats / std::max(1, span * C + 8), kMaxTileH, s.out_h });
        if (th >= std::min(8, s.out_h) || tw == 1) { fits = th >= 1; break; }
        tw = (tw + 1) / 2;
      }
    } else {
      th = std::min(s.out_h, 32); tw = 0;
      for (;;) {
        int span = max_span(iy, s.out_h, th, d.support[1], d.extent[1]);
        tw = std::min(kTmpFloats / std::max(1, span * C), s.out_w);
        if (tw >= std::min(16, s.out_w) || th == 1) { fits = tw >= 1; break; }
        th = (th + 1) / 2;
      }
    }
    if (!fits) {
      SetLastError("Resize: sample %d: filter footprint (%d x %d taps, %d channels) does not fit the on-chip tile",
                   i, d.support[0], d.support[1], C);
      return DALIB200_ERROR_UNSUPPORTED;
    }
    d.tile_h = th; d.tile_w = tw;
    d.tiles_x = (s.out_w + tw - 1) / tw; d.tiles_y = (s.out_h + th - 1) / th;
    // ---- row walk of the vertical pass (u8 input, vertical first): slots W such that output rows t and t + W never overlap
    d.walk_slots = 0;
    if (d.vfirst && in_dtype == DALIB200_UINT8) {
      const int Sy = d.support[1];
      int W = 0;
      for (int w = 1; w <= kWalkSlots && !W; w++) {
        bool ok = true;
        for (int t = 0; t + w < s.out_h && ok; t++) ok = std::abs(iy[t + w] - iy[t]) >= Sy;
        if (ok) W = w;
      }
      int maxJ = 0;
      for (int o = 0; o < s.out_h; o += th) {
        int a = iy[o], b = iy[std::min(o + th, s.out_h) - 1];
        maxJ = std::max(maxJ, std::max(a, b) + Sy - std::min(a, b));
      }
      d.walk_slots = W;
      d.tile_walk = W && maxJ <= kWalkMax;
      // ---- streaming kernel: strictly increasing source rows, strips whose row segment fits a ring slot
      bool inc = W > 0;
      for (int t = 0; t + 1 < s.out_h && inc; t++) inc = iy[t + 1] > iy[t];
      if (inc) {
        const int Sx = d.support[0];
        auto strip_bytes = [&](int o0, int cnt) {
          int a = ix[o0], b = ix[o0 + cnt - 1];
          int cmin = d.base[0] + std::min(std::max(std::min(a, b), 0), d.extent[0] - 1);
          int cmax = d.base[0] + std::min(std::max(std::max(a, b) + Sx - 1, 0), d.extent[0] - 1);
          // planar source: the strip is at most kPlPx pixels wide after aligning its start down and its width up to 32 pixels
          // (the crop offset is only known at launch: worst-case slack), expressed on the kStRowBytes scale
          if (p->planar_mode) return (cmax - cmin + 1 + 62 <= kPlPx) ? kStRowBytes : kStRowBytes + 1;
          return (((cmax + 1) * C + 15) & ~15) - ((cmin * C) & ~15);
        };
        int stw = 0;
        for (int nx = 1; nx <= s.out_w; nx++) {
          int t = (s.out_w + nx - 1) / nx;
          bool ok = true;
          for (int o = 0; o < s.out_w && ok; o += t) ok = strip_bytes(o, std::min(t, s.out_w - o)) <= kStRowBytes;
          if (ok) { stw = t; break; }
          if (t == 1) break;
        }
        const int seg = kStSeg;
        bool ok = stw > 0 && MaxChunkSteps(iy, s.out_h, Sy) <= kWalkMax;
        if (ok) {   // (ix / iy are not used below: the arena may move)
          auto wc = p->walk_cache.find(d.idx_off[1]);
          if (wc != p->walk_cache.end()) {
            d.walk_off = wc->second;
          } else {
            d.walk_off = BuildWalkRecords(p->tables, d.idx_off[1], d.coef_off[1], s.out_h, Sy, W);
            p->walk_cache[d.idx_off[1]] = d.walk_off;
          }
          ok = d.walk_off >= 0;
        }
        if (ok) {
          p->stream_ok[i] = 1;
          for (int o = 0; o < s.out_h; o += seg)
            for (int x0 = 0; x0 < s.out_w; x0 += stw)
              p->items.push_back(RsItem{ i, x0, std::min(stw, s.out_w - x0), o, std::min(o + seg, s.out_h) });
        }
      }
    }
    tiles += (int64_t)d.tiles_x * d.tiles_y;
  }
  p->n = n; p->in_dtype = in_dtype; p->out_dtype = out_dtype; p->total_tiles = tiles;
  // identical tables (the common fixed-size case) are not uploaded again
  p->tables_dirty = p->tables != p->uploaded_tables;
  return DALIB200_SUCCESS;
} DB_API_CATCH

int dalib200ResamplePlanSetupPlanar(dalib200ResamplePlan *p, int n, const dalib200ResampleSample *samples, uint8_t *planar_ok) try {
  DB_CHECK_ARG(p && samples && planar_ok, "ResamplePlanSetupPlanar: null argument");
  p->planar_mode = true;
  const int rc = dalib200ResamplePlanSetup(p, n, samples, DALIB200_UINT8, DALIB200_UINT8);
  p->planar_mode = false;
  if (rc) return rc;
  // eligible = what the streaming kernel takes (vertical pass first, strictly increasing source rows, strips that fit), 3 channels;
  // items exist for exactly those samples
  for (int i = 0; i < n; i++) planar_ok[i] = p->stream_ok[i] && samples[i].channels == 3 && samples[i].in_w > 4;
  std::vector<RsItem> keep;
  for (const RsItem &it : p->items) if (planar_ok[it.sample]) keep.push_back(it);
  p->items.swap(keep);
  for (int i = 0; i < n; i++) p->stream_ok[i] = planar_ok[i];
  return DALIB200_SUCCESS;
} DB_API_CATCH

int dalib200ResampleLaunchPlanar(dalib200ResamplePlan *p, const dalib200PlanarImage *srcs, void *const *out_ptrs, dalib200Stream_t stream) try {
  DB_CHECK_ARG(p && srcs && out_ptrs, "ResampleLaunchPlanar: null argument");
  if (p->n == 0 || p->items.empty()) return DALIB200_SUCCESS;
  RsDesc *hd;
  int rc = p->desc_arena.Stage(sizeof(RsDesc) * p->n, &hd);
  if (rc) return rc;
  int wmax = 1;
  for (int i = 0; i < p->n; i++) {
    hd[i] = p->descs[i];
    hd[i].in = nullptr;
    hd[i].out = out_ptrs[i];
    hd[i].neg_zero = -0.0f;
    hd[i].use_stream = p->stream_ok[i];
    p->path[i] = p->stream_ok[i] ? 2 : 0;
    if (!p->stream_ok[i]) continue;
    const dalib200PlanarImage &s = srcs[i];
    DB_CHECK_ARG(s.y && s.cb && s.cr && s.pitch_y % 16 == 0 && s.pitch_c % 16 == 0 &&
                 (reinterpret_cast<uintptr_t>(s.y) | reinterpret_cast<uintptr_t>(s.cb) | reinterpret_cast<uintptr_t>(s.cr)) % 16 == 0,
                 "ResampleLaunchPlanar: sample %d: planes must be 16-byte aligned with a pitch that is a multiple of 16", i);
    DB_CHECK_ARG(s.crop_x >= 0 && s.crop_y >= 0 && s.crop_x + hd[i].in_w <= s.width && s.crop_y + hd[i].in_h <= s.height,
                 "ResampleLaunchPlanar: sample %d: the window does not fit the image", i);
    hd[i].pl[0] = s.y; hd[i].pl[1] = s.cb; hd[i].pl[2] = s.cr;
    hd[i].pitch_y = s.pitch_y; hd[i].pitch_c = s.pitch_c; hd[i].img_w = s.width; hd[i].img_h = s.height;
    hd[i].crop_x = s.crop_x; hd[i].crop_y = s.crop_y;
    wmax = std::max(wmax, (int)hd[i].walk_slots);
  }
  if ((rc = UploadLaunchData(p, true, stream))) return rc;
  const auto *dd = reinterpret_cast<const RsDesc *>(p->desc_arena.dev);
  const auto *tb = reinterpret_cast<const int32_t *>(p->table_arena.dev);
  const auto *di = reinterpret_cast<const RsItem *>(p->item_arena.dev);
  const int nitems = (int)p->items.size();
  const int sgrid = std::min(nitems, NumSMs() * 2);
  auto slaunch = [&](auto kern, int slot) -> int {
    if (!p->smem_opted[slot]) {
      DB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, kPlSmemBytes));
      p->smem_opted[slot] = true;
    }
    Launch("resample_planar", kern, sgrid, kStThreads, kPlSmemBytes, stream, dd, tb, di, nitems);
    return DALIB200_SUCCESS;
  };
  if (wmax <= 2)      rc = slaunch(resample_planar_kernel<2>, 10);
  else if (wmax == 3) rc = slaunch(resample_planar_kernel<3>, 11);
  else                rc = slaunch(resample_planar_kernel<4>, 12);
  if (rc) return rc;
  DB_CUDA(cudaGetLastError());
  return DALIB200_SUCCESS;
} DB_API_CATCH

int dalib200ResampleLaunch(dalib200ResamplePlan *p, const void *const *in_ptrs, void *const *out_ptrs, dalib200Stream_t stream) try {
  DB_CHECK_ARG(p && in_ptrs && out_ptrs, "ResampleLaunch: null argument");
  if (p->n == 0 || p->total_tiles == 0) return DALIB200_SUCCESS;
  RsDesc *hd;
  int rc = p->desc_arena.Stage(sizeof(RsDesc) * p->n, &hd);
  if (rc) return rc;
  int nstream = 0;
  for (int i = 0; i < p->n; i++) {
    hd[i] = p->descs[i];
    hd[i].in = in_ptrs[i];
    hd[i].out = out_ptrs[i];
    hd[i].neg_zero = -0.0f;
    hd[i].aligned4 = (reinterpret_cast<uintptr_t>(in_ptrs[i]) % 4 == 0) && ((int64_t)hd[i].in_w * hd[i].C % 4 == 0);
    hd[i].use_stream = p->stream_ok[i] && (reinterpret_cast<uintptr_t>(in_ptrs[i]) % 16 == 0) && ((int64_t)hd[i].in_w * hd[i].C % 16 == 0);
    p->path[i] = hd[i].use_stream;
    nstream += hd[i].use_stream;
  }
  if ((rc = UploadLaunchData(p, nstream > 0, stream))) return rc;
  const auto *dd = reinterpret_cast<const RsDesc *>(p->desc_arena.dev);
  const auto *tb = reinterpret_cast<const int32_t *>(p->table_arena.dev);
  if (nstream > 0) {
    const auto *di = reinterpret_cast<const RsItem *>(p->item_arena.dev);
    const int nitems = (int)p->items.size();
    const int sgrid = std::min(nitems, NumSMs() * 2);
    auto slaunch = [&](auto kern, int slot) -> int {
      if (!p->smem_opted[slot]) {
        DB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, kStSmemBytes));
        p->smem_opted[slot] = true;
      }
      Launch("resample_stream", kern, sgrid, kStThreads, kStSmemBytes, stream, dd, tb, di, nitems);
      return DALIB200_SUCCESS;
    };
    int wmax = 1;
    for (int i = 0; i < p->n; i++) if (hd[i].use_stream) wmax = std::max(wmax, (int)hd[i].walk_slots);
    const bool u8o = p->out_dtype == DALIB200_UINT8;
    if (wmax <= 2)      rc = u8o ? slaunch(resample_stream_kernel<uint8_t, 2>, 4) : slaunch(resample_stream_kernel<float, 2>, 5);
    else if (wmax == 3) rc = u8o ? slaunch(resample_stream_kernel<uint8_t, 3>, 6) : slaunch(resample_stream_kernel<float, 3>, 7);
    else                rc = u8o ? slaunch(resample_stream_kernel<uint8_t, 4>, 8) : slaunch(resample_stream_kernel<float, 4>, 9);
    if (rc) return rc;
    DB_CUDA(cudaGetLastError());
    if (nstream == p->n) return DALIB200_SUCCESS;
  }
  const int smem = kTmpFloats * sizeof(float) + kTileTableBytes;
  int grid = (int)std::min<int64_t>(p->total_tiles, (int64_t)NumSMs() * 2 * 8);
  auto launch = [&](auto kern, int slot) -> int {
    if (!p->smem_opted[slot]) {
      DB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
      p->smem_opted[slot] = true;
    }
    Launch("resample_fused", kern, grid, 256, smem, stream, dd, tb, p->n, p->total_tiles);
    return DALIB200_SUCCESS;
  };
  if (p->in_dtype == DALIB200_UINT8 && p->out_dtype == DALIB200_UINT8) rc = launch(resample_fused_kernel<uint8_t, uint8_t>, 0);
  else if (p->in_dtype == DALIB200_UINT8) rc = launch(resample_fused_kernel<uint8_t, float>, 1);
  else rc = launch(resample_fused_kernel<float, float>, 2);
  if (rc) return rc;
  DB_CUDA(cudaGetLastError());
  return DALIB200_SUCCESS;
} DB_API_CATCH

}  // extern "C"
