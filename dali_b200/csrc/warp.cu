// dali_b200/csrc/warp.cu -- WarpAffine for sm_90a.
//
// Parity target: reference CPU kernel WarpCPU<AffineMapping2D>::RunImpl (dali/kernels/imgproc/warp_cpu.h:143-178)
// with Sampler<NN|LINEAR> (dali/kernels/imgproc/sampler.h:122-330):
//   * source coordinates: src_tile = M * (0.5, y + 0.5)        (transform.h:134-145: t + m0*x + m1*y, left to right)
//     then per 256-pixel tile   src_tile += 256 * dsdx          and per pixel   src += dsdx    -- the CPU kernel
//     ACCUMULATES coordinates; to be bit-exact the accumulation is replayed: one thread per output row walks the
//     tile and leaves the coordinates in shared memory, the whole CTA then samples from them.
//     (The reference GPU kernel recomputes M*(x+0.5, y+0.5) per pixel, block_warp.cuh:54-58, and therefore differs
//      from its own CPU backend in the last coordinate bits.)
//   * bilinear: x-=0.5; x0=floor; s0 = s00*(1-qx) + s01*qx; s1 = ...; out = s0 + (s1-s0)*qy   (mul/add unfused)
//   * border: clamp, or constant = ConvertSat<In>(fill_value)
//
// Algorithmic bytes per unit (SURVEY.md 8d): in_h*in_w*C + out_h*out_w*C*sizeof(Out).
#include "common.cuh"
#include <cuda.h>            // CUtensorMap (the encoder is resolved through cudaGetDriverEntryPoint: no libcuda link dependency)
#include <algorithm>
#include <cstring>

namespace dalib200 {

constexpr int kWarpTileW = 256;     // the reference's coordinate re-anchoring period (warp_cpu.h:160)
constexpr int kWarpTileH = 16;    // rows per tile: 16 threads replay coordinates while 4096 pixels are sampled by the CTA

struct WarpDesc {
  const uint8_t *in;
  void *out;
  int32_t in_h, in_w, C, out_h, out_w;
  int32_t tiles_x, tiles_y;
  int64_t first_tile;
  float m[6];
};

template <bool CLAMP>
__device__ __forceinline__ float warp_fetch(const uint8_t *__restrict__ in, int H, int W, int C, int x, int y, int c, float border) {
  if ((unsigned)x < (unsigned)W && (unsigned)y < (unsigned)H) return (float)__ldg(in + ((int64_t)y * W + x) * C + c);
  if (CLAMP) {
    const int cx = min(max(x, 0), W - 1), cy = min(max(y, 0), H - 1);
    return (float)__ldg(in + ((int64_t)cy * W + cx) * C + c);
  }
  return border;
}

template <typename Out> __device__ __forceinline__ Out warp_cvt(float v);
template <> __device__ __forceinline__ float warp_cvt<float>(float v) { return v; }
template <> __device__ __forceinline__ uint8_t warp_cvt<uint8_t>(float v) { return sat_u8_half_away(v); }

// One output pixel (all channels) from its replayed source coordinate.  Interior pixels (the whole 2x2 footprint inside the
// image) skip the per-tap bounds logic.
template <typename Out, bool LINEAR, bool CLAMP, int CMAX>
__device__ __forceinline__ void warp_pixel(const WarpDesc &d, float2 src, float border, int C, float *res) {
  const uint8_t *__restrict__ in = d.in;
  const int H = d.in_h, W = d.in_w;
  if (!LINEAR) {
    const int ix = (int)floorf(src.x), iy = (int)floorf(src.y);
#pragma unroll
    for (int c = 0; c < CMAX; c++) if (c < C) res[c] = warp_fetch<CLAMP>(in, H, W, C, ix, iy, c, border);
    return;
  }
  const float fx = sub_rn(src.x, 0.5f), fy = sub_rn(src.y, 0.5f);
  const float flx = floorf(fx), fly = floorf(fy);
  const int ix = (int)flx, iy = (int)fly;
  const float qx = sub_rn(fx, flx), px = sub_rn(1.0f, qx), qy = sub_rn(fy, fly);
  const bool interior = ix >= 0 && iy >= 0 && ix + 1 < W && iy + 1 < H;
  const uint8_t *p0 = in + ((int64_t)iy * W + ix) * C, *p1 = p0 + (int64_t)W * C;
  if (CMAX == 3 && interior && iy + 2 < H) {
    // 3 channels, interior (and not the last row pair, so that the 12-byte windows below stay inside the image): the two
    // pixels of a source row are 6 contiguous bytes -> three aligned 32-bit loads + funnel shifts instead of six byte loads
    float t0[6], t1[6];
#pragma unroll
    for (int r = 0; r < 2; r++) {
      const uint8_t *p = r ? p1 : p0;
      const uint32_t sh = (uint32_t)(reinterpret_cast<uintptr_t>(p) & 3u);
      const uint32_t *w = reinterpret_cast<const uint32_t *>(p - sh);
      const uint32_t w0 = __ldg(w), w1 = __ldg(w + 1), w2 = __ldg(w + 2);
      const uint32_t lo = __funnelshift_r(w0, w1, sh * 8u), hi = __funnelshift_r(w1, w2, sh * 8u);
      float *t = r ? t1 : t0;
      t[0] = u8_to_float(lo & 0xFFu); t[1] = u8_to_float((lo >> 8) & 0xFFu); t[2] = u8_to_float((lo >> 16) & 0xFFu);
      t[3] = u8_to_float(lo >> 24); t[4] = u8_to_float(hi & 0xFFu); t[5] = u8_to_float((hi >> 8) & 0xFFu);
    }
#pragma unroll
    for (int c = 0; c < 3; c++) {
      const float s0 = add_rn(mul_rn(t0[c], px), mul_rn(t0[3 + c], qx));
      const float s1 = add_rn(mul_rn(t1[c], px), mul_rn(t1[3 + c], qx));
      res[c] = add_rn(s0, mul_rn(sub_rn(s1, s0), qy));
    }
    return;
  }
#pragma unroll
  for (int c = 0; c < CMAX; c++) {
    if (c < C) {
      float s00, s01, s10, s11;
      if (interior) {
        s00 = u8_to_float(__ldg(p0 + c)); s01 = u8_to_float(__ldg(p0 + C + c)); s10 = u8_to_float(__ldg(p1 + c)); s11 = u8_to_float(__ldg(p1 + C + c));
      } else {
        s00 = warp_fetch<CLAMP>(in, H, W, C, ix, iy, c, border);
        s01 = warp_fetch<CLAMP>(in, H, W, C, ix + 1, iy, c, border);
        s10 = warp_fetch<CLAMP>(in, H, W, C, ix, iy + 1, c, border);
        s11 = warp_fetch<CLAMP>(in, H, W, C, ix + 1, iy + 1, c, border);
      }
      const float s0 = add_rn(mul_rn(s00, px), mul_rn(s01, qx));
      const float s1 = add_rn(mul_rn(s10, px), mul_rn(s11, qx));
      res[c] = add_rn(s0, mul_rn(sub_rn(s1, s0), qy));
    }
  }
}

template <typename Out, bool LINEAR, bool CLAMP>
__global__ void __launch_bounds__(256) warp_affine_kernel(const WarpDesc *__restrict__ descs, int n, int64_t total_tiles,
                                                          float border) {
  __shared__ float2 coords[kWarpTileH][kWarpTileW];
  __shared__ int s_first;
  // contiguous range of tiles per CTA: the sample is searched once and then only advanced
  const int64_t per_cta = (total_tiles + gridDim.x - 1) / gridDim.x;
  const int64_t t0 = (int64_t)blockIdx.x * per_cta, t1 = min(total_tiles, t0 + per_cta);
  if (t0 >= t1) return;
  if (threadIdx.x == 0) s_first = last_at_most(descs, 0, n - 1, t0, [](const WarpDesc &d) { return d.first_tile; });
  __syncthreads();
  int s = s_first;
  for (int64_t tile = t0; tile < t1; tile++) {
    while (s + 1 < n && descs[s + 1].first_tile <= tile) s++;
    const WarpDesc &d = descs[s];
    const int64_t tl = tile - d.first_tile;
    const int ty = (int)((uint32_t)tl / (uint32_t)d.tiles_x), tx = (int)((uint32_t)tl - (uint32_t)ty * (uint32_t)d.tiles_x);
    const int y0 = ty * kWarpTileH, x0 = tx * kWarpTileW;
    const int th = min(kWarpTileH, d.out_h - y0), tw = min(kWarpTileW, d.out_w - x0);
    // ---- stage 1: replay the reference's coordinate accumulation, one thread per row
    if (threadIdx.x < th) {
      const int y = y0 + threadIdx.x;
      const float vx = 0.5f, vy = (float)y + 0.5f;
      float sx = add_rn(add_rn(d.m[2], mul_rn(d.m[0], vx)), mul_rn(d.m[1], vy));
      float sy = add_rn(add_rn(d.m[5], mul_rn(d.m[3], vx)), mul_rn(d.m[4], vy));
      const float dx = d.m[0], dy = d.m[3];
      const float tdx = mul_rn(256.0f, dx), tdy = mul_rn(256.0f, dy);
      for (int t = 0; t < tx; t++) { sx = add_rn(sx, tdx); sy = add_rn(sy, tdy); }
      for (int j = 0; j < tw; j++) {
        coords[threadIdx.x][j] = make_float2(sx, sy);
        sx = add_rn(sx, dx); sy = add_rn(sy, dy);
      }
    }
    __syncthreads();
    // ---- stage 2: sample; one thread = 4 consecutive pixels of a row (u8, 3 channels: three 32-bit stores)
    const int C = d.C;
    Out *out = static_cast<Out *>(d.out);
    const int gpr = (tw + 3) >> 2;
    for (int e = threadIdx.x; e < th * gpr; e += blockDim.x) {
      const int r = e / gpr, j0 = (e - r * gpr) << 2;
      const int np = min(4, tw - j0);
      Out *o = out + ((int64_t)(y0 + r) * d.out_w + x0 + j0) * C;
      if (sizeof(Out) == 1 && C == 3 && np == 4 && (reinterpret_cast<uintptr_t>(o) & 3) == 0) {
        uint32_t b[12];
#pragma unroll
        for (int k = 0; k < 4; k++) {
          float res[3];
          warp_pixel<Out, LINEAR, CLAMP, 3>(d, coords[r][j0 + k], border, 3, res);
#pragma unroll
          for (int c = 0; c < 3; c++) b[3 * k + c] = (uint32_t)sat_u8_half_away(res[c]);
        }
        uint32_t *o4 = reinterpret_cast<uint32_t *>(o);
        o4[0] = b[0] | (b[1] << 8) | (b[2] << 16) | (b[3] << 24);
        o4[1] = b[4] | (b[5] << 8) | (b[6] << 16) | (b[7] << 24);
        o4[2] = b[8] | (b[9] << 8) | (b[10] << 16) | (b[11] << 24);
      } else {
        for (int k = 0; k < np; k++) {
          float res[8];
          warp_pixel<Out, LINEAR, CLAMP, 8>(d, coords[r][j0 + k], border, C, res);
          for (int c = 0; c < C; c++) o[k * C + c] = warp_cvt<Out>(res[c]);
        }
      }
    }
    __syncthreads();
  }
}

// =============================================================================================
// Band kernel: bilinear, 3-channel u8 -> u8 (the C3 hot case).
//
// The reference's coordinate accumulation is a serial recurrence per (row, 256-pixel block); with one thread per row of a 16-row
// tile only half a warp works on it while the other warps wait, and it then costs more than the sampling.  Here a CTA owns a BAND
// of 32 output rows x up to 2048 columns:
//   phase 1  one thread per (row, 256-block) -- 256 independent chains, all lanes busy -- replays the recurrence and keeps every
//            16th coordinate (an ANCHOR) in shared memory (32 x 129 float2);
//   phase 2  the band is walked in 32 x 128 tiles; a thread owns one 16-pixel run of a row: it restarts the recurrence at the run's
//            anchor (15 more adds -- the very same additions the reference performs) and samples as it goes, so the coordinates
//            of the other 15 pixels never touch memory; it writes its 48 output bytes as three 16-byte stores.
// With a tensor map (uniform batches: frames of one shape at a constant stride) the source box of tile t + 2 is fetched by ONE
// tiled TMA load (cp.async.bulk.tensor.3d, SASS UTMALDG.3D) into a two-deep shared-memory ring while tile t is sampled, and the
// taps come from shared memory; the box (448 bytes x 64 rows) covers rotations of about +-12 degrees at unit scale.  A pixel whose
// footprint is not inside the loaded box (large angles, down-scaling maps, image borders, no tensor map at all) takes the generic
// tap path of warp_pixel -- decided per pixel from its replayed coordinate, so a wrong box estimate can cost time, not correctness.
// The box must START on a 16-byte boundary of the innermost dimension: a tile coordinate with (c0 * 4) % 16 != 0 faults with
// "illegal instruction" at the UTMALDG (measured, tools/probe/tma_probe.cu), so the byte column of the box is aligned down to 16.
constexpr int kBandH = 32, kBandW = 2048, kBandTileW = 128, kRun = 16;
constexpr int kAnchorPitch = kBandW / kRun + 1;                       // float2 per row (+1: conflict-free column accesses)
constexpr int kTmaBoxBytes = 448, kTmaBoxRows = 64;
constexpr size_t kBandSmem = sizeof(float2) * kBandH * kAnchorPitch + 2 * (size_t)kTmaBoxRows * kTmaBoxBytes + 128;

struct BoxInfo { int use, bx, by; };

// the rare path of the band kernel (borders, pixels outside the loaded box), kept OUT of line: inlined into the 16-times unrolled
// pixel loop it grew the kernel to 4 096 instructions and the warps stalled on instruction fetch (ncu: no_instruction top stall)
template <bool CLAMP>
__device__ __noinline__ void warp_pixel_outline(const WarpDesc &d, float sx, float sy, float border, float *res) {
  warp_pixel<uint8_t, true, CLAMP, 3>(d, make_float2(sx, sy), border, 3, res);
}

template <bool CLAMP>
__global__ void __launch_bounds__(256, 2) warp_affine_band_kernel(const WarpDesc *__restrict__ descs, int n, int64_t total_items, float border,
                                                                  const __grid_constant__ CUtensorMap tmap, int use_tma) {
  extern __shared__ __align__(128) uint8_t band_smem[];
  uint8_t *box0 = band_smem;                                                       // 2 boxes, 128-byte aligned
  float2 *anchors = reinterpret_cast<float2 *>(band_smem + 2 * kTmaBoxRows * kTmaBoxBytes);
  __shared__ __align__(8) uint64_t bars[2];
  __shared__ BoxInfo binfo[2];
  __shared__ int s_first;
  const int tid = threadIdx.x;
  const int64_t per_cta = (total_items + gridDim.x - 1) / gridDim.x;
  const int64_t i0 = (int64_t)blockIdx.x * per_cta, i1 = min(total_items, i0 + per_cta);
  if (i0 >= i1) return;
  if (tid == 0) {
    s_first = last_at_most(descs, 0, n - 1, i0, [](const WarpDesc &d) { return d.first_tile; });
    mbar_init(&bars[0], 1); mbar_init(&bars[1], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  int s = s_first;
  uint32_t phase[2] = {0u, 0u};
  for (int64_t item = i0; item < i1; item++) {
    while (s + 1 < n && descs[s + 1].first_tile <= item) s++;
    const WarpDesc &d = descs[s];
    const int64_t li = item - d.first_tile;
    const int by_ = (int)((uint32_t)li / (uint32_t)d.tiles_x), gx = (int)((uint32_t)li - (uint32_t)by_ * (uint32_t)d.tiles_x);
    const int y0 = by_ * kBandH, X0 = gx * kBandW;
    const int bh = min(kBandH, d.out_h - y0), bw = min(kBandW, d.out_w - X0);
    const float dx = d.m[0], dy = d.m[3];
    // ---- phase 1: anchors.  thread = (row, 256-block of the band)
    {
      const int r = tid & 31, k = tid >> 5;                       // 8 blocks of 256 columns
      if (r < bh && k * 256 < bw) {
        const float vy = (float)(y0 + r) + 0.5f;
        float sx = add_rn(add_rn(d.m[2], mul_rn(d.m[0], 0.5f)), mul_rn(d.m[1], vy));
        float sy = add_rn(add_rn(d.m[5], mul_rn(d.m[3], 0.5f)), mul_rn(d.m[4], vy));
        const float tdx = mul_rn(256.0f, dx), tdy = mul_rn(256.0f, dy);
        for (int t = 0; t < (X0 >> 8) + k; t++) { sx = add_rn(sx, tdx); sy = add_rn(sy, tdy); }
        const int steps = min(256, bw - k * 256);
        float2 *arow = anchors + r * kAnchorPitch + k * (256 / kRun);
        for (int j = 0; j < steps; j += kRun) {
          arow[j / kRun] = make_float2(sx, sy);
#pragma unroll
          for (int q = 0; q < kRun; q++) { sx = add_rn(sx, dx); sy = add_rn(sy, dy); }
        }
      }
    }
    __syncthreads();
    // ---- phase 2: 32 x 128 tiles, two boxes in flight
    const int ntiles = (bw + kBandTileW - 1) / kBandTileW;
    auto issue = [&](int t) {                                     // thread 0 only: source box of tile t -> ring slot t & 1
      const int slot = t & 1;
      BoxInfo bi; bi.use = 0; bi.bx = 0; bi.by = 0;
      if (use_tma) {
        const int tx0 = X0 + t * kBandTileW, tw = min(kBandTileW, bw - t * kBandTileW);
        // the map is affine: the extremes of the tile's footprint sit at its corners (exact map here; the replayed coordinates
        // drift from it by far less than the one-pixel margin, and a pixel outside the box falls back to the generic taps anyway)
        float minx = 3.0e38f, maxx = -3.0e38f, miny = 3.0e38f, maxy = -3.0e38f;
#pragma unroll
        for (int c = 0; c < 4; c++) {
          const float ux = (float)(tx0 + ((c & 1) ? tw - 1 : 0)) + 0.5f, uy = (float)(y0 + ((c & 2) ? bh - 1 : 0)) + 0.5f;
          const float px = d.m[2] + d.m[0] * ux + d.m[1] * uy, py = d.m[5] + d.m[3] * ux + d.m[4] * uy;
          minx = fminf(minx, px); maxx = fmaxf(maxx, px); miny = fminf(miny, py); maxy = fmaxf(maxy, py);
        }
        if (fabsf(minx) < 1.0e6f && fabsf(maxx) < 1.0e6f && fabsf(miny) < 1.0e6f && fabsf(maxy) < 1.0e6f) {
          const int ix0 = (int)floorf(minx - 0.5f) - 1, iy0 = (int)floorf(miny - 0.5f) - 1;
          const int iy1 = (int)floorf(maxy - 0.5f) + 2;
          bi.bx = (ix0 * 3) & ~15;                                  // 16-byte aligned start (TMA requirement)
          bi.by = iy0;
          // worth fetching only if the box can hold most of the footprint; each pixel re-checks its own taps
          bi.use = ((int)floorf(maxx - 0.5f) + 4) * 3 - bi.bx <= kTmaBoxBytes + 96 && iy1 - iy0 + 1 <= kTmaBoxRows + 8 &&
                   bi.bx + kTmaBoxBytes > 0 && bi.bx < d.in_w * 3 && iy0 + kTmaBoxRows > 0 && iy0 < d.in_h;
        }
      }
      binfo[slot] = bi;
      if (bi.use) {
        mbar_expect_tx(&bars[slot], kTmaBoxRows * kTmaBoxBytes);
        tma_load_3d(box0 + slot * kTmaBoxRows * kTmaBoxBytes, &tmap, bi.bx >> 2, bi.by, s, &bars[slot]);
      }
    };
    if (tid == 0) { issue(0); if (ntiles > 1) issue(1); }
    __syncthreads();
    const int row = tid >> 3, seg = tid & 7;
    uint8_t *out = static_cast<uint8_t *>(d.out);
    for (int t = 0; t < ntiles; t++) {
      const int slot = t & 1;
      const BoxInfo bi = binfo[slot];
      if (bi.use) { mbar_wait(&bars[slot], phase[slot]); phase[slot] ^= 1u; }
      const int lx = t * kBandTileW + seg * kRun;                  // column of the run inside the band
      if (row < bh && lx < bw) {
        const int np = min(kRun, bw - lx);
        const float2 a = anchors[row * kAnchorPitch + lx / kRun];
        float sx = a.x, sy = a.y;
        const uint32_t a_box = smem_u32(box0 + slot * kTmaBoxRows * kTmaBoxBytes);
        uint32_t w[12];
#pragma unroll
        for (int q = 0; q < 12; q++) w[q] = 0u;
#pragma unroll
        for (int k = 0; k < kRun; k++) {
          if (k < np) {
            float res[3];
            const float fx = sub_rn(sx, 0.5f), fy = sub_rn(sy, 0.5f);
            const float flx = floorf(fx), fly = floorf(fy);
            const int ix = (int)flx, iy = (int)fly;
            const int col = ix * 3 - bi.bx, rr0 = iy - bi.by;
            // taps (ix, ix + 1) x (iy, iy + 1) inside the image AND their 12-byte windows inside the loaded box
            const bool in_box = bi.use && (unsigned)col <= (unsigned)(kTmaBoxBytes - 12) && (unsigned)rr0 < (unsigned)(kTmaBoxRows - 1) &&
                                (unsigned)ix < (unsigned)(d.in_w - 1) && (unsigned)iy < (unsigned)(d.in_h - 1);
            if (in_box) {
              const float qx = sub_rn(fx, flx), px = sub_rn(1.0f, qx), qy = sub_rn(fy, fly);
              // products without converting the bytes: 0x4B0000bb is the float 2^23 + b, and fma(2^23 + b, p, -2^23 p) = RN(b p)
              // exactly (2^23 p is exact) -- one PRMT per byte instead of extract + bias subtract, the product is one FFMA
              const float npx = mul_rn(px, -8388608.0f), nqx = mul_rn(qx, -8388608.0f);
              float s[2][3];
#pragma unroll
              for (int rr = 0; rr < 2; rr++) {
                const uint32_t off = (uint32_t)((rr0 + rr) * kTmaBoxBytes + col);
                const uint32_t sh = off & 3u, ad = a_box + (off & ~3u);
                const uint32_t w0 = lds_u32(ad), w1 = lds_u32(ad + 4), w2 = lds_u32(ad + 8);
                const uint32_t lo = __funnelshift_r(w0, w1, sh * 8u), hi = __funnelshift_r(w1, w2, sh * 8u);
                const float b0 = __uint_as_float(__byte_perm(lo, 0x4B000000u, 0x7440)), b1 = __uint_as_float(__byte_perm(lo, 0x4B000000u, 0x7441));
                const float b2 = __uint_as_float(__byte_perm(lo, 0x4B000000u, 0x7442)), b3 = __uint_as_float(__byte_perm(lo, 0x4B000000u, 0x7443));
                const float b4 = __uint_as_float(__byte_perm(hi, 0x4B000000u, 0x7440)), b5 = __uint_as_float(__byte_perm(hi, 0x4B000000u, 0x7441));
                s[rr][0] = add_rn(__fmaf_rn(b0, px, npx), __fmaf_rn(b3, qx, nqx));
                s[rr][1] = add_rn(__fmaf_rn(b1, px, npx), __fmaf_rn(b4, qx, nqx));
                s[rr][2] = add_rn(__fmaf_rn(b2, px, npx), __fmaf_rn(b5, qx, nqx));
              }
#pragma unroll
              for (int c = 0; c < 3; c++) res[c] = add_rn(s[0][c], mul_rn(sub_rn(s[1][c], s[0][c]), qy));
            } else {
              warp_pixel_outline<CLAMP>(d, sx, sy, border, res);
            }
#pragma unroll
            for (int c = 0; c < 3; c++) {
              const int bidx = 3 * k + c;
              w[bidx >> 2] = __byte_perm(w[bidx >> 2], round_u8_bits(res[c]), (bidx & 3) == 0 ? 0x3214 : (bidx & 3) == 1 ? 0x3240 : (bidx & 3) == 2 ? 0x3410 : 0x4210);
            }
            sx = add_rn(sx, dx); sy = add_rn(sy, dy);
          }
        }
        uint8_t *o = out + ((int64_t)(y0 + row) * d.out_w + X0 + lx) * 3;
        if (np == kRun && (reinterpret_cast<uintptr_t>(o) & 15) == 0) {
          uint4 *o16 = reinterpret_cast<uint4 *>(o);
          o16[0] = make_uint4(w[0], w[1], w[2], w[3]); o16[1] = make_uint4(w[4], w[5], w[6], w[7]); o16[2] = make_uint4(w[8], w[9], w[10], w[11]);
        } else if (np == kRun && (reinterpret_cast<uintptr_t>(o) & 3) == 0) {
          uint32_t *o4 = reinterpret_cast<uint32_t *>(o);
#pragma unroll
          for (int q = 0; q < 12; q++) o4[q] = w[q];
        } else {
#pragma unroll
          for (int q = 0; q < kRun * 3; q++)
            if (q < np * 3) o[q] = (uint8_t)(w[q >> 2] >> (8 * (q & 3)));
        }
      }
      __syncthreads();                                             // every reader of ring slot `slot` is done
      if (tid == 0 && t + 2 < ntiles) issue(t + 2);
    }
    __syncthreads();                                               // anchors and binfo are rewritten by the next item
  }
}

}  // namespace dalib200

using namespace dalib200;  // NOLINT

struct dalib200WarpPlan {
  int max_batch = 0, n = 0;
  int interp = 1, use_fill = 0, out_dtype = DALIB200_UINT8;
  float border = 0;
  int64_t total_tiles = 0;
  DescArena arena;
  // band kernel / tensor-map path: the map is cached per (base, stride, shape)
  std::vector<dalib200WarpSample> samples;
  CUtensorMap tmap;
  const void *tmap_base = nullptr; size_t tmap_stride = 0; int tmap_h = 0, tmap_w = 0, tmap_n = 0;
  int path = 0;                  // last launch: 0 generic kernel, 1 band kernel with tensor-map TMA boxes, 2 band kernel without
  bool smem_set = false;         // the band kernel's dynamic shared-memory attribute is set (on this plan's device)
};

namespace {
typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *,
                                  const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                                  CUtensorMapFloatOOBfill);
EncodeTiledFn GetEncodeTiled() {
  static EncodeTiledFn fn = []() -> EncodeTiledFn {
    void *p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess) return nullptr;
    return reinterpret_cast<EncodeTiledFn>(p);
  }();
  return fn;
}
}  // namespace

extern "C" {

int dalib200WarpPlanGetPath(const dalib200WarpPlan *p) { return p ? p->path : -1; }

void dalib200AffineInverse(const float *M, float *out) {
  // include/dali/core/geom/transform.h:166-174 + mat.h:611-623: m = adj(2x2)/det ; t = (-m) * t
  const float det = M[0] * M[4] - M[1] * M[3];
  const float m00 = M[4] / det, m01 = -M[1] / det, m10 = -M[3] / det, m11 = M[0] / det;
  const float n00 = -m00, n01 = -m01, n10 = -m10, n11 = -m11;
  volatile float a = n00 * M[2], b = n01 * M[5];
  const float t0 = a + b;
  volatile float c = n10 * M[2], d = n11 * M[5];
  const float t1 = c + d;
  out[0] = m00; out[1] = m01; out[2] = t0; out[3] = m10; out[4] = m11; out[5] = t1;
}

int dalib200WarpPlanCreate(dalib200WarpPlan **plan, int max_batch) try {
  DB_CHECK_ARG(plan && max_batch > 0, "WarpPlanCreate: bad arguments");
  auto *p = new dalib200WarpPlan();
  p->max_batch = max_batch;
  int rc = p->arena.Reserve(sizeof(WarpDesc) * max_batch);
  if (rc) { delete p; return rc; }
  *plan = p;
  return DALIB200_SUCCESS;
} DB_API_CATCH

int dalib200WarpPlanDestroy(dalib200WarpPlan *p) try {
  if (!p) return DALIB200_SUCCESS;
  p->arena.Free();
  delete p;
  return DALIB200_SUCCESS;
} DB_API_CATCH

int dalib200WarpPlanSetup(dalib200WarpPlan *p, int n, const dalib200WarpSample *samples, int interp, int use_fill,
                          float fill_value, int out_dtype) try {
  DB_CHECK_ARG(p && samples && n >= 0, "WarpPlanSetup: null argument");
  DB_CHECK_ARG(n <= p->max_batch, "WarpPlanSetup: batch %d exceeds plan capacity %d", n, p->max_batch);
  DB_CHECK_ARG(interp == 0 || interp == 1, "WarpAffine: only NN and LINEAR interpolation are supported (got %d)", interp);
  DB_CHECK_ARG(out_dtype == DALIB200_UINT8 || out_dtype == DALIB200_FLOAT, "WarpAffine: output type %d not supported", out_dtype);
  WarpDesc *descs;
  if (int rc = p->arena.Stage(sizeof(WarpDesc) * n, &descs)) return rc;
  p->samples.assign(samples, samples + n);
  int64_t tiles = 0;
  for (int i = 0; i < n; i++) {
    const auto &s = samples[i];
    DB_CHECK_ARG(s.in_h > 0 && s.in_w > 0 && s.channels >= 1 && s.channels <= 8 && s.out_h >= 0 && s.out_w >= 0,
                 "WarpAffine: sample %d has unsupported shapes", i);
    WarpDesc &d = descs[i];
    memset(&d, 0, sizeof(d));
    d.in_h = s.in_h; d.in_w = s.in_w; d.C = s.channels; d.out_h = s.out_h; d.out_w = s.out_w;
    DB_CHECK_ARG(ElementsFit31(s.in_h, s.in_w, s.channels) && ElementsFit31(s.out_h, s.out_w, s.channels),
                 "WarpAffine: sample %d: images of 2^31 elements or more are not supported", i);
    d.tiles_x = static_cast<int>((static_cast<int64_t>(s.out_w) + kWarpTileW - 1) / kWarpTileW);
    d.tiles_y = static_cast<int>((static_cast<int64_t>(s.out_h) + kWarpTileH - 1) / kWarpTileH);
    d.first_tile = tiles;
    tiles += (int64_t)d.tiles_x * d.tiles_y;
    memcpy(d.m, s.matrix, sizeof(d.m));
  }
  p->n = n; p->interp = interp; p->use_fill = use_fill != 0; p->out_dtype = out_dtype; p->total_tiles = tiles;
  // ConvertSat<uint8_t>(fill_value): round half away, clamp (warp.h:268, convert.h:306-324)
  float r = std::round(fill_value);
  p->border = r <= 0 ? 0.0f : r >= 255 ? 255.0f : r;
  return DALIB200_SUCCESS;
} DB_API_CATCH

int dalib200WarpLaunch(dalib200WarpPlan *p, const void *const *in_ptrs, void *const *out_ptrs, dalib200Stream_t stream) try {
  DB_CHECK_ARG(p && in_ptrs && out_ptrs, "WarpLaunch: null argument");
  if (p->n == 0 || p->total_tiles == 0) return DALIB200_SUCCESS;
  WarpDesc *descs;
  if (int rc = p->arena.Stage(sizeof(WarpDesc) * p->n, &descs)) return rc;
  for (int i = 0; i < p->n; i++) { descs[i].in = static_cast<const uint8_t *>(in_ptrs[i]); descs[i].out = out_ptrs[i]; }
  // ---- band kernel: bilinear u8 -> u8, every sample 3-channel (DALIB200_WARP_GENERIC=1 forces the generic kernel: A/B runs) ...
  bool band = p->interp == 1 && p->out_dtype == DALIB200_UINT8 && !getenv("DALIB200_WARP_GENERIC");
  for (int i = 0; i < p->n && band; i++) band = p->samples[i].channels == 3;
  // ---- ... with tensor-map TMA source boxes: the batch must be uniform (frames of one shape laid out at a constant stride).
  // Without the boxes the band kernel measures slower than the generic kernel (every pixel takes the out-of-line tap path), so it
  // is only used together with them unless DALIB200_WARP_BAND=1 asks for it.
  bool tma = band && !getenv("DALIB200_WARP_NO_TMA") && GetEncodeTiled() != nullptr;
  const auto &s0 = p->samples[0];
  size_t stride = 0;
  if (tma) {
    tma = (s0.in_w * 3) % 16 == 0 && reinterpret_cast<uintptr_t>(in_ptrs[0]) % 16 == 0 && s0.in_w * 3 >= kTmaBoxBytes;
    if (tma && p->n > 1) {
      stride = static_cast<const uint8_t *>(in_ptrs[1]) - static_cast<const uint8_t *>(in_ptrs[0]);
      tma = static_cast<const uint8_t *>(in_ptrs[1]) > static_cast<const uint8_t *>(in_ptrs[0]) && stride % 16 == 0 &&
            stride >= (size_t)s0.in_h * s0.in_w * 3;
    } else if (tma) {
      stride = (size_t)s0.in_h * s0.in_w * 3;
    }
    for (int i = 0; i < p->n && tma; i++) {
      const auto &s = p->samples[i];
      tma = s.in_h == s0.in_h && s.in_w == s0.in_w &&
            static_cast<const uint8_t *>(in_ptrs[i]) == static_cast<const uint8_t *>(in_ptrs[0]) + (size_t)i * stride;
    }
  }
  if (tma && (p->tmap_base != in_ptrs[0] || p->tmap_stride != stride || p->tmap_h != s0.in_h || p->tmap_w != s0.in_w || p->tmap_n != p->n)) {
    // the batch as a rank-3 tensor of 32-bit words: [frame][row][word]; box = 112 words x 64 rows x 1 frame
    const cuuint64_t dims[3] = { (cuuint64_t)s0.in_w * 3 / 4, (cuuint64_t)s0.in_h, (cuuint64_t)p->n };
    const cuuint64_t strides[2] = { (cuuint64_t)s0.in_w * 3, (cuuint64_t)stride };
    const cuuint32_t box[3] = { kTmaBoxBytes / 4, kTmaBoxRows, 1 }, estr[3] = { 1, 1, 1 };
    const CUresult r = GetEncodeTiled()(&p->tmap, CU_TENSOR_MAP_DATA_TYPE_UINT32, 3, const_cast<void *>(in_ptrs[0]), dims, strides, box, estr,
                                        CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
      tma = false; p->tmap_base = nullptr;
    } else {
      p->tmap_base = in_ptrs[0]; p->tmap_stride = stride; p->tmap_h = s0.in_h; p->tmap_w = s0.in_w; p->tmap_n = p->n;
    }
  }
  if (!tma && !getenv("DALIB200_WARP_BAND")) band = false;
  p->path = !band ? 0 : tma ? 1 : 2;
  int64_t total_tiles = 0;
  for (int i = 0; i < p->n; i++) {        // work items: 32-row bands x 2048-column groups, or the generic kernel's 16 x 256 tiles
    descs[i].tiles_x = band ? (descs[i].out_w + kBandW - 1) / kBandW : (descs[i].out_w + kWarpTileW - 1) / kWarpTileW;
    descs[i].tiles_y = band ? (descs[i].out_h + kBandH - 1) / kBandH : (descs[i].out_h + kWarpTileH - 1) / kWarpTileH;
    descs[i].first_tile = total_tiles;
    total_tiles += (int64_t)descs[i].tiles_x * descs[i].tiles_y;
  }
  int rc = p->arena.Upload(sizeof(WarpDesc) * p->n, stream);
  if (rc) return rc;
  const auto *dd = reinterpret_cast<const WarpDesc *>(p->arena.dev);
  const bool lin = p->interp == 1, clampb = !p->use_fill, u8 = p->out_dtype == DALIB200_UINT8;
  if (band) {
    // the shared-memory attribute belongs to the kernel on the current device, so it is set once per PLAN, not once per process: a
    // plan's descriptor arena lives on the device it was created on, and a process warping on two devices has a plan on each
    if (!p->smem_set) {
      DB_CUDA(cudaFuncSetAttribute(warp_affine_band_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kBandSmem));
      DB_CUDA(cudaFuncSetAttribute(warp_affine_band_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kBandSmem));
      p->smem_set = true;
    }
    const int grid = (int)std::min<int64_t>(total_tiles, (int64_t)NumSMs() * 2);
    Launch(tma ? "warp_affine_tma" : "warp_affine_band", clampb ? warp_affine_band_kernel<true> : warp_affine_band_kernel<false>, grid, 256, kBandSmem,
           stream, dd, p->n, total_tiles, p->border, p->tmap, tma ? 1 : 0);
    DB_CUDA(cudaGetLastError());
    return DALIB200_SUCCESS;
  }
  const int grid = (int)std::min<int64_t>(total_tiles, (int64_t)NumSMs() * 16);
  const auto kernel = u8 ? (lin ? (clampb ? warp_affine_kernel<uint8_t, true, true> : warp_affine_kernel<uint8_t, true, false>)
                                : (clampb ? warp_affine_kernel<uint8_t, false, true> : warp_affine_kernel<uint8_t, false, false>))
                         : (lin ? (clampb ? warp_affine_kernel<float, true, true> : warp_affine_kernel<float, true, false>)
                                : (clampb ? warp_affine_kernel<float, false, true> : warp_affine_kernel<float, false, false>));
  Launch("warp_affine", kernel, grid, 256, 0, stream, dd, p->n, total_tiles, p->border);
  DB_CUDA(cudaGetLastError());
  return DALIB200_SUCCESS;
} DB_API_CATCH

}  // extern "C"
