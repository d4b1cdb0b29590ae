// dali_b200/csrc/audio.cu -- Spectrogram (framing + window + FFT + |X|^p) and MelFilterBank for sm_90a.
//
// Spectrogram: the reference GPU path (dali/kernels/signal/fft/stft_gpu_impl.cu:200-294) runs three kernels plus
// cuFFT with HBM round trips of the framed (2x oversampled) signal and of the complex spectrum.  Here one CTA
// frames F consecutive windows straight from the signal (reflect-101 / zero padding, window function, window
// centred in the nfft buffer: dali/kernels/signal/window/extract_windows_cpu.cc:97-146,
// fft_cpu_impl_ffts.cc:111), runs a radix-2 FFT in shared memory and writes |X|^2 or |X| -- the signal is read
// once and only the nfft/2+1 output bins are written.  Parity with the reference CPU backend (FFTS, fp32) is by
// tolerance: the oracle evaluates the DFT of each float32 windowed frame x_f in double precision; tests bound each frame's amplitude
// error by 8 ceil(log2 nfft) 2^-24 sqrt(nfft) ||x_f|| + 2^-22 |X| (what a float32 FFT of that frame alone achieves), so an all-zero
// frame must come out exactly 0.
//
// MelFilterBank: parity target MelFilterBankCpu::ComputeFreqMajor (dali/kernels/audio/mel_scale/
// mel_filter_bank_cpu.cc:77-111) with the filter tables of MelFilterImplBase (mel_scale.h:76-131): every output
// accumulates its (at most two triangles') bins in ascending bin order with unfused mul/add, which makes this
// kernel BIT-EXACT against the CPU backend.  (A dense tensor-core GEMM formulation reorders the sums; see
// DESIGN.md for why the exact banded kernel is the default.)
//
// Algorithmic bytes per unit (SURVEY.md 8d): STFT len*4 + nbin*nwin*4 ; mel nbin*nwin*4 + nfilter*nwin*4.
#include "common.cuh"
#include <algorithm>
#include <cmath>
#include <cstring>

namespace dalib200 {

struct SpecDesc {
  const float *in;
  float *out;
  int64_t len;
  int64_t nwin;
  int64_t first_group;     // first CTA work item (group of F frames)
  float preemph;           // pre-emphasis coefficient (kernels instantiated with PRE)
};

struct SpecParams {
  int nfft, log2n, win_len, step, power, center_off, padding /*0 none,1 zero,2 reflect*/, layout_ft, frames_per_cta, nbin;
  int in_win_start;
  int pre_border;          // DALIB200_BORDER_* of the fused pre-emphasis
};

__device__ __forceinline__ int64_t reflect101(int64_t i, int64_t n) {
  if (n < 2) return n - 1;
  for (;;) {
    if (i < 0) i = -i;
    else if (i >= n) i = 2 * n - 2 - i;
    else break;
  }
  return i;
}

// Two real frames per complex FFT (frame 2p = real part, 2p + 1 = imaginary part; the spectra are separated afterwards from
// Z[k] and Z[N - k]), radix-2 DIT stages fused in pairs (a thread carries 4 points through 2 stages: half the barriers and half
// the shared-memory traffic), twiddles in shared memory.  Element i of a buffer lives at i + (i >> 5): the bit-reversed
// scatter of the framing step (stride N/32 elements between lanes) would otherwise hit one bank 32 times.
// smem: [F/2 pairs][N + N/32] float2 | twiddle[N/2] = exp(-2 pi i k / N), computed in double on the host.
__device__ __forceinline__ int pad32(int i) { return i + (i >> 5); }

// PRE: the signal is the pre-emphasised input y (preemph_at), so the padding applies to y -- reflect reads y at the reflected index
template <bool PRE>
__device__ __forceinline__ float spec_sample(const SpecDesc &d, const SpecParams &P, const float *__restrict__ window, int64_t frame, int t) {
  int64_t si = frame * (int64_t)P.step - P.center_off + t;
  if (si < 0 || si >= d.len) {
    if (P.padding != 2) return 0.0f;
    si = reflect101(si, d.len);
  }
  return mul_rn(window[t], PRE ? preemph_at(d.in, si, d.len, d.preemph, P.pre_border) : __ldg(d.in + si));
}

// Per-frame scaling of the paired FFTs.  A float32 FFT's rounding error scales with the norm of its whole complex input, so without
// it the separated spectrum of a quiet frame carries error proportional to its loud partner's energy (and an all-zero frame comes out
// non-zero).  Each frame is multiplied by an exact power of two that brings its largest |windowed sample| to [1, 2) before packing,
// and the scale is undone on |X| or |X|^2 after separation.  `amax` = bits of that largest |sample| (0: the frame is all zero).
__device__ __forceinline__ int spec_shift(unsigned amax) {           // clamped so that 2^shift stays a normal float
  return min(126, max(-126, 127 - (int)(amax >> 23)));
}
__device__ __forceinline__ float spec_scale(unsigned amax) { return __int_as_float((127 + spec_shift(amax)) << 23); }
// |X| (power 1) or |X|^2 (power 2) of the scaled frame -> that of the frame itself; an all-zero frame gives exactly 0.  Products with
// powers of two are exact unless the result is subnormal, so a power comes out within one subnormal step (2^-149) of rounding once.
__device__ __forceinline__ float spec_unscale(float v, unsigned amax, int power) {
  if (amax == 0) return 0.0f;
  const float inv = __int_as_float((127 - spec_shift(amax)) << 23);
  v *= inv;
  return power == 2 ? v * inv : v;
}

__device__ __forceinline__ float2 cmul(float2 c, float2 w) {          // c * (w.x - i w.y), w = (cos, sin)
  return make_float2(c.x * w.x + c.y * w.y, c.y * w.x - c.x * w.y);
}

template <bool PRE>
__global__ void __launch_bounds__(256) spectrogram_kernel(const SpecDesc *__restrict__ descs, int n, int64_t total_groups,
                                                          SpecParams P, const float *__restrict__ window,
                                                          const float2 *__restrict__ twiddle) {
  extern __shared__ float2 buf[];
  __shared__ unsigned amax[16];                              // per frame of the group (F <= 16): see spec_shift
  const int N = P.nfft, F = P.frames_per_cta, L = P.log2n, NPAD = N + (N >> 5);
  float2 *tw = buf + (size_t)(F >> 1) * NPAD;
  for (int i = threadIdx.x; i < (N >> 1); i += blockDim.x) tw[i] = twiddle[i];
  __syncthreads();
  for (int64_t grp = blockIdx.x; grp < total_groups; grp += gridDim.x) {
    const int s = last_at_most(descs, 0, n - 1, grp, [](const SpecDesc &d) { return d.first_group; });
    const SpecDesc &d = descs[s];
    const int64_t w0 = (grp - d.first_group) * F;
    const int nf = (int)min((int64_t)F, d.nwin - w0);
    const int np = (nf + 1) >> 1;
    if (threadIdx.x < F) amax[threadIdx.x] = 0;
    __syncthreads();
    // ---- framing: sample t of a frame lands at the bit-reversed index of (in_win_start + t); everything else is zero
    for (int e = threadIdx.x; e < np * N; e += blockDim.x) {
      const int p = e / N, i = e - p * N;
      const int t = i - P.in_win_start;
      float va = 0.0f, vb = 0.0f;
      if (t >= 0 && t < P.win_len) {
        va = spec_sample<PRE>(d, P, window, w0 + 2 * p, t);
        if (2 * p + 1 < nf) vb = spec_sample<PRE>(d, P, window, w0 + 2 * p + 1, t);
      }
      const int r = (int)(__brev((unsigned)i) >> (32 - L));
      buf[p * NPAD + pad32(r)] = make_float2(va, vb);
      unsigned ua = __float_as_uint(va) & 0x7fffffffu, ub = __float_as_uint(vb) & 0x7fffffffu;
      if (N >= 32) {                  // whole warps, each inside one pair's row (N and blockDim are multiples of 32)
        ua = __reduce_max_sync(0xffffffffu, ua); ub = __reduce_max_sync(0xffffffffu, ub);
        if ((threadIdx.x & 31) == 0) { atomicMax(&amax[2 * p], ua); atomicMax(&amax[2 * p + 1], ub); }
      } else {
        atomicMax(&amax[2 * p], ua); atomicMax(&amax[2 * p + 1], ub);
      }
    }
    __syncthreads();
    for (int e = threadIdx.x; e < np * N; e += blockDim.x) {
      const int p = e / N;
      float2 &v = buf[p * NPAD + pad32(e - p * N)];
      v.x *= spec_scale(amax[2 * p]); v.y *= spec_scale(amax[2 * p + 1]);
    }
    __syncthreads();
    // ---- in-place radix-2 DIT, two stages per pass
    int st = 0;
    for (; st + 1 < L; st += 2) {
      const int half = 1 << st;
      for (int e = threadIdx.x; e < np * (N >> 2); e += blockDim.x) {
        const int p = e / (N >> 2), q = e - p * (N >> 2);
        const int k = q & (half - 1);
        const int base = ((q >> st) << (st + 2)) + k;
        float2 *fb = buf + p * NPAD;
        const int i0 = pad32(base), i1 = pad32(base + half), i2 = pad32(base + 2 * half), i3 = pad32(base + 3 * half);
        const float2 e0 = fb[i0], e1 = fb[i1], e2 = fb[i2], e3 = fb[i3];
        const float2 w1 = tw[k << (L - 1 - st)];
        const float2 t1 = cmul(e1, w1), t3 = cmul(e3, w1);
        const float2 a0 = make_float2(e0.x + t1.x, e0.y + t1.y), a1 = make_float2(e0.x - t1.x, e0.y - t1.y);
        const float2 a2 = make_float2(e2.x + t3.x, e2.y + t3.y), a3 = make_float2(e2.x - t3.x, e2.y - t3.y);
        const float2 wa = tw[k << (L - 2 - st)], wb = tw[(k + half) << (L - 2 - st)];
        const float2 ta = cmul(a2, wa), tb = cmul(a3, wb);
        fb[i0] = make_float2(a0.x + ta.x, a0.y + ta.y);
        fb[i2] = make_float2(a0.x - ta.x, a0.y - ta.y);
        fb[i1] = make_float2(a1.x + tb.x, a1.y + tb.y);
        fb[i3] = make_float2(a1.x - tb.x, a1.y - tb.y);
      }
      __syncthreads();
    }
    if (st < L) {                                            // odd log2(nfft): one plain radix-2 stage is left
      const int half = 1 << st;
      for (int e = threadIdx.x; e < np * (N >> 1); e += blockDim.x) {
        const int p = e / (N >> 1), b = e - p * (N >> 1);
        const int k = b & (half - 1);
        const int j0 = ((b >> st) << (st + 1)) + k;
        float2 *fb = buf + p * NPAD;
        const int i0 = pad32(j0), i1 = pad32(j0 + half);
        const float2 a = fb[i0], t = cmul(fb[i1], tw[k << (L - 1 - st)]);
        fb[i0] = make_float2(a.x + t.x, a.y + t.y);
        fb[i1] = make_float2(a.x - t.x, a.y - t.y);
      }
      __syncthreads();
    }
    // ---- separate the two frames of a pair, magnitude / power, store
    for (int e = threadIdx.x; e < nf * P.nbin; e += blockDim.x) {
      int f, k;
      if (P.layout_ft) { k = e / nf; f = e - k * nf; } else { f = e / P.nbin; k = e - f * P.nbin; }
      const float2 *fb = buf + (f >> 1) * NPAD;
      const float2 zk = fb[pad32(k)], zn = fb[pad32((N - k) & (N - 1))];
      const float2 x = (f & 1) ? make_float2(0.5f * (zk.y + zn.y), 0.5f * (zn.x - zk.x))
                               : make_float2(0.5f * (zk.x + zn.x), 0.5f * (zk.y - zn.y));
      const float pw = x.x * x.x + x.y * x.y;
      const float v = spec_unscale(P.power == 2 ? pw : sqrtf(pw), amax[f], P.power);
      if (P.layout_ft) d.out[(int64_t)k * d.nwin + w0 + f] = v;
      else d.out[(w0 + f) * (int64_t)P.nbin + k] = v;
    }
    __syncthreads();
  }
}

// ---------------------------------------------------------------------------------------------
// nfft NOT a power of two (the reference hands those to FFTS' complex transform, fft_cpu_impl_ffts.cc:38-86): a direct DFT from shared
// memory -- O(nfft^2 / 2) per frame, meant for the occasional odd nfft (400, 600, 1000 ...), not for the hot configurations.  One thread
// = one (frame, bin); the twiddle e^(-2 pi i k t / n) is read from a full-period table with an incrementally wrapped index (no
// trigonometry in the loop), sums are accumulated in double so that the result stays inside the stated STFT tolerance for any nfft.
template <bool PRE>
__global__ void __launch_bounds__(256) spectrogram_dft_kernel(const SpecDesc *__restrict__ descs, int n, int64_t total_groups, SpecParams P,
                                                              const float *__restrict__ window, const float2 *__restrict__ twiddle_full) {
  extern __shared__ float2 dbuf[];
  const int N = P.nfft, F = P.frames_per_cta;
  float2 *tw = dbuf;                                   // [N] (cos, sin)(2 pi j / N)
  float *fr = reinterpret_cast<float *>(dbuf + N);     // [F][N]
  for (int i = threadIdx.x; i < N; i += blockDim.x) tw[i] = twiddle_full[i];
  for (int64_t grp = blockIdx.x; grp < total_groups; grp += gridDim.x) {
    const int s = last_at_most(descs, 0, n - 1, grp, [](const SpecDesc &d) { return d.first_group; });
    const SpecDesc &d = descs[s];
    const int64_t w0 = (grp - d.first_group) * F;
    const int nf = (int)min((int64_t)F, d.nwin - w0);
    __syncthreads();
    for (int e = threadIdx.x; e < nf * N; e += blockDim.x) {
      const int f = e / N, i = e - f * N;
      const int t = i - P.in_win_start;
      fr[f * N + i] = (t >= 0 && t < P.win_len) ? spec_sample<PRE>(d, P, window, w0 + f, t) : 0.0f;
    }
    __syncthreads();
    for (int e = threadIdx.x; e < nf * P.nbin; e += blockDim.x) {
      int f, k;
      if (P.layout_ft) { k = e / nf; f = e - k * nf; } else { f = e / P.nbin; k = e - f * P.nbin; }
      const float *x = fr + f * N;
      double re = 0.0, im = 0.0;
      int idx = 0;
      for (int t = 0; t < N; t++) {
        const float2 w = tw[idx];
        const double xv = (double)x[t];
        re += xv * (double)w.x; im -= xv * (double)w.y;
        idx += k; if (idx >= N) idx -= N;
      }
      const double pw = re * re + im * im;             // in double: a float |X|^2 underflows for quiet frames
      const float v = (float)(P.power == 2 ? pw : sqrt(pw));
      if (P.layout_ft) d.out[(int64_t)k * d.nwin + w0 + f] = v;
      else d.out[(w0 + f) * (int64_t)P.nbin + k] = v;
    }
  }
}

// ---------------------------------------------------------------------------------------------
struct MelDesc {
  const float *in;
  float *out;
  int64_t nwin;
  int64_t first_item;      // first (filter, 128-column chunk) work item
};

// ---------------------------------------------------------------------------------------------
// nfft = 1024: the FFT lives in REGISTERS.  One warp transforms one pair of frames (frame 2p = real part, 2p + 1 = imaginary part)
// as 1024 = 32 x 32 (Cooley-Tukey, n = 32 n1 + n2, k = k1 + 32 k2):
//   step 1  lane = n2 holds x[32 n1 + n2], n1 = 0..31 (every load is one coalesced 128-byte row of the frame) and runs a
//           32-point DFT over n1 in registers (5 fully unrolled radix-2 DIF stages, constant twiddles);
//   step 2  multiplies Y[k1] by W_1024^(n2 k1) (32 x 32 table in shared memory, row k1 read conflict-free);
//   step 3  transposes through a warp-private 32 x 33 tile (the only shared-memory round trip, __syncwarp only) so that lane = k1
//           holds Y[k1][n2], and runs the second 32-point DFT over n2: X[k1 + 32 k2].
// The two real spectra are separated with one shuffle per bin (the partner bin N - k sits in lane 32 - k1, register 31 - k2).
// Against the shared-memory radix-2 kernel above: 1 shared round trip instead of 5, no block-wide barrier, ~64 independent values
// per thread in flight.  With `mel` the power spectrum of the pair never leaves the SM: it is parked in the (now free) tile and
// the mel filters are applied there, in the summation order of mel_kernel below -- STFT -> mel in ONE kernel, 128 x T written once.
__device__ __forceinline__ float w32c(int j) {      // cos(2 pi j / 32)
  switch (j) {
    case 0: return 1.0f; case 1: return 0.98078528040323043f; case 2: return 0.92387953251128674f; case 3: return 0.83146961230254524f;
    case 4: return 0.70710678118654757f; case 5: return 0.55557023301960229f; case 6: return 0.38268343236508984f;
    case 7: return 0.19509032201612833f; case 8: return 0.0f; case 9: return -0.19509032201612819f; case 10: return -0.38268343236508973f;
    case 11: return -0.55557023301960196f; case 12: return -0.70710678118654746f; case 13: return -0.83146961230254535f;
    case 14: return -0.92387953251128674f; default: return -0.98078528040323043f;
  }
}

template <int HALF>
__device__ __forceinline__ void fft32_stage(float (&re)[32], float (&im)[32]) {
#pragma unroll
  for (int i = 0; i < 32; i += 2 * HALF) {
#pragma unroll
    for (int j = 0; j < HALF; j++) {
      const int a = i + j, b = a + HALF;
      const float ar = re[a], ai = im[a], br = re[b], bi = im[b];
      re[a] = ar + br; im[a] = ai + bi;
      float tr = ar - br, ti = ai - bi;
      const int tw = j * (16 / HALF);                  // times W_32^tw = exp(-2 pi i tw / 32)
      if (tw == 8) { const float t = tr; tr = ti; ti = -t; }
      else if (tw != 0) {
        const float c = w32c(tw), sn = w32c(tw <= 8 ? 8 - tw : tw - 8);      // sin(2 pi tw / 32) = cos(2 pi (8 - tw) / 32)
        const float r2 = tr * c + ti * sn, i2 = ti * c - tr * sn;
        tr = r2; ti = i2;
      }
      re[b] = tr; im[b] = ti;
    }
  }
}
// natural order in, bit-reversed order out: X[k] = v[brev5(k)]
__device__ __forceinline__ void fft32(float (&re)[32], float (&im)[32]) {
  fft32_stage<16>(re, im); fft32_stage<8>(re, im); fft32_stage<4>(re, im); fft32_stage<2>(re, im); fft32_stage<1>(re, im);
}
__device__ __forceinline__ constexpr int brev5(int k) { return ((k & 1) << 4) | ((k & 2) << 2) | (k & 4) | ((k & 8) >> 2) | ((k & 16) >> 4); }

constexpr int kF1024Warps = 8;                       // 16 frames per CTA, like the radix-2 kernel's grouping at nfft = 1024
constexpr int kF1024Tile = 32 * 33;                  // float2 per warp
constexpr size_t kF1024Smem = sizeof(float2) * (1024 + (size_t)kF1024Warps * kF1024Tile);

struct MelTables { const int32_t *ends; const float *w_up, *w_down; int nfilter; };

template <bool MEL, bool PRE>
__global__ void __launch_bounds__(kF1024Warps * 32, 2) spectrogram1024_kernel(const SpecDesc *__restrict__ descs, int n, int64_t total_groups,
                                                                              SpecParams P, const float *__restrict__ window,
                                                                              const float2 *__restrict__ twiddle1024, MelTables mt,
                                                                              const MelDesc *__restrict__ mdescs, int write_spec) {
  extern __shared__ float2 fbuf[];
  float2 *tw = fbuf;                                 // [k1][n2] = W_1024^(k1 n2)
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float2 *tile = fbuf + 1024 + warp * kF1024Tile;
  for (int e = threadIdx.x; e < 1024; e += blockDim.x) {
    const int idx = (e >> 5) * (e & 31);             // < 1024; W^(idx) from the half table: W^(idx) = -W^(idx - 512)
    const float2 t = twiddle1024[idx & 511];
    tw[e] = idx < 512 ? t : make_float2(-t.x, -t.y);
  }
  __syncthreads();
  for (int64_t grp = blockIdx.x; grp < total_groups; grp += gridDim.x) {
    const int s = last_at_most(descs, 0, n - 1, grp, [](const SpecDesc &d) { return d.first_group; });
    const SpecDesc &d = descs[s];
    const int64_t w0 = (grp - d.first_group) * (2 * kF1024Warps) + 2 * warp;
    if (w0 >= d.nwin) continue;
    const bool two = w0 + 1 < d.nwin;
    float re[32], im[32];
    // ---- framing (window applied here); interior pairs skip the per-sample bounds logic
    {
      const int64_t start = w0 * (int64_t)P.step - P.center_off - P.in_win_start;      // signal index of FFT sample 0 of frame w0
      // with PRE, sample 0 of the pair also reads its predecessor: start >= 1 keeps the interior path off the border rule
      const bool interior = two && P.in_win_start == 0 && P.win_len == 1024 && start >= (PRE ? 1 : 0) && start + P.step + 1024 <= d.len;
      if (interior) {
        const float *pa = d.in + start + lane, *pb = pa + P.step;
#pragma unroll
        for (int n1 = 0; n1 < 32; n1++) {
          const float wv = __ldg(window + 32 * n1 + lane);
          if (PRE) {
            const float c = d.preemph;
            const float xa = __ldg(pa + 32 * n1), xb = __ldg(pb + 32 * n1);
            re[n1] = mul_rn(wv, c == 0.0f ? xa : sub_rn(xa, mul_rn(c, __ldg(pa + 32 * n1 - 1))));
            im[n1] = mul_rn(wv, c == 0.0f ? xb : sub_rn(xb, mul_rn(c, __ldg(pb + 32 * n1 - 1))));
          } else {
            re[n1] = mul_rn(wv, __ldg(pa + 32 * n1));
            im[n1] = mul_rn(wv, __ldg(pb + 32 * n1));
          }
        }
      } else {
#pragma unroll
        for (int n1 = 0; n1 < 32; n1++) {
          const int t = 32 * n1 + lane - P.in_win_start;
          float va = 0.0f, vb = 0.0f;
          if (t >= 0 && t < P.win_len) {
            va = spec_sample<PRE>(d, P, window, w0, t);
            if (two) vb = spec_sample<PRE>(d, P, window, w0 + 1, t);
          }
          re[n1] = va; im[n1] = vb;
        }
      }
    }
    // ---- per-frame scale (spec_shift) from the largest |windowed sample| of each frame of the pair
    unsigned amax_a = 0, amax_b = 0;
#pragma unroll
    for (int n1 = 0; n1 < 32; n1++) {
      amax_a = max(amax_a, __float_as_uint(re[n1]) & 0x7fffffffu);
      amax_b = max(amax_b, __float_as_uint(im[n1]) & 0x7fffffffu);
    }
    amax_a = __reduce_max_sync(0xffffffffu, amax_a);
    amax_b = __reduce_max_sync(0xffffffffu, amax_b);
    {
      const float sa = spec_scale(amax_a), sb = spec_scale(amax_b);
#pragma unroll
      for (int n1 = 0; n1 < 32; n1++) { re[n1] *= sa; im[n1] *= sb; }
    }
    fft32(re, im);                                   // Y[k1] (for this lane's n2) = v[brev5(k1)]
    __syncwarp();                                    // the tile may still be read as the previous pair's power spectrum
#pragma unroll
    for (int k1 = 0; k1 < 32; k1++) {
      const float2 w = tw[k1 * 32 + lane];
      const float yr = re[brev5(k1)], yi = im[brev5(k1)];
      tile[k1 * 33 + lane] = make_float2(yr * w.x + yi * w.y, yi * w.x - yr * w.y);     // * (cos - i sin)
    }
    __syncwarp();
#pragma unroll
    for (int n2 = 0; n2 < 32; n2++) {
      const float2 v = tile[lane * 33 + n2];
      re[n2] = v.x; im[n2] = v.y;
    }
    fft32(re, im);                                   // Z[lane + 32 k2] = v[brev5(k2)]
    __syncwarp();
    // ---- separate the two real spectra, power / magnitude.  Bins k = lane + 32 k2, k2 = 0..15, and k = 512 (lane 0, k2 = 16).
    float *pw = reinterpret_cast<float *>(tile);     // [2][520] floats: the pair's spectra, parked for the mel filters
    const int src = (32 - lane) & 31;
#pragma unroll
    for (int k2 = 0; k2 <= 16; k2++) {
      // partner bin N - k: lane (32 - k1) % 32, k2' = 31 - k2 -- for k1 = 0 it stays in lane 0 with k2' = (32 - k2) % 32
      const float zr = re[brev5(k2)], zi = im[brev5(k2)];
      float pr = __shfl_sync(0xffffffffu, re[brev5(31 - k2)], src);
      float pi = __shfl_sync(0xffffffffu, im[brev5(31 - k2)], src);
      if (lane == 0) { pr = re[brev5((32 - k2) & 31)]; pi = im[brev5((32 - k2) & 31)]; }
      if (k2 == 16 && lane != 0) continue;
      const float ax = 0.5f * (zr + pr), ay = 0.5f * (zi - pi);       // frame 2p
      const float bx = 0.5f * (zi + pi), by = 0.5f * (pr - zr);       // frame 2p + 1
      float va = ax * ax + ay * ay, vb = bx * bx + by * by;
      if (P.power != 2) { va = sqrtf(va); vb = sqrtf(vb); }
      va = spec_unscale(va, amax_a, P.power);
      vb = spec_unscale(vb, amax_b, P.power);
      const int k = lane + 32 * k2;
      if (write_spec) {
        if (P.layout_ft) {
          float *o = d.out + (int64_t)k * d.nwin + w0;
          o[0] = va;
          if (two) o[1] = vb;
        } else {
          d.out[w0 * (int64_t)P.nbin + k] = va;
          if (two) d.out[(w0 + 1) * (int64_t)P.nbin + k] = vb;
        }
      }
      if (MEL) { pw[k] = va; pw[520 + k] = vb; }
    }
    if (MEL) {
      __syncwarp();
      float *mo = mdescs[s].out;
      for (int m = lane; m < mt.nfilter; m += 32) {
        const int b0 = mt.ends[m], b1 = mt.ends[m + 1], b2 = mt.ends[m + 2];
        float acca = 0.0f, accb = 0.0f;
        for (int b = b0; b < b1; b++) { const float w = __ldg(mt.w_up + b); acca = add_rn(acca, mul_rn(w, pw[b])); accb = add_rn(accb, mul_rn(w, pw[520 + b])); }
        for (int b = b1; b < b2; b++) { const float w = __ldg(mt.w_down + b); acca = add_rn(acca, mul_rn(w, pw[b])); accb = add_rn(accb, mul_rn(w, pw[520 + b])); }
        mo[(int64_t)m * d.nwin + w0] = acca;
        if (two) mo[(int64_t)m * d.nwin + w0 + 1] = accb;
      }
    }
  }
}

// tables: ends[nfilter+2] (int, interval boundaries in bins), w_up[nbin], w_down[nbin] (already normalised)
__global__ void __launch_bounds__(128) mel_kernel(const MelDesc *__restrict__ descs, int n, int64_t total_items, int nfilter,
                                                  const int32_t *__restrict__ ends, const float *__restrict__ w_up,
                                                  const float *__restrict__ w_down) {
  for (int64_t item = blockIdx.x; item < total_items; item += gridDim.x) {
    const int s = last_at_most(descs, 0, n - 1, item, [](const MelDesc &d) { return d.first_item; });
    const MelDesc &d = descs[s];
    const int64_t li = item - d.first_item;
    const int64_t chunks = (d.nwin + 127) / 128;
    const int m = (int)(li / chunks);
    const int64_t t = (li % chunks) * 128 + threadIdx.x;
    if (t >= d.nwin) continue;
    const int b0 = ends[m], b1 = ends[m + 1], b2 = ends[m + 2];
    float acc = 0.0f;
    for (int b = b0; b < b1; b++) acc = add_rn(acc, mul_rn(w_up[b], __ldg(d.in + (int64_t)b * d.nwin + t)));
    for (int b = b1; b < b2; b++) acc = add_rn(acc, mul_rn(w_down[b], __ldg(d.in + (int64_t)b * d.nwin + t)));
    d.out[(int64_t)m * d.nwin + t] = acc;
  }
}

// ---------------------------------------------------------------------------------------------
// Optional tensor-core path of MelFilterBank (dalib200MelPlanSetTensorCores): the banded sums as ONE dense GEMM
//   out[nfilter x nwin] = W[nfilter x nbin] * S[nbin x nwin]            per sample
// on the tensor cores (mma.sync m16n8k8, TF32 inputs, FP32 accumulate).  FP32 accuracy is kept with the 3-term split
// a = a_hi + a_lo (both TF32): a*b ~= a_hi*b_hi + a_lo*b_hi + a_hi*b_lo, error ~2^-21 relative.  The summation ORDER differs
// from the reference CPU kernel, so this path is a tolerance path (tests: 8e-6 of the row maximum); the default banded kernel
// above stays bit exact.  A CTA = 128 filters x 64 windows, K streamed in chunks of 32 bins through shared memory (row pitches
// 36 / 72 floats: the m16n8k8 fragment loads are bank-conflict free); chunks outside the filters' bands are skipped.
constexpr int kMmM = 128, kMmN = 64, kMmK = 32, kMmWP = kMmK + 4, kMmSP = kMmN + 8;

__device__ __forceinline__ uint32_t to_tf32(float x) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return r;
}
__device__ __forceinline__ void mma_tf32(float (&d)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
  asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}

// dense: [mpad][kpad] row-major, zero padded; kr: per 128-row block {first chunk, end chunk}
__global__ void __launch_bounds__(256) mel_mma_kernel(const MelDesc *__restrict__ descs, int n, int64_t total_items, int nfilter, int nbin,
                                                      int kpad, const float *__restrict__ dense, const int2 *__restrict__ kr) {
  __shared__ __align__(16) float s_w[kMmM * kMmWP];
  __shared__ __align__(16) float s_s[kMmK * kMmSP];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, gid = lane >> 2, tig = lane & 3;
  const int mblocks = (nfilter + kMmM - 1) / kMmM;
  for (int64_t item = blockIdx.x; item < total_items; item += gridDim.x) {
    const int s = last_at_most(descs, 0, n - 1, item, [](const MelDesc &d) { return d.first_item; });
    const MelDesc &d = descs[s];
    const int64_t li = item - d.first_item;
    const int mb = (int)(li % mblocks);
    const int64_t t0 = (li / mblocks) * kMmN;
    float acc[kMmN / 8][4];
#pragma unroll
    for (int j = 0; j < kMmN / 8; j++) acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0.0f;
    const int2 range = kr[mb];
    for (int kc = range.x; kc < range.y; kc++) {
      const int k0 = kc * kMmK;
      // W chunk: 128 x 32 (float4, coalesced per row)
      for (int e = threadIdx.x; e < kMmM * kMmK / 4; e += blockDim.x) {
        const int r = e / (kMmK / 4), c4 = e % (kMmK / 4);
        const float4 v = __ldg(reinterpret_cast<const float4 *>(dense + (size_t)(mb * kMmM + r) * kpad + k0) + c4);
        *reinterpret_cast<float4 *>(s_w + r * kMmWP + 4 * c4) = v;
      }
      // S chunk: 32 bins x 64 windows (zero outside the spectrogram)
      for (int e = threadIdx.x; e < kMmK * kMmN; e += blockDim.x) {
        const int r = e / kMmN, c = e % kMmN;
        const int64_t t = t0 + c;
        s_s[r * kMmSP + c] = (k0 + r < nbin && t < d.nwin) ? __ldg(d.in + (int64_t)(k0 + r) * d.nwin + t) : 0.0f;
      }
      __syncthreads();
#pragma unroll
      for (int ks = 0; ks < kMmK / 8; ks++) {
        const float *wr = s_w + (warp * 16 + gid) * kMmWP + ks * 8 + tig;
        const float af[4] = { wr[0], wr[8 * kMmWP], wr[4], wr[8 * kMmWP + 4] };
        uint32_t ah[4], al[4];
#pragma unroll
        for (int q = 0; q < 4; q++) { ah[q] = to_tf32(af[q]); al[q] = to_tf32(af[q] - __uint_as_float(ah[q])); }
#pragma unroll
        for (int j = 0; j < kMmN / 8; j++) {
          const float *sr = s_s + (ks * 8 + tig) * kMmSP + j * 8 + gid;
          const float bf[2] = { sr[0], sr[4 * kMmSP] };
          uint32_t bh[2], bl[2];
#pragma unroll
          for (int q = 0; q < 2; q++) { bh[q] = to_tf32(bf[q]); bl[q] = to_tf32(bf[q] - __uint_as_float(bh[q])); }
          mma_tf32(acc[j], al, bh);
          mma_tf32(acc[j], ah, bl);
          mma_tf32(acc[j], ah, bh);
        }
      }
      __syncthreads();
    }
    const int m0 = mb * kMmM + warp * 16 + gid;
#pragma unroll
    for (int j = 0; j < kMmN / 8; j++) {
      const int64_t t = t0 + j * 8 + 2 * tig;
#pragma unroll
      for (int h = 0; h < 2; h++) {
        const int m = m0 + 8 * h;
        if (m < nfilter) {
          if (t < d.nwin) d.out[(int64_t)m * d.nwin + t] = acc[j][2 * h];
          if (t + 1 < d.nwin) d.out[(int64_t)m * d.nwin + t + 1] = acc[j][2 * h + 1];
        }
      }
    }
  }
}

}  // namespace dalib200

using namespace dalib200;  // NOLINT

struct dalib200SpectrogramPlan {
  int max_batch = 0, n = 0;
  SpecParams P{};
  std::vector<SpecDesc> descs;
  int64_t total_groups = 0;
  DescArena arena;           // descriptors
  float *d_window = nullptr; float2 *d_twiddle = nullptr;
  int tw_nfft = 0;
  size_t win_cap = 0;
  std::vector<float> window;
  bool window_dirty = true;
  size_t smem = 0;
  bool smem_set = false;
  std::vector<float> preemph;    // per-sample coefficients of the fused pre-emphasis; empty = off
};

struct dalib200MelPlan {
  int max_batch = 0, n = 0, nfilter = 0, nbin = 0;
  std::vector<MelDesc> descs;
  int64_t total_items = 0;
  DescArena arena;
  DescArena tables;          // ends | w_up | w_down
  std::vector<int32_t> h_ends; std::vector<float> h_up, h_down;
  bool tables_dirty = true;
  bool tensor_cores = false;     // dense TF32x3 GEMM on the tensor cores instead of the bit-exact banded sums
  DescArena dense;               // [mpad][kpad] weights | int2 chunk range per 128-filter block
  bool dense_dirty = true;
  int kpad = 0, mpad = 0;
  int64_t total_items_mma = 0;
  std::vector<int64_t> first_item_mma;
  dalib200MelArgs args{};
};

namespace {

// mel_scale.h:28-74 (T = float)
struct Slaney {
  static float hz_to_mel(float hz) {
    const float fsp = 200.0 / 3.0, min_log_hz = 1000.0, min_log_mel = (min_log_hz - 0) / fsp, step_log = 0.068751777;
    return hz >= min_log_hz ? min_log_mel + std::log(hz / min_log_hz) / step_log : (hz - 0) / fsp;
  }
  static float mel_to_hz(float mel) {
    const float fsp = 200.0 / 3.0, min_log_hz = 1000.0, min_log_mel = (min_log_hz - 0) / fsp, step_log = 0.068751777;
    return mel >= min_log_mel ? min_log_hz * std::exp(step_log * (mel - min_log_mel)) : 0 + mel * fsp;
  }
};
struct Htk {
  static float hz_to_mel(float hz) { return 1127.0f * std::log(1.0f + hz / 700.0f); }
  static float mel_to_hz(float mel) { return 700.0f * (std::exp(mel / 1127.0f) - 1.0f); }
};

// mel_scale.h:76-131 + mel_filter_bank_cpu.cc:40-69, producing per-bin weights already multiplied by the
// normalisation factor of the filter they feed (as ComputeFreqMajor does on the fly, :88-104).
template <typename Scale>
void BuildMel(const dalib200MelArgs &a, int nfft, std::vector<int32_t> &ends, std::vector<float> &up, std::vector<float> &down) {
  const int nfilter = a.nfilter;
  const double mel_low = Scale::hz_to_mel(a.freq_low), mel_high = Scale::hz_to_mel(a.freq_high);
  const double hz_step = static_cast<double>(a.sample_rate) / nfft;
  const double mel_delta = (mel_high - mel_low) / (nfilter + 1);
  const int nbin = nfft / 2 + 1;
  const double inv_hz_step = 1.0 / hz_step;
  const int bin_start = (int)std::ceil(a.freq_low * inv_hz_step);
  int bin_end = (int)std::ceil(a.freq_high * inv_hz_step);
  if (bin_end > nbin) bin_end = nbin;
  std::vector<float> wd(nbin, 0.0f), norm(nfilter, 1.0f);
  double mel0 = mel_low, mel1 = mel_low + mel_delta;
  int bin = bin_start;
  double f = bin * hz_step;
  for (int interval = 0; interval <= nfilter; interval++, mel0 = mel1, mel1 += mel_delta) {
    if (interval == nfilter) mel1 = mel_high;
    double f0 = Scale::mel_to_hz((float)mel0), f1 = Scale::mel_to_hz((float)mel1);
    if (a.normalize && interval < nfilter) {
      double f2 = Scale::mel_to_hz((float)(mel1 + mel_delta));
      norm[interval] = (float)(2.0 / (f2 - f0));
    }
    double slope = 1. / (f1 - f0);
    for (; bin < bin_end && f < f1; bin++, f = bin * hz_step) wd[bin] = (float)((f1 - f) * slope);
  }
  std::vector<int> intervals(nbin, -1);
  bin = bin_start; f = bin * hz_step;
  double mel = mel_low + mel_delta;
  for (int interval = 0; interval < nfilter + 1; interval++, mel += mel_delta) {
    double freq = Scale::mel_to_hz((float)(interval == nfilter ? mel_high : mel));
    for (; bin < bin_end && f < freq; bin++, f = bin * hz_step) intervals[bin] = interval;
  }
  // interval boundaries in bins, derived from the per-bin interval ids (so both loops agree exactly)
  ends.assign(nfilter + 2, bin_end);
  ends[0] = bin_start;
  for (int iv = 1; iv <= nfilter; iv++) {
    int b = bin_start;
    while (b < bin_end && intervals[b] < iv) b++;
    ends[iv] = b;
  }
  ends[nfilter + 1] = bin_end;
  up.assign(nbin, 0.0f); down.assign(nbin, 0.0f);
  for (int b = bin_start; b < bin_end; b++) {
    const int fu = intervals[b], fd = fu - 1;
    float wu = 1.0f - wd[b], wdn = wd[b];
    if (fd >= 0) { if (a.normalize) wdn *= norm[fd]; down[b] = wdn; }
    if (fu >= 0 && fu < nfilter) { if (a.normalize) wu *= norm[fu]; up[b] = wu; }
  }
}

}  // namespace

extern "C" {

void dalib200HannWindow(float *out, int n) {     // window_functions.h:26-33
  const double a = (2 * M_PI / n);
  for (int t = 0; t < n; t++) out[t] = static_cast<float>(0.5 * (1.0 - std::cos(a * (t + 0.5))));
}

int dalib200SpectrogramPlanCreate(dalib200SpectrogramPlan **plan, int max_batch) try {
  DB_CHECK_ARG(plan && max_batch > 0, "SpectrogramPlanCreate: bad arguments");
  auto *p = new dalib200SpectrogramPlan();
  p->max_batch = max_batch;
  int rc = p->arena.Reserve(sizeof(SpecDesc) * max_batch);
  if (rc) { delete p; return rc; }
  *plan = p;
  return DALIB200_SUCCESS;
} DB_API_CATCH

int dalib200SpectrogramPlanDestroy(dalib200SpectrogramPlan *p) try {
  if (!p) return DALIB200_SUCCESS;
  p->arena.Free();
  if (p->d_window) cudaFree(p->d_window);
  if (p->d_twiddle) cudaFree(p->d_twiddle);
  delete p;
  return DALIB200_SUCCESS;
} DB_API_CATCH

int dalib200SpectrogramPlanSetup(dalib200SpectrogramPlan *p, const dalib200SpectrogramArgs *a, const float *window_fn, int n,
                                 const int64_t *lengths) try {
  DB_CHECK_ARG(p && a && lengths && n >= 0 && n <= p->max_batch, "SpectrogramPlanSetup: bad arguments");
  DB_CHECK_ARG(a->window_length > 0, "Spectrogram: invalid window length %d", a->window_length);
  DB_CHECK_ARG(a->window_step > 0, "Spectrogram: invalid window step %d", a->window_step);
  DB_CHECK_ARG(a->power == 1 || a->power == 2, "Spectrogram: power must be 1 or 2, got %d", a->power);
  const int nfft = a->nfft > 0 ? a->nfft : a->window_length;
  DB_CHECK_ARG(nfft >= a->window_length, "Spectrogram: nfft (%d) must not be smaller than window_length (%d)", nfft, a->window_length);
  const bool pow2 = (nfft & (nfft - 1)) == 0;
  if (nfft < 2 || (pow2 && nfft > 8192) || (!pow2 && nfft > 4096)) {
    SetLastError("Spectrogram: nfft=%d -- the GPU path supports powers of two up to 8192 and other sizes up to 4096", nfft);
    return DALIB200_ERROR_UNSUPPORTED;
  }
  SpecParams &P = p->P;
  P.nfft = nfft; P.log2n = 0; while ((1 << P.log2n) < nfft) P.log2n++;
  P.win_len = a->window_length; P.step = a->window_step; P.power = a->power;
  P.padding = a->center ? (a->reflect ? 2 : 1) : 0;
  P.center_off = a->center ? a->window_length / 2 : 0;
  P.layout_ft = a->layout_ft != 0;
  P.nbin = nfft / 2 + 1;
  P.in_win_start = a->window_length < nfft ? (nfft - a->window_length) / 2 : 0;
  // two frames share one complex buffer: 16 frames (8 buffers of nfft + nfft/32 float2) per CTA at nfft = 1024 -> 3 CTAs / SM
  P.frames_per_cta = 2 * std::max(1, std::min(8, (64 * 1024) / (nfft * 8)));
  p->smem = (size_t)(P.frames_per_cta / 2) * (nfft + nfft / 32) * sizeof(float2) + (size_t)(nfft / 2) * sizeof(float2);
  if (!pow2) {                       // direct DFT: full twiddle period + F windowed frames in shared memory
    P.frames_per_cta = std::max(1, std::min(8, (int)((160 * 1024 - (size_t)nfft * 8) / ((size_t)nfft * 4))));
    p->smem = (size_t)nfft * sizeof(float2) + (size_t)P.frames_per_cta * nfft * sizeof(float);
  }
  std::vector<float> w(a->window_length);
  if (window_fn) memcpy(w.data(), window_fn, sizeof(float) * a->window_length);
  else dalib200HannWindow(w.data(), a->window_length);
  if (w != p->window) { p->window = w; p->window_dirty = true; }
  p->descs.assign(n, SpecDesc());
  int64_t groups = 0;
  for (int i = 0; i < n; i++) {
    DB_CHECK_ARG(lengths[i] > 0, "Spectrogram does not support empty (0-volume) samples (sample %d)", i);
    int64_t len = lengths[i];
    int64_t nwin = (P.padding ? len : len - P.win_len) / P.step + 1;     // extract_windows_args.h:41-45
    DB_CHECK_ARG(nwin > 0 && (P.padding || len >= P.win_len), "Spectrogram: signal is too short (%lld) for sample %d", (long long)len, i);
    if (P.padding == 2) DB_CHECK_ARG(len >= 2 || true, "unreachable");
    SpecDesc &d = p->descs[i];
    d.in = nullptr; d.out = nullptr; d.len = len; d.nwin = nwin; d.first_group = groups;
    groups += (nwin + P.frames_per_cta - 1) / P.frames_per_cta;
  }
  p->n = n; p->total_groups = groups;
  p->preemph.clear(); P.pre_border = 0;
  return DALIB200_SUCCESS;
} DB_API_CATCH

int dalib200SpectrogramPlanSetPreemphasis(dalib200SpectrogramPlan *p, const float *coeffs, int border) try {
  DB_CHECK_ARG(p, "SpectrogramPlanSetPreemphasis: null plan");
  DB_CHECK_ARG(border == DALIB200_BORDER_ZERO || border == DALIB200_BORDER_CLAMP || border == DALIB200_BORDER_REFLECT,
               "SpectrogramPlanSetPreemphasis: unknown border type %d", border);
  if (coeffs) p->preemph.assign(coeffs, coeffs + p->n); else p->preemph.clear();
  p->P.pre_border = border;
  return DALIB200_SUCCESS;
} DB_API_CATCH

int64_t dalib200SpectrogramNumWindows(const dalib200SpectrogramPlan *p, int sample) {
  if (!p || sample < 0 || sample >= p->n) return -1;
  return p->descs[sample].nwin;
}

static int MelUploadTables(dalib200MelPlan *p, dalib200Stream_t stream, size_t *o_up_out, size_t *o_down_out);

// mel != nullptr: STFT -> mel in one kernel (nfft = 1024 only); out_ptrs may then be null (the spectrogram is not written)
static int SpectrogramLaunchImpl(dalib200SpectrogramPlan *p, const void *const *in_ptrs, void *const *out_ptrs, dalib200MelPlan *mel,
                                 void *const *mel_out_ptrs, dalib200Stream_t stream) {
  if (p->n == 0 || p->total_groups == 0) return DALIB200_SUCCESS;
  const SpecParams &P = p->P;
  const bool pow2 = (P.nfft & (P.nfft - 1)) == 0;
  if (p->tw_nfft != P.nfft) {
    if (p->d_twiddle) cudaFree(p->d_twiddle);
    p->d_twiddle = nullptr;
    const int ntw = pow2 ? P.nfft / 2 : P.nfft;          // half period for the FFT kernels, the full one for the direct DFT
    DB_CUDA(cudaMalloc(reinterpret_cast<void **>(&p->d_twiddle), sizeof(float2) * ntw));
    std::vector<float2> tw(ntw);
    for (int k = 0; k < ntw; k++) {
      const double ang = 2.0 * M_PI * k / P.nfft;
      tw[k] = make_float2((float)std::cos(ang), (float)std::sin(ang));
    }
    DB_CUDA(cudaMemcpyAsync(p->d_twiddle, tw.data(), sizeof(float2) * tw.size(), cudaMemcpyHostToDevice, stream));
    DB_CUDA(cudaStreamSynchronize(stream));      // tw is a stack object; one-time cost per nfft
    p->tw_nfft = P.nfft;
  }
  if (p->window_dirty) {
    if (int rc = GrowDevice(p->d_window, p->win_cap, (size_t)P.win_len)) return rc;
    DB_CUDA(cudaMemcpyAsync(p->d_window, p->window.data(), sizeof(float) * P.win_len, cudaMemcpyHostToDevice, stream));
    DB_CUDA(cudaStreamSynchronize(stream));
    p->window_dirty = false;
  }
  const bool pre = !p->preemph.empty();
  SpecDesc *hd;
  int rc = p->arena.Stage(sizeof(SpecDesc) * p->n, &hd);
  if (rc) return rc;
  for (int i = 0; i < p->n; i++) {
    hd[i] = p->descs[i]; hd[i].in = static_cast<const float *>(in_ptrs[i]);
    hd[i].out = out_ptrs ? static_cast<float *>(out_ptrs[i]) : nullptr;
    hd[i].preemph = pre ? p->preemph[i] : 0.0f;
  }
  if ((rc = p->arena.Upload(sizeof(SpecDesc) * p->n, stream))) return rc;
  static const bool radix2_only = getenv("DALIB200_STFT_RADIX2") != nullptr;
  if (P.nfft == 1024 && (!radix2_only || mel)) {
    // register-resident 32 x 32 FFT, one warp per pair of frames (16 frames per CTA = the grouping the descriptors were built with)
    // the shared-memory attribute belongs to the kernel on the current device, so it is set once per PLAN, not once per process: a
    // plan's descriptor arena lives on the device it was created on, and a process running on two devices has a plan on each
    if (!p->smem_set) {
      DB_CUDA(cudaFuncSetAttribute(spectrogram1024_kernel<false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kF1024Smem));
      DB_CUDA(cudaFuncSetAttribute(spectrogram1024_kernel<true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kF1024Smem));
      DB_CUDA(cudaFuncSetAttribute(spectrogram1024_kernel<false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kF1024Smem));
      DB_CUDA(cudaFuncSetAttribute(spectrogram1024_kernel<true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kF1024Smem));
      p->smem_set = true;
    }
    const int grid = (int)std::min<int64_t>(p->total_groups, (int64_t)NumSMs() * 2);
    MelTables mt{};
    if (mel) {
      size_t o_up = 0, o_down = 0;
      if ((rc = MelUploadTables(mel, stream, &o_up, &o_down))) return rc;
      MelDesc *md;
      if ((rc = mel->arena.Stage(sizeof(MelDesc) * mel->n, &md))) return rc;
      for (int i = 0; i < mel->n; i++) { md[i] = mel->descs[i]; md[i].in = nullptr; md[i].out = static_cast<float *>(mel_out_ptrs[i]); }
      if ((rc = mel->arena.Upload(sizeof(MelDesc) * mel->n, stream))) return rc;
      mt.ends = reinterpret_cast<const int32_t *>(mel->tables.dev);
      mt.w_up = reinterpret_cast<const float *>(mel->tables.dev + o_up);
      mt.w_down = reinterpret_cast<const float *>(mel->tables.dev + o_down);
      mt.nfilter = mel->nfilter;
      Launch(pre ? "preemph_spectrogram_mel_fused" : "spectrogram_mel_fused", pre ? spectrogram1024_kernel<true, true> : spectrogram1024_kernel<true, false>,
             grid, kF1024Warps * 32, kF1024Smem, stream, reinterpret_cast<const SpecDesc *>(p->arena.dev), p->n, p->total_groups, P, p->d_window,
             p->d_twiddle, mt, reinterpret_cast<const MelDesc *>(mel->arena.dev), out_ptrs ? 1 : 0);
    } else {
      Launch(pre ? "preemph_spectrogram_stft" : "spectrogram_stft", pre ? spectrogram1024_kernel<false, true> : spectrogram1024_kernel<false, false>,
             grid, kF1024Warps * 32, kF1024Smem, stream, reinterpret_cast<const SpecDesc *>(p->arena.dev), p->n, p->total_groups, P, p->d_window,
             p->d_twiddle, mt, nullptr, 1);
    }
    DB_CUDA(cudaGetLastError());
    return DALIB200_SUCCESS;
  }
  if (!pow2) {
    auto *k = pre ? spectrogram_dft_kernel<true> : spectrogram_dft_kernel<false>;
    DB_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)std::max<size_t>(p->smem, 48 * 1024)));
    const int gridd = (int)std::min<int64_t>(p->total_groups, (int64_t)NumSMs() * 4);
    Launch(pre ? "preemph_spectrogram_dft" : "spectrogram_dft", k, gridd, 256, p->smem, stream, reinterpret_cast<const SpecDesc *>(p->arena.dev), p->n,
           p->total_groups, P, p->d_window, p->d_twiddle);
    DB_CUDA(cudaGetLastError());
    return DALIB200_SUCCESS;
  }
  auto *k = pre ? spectrogram_kernel<true> : spectrogram_kernel<false>;
  DB_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)std::max<size_t>(p->smem, 96 * 1024)));
  const int grid = (int)std::min<int64_t>(p->total_groups, (int64_t)NumSMs() * 8);
  Launch(pre ? "preemph_spectrogram_stft_radix2" : "spectrogram_stft_radix2", k, grid, 256, p->smem, stream, reinterpret_cast<const SpecDesc *>(p->arena.dev),
         p->n, p->total_groups, P, p->d_window, p->d_twiddle);
  DB_CUDA(cudaGetLastError());
  return DALIB200_SUCCESS;
}

int dalib200SpectrogramLaunch(dalib200SpectrogramPlan *p, const void *const *in_ptrs, void *const *out_ptrs, dalib200Stream_t stream) try {
  DB_CHECK_ARG(p && in_ptrs && out_ptrs, "SpectrogramLaunch: null argument");
  return SpectrogramLaunchImpl(p, in_ptrs, out_ptrs, nullptr, nullptr, stream);
} DB_API_CATCH

int dalib200SpectrogramMelSupported(const dalib200SpectrogramPlan *p, const dalib200MelPlan *m) try {
  if (!p || !m || p->P.nfft != 1024 || !p->P.layout_ft || m->nbin != p->P.nbin || m->n != p->n || m->tensor_cores) return 0;
  for (int i = 0; i < p->n; i++) if (m->descs[i].nwin != p->descs[i].nwin) return 0;
  return 1;
} DB_API_CATCH

int dalib200SpectrogramMelLaunch(dalib200SpectrogramPlan *p, dalib200MelPlan *m, const void *const *in_ptrs, void *const *spec_out_ptrs,
                                 void *const *mel_out_ptrs, dalib200Stream_t stream) try {
  DB_CHECK_ARG(p && m && in_ptrs && mel_out_ptrs, "SpectrogramMelLaunch: null argument");
  DB_CHECK_ARG(dalib200SpectrogramMelSupported(p, m), "SpectrogramMelLaunch: the fused kernel needs nfft = 1024, the (f, t) layout and a mel "
               "plan set up for the same batch (check dalib200SpectrogramMelSupported)");
  return SpectrogramLaunchImpl(p, in_ptrs, spec_out_ptrs, m, mel_out_ptrs, stream);
} DB_API_CATCH

int dalib200MelPlanCreate(dalib200MelPlan **plan, int max_batch) try {
  DB_CHECK_ARG(plan && max_batch > 0, "MelPlanCreate: bad arguments");
  auto *p = new dalib200MelPlan();
  p->max_batch = max_batch;
  int rc = p->arena.Reserve(sizeof(MelDesc) * max_batch);
  if (rc) { delete p; return rc; }
  *plan = p;
  return DALIB200_SUCCESS;
} DB_API_CATCH

int dalib200MelPlanDestroy(dalib200MelPlan *p) try {
  if (!p) return DALIB200_SUCCESS;
  p->arena.Free(); p->tables.Free(); p->dense.Free();
  delete p;
  return DALIB200_SUCCESS;
} DB_API_CATCH

int dalib200MelPlanSetTensorCores(dalib200MelPlan *p, int enable) try {
  DB_CHECK_ARG(p, "MelPlanSetTensorCores: null plan");
  p->tensor_cores = enable != 0;
  return DALIB200_SUCCESS;
} DB_API_CATCH

int dalib200MelPlanSetup(dalib200MelPlan *p, const dalib200MelArgs *args, int nbin, int n, const int64_t *nwin) try {
  DB_CHECK_ARG(p && args && nwin && n >= 0 && n <= p->max_batch, "MelPlanSetup: bad arguments");
  DB_CHECK_ARG(args->nfilter > 0, "MelFilterBank: nfilter must be positive");
  DB_CHECK_ARG(nbin >= 2 && nbin <= (1 << 24), "MelFilterBank: the frequency axis must have 2 .. 2^24 bins (got %d)", nbin);
  DB_CHECK_ARG(args->nfilter >= 1 && args->nfilter <= (1 << 20), "MelFilterBank: nfilter must be in 1 .. 2^20 (got %d)", args->nfilter);
  dalib200MelArgs a = *args;
  DB_CHECK_ARG(a.sample_rate > 0 && a.sample_rate <= 1e9f, "MelFilterBank: sample_rate must be positive and finite");
  if (a.freq_high <= 0) a.freq_high = a.sample_rate / 2;
  DB_CHECK_ARG(a.freq_low >= 0 && a.freq_low <= a.sample_rate / 2, "MelFilterBank: freq_low out of range");
  DB_CHECK_ARG(a.freq_high >= 0 && a.freq_high <= a.sample_rate / 2, "MelFilterBank: freq_high out of range");
  const bool same = p->nbin == nbin && memcmp(&a, &p->args, sizeof(a)) == 0 && !p->h_ends.empty();
  if (!same) {
    const int nfft = 2 * (nbin - 1);
    if (a.htk) BuildMel<Htk>(a, nfft, p->h_ends, p->h_up, p->h_down);
    else BuildMel<Slaney>(a, nfft, p->h_ends, p->h_up, p->h_down);
    p->args = a; p->nbin = nbin; p->nfilter = a.nfilter;
    p->tables_dirty = true; p->dense_dirty = true;
  }
  p->descs.assign(n, MelDesc());
  int64_t items = 0;
  for (int i = 0; i < n; i++) {
    DB_CHECK_ARG(nwin[i] >= 0, "MelFilterBank: negative number of windows");
    p->descs[i].nwin = nwin[i]; p->descs[i].first_item = items;
    items += (int64_t)a.nfilter * ((nwin[i] + 127) / 128);
  }
  p->first_item_mma.assign(n, 0);
  int64_t items2 = 0;
  for (int i = 0; i < n; i++) {
    p->first_item_mma[i] = items2;
    items2 += (int64_t)((a.nfilter + kMmM - 1) / kMmM) * ((nwin[i] + kMmN - 1) / kMmN);
  }
  p->total_items_mma = items2;
  p->n = n; p->total_items = items;
  return DALIB200_SUCCESS;
} DB_API_CATCH

static int MelUploadTables(dalib200MelPlan *p, dalib200Stream_t stream, size_t *o_up_out, size_t *o_down_out) {
  const size_t o_up = (p->h_ends.size() * 4 + 15) / 16 * 16, o_down = o_up + (p->h_up.size() * 4 + 15) / 16 * 16;
  const size_t tbytes = o_down + p->h_down.size() * 4;
  *o_up_out = o_up; *o_down_out = o_down;
  if (p->tables_dirty) {
    uint8_t *h;
    int rc = p->tables.Stage(tbytes, &h);
    if (rc) return rc;
    memcpy(h, p->h_ends.data(), p->h_ends.size() * 4);
    memcpy(h + o_up, p->h_up.data(), p->h_up.size() * 4);
    memcpy(h + o_down, p->h_down.data(), p->h_down.size() * 4);
    rc = p->tables.Upload(tbytes, stream);
    if (rc) return rc;
    p->tables_dirty = false;
  }
  return DALIB200_SUCCESS;
}

int dalib200MelLaunch(dalib200MelPlan *p, const void *const *in_ptrs, void *const *out_ptrs, dalib200Stream_t stream) try {
  DB_CHECK_ARG(p && in_ptrs && out_ptrs, "MelLaunch: null argument");
  if (p->n == 0 || p->total_items == 0) return DALIB200_SUCCESS;
  size_t o_up = 0, o_down = 0;
  int rc = MelUploadTables(p, stream, &o_up, &o_down);
  if (rc) return rc;
  MelDesc *hd;
  if ((rc = p->arena.Stage(sizeof(MelDesc) * p->n, &hd))) return rc;
  for (int i = 0; i < p->n; i++) {
    hd[i] = p->descs[i]; hd[i].in = static_cast<const float *>(in_ptrs[i]); hd[i].out = static_cast<float *>(out_ptrs[i]);
    if (p->tensor_cores) hd[i].first_item = p->first_item_mma[i];
  }
  if ((rc = p->arena.Upload(sizeof(MelDesc) * p->n, stream))) return rc;
  if (p->tensor_cores) {
    const int mblocks = (p->nfilter + kMmM - 1) / kMmM;
    if (p->dense_dirty) {
      p->kpad = (p->nbin + kMmK - 1) / kMmK * kMmK; p->mpad = mblocks * kMmM;
      const size_t wbytes = (size_t)p->mpad * p->kpad * 4, total = wbytes + sizeof(int2) * mblocks;
      float *w;
      if ((rc = p->dense.Stage(total, &w))) return rc;
      memset(w, 0, wbytes);
      for (int m = 0; m < p->nfilter; m++) {
        for (int b = p->h_ends[m]; b < p->h_ends[m + 1]; b++) w[(size_t)m * p->kpad + b] = p->h_up[b];
        for (int b = p->h_ends[m + 1]; b < p->h_ends[m + 2]; b++) w[(size_t)m * p->kpad + b] = p->h_down[b];
      }
      int2 *kr = reinterpret_cast<int2 *>(reinterpret_cast<uint8_t *>(w) + wbytes);
      for (int mb = 0; mb < mblocks; mb++) {
        const int m0 = mb * kMmM, m1 = std::min(p->nfilter, m0 + kMmM);
        kr[mb] = make_int2(p->h_ends[m0] / kMmK, (p->h_ends[m1 + 1] + kMmK - 1) / kMmK);
      }
      rc = p->dense.Upload(total, stream);
      if (rc) return rc;
      p->dense_dirty = false;
    }
    const int grid = (int)std::min<int64_t>(p->total_items_mma, (int64_t)NumSMs() * 8);
    Launch("mel_filter_bank_mma", mel_mma_kernel, grid, 256, 0, stream, reinterpret_cast<const MelDesc *>(p->arena.dev), p->n, p->total_items_mma,
           p->nfilter, p->nbin, p->kpad, reinterpret_cast<const float *>(p->dense.dev),
           reinterpret_cast<const int2 *>(p->dense.dev + (size_t)p->mpad * p->kpad * 4));
    DB_CUDA(cudaGetLastError());
    return DALIB200_SUCCESS;
  }
  const int grid = (int)std::min<int64_t>(p->total_items, (int64_t)NumSMs() * 32);
  Launch("mel_filter_bank", mel_kernel, grid, 128, 0, stream, reinterpret_cast<const MelDesc *>(p->arena.dev), p->n, p->total_items, p->nfilter,
         reinterpret_cast<const int32_t *>(p->tables.dev), reinterpret_cast<const float *>(p->tables.dev + o_up),
         reinterpret_cast<const float *>(p->tables.dev + o_down));
  DB_CUDA(cudaGetLastError());
  return DALIB200_SUCCESS;
} DB_API_CATCH

}  // extern "C"
