// dali_b200/csrc/jpeg.cu -- baseline JPEG decode on sm_90a: Huffman + dequant + IDCT + upsample + colour.
//
// Replaces the reference's mixed-backend image decoder (dali/operators/imgcodec/image_decoder.h:613-882), whose
// arithmetic lives in nvImageCodec / nvJPEG / libjpeg-turbo (not in the reference tree).  Parity target =
// the reference CPU backend = libjpeg-turbo defaults: islow integer IDCT, "fancy" (triangle) chroma
// upsampling (image_decoder.h:297-304: CPU always fancy), fixed-point YCbCr->RGB; oracle/jpeg_oracle.c
// restates it and is pinned bit-exactly against cv2.imdecode.
//
// Host (PlanSetup): marker / table parse only (ITU-T T.81 Annex B), packing of the entropy-coded
// segments into pinned staging.  Everything else runs on the device:
//   U1/U2/U3  byte un-stuffing (FF 00 -> FF) of every entropy-coded segment into a clean, word-swapped stream
//   H1        speculative Huffman decode of 2^k-byte subsequences + intra-block self-synchronisation
//   H2        inter-block synchronisation, per-segment exclusive scan of the coefficient counts
//   H3        final decode pass writing quantised coefficients (natural order, DC still differential)
//   D1        DC prediction (prefix sum per component, reset at restart intervals)
//   I1        dequantisation + islow IDCT -> planar component samples
//   C1        chroma upsampling (fancy / box) + colour conversion (YCbCr, RGB, CMYK, YCCK) -> interleaved HWC u8
//   I1 + C1   fused, without the planes, for 4:2:0 YCbCr with fancy upsampling to RGB / BGR (idct_color_420)
// The parallel entropy decode follows the self-synchronising scheme of Weissenberger & Schmidt
// ("Accelerating JPEG decompression on GPUs", 2021): a decoder started at a wrong bit position
// re-synchronises with the true symbol sequence after a few symbols, so every subsequence is first
// decoded speculatively and the exit states are then chained until they agree.
//
// Algorithmic bytes per unit (SURVEY.md 8d): J (encoded bytes) + H*W*3 (decoded image).
//
// The plan also takes PNG, TIFF, lossy WebP, BMP and PNM streams (detected by their signatures): the stage of each format (png.h,
// tiff.h, webp.h, bitmap.h; decode_stage.h) plans them at set-up and decodes them into the same decode windows on a stream of its own,
// and the post pass below serves every format.  Such a sample has no units, subsequences or MCUs, so every kernel of this file skips it.
// A lossless JPEG (SOF3) sample is parsed here and planned by the lossless stage (ljpeg.h): its restart intervals join U1 - U3 as units
// of no JPEG image, and the stage decodes their clean streams on a stream forked behind U3.
#include "common.cuh"
#include "jpeg_recon.h"
#include "jpeg_idct_core.h"
#include "jpeg_huff_core.h"
#include <algorithm>
#include <array>
#include <cstring>
#include <map>
#include <thread>

namespace dalib200 {

constexpr int kSyncThreads = 256;            // subsequences per synchronisation block
constexpr int kMaxLog2Sub = 10;              // largest subsequence: 2^10 bits = 128 bytes

// Huffman tables as the device sees them (jpeg_huff_core.h).  The first-level LUTs are copied to shared memory by every block; the
// canonical tables for longer codes stay in global memory.
struct TableSet {             // the 4 tables a baseline scan can reference: DC0, DC1, AC0, AC1
  uint32_t lut[kLutWords];    // at LutOffset(t)
  HuffSlow slow[4];
};

// Post pass of one sample (decoders.image with output_type / dtype / orientation / unaligned ROI handling): gathers the
// oriented region of interest from the decoded window and converts colour space and type
// (dali/operators/imgcodec/util/convert.h:255-316 ApplyOrientation + ConvertPixel, convert_gpu.cu:75-123).
struct JpegPost {
  const uint8_t *src; void *dst;
  int32_t src_w, src_c;                    // window pitch in pixels, channels (1 or 3: GRAY / RGB)
  int32_t img_w, img_h;                    // un-oriented image size
  int32_t win_x0, win_y0;
  int32_t out_x0, out_y0, out_w, out_h;    // region of interest in ORIENTED image coordinates
  int32_t orientation;                     // EXIF 1..8
  int32_t out_type, dtype;                 // DALIB200_RGB.. / DALIB200_UINT8 | DALIB200_FLOAT
  int64_t first_px;
};

__constant__ uint8_t c_zigzag[64] = {
   0,  1,  8, 16,  9,  2,  3, 10, 17, 24, 32, 25, 18, 11,  4,  5,
  12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13,  6,  7, 14, 21, 28,
  35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51,
  58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63 };

// ============================================================================================
// U1..U3: byte un-stuffing
// a byte is dropped when it is the 0x00 that follows a 0xFF.  Word-at-a-time: bit 8k+7.. of the result marks byte k of
// `w` as dropped; `prev` is the byte in front of the word (0 at the start of a unit).
__device__ __forceinline__ uint32_t dropped_mask(uint32_t w, uint32_t prev) {
  const uint32_t is00 = __vcmpeq4(w, 0u);                      // 0xFF per byte that is 0x00
  const uint32_t pw = (w << 8) | prev;                         // byte k = the byte in front of byte k of w
  const uint32_t isff = __vcmpeq4(pw, 0xFFFFFFFFu);
  return is00 & isff;
}

// 4 raw bytes at offset i of a chunk (bytes at or beyond `len` read as 0x01: never dropped, never a 0xFF prefix).  Units that
// start behind a restart marker are not word aligned: those take the byte path.
__device__ __forceinline__ uint32_t load_raw_word(const uint8_t *p, uint32_t i, uint32_t len) {
  uint32_t w;
  if ((reinterpret_cast<uintptr_t>(p + i) & 3u) == 0 && i + 4 <= len) {
    w = *reinterpret_cast<const uint32_t *>(p + i);
  } else {
    w = 0;
#pragma unroll
    for (int k = 0; k < 4; k++) w |= (uint32_t)(i + k < len ? p[i + k] : 1u) << (8 * k);
  }
  return w;
}

// One chunk = 4096 raw bytes = 4 rounds of 256 words: thread t owns words t, 256 + t, 512 + t, 768 + t, so that the lanes of a warp
// always touch consecutive words (coalesced loads, conflict-free shared-memory byte stores in the scatter pass).
constexpr int kChunkRounds = kChunkBytes / (256 * 4);

struct ChunkWords { uint32_t w[kChunkRounds], dm[kChunkRounds]; int nk[kChunkRounds]; };

__device__ __forceinline__ ChunkWords load_chunk(const uint8_t *__restrict__ p, uint32_t c0, uint32_t len) {
  ChunkWords cw;
#pragma unroll
  for (int r = 0; r < kChunkRounds; r++) {
    const uint32_t i = (uint32_t)r * 1024u + threadIdx.x * 4u;
    cw.w[r] = 0; cw.dm[r] = 0; cw.nk[r] = 0;
    if (i < len) {
      cw.w[r] = load_raw_word(p, i, len);
      const uint32_t prev = c0 + i > 0 ? p[(int64_t)i - 1] : 0u;      // the chunk is not the first of its unit when c0 > 0
      cw.dm[r] = dropped_mask(cw.w[r], prev);
      cw.nk[r] = (int)min(4u, len - i) - (__popc(cw.dm[r]) >> 3);
    }
  }
  return cw;
}

__global__ void __launch_bounds__(256) unstuff_count_kernel(const uint8_t *__restrict__ raw, const JpegUnit *__restrict__ units,
                                                            int nunits, uint32_t nchunks, uint32_t *__restrict__ chunk_cnt) {
  __shared__ int wsum[8];
  __shared__ int s_ui;
  // contiguous range of chunks per CTA: the unit is searched once and then only advanced
  const uint32_t per = (nchunks + gridDim.x - 1) / gridDim.x;
  const uint32_t ch0 = blockIdx.x * per, ch1 = min(nchunks, ch0 + per);
  if (ch0 >= ch1) return;
  if (threadIdx.x == 0) s_ui = last_at_most(units, 0, nunits - 1, ch0, [](const JpegUnit &u) { return u.first_chunk; });
  __syncthreads();
  int ui = s_ui;
  for (uint32_t chunk = ch0; chunk < ch1; chunk++) {
    while (ui + 1 < nunits && units[ui + 1].first_chunk <= chunk) ui++;
    const JpegUnit &u = units[ui];
    const uint32_t c0 = (chunk - u.first_chunk) * kChunkBytes;
    const uint32_t len = min((uint32_t)kChunkBytes, u.raw_len - c0);
    const ChunkWords cw = load_chunk(raw + u.raw_off + c0, c0, len);
    int cnt = 0;
#pragma unroll
    for (int r = 0; r < kChunkRounds; r++) cnt += __popc(cw.dm[r]) >> 3;
    for (int o = 16; o; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
    if ((threadIdx.x & 31) == 0) wsum[threadIdx.x >> 5] = cnt;
    __syncthreads();
    if (threadIdx.x == 0) { int s = 0; for (int w = 0; w < 8; w++) s += wsum[w]; chunk_cnt[chunk] = (uint32_t)s; }
    __syncthreads();
  }
}

// one warp per unit: exclusive scan of the dropped-byte counts of its chunks
__global__ void __launch_bounds__(256) unstuff_scan_kernel(const JpegUnit *__restrict__ units, int nunits, uint32_t *__restrict__ chunk_cnt,
                                                           uint32_t *__restrict__ unit_clean_len) {
  const uint32_t lane = threadIdx.x & 31u;
  const int nwarps = (int)((gridDim.x * blockDim.x) >> 5);
  for (int ui = (int)((blockIdx.x * blockDim.x + threadIdx.x) >> 5); ui < nunits; ui += nwarps) {
    const JpegUnit &u = units[ui];
    const uint32_t nch = (u.raw_len + kChunkBytes - 1) / kChunkBytes;
    uint32_t run = 0;
    for (uint32_t base = 0; base < nch; base += 32) {
      const uint32_t c = base + lane;
      const uint32_t v = c < nch ? chunk_cnt[u.first_chunk + c] : 0u;
      uint32_t incl = v;
      for (int o = 1; o < 32; o <<= 1) { const uint32_t x = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= (uint32_t)o) incl += x; }
      if (c < nch) chunk_cnt[u.first_chunk + c] = run + incl - v;
      run += __shfl_sync(0xffffffffu, incl, 31);
    }
    if (lane == 0) unit_clean_len[ui] = u.raw_len - run;
  }
}

// Writes the clean stream with every 32-bit word byte-swapped (address ^ 3), so that a plain 32-bit
// load returns the big-endian bit order the Huffman reader wants.  The kept bytes of a chunk are compacted in shared
// memory (byte stores, consecutive lanes -> consecutive words) and leave as whole swapped words; only the two words a
// chunk shares with its neighbours are written byte by byte.
__global__ void __launch_bounds__(256) unstuff_scatter_kernel(const uint8_t *__restrict__ raw, const JpegUnit *__restrict__ units,
                                                              int nunits, uint32_t nchunks, const uint32_t *__restrict__ chunk_drop,
                                                              uint8_t *__restrict__ clean) {
  __shared__ int wsum[8][kChunkRounds];
  __shared__ uint32_t obuf[kChunkBytes / 4 + 2];
  __shared__ int s_ui;
  const uint32_t lane = threadIdx.x & 31u, wid = threadIdx.x >> 5;
  const uint32_t per = (nchunks + gridDim.x - 1) / gridDim.x;
  const uint32_t ch0 = blockIdx.x * per, ch1 = min(nchunks, ch0 + per);
  if (ch0 >= ch1) return;
  if (threadIdx.x == 0) s_ui = last_at_most(units, 0, nunits - 1, ch0, [](const JpegUnit &u) { return u.first_chunk; });
  __syncthreads();
  int ui = s_ui;
  for (uint32_t chunk = ch0; chunk < ch1; chunk++) {
    while (ui + 1 < nunits && units[ui + 1].first_chunk <= chunk) ui++;
    const JpegUnit &u = units[ui];
    const uint32_t c0 = (chunk - u.first_chunk) * kChunkBytes;
    const uint32_t len = min((uint32_t)kChunkBytes, u.raw_len - c0);
    const uint32_t out_base = u.clean_off + c0 - chunk_drop[chunk];
    const ChunkWords cw = load_chunk(raw + u.raw_off + c0, c0, len);
    int incl[kChunkRounds];
#pragma unroll
    for (int r = 0; r < kChunkRounds; r++) incl[r] = cw.nk[r];
    for (int o = 1; o < 32; o <<= 1) {
#pragma unroll
      for (int r = 0; r < kChunkRounds; r++) { const int v = __shfl_up_sync(0xffffffffu, incl[r], o); if (lane >= (uint32_t)o) incl[r] += v; }
    }
    if (lane == 31) {
#pragma unroll
      for (int r = 0; r < kChunkRounds; r++) wsum[wid][r] = incl[r];
    }
    __syncthreads();
    const uint32_t head = out_base & 3u;                      // obuf word k <-> clean word (out_base >> 2) + k
    uint32_t total = 0;
    uint8_t *ob = reinterpret_cast<uint8_t *>(obuf);
#pragma unroll
    for (int r = 0; r < kChunkRounds; r++) {
      int woff = 0, tot = 0;
#pragma unroll
      for (int w = 0; w < 8; w++) { if (w < (int)wid) woff += wsum[w][r]; tot += wsum[w][r]; }
      uint32_t pos = head + total + (uint32_t)(woff + incl[r] - cw.nk[r]);
      const uint32_t i = (uint32_t)r * 1024u + threadIdx.x * 4u;
#pragma unroll
      for (int k = 0; k < 4; k++)
        if (i + k < len && !((cw.dm[r] >> (8 * k)) & 1u)) ob[pos++] = (uint8_t)(cw.w[r] >> (8 * k));
      total += (uint32_t)tot;
    }
    __syncthreads();
    const uint32_t nwords = (head + total + 3u) >> 2, tailb = (head + total) & 3u;
    uint32_t *cw32 = reinterpret_cast<uint32_t *>(clean) + (out_base >> 2);
    for (uint32_t wd = threadIdx.x; wd < nwords; wd += blockDim.x) {
      const uint32_t v = obuf[wd];
      const bool full = (wd > 0 || head == 0) && (wd + 1 < nwords || tailb == 0);
      if (full) {
        cw32[wd] = __byte_perm(v, 0u, 0x0123);
      } else {
        const uint32_t lo = wd == 0 ? head : 0u, hi = (wd + 1 == nwords && tailb) ? tailb : 4u;
        for (uint32_t b = lo; b < hi; b++) reinterpret_cast<uint8_t *>(cw32 + wd)[3u - b] = (uint8_t)(v >> (8 * b));
      }
    }
    if (c0 + kChunkBytes >= u.raw_len) {
      // last chunk of the unit: zero the pad behind the clean bytes (the bit reader peeks a few bytes past the end); the
      // clean buffer itself is never memset
      const uint32_t e0 = out_base + total, e1 = u.clean_off + ((u.raw_len + kCleanPad + 15u) & ~15u);
      for (uint32_t q = e0 + threadIdx.x; q < e1; q += blockDim.x) clean[(q & ~3u) | (3u - (q & 3u))] = 0;
    }
    __syncthreads();
  }
}

// ============================================================================================
// Huffman decoding
//
// Bit source: the clean (un-stuffed, word-swapped) stream of a unit.  The sync-intra pass stages the CTA's subsequences
// (+ look-ahead columns) into shared memory with coalesced 16-byte loads; word g of the staged run sits at
// g ^ ((g >> lsw) & 31) so that the 32 lanes of a warp, each inside its own subsequence, always hit 32 different banks.  The write
// pass reads the stream straight from global memory through a register window (StreamWindow below); the chain walk copies a
// subsequence into a private shared-memory column (ColSrc) or reads words from global (GlobalSrc).
struct SmemSrc {
  uint32_t base; int lsw;                  // shared-window address of the staged run
  __device__ __forceinline__ uint32_t load(uint32_t g) const { return lds_u32(base + ((g ^ ((g >> lsw) & 31u)) << 2)); }
};
// table accessors: first-level LUT (32-bit entries) and the per-block (dc | ac << 16) table offsets
struct SmemLut { uint32_t base; __device__ __forceinline__ uint32_t load(uint32_t i) const { return lds_u32(base + (i << 2)); } };
struct GlobalLut { const uint32_t *p; __device__ __forceinline__ uint32_t load(uint32_t i) const { return __ldg(p + i); } };
template <int STRIDE> struct SmemTbl { uint32_t base; __device__ __forceinline__ uint32_t load(int c) const { return lds_u32(base + (uint32_t)c * (STRIDE * 4u)); } };
struct GlobalSrc {
  const uint32_t *w;
  __device__ __forceinline__ uint32_t load(uint32_t g) const { return __ldg(w + g); }
};

// 64-bit MSB-aligned window in two registers: `hi` always holds the next 32 bits.  The refill is written with selects:
// the 32 lanes of a warp sit at unrelated bit positions, so a branch here would be divergent on almost every symbol.
template <class Src>
struct BitWindow {
  Src s;
  uint32_t hi, lo, g;
  int avail;
  __device__ __forceinline__ void init(const Src &src, uint32_t word, uint32_t sh) {
    s = src;
    const uint32_t w0 = s.load(word), w1 = s.load(word + 1);
    hi = __funnelshift_l(w1, w0, sh);
    lo = w1 << sh;
    avail = 64 - (int)sh;
    g = word + 2;
  }
  __device__ __forceinline__ void consume(uint32_t e) {      // e & 31 = bits to drop, 0..31
    hi = __funnelshift_l(lo, hi, e);
    lo = __funnelshift_l(0u, lo, e);
    avail -= (int)(e & 31u);
    const uint32_t w = s.load(g);                  // the same word is re-read until it is taken
    const bool need = avail < 32;                  // then 1 <= avail <= 31 and lo == 0
    const uint32_t a = (uint32_t)avail & 31u;
    hi |= (need ? w : 0u) >> a;
    lo = need ? (w << ((32u - a) & 31u)) : lo;
    avail += need ? 32 : 0;
    g += need ? 1u : 0u;
  }
};

// The same window fed from global memory without shared memory.  The unit's stream is read in 16-byte chunks (ld.global.nc, always
// aligned: units start 16-byte aligned in the clean buffer) into registers: a queue c0..c4 of up to 5 words (c0 = the word the
// next refill takes; a refill moves the others up by one with selects, no branch) and the next chunk `nxt`, in flight.
// A load's destination registers carry a scoreboard for the whole warp, so `nxt` is only ever read at warp-uniform points: every
// second iteration of a warp-uniform symbol loop (top_up), where the lanes with at most one word left append `nxt` to their queue
// and request the chunk behind it.  A refill takes at most one word per symbol, so a lane never runs dry between two top-ups, and
// every load has had two loop iterations to arrive before its registers are read (huff_write's loop is warp-uniform).
//
// Read bound.  Window invariant: 32 * T = pos + avail, T = words taken by the window, 32 <= avail <= 64 after every consume, pos =
// the unit bit position of `hi`'s MSB.  The decode loops only start a symbol at pos < clean_bits (= 8 * L, L = the unit's clean
// length) and a symbol takes at most 31 bits, so pos <= 8L + 30 and T <= (8L + 94) / 32: every word the window takes lies within
// L + 12 bytes, inside the unit's zero pad (>= kCleanPad bytes) -- the window never sees a byte of the next unit.  The queue ends
// at word T + 4 at most, and the chunk loaded last is the one behind it: every load lies below 16 * ((T + 4) / 4 + 2) <= 4T + 48
// <= L + 60 bytes behind the start of the unit.
constexpr uint32_t kStreamReadBehind = 60;     // StreamWindow loads stay below clean_off + L + kStreamReadBehind (see above)
// Predicated 16-byte load of the next chunk into `v` itself, read-only path, the L2 fetches the whole 128-byte line.  The
// destination is tied to the registers that hold `v` across the loop: with a plain load the compiler picked other registers and
// copied the result over right behind the load, which waits for it.
__device__ __forceinline__ void ldg_stream(bool pred, uint4 &v, const uint4 *p) {
  asm volatile("{\n\t.reg .pred q;\n\tsetp.ne.u32 q, %5, 0;\n\t@q ld.global.nc.L2::128B.v4.u32 {%0, %1, %2, %3}, [%4];\n\t}"
               : "+r"(v.x), "+r"(v.y), "+r"(v.z), "+r"(v.w) : "l"(p), "r"((uint32_t)pred));
}
// plain (weak) global stores to a 64-bit global address
__device__ __forceinline__ void stg_u16(uint64_t a, uint32_t v) { asm volatile("st.global.u16 [%0], %1;" :: "l"(a), "h"((unsigned short)v)); }
__device__ __forceinline__ void stg_v4(uint64_t a, uint4 v) {
  asm volatile("st.global.v4.u32 [%0], {%1, %2, %3, %4};" :: "l"(a), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w));
}
__device__ __forceinline__ uint4 lds_v4(uint32_t a) {
  uint4 v;
  asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(a));
  return v;
}
__device__ __forceinline__ void sts_v4(uint32_t a, uint4 v) {
  asm volatile("st.shared.v4.u32 [%0], {%1, %2, %3, %4};" :: "r"(a), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
struct StreamWindow {
  uint32_t hi, lo;
  int avail;
  uint32_t left;                   // valid words in the queue c0..c4
  uint32_t c0, c1, c2, c3, c4;
  uint4 nxt;
  const uint4 *p;                  // the chunk behind `nxt`
  __device__ __forceinline__ void clear() { left = 5; }            // a lane without a stream: top_up never loads
  // window at unit bit position `pos`; `unit` = the unit's clean stream
  __device__ __forceinline__ void init(const uint8_t *unit, uint32_t pos) {
    const uint4 *q = reinterpret_cast<const uint4 *>(unit) + (pos >> 7);
    const uint4 a = __ldg(q);
    nxt = __ldg(q + 1);
    p = q + 2;
    hi = a.x; lo = a.y; avail = 64;
    c0 = a.z; c1 = a.w; c2 = c3 = c4 = 0; left = 2;
    for (uint32_t d = pos & 127u; d;) {            // skip to pos inside the chunk: at most 5 steps, once per window
      const uint32_t e = min(d, 31u);
      consume(e);
      top_up();
      d -= e;
    }
  }
  __device__ __forceinline__ void consume(uint32_t e) {      // e & 31 = bits to drop, 0..31
    hi = __funnelshift_l(lo, hi, e);
    lo = __funnelshift_l(0u, lo, e);
    avail -= (int)(e & 31u);
    const bool need = avail < 32;                  // then 1 <= avail <= 31 and lo == 0
    const uint32_t a = (uint32_t)avail & 31u;
    hi |= (need ? c0 : 0u) >> a;
    lo = need ? (c0 << ((32u - a) & 31u)) : lo;
    avail += need ? 32 : 0;
    c0 = need ? c1 : c0; c1 = need ? c2 : c1; c2 = need ? c3 : c2; c3 = need ? c4 : c3;
    left -= need ? 1u : 0u;
  }
  __device__ __forceinline__ void top_up() {
    const bool take = left <= 1;
    if (take) {
      const bool one = left != 0;
      c0 = one ? c0 : nxt.x; c1 = one ? nxt.x : nxt.y; c2 = one ? nxt.y : nxt.z; c3 = one ? nxt.z : nxt.w; c4 = nxt.w;
      left += 4;
    }
    ldg_stream(take, nxt, p);
    p += take ? 1 : 0;
  }
};

// Per-subsequence record of the synchronisation (one 64-bit word, updated with atomicMax in the chain walk):
//   [31:0] exit bit position  [35:32] block in MCU (c)  [41:36] zig-zag index (z)  [51:42] blocks completed in the subsequence
//   [63:52] priority t = distance of the chain that wrote the record from its origin (x - origin): the larger, the further
//   left the chain started, the better informed it is.  The state proper is the low 42 bits.
// A chain stops when its priority is full (t = kMaxChainLen).  Valid data can get there: a segment in which no speculative decoder
// meets the true one for 4095 subsequences (e.g. all-zero bits under tables whose all-zero codes are real codes, with an odd MCU
// length above 4096 bits).  The records up to subsequence kMaxChainLen - 1 of a unit are then still right; H2b re-decodes the rest of
// the unit sequentially from there (resync_unit).
constexpr uint64_t kStateMask = (1ull << 42) - 1;
constexpr uint32_t kMaxChainLen = 4095;
__device__ __forceinline__ uint64_t pack_state(uint32_t p, int c, int z, uint32_t cnt = 0, uint32_t t = 0) {
  return (uint64_t)p | ((uint64_t)(uint32_t)c << 32) | ((uint64_t)(uint32_t)z << 36) | ((uint64_t)min(cnt, 1023u) << 42) | ((uint64_t)t << 52);
}
__device__ __forceinline__ uint32_t state_count(uint64_t s) { return (uint32_t)(s >> 42) & 1023u; }

// codes longer than the first-level LUT (std tables: AC codes of 12..16 bits, < 1 % of the symbols): canonical search,
// T.81 F.2.2.3.  `toff` = LUT word offset of the table, which identifies it.  Returns the entry of the code (a single step,
// huff_entry); a window that matches no code gives 17 bits and symbol 0, which the 5-bit bit counts and the >= 32-bit window hold.
// The sync, walk and write passes all decode through here, so they stay in step on damaged data.
__device__ __noinline__ uint32_t slow_lookup(const HuffSlow *__restrict__ slow, uint32_t toff, uint32_t hi, bool is_dc) {
  const int tbl = toff < 2u * kDcLutSize ? (int)(toff / kDcLutSize) : 2 + (int)((toff - 2u * kDcLutSize) / kAcLutSize);
  const HuffSlow *sl = slow + tbl;
  const int32_t code16 = (int32_t)(hi >> 16);
  uint32_t len, sym = 0;
  if (sl->long_n > 0) {
    const int idx = min(max(code16 - sl->long_base, 0), sl->long_n - 1);
    const uint32_t e = sl->long_lut[idx];
    len = e ? (e & 0xFFu) : 17u;                             // not a code: 17 bits, symbol 0 (libjpeg jpeg_huff_decode)
    sym = e >> 8;
  } else {
    len = (is_dc ? kDcLutBits : kAcLutBits) + 1;
    while (len <= 16 && code16 >= sl->maxcode[len]) len++;
    if (len > 16) len = 17;                                  // not a code: 17 bits, symbol 0, as libjpeg (jpeg_huff_decode)
    else sym = sl->vals[(sl->valoff[len] + (code16 >> (16 - len))) & 0xFF];
  }
  return huff_entry(len, sym, is_dc);
}

// Decodes the symbols that START before `end` (absolute bit positions inside the unit) without producing coefficients: the
// synchronisation only needs the state (pos, c, z) and `nb`, the number of completed blocks.  Branch-free apart from the loop
// and the rare long-code path.  A step decodes one symbol or two of one block (huff_step); a block ends at most once per step.
template <class Win, class Lut, class Tbl>
__device__ __forceinline__ void decode_span(Win &win, const Lut &lut, const HuffSlow *__restrict__ slow,
                                            const Tbl &tbl, int bpm, uint32_t &pos, uint32_t end, int &c, int &z, uint32_t &nb) {
  uint32_t tb12 = tbl.load(c);                                // dc table offset | ac table offset << 16 (in LUT words)
  while (pos < end) {
    const uint32_t thr = pair_threshold(z, pos, end);
    // the AC entry is fetched before z is known (it is the common case and sits on the loop-carried path); the DC entry only
    // by the lanes that start a block, so that its random-bank lookup costs one shared-memory wavefront instead of three
    const uint32_t e_ac = lut.load((tb12 >> 16) + (win.hi >> (32 - kAcLutBits)));
    const bool is_dc = z == 0;
    uint32_t e = e_ac;
    if (is_dc) e = lut.load((tb12 & 0xFFFFu) + (win.hi >> (32 - kDcLutBits)));
    if (__builtin_expect(e == 0, 0)) e = slow_lookup(slow, is_dc ? (tb12 & 0xFFFFu) : (tb12 >> 16), win.hi, is_dc);
    const uint32_t st = huff_step(e, thr);
    win.consume(st);
    pos += step_bits(st);
    z += (int)step_adv(st);
    const bool endb = z >= 64;                                // block finished (EOB, 64th coefficient, or garbage overrun)
    const int c1 = c + 1 == bpm ? 0 : c + 1;
    nb += endb ? 1u : 0u;
    c = endb ? c1 : c;
    z = endb ? 0 : z;
    if (endb) tb12 = tbl.load(c);
  }
}

struct HuffCtx {
  const JpegImage *images; int nimages;
  const int32_t *block_image;           // sync block -> image
  const int32_t *wblock_image;          // write block -> image
  const JpegUnit *units;
  const uint32_t *unit_clean_len;
  const TableSet *tables;
  const uint8_t *clean;
  uint64_t *s_state;       // per subsequence: packed record (pack_state)
  uint32_t *s_n;           // per subsequence: exclusive prefix (per unit) of the completed-block counts (H2b)
  int16_t *coef;
  int16_t *dc;             // compact DC array: one int16 per block, same block order as coef
  int log2_sub;            // log2 of the subsequence size in BITS
  int32_t *status;         // per image: 0 ok, 1 = block count mismatch (corrupt stream)
  uint32_t *unit_nblk;     // per unit: blocks actually decoded (H2b), <= the unit's block count
  // live chains of the synchronisation: record = (bit position, c | z << 8 | t << 16, target subsequence, image)
  uint4 *chains[3];        // [0] filled by H1, [1] survivors of the first walk step, [2] survivors of the second
  uint32_t *chain_count;   // [3]
  uint32_t *chain_cut;     // per image: nonzero when a chain of one of its units stopped at kMaxChainLen before the unit's end
};

__device__ __forceinline__ uint32_t tbl_word(const JpegImage &im, int b) {
  return (uint32_t)LutOffset(im.blk_dc[b]) | ((uint32_t)LutOffset(im.blk_ac[b]) << 16);
}

// Shared memory of the sync-block kernels.
struct SyncSmem {
  uint32_t *lut, *sw, *cnt, *tbl, *col_end, *blkbuf;
  uint64_t *exitst;
  const uint8_t **colptr;
  uint8_t *zig, *col_cont;
  HuffSlow *slow;                // shared-memory copy of the canonical tables (the long-code path is latency critical)
};
// Columns staged behind the sync block: 256 bytes worth.  A block is at most 63 x 26 + 20 bits = 208 bytes long and the
// write pass completes the last block of the last column past the end of the sync block.
constexpr int kMaxLookAheadCols = 8;          // 32-byte subsequences
__host__ __device__ inline int look_ahead_cols(int log2_sub) { return 256 >> (log2_sub - 3); }
__host__ __device__ inline size_t sync_sw_words(int log2_sub) { return (size_t)(kSyncThreads + look_ahead_cols(log2_sub)) << (log2_sub - 5); }
__host__ __device__ inline size_t sync_smem_bytes(int log2_sub, bool with_block_buffers) {
  return kLutWords * 4 + sync_sw_words(log2_sub) * 4 + kSyncThreads * 8 /*exit*/ + (kSyncThreads + kMaxLookAheadCols) * 8 /*colptr*/ +
         kSyncThreads * 4 * 2 /*cnt, col_end*/ + 16 * 4 /*tbl*/ + 64 /*zig*/ + kSyncThreads /*col_cont*/ + 4 * sizeof(HuffSlow) +
         (with_block_buffers ? (size_t)kSyncThreads * 128 : 0) /*block buffers (H3)*/;
}
__device__ __forceinline__ SyncSmem carve_sync_smem(uint32_t *base, int log2_sub) {
  SyncSmem s;
  s.lut = base;
  s.sw = s.lut + kLutWords;
  s.exitst = reinterpret_cast<uint64_t *>(s.sw + sync_sw_words(log2_sub));     // both word counts are multiples of 8
  s.colptr = reinterpret_cast<const uint8_t **>(s.exitst + kSyncThreads);
  s.cnt = reinterpret_cast<uint32_t *>(s.colptr + kSyncThreads + kMaxLookAheadCols);
  s.col_end = s.cnt + kSyncThreads;
  s.tbl = s.col_end + kSyncThreads;
  s.zig = reinterpret_cast<uint8_t *>(s.tbl + 16);
  s.col_cont = s.zig + 64;
  s.slow = reinterpret_cast<HuffSlow *>(s.col_cont + kSyncThreads);       // 4-byte aligned: all sizes above are multiples of 4
  s.blkbuf = reinterpret_cast<uint32_t *>(s.slow + 4);
  return s;
}

// Common prologue of H1 / H3: tables into shared memory, per-thread subsequence geometry, cooperative staging of the stream.
struct SubGeom { bool valid; int ui; uint32_t jl, nsub_eff, clean_bits; int64_t g; };

__device__ __forceinline__ SubGeom sync_block_prologue(const HuffCtx &cx, const JpegImage &im, const SyncSmem &sm) {
  const int lsw = cx.log2_sub - 5;
  {
    const uint4 *src = reinterpret_cast<const uint4 *>(cx.tables[im.table_set].lut);
    uint4 *dst = reinterpret_cast<uint4 *>(sm.lut);
    for (int i = threadIdx.x; i < kLutWords / 4; i += blockDim.x) dst[i] = __ldg(src + i);
    if (threadIdx.x < kMaxBlocksPerMcu) sm.tbl[threadIdx.x] = tbl_word(im, threadIdx.x);
    if (threadIdx.x < 64) sm.zig[threadIdx.x] = c_zigzag[threadIdx.x];
    const uint32_t *ssrc = reinterpret_cast<const uint32_t *>(cx.tables[im.table_set].slow);
    uint32_t *sdst = reinterpret_cast<uint32_t *>(sm.slow);
    for (int i = threadIdx.x; i < (int)(4 * sizeof(HuffSlow) / 4); i += blockDim.x) sdst[i] = __ldg(ssrc + i);
  }
  SubGeom sg;
  const int j = (blockIdx.x - im.block_begin) * kSyncThreads + threadIdx.x;     // image-local subsequence
  sg.valid = j < im.nsub;
  sg.ui = 0; sg.jl = 0; sg.nsub_eff = 0; sg.clean_bits = 0;
  sg.g = (int64_t)im.subseq_begin + j;
  const uint8_t *ptr = nullptr;
  if (sg.valid) {
    sg.ui = im.unit_end - im.unit_begin == 1 ? im.unit_begin : last_at_most(cx.units, im.unit_begin, im.unit_end - 1, j, [](const JpegUnit &u) { return u.first_subseq; });
    const JpegUnit &u = cx.units[sg.ui];
    sg.clean_bits = cx.unit_clean_len[sg.ui] * 8u;
    sg.nsub_eff = (sg.clean_bits + (1u << cx.log2_sub) - 1) >> cx.log2_sub;
    sg.jl = (uint32_t)(j - u.first_subseq);
    sg.valid = sg.jl < sg.nsub_eff;
    if (sg.valid) ptr = cx.clean + u.clean_off + ((size_t)sg.jl << (cx.log2_sub - 3));
  }
  sm.colptr[threadIdx.x] = ptr;
  sm.col_end[threadIdx.x] = min((sg.jl + 1) << cx.log2_sub, sg.clean_bits);
  sm.col_cont[threadIdx.x] = sg.valid && sg.jl + 1 < sg.nsub_eff;             // the unit continues behind this column
  const int la_cols = look_ahead_cols(cx.log2_sub);
  if (threadIdx.x == kSyncThreads - 1)
    for (int q = 1; q <= la_cols; q++) sm.colptr[kSyncThreads - 1 + q] = ptr ? ptr + ((size_t)q << (cx.log2_sub - 3)) : nullptr;
  __syncthreads();
  const int cpc = 1 << (cx.log2_sub - 7);                    // 16-byte chunks per column
  for (int ch = threadIdx.x; ch < (kSyncThreads + la_cols) * cpc; ch += blockDim.x) {
    const int col = ch / cpc, o = ch - col * cpc;
    const uint8_t *p = sm.colptr[col];
    if (p) {
      const uint4 v = __ldg(reinterpret_cast<const uint4 *>(p) + o);
      const uint32_t g = ((uint32_t)col << lsw) + 4u * o, x = (uint32_t)col & 31u;
      sm.sw[(g + 0) ^ x] = v.x; sm.sw[(g + 1) ^ x] = v.y; sm.sw[(g + 2) ^ x] = v.z; sm.sw[(g + 3) ^ x] = v.w;
    }
  }
  __syncthreads();
  return sg;
}

__device__ __forceinline__ void push_chain(const HuffCtx &cx, int list, uint32_t pos, int c, int z, uint32_t t, int64_t g, int img) {
  const uint32_t k = atomicAdd(&cx.chain_count[list], 1u);
  cx.chains[list][k] = make_uint4(pos, (uint32_t)c | ((uint32_t)z << 8) | (t << 16), (uint32_t)g, (uint32_t)img);
}

// H1: every thread decodes its own subsequence speculatively from (c, z) = (0, 0) (round 0) and then the following one from
// its exit state (round 1).  A chain whose exit state does not yet agree with what the owner of that subsequence found is
// still "live": it is handed to the chain walk (H2a).  Records carry the priority t = (subsequence - origin of the chain that
// wrote it): 0 for the owner's own speculative decode, 1 for the visit of the left neighbour.
__global__ void __launch_bounds__(kSyncThreads) huff_sync_intra_kernel(HuffCtx cx) {
  extern __shared__ __align__(16) uint32_t hsm[];
  const SyncSmem sm = carve_sync_smem(hsm, cx.log2_sub);
  const int img_i = cx.block_image[blockIdx.x];
  const JpegImage &im = cx.images[img_i];
  const SubGeom sg = sync_block_prologue(cx, im, sm);
  const HuffSlow *slow = sm.slow;
  const int lsw = cx.log2_sub - 5;
  const SmemSrc src{smem_u32(sm.sw), lsw};
  const SmemLut lut{smem_u32(sm.lut)};
  const SmemTbl<1> tbl{smem_u32(sm.tbl)};
  BitWindow<SmemSrc> win;
  uint32_t pos = sg.jl << cx.log2_sub, nb = 0;
  int c = 0, z = 0;
  // ---- round 0
  if (sg.valid) {
    win.init(src, (uint32_t)threadIdx.x << lsw, 0);
    decode_span(win, lut, slow, tbl, im.bpm, pos, sm.col_end[threadIdx.x], c, z, nb);
    sm.exitst[threadIdx.x] = pack_state(pos, c, z);
    sm.cnt[threadIdx.x] = nb;
  }
  __syncthreads();
  // ---- round 1: the window simply continues into the next column; the last thread's next column belongs to the next block
  if (sm.col_cont[threadIdx.x]) {
    if (threadIdx.x + 1 == kSyncThreads) {
      push_chain(cx, 0, pos, c, z, 1u, sg.g + 1, img_i);
    } else {
      const uint32_t x = threadIdx.x + 1;
      nb = 0;
      decode_span(win, lut, slow, tbl, im.bpm, pos, sm.col_end[x], c, z, nb);
      const uint64_t ns = pack_state(pos, c, z);
      // The record is ALWAYS rewritten: a chain that merely converged inside this subsequence entered it in a different
      // state than the previous visitor; the chain that started further left is the better informed one.
      const bool same = sm.exitst[x] == ns;
      sm.exitst[x] = ns; sm.cnt[x] = nb;
      if (!same && sm.col_cont[x]) push_chain(cx, 0, pos, c, z, 2u, sg.g + 2, img_i);
    }
  }
  __syncthreads();
  if (sg.valid) {
    const uint32_t t = threadIdx.x > 0 && sm.col_cont[threadIdx.x - 1] ? 1u : 0u;       // visited by the left neighbour above
    cx.s_state[sg.g] = sm.exitst[threadIdx.x] | ((uint64_t)min(sm.cnt[threadIdx.x], 1023u) << 42) | ((uint64_t)t << 52);
  }
}

// H2a: the chain walk.  One thread per live chain; a visit decodes ONE subsequence from the chain's state, publishes the
// result with atomicMax on the packed record (priority in the top bits) and compares with the record it replaced:
//   * the old record has a higher priority -> a better informed chain (one that started further left) has already been here;
//     it covers everything this chain would do: the chain dies without having modified the record;
//   * equal states -> synchronised: everything to the right was decoded from the right entry state: the chain dies;
//   * otherwise the chain moves on to the next subsequence with priority + 1.
// The record of a subsequence therefore always belongs to the best informed visitor so far, whatever the order of arrival:
// no rounds, no grid-wide barriers (the previous version spent 34 stall cycles per issue in grid.sync()), and the result
// is deterministic because max() is.  The true chain of a unit (origin = its first subsequence) has the highest priority
// everywhere, is never overtaken and only stops where the record already equals the true state -- which was then written
// by a visitor that carries it on.  The walk is issued as three launches over compacted lists: two single-visit steps
// (30 % / 8 % of the subsequences still carry a live chain) keep the warps full, the last launch follows the few long
// chains to their end.  Every thread copies its subsequence (+ look-ahead) into a private shared-memory column
// ([word][thread]: bank = thread, conflict free); the tables are shared by the CTA.
constexpr int kTailThreads = 256;
constexpr int kTailColWords = 36;          // 128-byte subsequence + 16 bytes of look-ahead
// Bytes behind clean_off + L (L = a unit's clean length) that the Huffman passes may load: the sync-intra staging reads the
// look-ahead columns (256 bytes) behind a subsequence that starts below L; a column of the walk spans the subsequence + 16
// bytes; StreamWindow stays below kStreamReadBehind.  The clean buffer is allocated with this much minus kCleanPad of slack behind
// the last unit (every unit has at least kCleanPad bytes of pad of its own).
__host__ __device__ inline uint32_t clean_read_behind(int log2_sub) {
  const uint32_t sub = 1u << (log2_sub - 3), staged = sub + (uint32_t)look_ahead_cols(log2_sub) * sub;
  return staged > kStreamReadBehind ? staged : kStreamReadBehind;
}
struct ColSrc {
  uint32_t base;                           // shared-window address of column[0][threadIdx.x]
  __device__ __forceinline__ uint32_t load(uint32_t g) const { return lds_u32(base + g * (kTailThreads * 4u)); }
};

__device__ __forceinline__ void walk_chain(const HuffCtx &cx, const uint4 rec, int out_list, int max_visits, const uint32_t *s_lut,
                                           const HuffSlow *s_slow, int s_table_set, uint32_t *col, uint32_t *tblcol) {
  const int img_i = (int)rec.w;
  const JpegImage &im = cx.images[img_i];
  int64_t g = rec.z;
  const int j = (int)(g - im.subseq_begin);
  const int ui = im.unit_end - im.unit_begin == 1 ? im.unit_begin : last_at_most(cx.units, im.unit_begin, im.unit_end - 1, j, [](const JpegUnit &u) { return u.first_subseq; });
  const JpegUnit &u = cx.units[ui];
  const uint32_t clean_bits = cx.unit_clean_len[ui] * 8u;
  const uint32_t nsub_eff = (clean_bits + (1u << cx.log2_sub) - 1) >> cx.log2_sub;
  uint32_t jl = (uint32_t)(j - u.first_subseq);
#pragma unroll
  for (int b = 0; b < kMaxBlocksPerMcu; b++) tblcol[b * kTailThreads] = tbl_word(im, b);       // private column: bank = thread
  const bool shared_tables = im.table_set == s_table_set;
  uint32_t pos = rec.x, t = rec.y >> 16;
  int c = (int)(rec.y & 0xFF), z = (int)((rec.y >> 8) & 0xFF);
  const int sub_words = 1 << (cx.log2_sub - 5);
  for (int visit = 0;;) {
    uint32_t nb = 0;
    const uint32_t end = min((jl + 1) << cx.log2_sub, clean_bits);
    if (shared_tables && sub_words + 4 <= kTailColWords) {
      // private column: words [0, sub_words + 4) of this subsequence
      const uint4 *p4 = reinterpret_cast<const uint4 *>(cx.clean + u.clean_off + ((size_t)jl << (cx.log2_sub - 3)));
      for (int q = 0; q < sub_words / 4 + 1; q++) {
        const uint4 v = __ldg(p4 + q);
        col[(4 * q + 0) * kTailThreads] = v.x; col[(4 * q + 1) * kTailThreads] = v.y;
        col[(4 * q + 2) * kTailThreads] = v.z; col[(4 * q + 3) * kTailThreads] = v.w;
      }
      const ColSrc src{smem_u32(col)};
      const uint32_t rel = pos - (jl << cx.log2_sub);
      BitWindow<ColSrc> win;
      win.init(src, rel >> 5, rel & 31u);
      decode_span(win, SmemLut{smem_u32(s_lut)}, s_slow, SmemTbl<kTailThreads>{smem_u32(tblcol)}, im.bpm, pos, end, c, z, nb);
    } else {
      // another table set than the one this CTA keeps in shared memory (mixed batches), or an oversized subsequence: global path
      const GlobalSrc src{reinterpret_cast<const uint32_t *>(cx.clean + u.clean_off)};
      BitWindow<GlobalSrc> win;
      win.init(src, pos >> 5, pos & 31u);
      decode_span(win, GlobalLut{cx.tables[im.table_set].lut}, cx.tables[im.table_set].slow, SmemTbl<kTailThreads>{smem_u32(tblcol)},
                  im.bpm, pos, end, c, z, nb);
    }
    const uint64_t ns = pack_state(pos, c, z, nb, t);
    const uint64_t old = atomicMax(reinterpret_cast<unsigned long long *>(cx.s_state + g), (unsigned long long)ns);
    if ((uint32_t)(old >> 52) >= t) break;                    // overtaken by a better informed chain
    if (((old ^ ns) & kStateMask) == 0) break;                // synchronised
    if (jl + 1 >= nsub_eff) break;                            // end of the unit
    if (t >= kMaxChainLen) { cx.chain_cut[img_i] = 1u; break; }   // the priority is full: H2b finishes the unit (resync_unit)
    g++; jl++; t++;
    if (++visit >= max_visits) { push_chain(cx, out_list, pos, c, z, t, g, img_i); break; }
  }
}

__global__ void __launch_bounds__(kTailThreads) huff_sync_walk_kernel(HuffCtx cx, int in_list, int out_list, int max_visits) {
  extern __shared__ __align__(16) uint32_t tsm[];
  const uint32_t n = cx.chain_count[in_list];
  if (blockIdx.x * blockDim.x >= n) return;                  // launched for an upper bound of the list length
  uint32_t *s_lut = tsm;
  HuffSlow *s_slow = reinterpret_cast<HuffSlow *>(s_lut + kLutWords);
  uint32_t *col = reinterpret_cast<uint32_t *>(s_slow + 4) + threadIdx.x;
  uint32_t *tblcol = reinterpret_cast<uint32_t *>(s_slow + 4) + kTailColWords * kTailThreads + threadIdx.x;
  const int s_table_set = cx.images[0].table_set;
  {
    const uint4 *src = reinterpret_cast<const uint4 *>(cx.tables[s_table_set].lut);
    uint4 *dst = reinterpret_cast<uint4 *>(s_lut);
    for (int i = threadIdx.x; i < kLutWords / 4; i += blockDim.x) dst[i] = __ldg(src + i);
    const uint32_t *ssrc = reinterpret_cast<const uint32_t *>(cx.tables[s_table_set].slow);
    uint32_t *sdst = reinterpret_cast<uint32_t *>(s_slow);
    for (int i = threadIdx.x; i < (int)(4 * sizeof(HuffSlow) / 4); i += blockDim.x) sdst[i] = __ldg(ssrc + i);
  }
  __syncthreads();
  const uint32_t gtid = blockIdx.x * blockDim.x + threadIdx.x, gsize = gridDim.x * blockDim.x;
  for (uint32_t i = gtid; i < n; i += gsize) walk_chain(cx, cx.chains[in_list][i], out_list, max_visits, s_lut, s_slow, s_table_set, col, tblcol);
}

// The per-block table offsets of an image, read from its descriptor (resync_unit: one thread, no shared copy).
struct ImageTbl {
  const JpegImage *im;
  __device__ __forceinline__ uint32_t load(int c) const { return tbl_word(*im, c); }
};

// A unit whose true chain may have stopped at kMaxChainLen (walk_chain): its records up to subsequence kMaxChainLen - 1 are right (a
// chain only stops at t >= kMaxChainLen, so no stop can reach further left); the records behind are re-decoded sequentially from there.
// Not inlined, and given the few fields it reads by value (a reference to the kernel's HuffCtx would put the context on the stack):
// the scan keeps its registers and no spill of this rare path reaches it.
__device__ __noinline__ void resync_unit(const JpegImage *__restrict__ imp, const JpegUnit *__restrict__ units,
                                         const uint32_t *__restrict__ unit_clean_len, const TableSet *__restrict__ tables,
                                         const uint8_t *__restrict__ clean, uint64_t *__restrict__ s_state, int log2_sub, int ui) {
  const JpegImage &im = *imp;
  const JpegUnit &u = units[ui];
  const uint32_t clean_bits = unit_clean_len[ui] * 8u;
  const uint32_t nsub_eff = (clean_bits + (1u << log2_sub) - 1) >> log2_sub;
  if (nsub_eff <= kMaxChainLen) return;
  const int64_t g0 = (int64_t)im.subseq_begin + u.first_subseq;
  const uint64_t st = s_state[g0 + kMaxChainLen - 1];
  uint32_t pos = (uint32_t)st;
  int c = (int)((st >> 32) & 15u), z = (int)((st >> 36) & 63u);
  BitWindow<GlobalSrc> win;
  win.init(GlobalSrc{reinterpret_cast<const uint32_t *>(clean + u.clean_off)}, pos >> 5, pos & 31u);
  const TableSet &ts = tables[im.table_set];
  for (uint32_t jl = kMaxChainLen; jl < nsub_eff; jl++) {
    uint32_t nb = 0;
    decode_span(win, GlobalLut{ts.lut}, ts.slow, ImageTbl{&im}, im.bpm, pos, min((jl + 1) << log2_sub, clean_bits), c, z, nb);
    s_state[g0 + jl] = pack_state(pos, c, z, nb);
  }
}

// H2b: one CTA per image: per-unit exclusive scan of the block counts (in place), status check.
// Two 1024-thread CTAs per SM (32 registers).  The bound binds resync_unit too: it spills in its own frame, and the scan saves a few
// registers around the call, inside the flagged branch only; the scan loop itself has no local-memory access.
__global__ void __launch_bounds__(1024, 2) huff_scan_kernel(HuffCtx cx) {
  __shared__ uint32_t warp_tot[32];
  __shared__ uint32_t carry;
  const JpegImage &im = cx.images[blockIdx.x];
  const uint32_t sub_bits = 1u << cx.log2_sub;
  const int unit_begin = im.unit_begin, unit_end = im.unit_end;    // read first: these loads and the flag's are in flight together
  if (cx.chain_cut[blockIdx.x]) {                            // rare: only streams built to defeat the synchronisation get here
    for (int ui = unit_begin + (int)threadIdx.x; ui < unit_end; ui += blockDim.x) 
      resync_unit(&im, cx.units, cx.unit_clean_len, cx.tables, cx.clean, cx.s_state, cx.log2_sub, ui);
    __syncthreads();
  }
  for (int ui = unit_begin; ui < unit_end; ui++) {
    const JpegUnit &u = cx.units[ui];
    const uint32_t clean_bits = cx.unit_clean_len[ui] * 8u;
    const uint32_t nsub_eff = (clean_bits + sub_bits - 1) >> cx.log2_sub;
    const int64_t g0 = (int64_t)im.subseq_begin + u.first_subseq;
    __syncthreads();
    if (threadIdx.x == 0) carry = 0;
    __syncthreads();
    for (uint32_t base = 0; base < nsub_eff; base += blockDim.x) {
      const uint32_t i = base + threadIdx.x;
      const uint32_t v = i < nsub_eff ? state_count(cx.s_state[g0 + i]) : 0u;
      uint32_t incl = v;
      for (int o = 1; o < 32; o <<= 1) { uint32_t x = __shfl_up_sync(0xffffffffu, incl, o); if ((threadIdx.x & 31) >= o) incl += x; }
      if ((threadIdx.x & 31) == 31) warp_tot[threadIdx.x >> 5] = incl;
      __syncthreads();
      uint32_t woff = 0, tot = 0;
      for (int w = 0; w < (int)(blockDim.x >> 5); w++) { if (w < (int)(threadIdx.x >> 5)) woff += warp_tot[w]; tot += warp_tot[w]; }
      if (i < nsub_eff) cx.s_n[g0 + i] = carry + woff + incl - v;
      __syncthreads();
      if (threadIdx.x == 0) carry += tot;
      __syncthreads();
    }
    // trailing pad bits may decode into a few extra symbols, so only a SHORT count is an error
    if (threadIdx.x == 0) {
      if ((int64_t)carry * 64 < u.nslots) cx.status[blockIdx.x] = 1;
      cx.unit_nblk[ui] = (uint32_t)min((int64_t)carry, u.nslots >> 6);
    }
  }
}

// H3: final pass -- every subsequence is decoded from its now-correct entry state and writes coefficients.
//
// A block belongs to the thread in whose subsequence it STARTS: a thread skips the tail of the block that is open at its
// entry and runs past its own end until its last block is complete (its window simply reads on into the following
// subsequences).  Every block therefore has exactly one writer, which assembles it in a private 128-byte shared-memory buffer
// (16-byte chunk k of lane l at l * 8 + (k ^ (l & 7))) and the warp writes each finished block to HBM as ONE coalesced 128-byte
// line: no memset of the coefficient arena, no 2-byte read-modify-write traffic, ~12x fewer store wavefronts than a per-symbol
// scatter.  A flush step moves four blocks, one per quarter-warp, each lane a 16-byte chunk: the swizzle puts the 8 chunks a
// quarter reads in 8 different bank groups, and spreads the per-symbol 16-bit scatter of lanes at the same position over them.
//
// The loop is a chain of dependent fixed-latency instructions (its stalls are fixed-latency waits and short scoreboards):
// throughput scales with resident warps.  The pass therefore runs its own block shape -- kWriteThreads subsequences per CTA,
// and the stream read from global memory (StreamWindow), so that shared memory holds only the tables and the block buffers:
// 20.1 KB + 128 B per thread.
//
// Every instruction of the symbol loop runs on every trip, so the loop holds no per-phase tests.  A thread passes through three
// phases -- skip the tail of the block open at its entry, decode its own blocks while symbols start inside its subsequence, finish
// the last one behind it -- and each is a value, not a branch: the block index carries kSkipBlock while the entry's open block is
// decoded (its coefficients go to the lane's buffer like any others and the flush clears them without writing the line), and the
// decode limit `lim` is hard_end inside a block and, where a block is about to start, the subsequence end or 0 (blk_limit reached).
// The DC difference is stored into the buffer at natural position 0 like a coefficient, and the flush moves it to the DC array.
constexpr int kWriteThreads = 384;
constexpr int kWriteCtasPerSm = 3;       // 3 x (68.1 KB + 1 KB reserved) of the 228 KB per SM
constexpr uint32_t kSkipBlock = 1u << 31;   // block indices stay below 2^31: the arena would hold 256 GB of coefficients
struct WriteSmem {
  uint32_t *lut, *tbl, *blkbuf; uint8_t *zig;
};
__host__ __device__ inline size_t write_smem_bytes() { return kLutWords * 4 + 16 * 4 /*tbl*/ + 64 /*zig*/ + (size_t)kWriteThreads * 128; }
__device__ __forceinline__ WriteSmem carve_write_smem(uint32_t *base) {
  WriteSmem s;
  s.lut = base;
  s.tbl = base + kLutWords;
  s.zig = reinterpret_cast<uint8_t *>(s.tbl + 16);
  s.blkbuf = reinterpret_cast<uint32_t *>(s.zig + 64);                       // 16-byte aligned: every size above is a multiple of 16
  return s;
}

__global__ void __launch_bounds__(kWriteThreads, kWriteCtasPerSm) huff_write_kernel(HuffCtx cx) {
  extern __shared__ __align__(16) uint32_t hsm[];
  const WriteSmem sm = carve_write_smem(hsm);
  const JpegImage &im = cx.images[cx.wblock_image[blockIdx.x]];
  // ---- prologue: tables, per-thread subsequence geometry
  {
    const uint4 *src = reinterpret_cast<const uint4 *>(cx.tables[im.table_set].lut);
    uint4 *dst = reinterpret_cast<uint4 *>(sm.lut);
    for (int i = threadIdx.x; i < kLutWords / 4; i += blockDim.x) dst[i] = __ldg(src + i);
    // table word of block b of the MCU, with the next block's index in the free bits [15:12] (DC offsets are < 1024): the loop
    // follows the MCU through this word alone
    if (threadIdx.x < kMaxBlocksPerMcu) {
      const int b = threadIdx.x, next = b + 1 == im.bpm ? 0 : b + 1;
      sm.tbl[b] = tbl_word(im, b) | ((uint32_t)next << 12);
    }
    // byte offset of each zig-zag position in a block buffer (2 x natural position), before the lane's swizzle
    if (threadIdx.x < 64) sm.zig[threadIdx.x] = (uint8_t)(2 * c_zigzag[threadIdx.x]);
  }
  SubGeom sg;
  {
    const int j = (blockIdx.x - im.wblock_begin) * kWriteThreads + threadIdx.x;     // image-local subsequence
    sg.valid = j < im.nsub;
    sg.ui = 0; sg.jl = 0; sg.nsub_eff = 0; sg.clean_bits = 0;
    sg.g = (int64_t)im.subseq_begin + j;
    if (sg.valid) {
      sg.ui = im.unit_end - im.unit_begin == 1 ? im.unit_begin : last_at_most(cx.units, im.unit_begin, im.unit_end - 1, j, [](const JpegUnit &u) { return u.first_subseq; });
      const JpegUnit &u = cx.units[sg.ui];
      sg.clean_bits = cx.unit_clean_len[sg.ui] * 8u;
      sg.nsub_eff = (sg.clean_bits + (1u << cx.log2_sub) - 1) >> cx.log2_sub;
      sg.jl = (uint32_t)(j - u.first_subseq);
      sg.valid = sg.jl < sg.nsub_eff;
    }
  }
  // long codes (~1 % of the symbols) are looked up in global memory (L1-resident, one load with the direct table): a shared-memory
  // copy cost 5.7 KB per CTA and made the compiler rebuild the generic address of the copy inside the symbol loop
  const HuffSlow *slow = cx.tables[im.table_set].slow;
  const uint32_t lane = threadIdx.x & 31u;
  // shared-window addresses (plain integers inside the loop, see lds_u32)
  const uint32_t a_lut = smem_u32(sm.lut), a_tbl = smem_u32(sm.tbl), a_zig = smem_u32(sm.zig);
  const uint32_t a_wbuf = smem_u32(sm.blkbuf) + (threadIdx.x & ~31u) * 128u;     // this warp's 32 block buffers (128 bytes each)
  const uint32_t a_mybuf = a_wbuf + lane * 128u;
#pragma unroll
  for (int j = 0; j < 32; j++) sts_u32(a_mybuf + 4u * j, 0u);
  __syncwarp();
  uint32_t pos = 0, end = 0, hard_end = 0, blk = 0, blk_limit = 0, lim = 0;
  int c = 0, z = 0;
  if (sg.valid) {
    const JpegUnit &u = cx.units[sg.ui];
    if (sg.jl > 0) {
      const uint64_t prev = cx.s_state[sg.g - 1];
      pos = (uint32_t)prev; c = (int)((prev >> 32) & 15u); z = (int)((prev >> 36) & 63u);
    }
    end = min((sg.jl + 1) << cx.log2_sub, sg.clean_bits);
    hard_end = sg.clean_bits;
    const uint32_t ublk = (uint32_t)(u.slot_base >> 6);
    const uint32_t blk0 = ublk + cx.s_n[sg.g];
    blk_limit = ublk + (uint32_t)(u.nslots >> 6);
    blk = blk0 | (z != 0 ? kSkipBlock : 0u);                  // z != 0: the entry is inside a block of the previous thread
    lim = blk0 < blk_limit ? end : 0u;                        // pad bits behind the last block of a unit are not symbols
  }
  StreamWindow win;
  win.clear();
  if (pos < lim) win.init(cx.clean + cx.units[sg.ui].clean_off, pos);
  __syncthreads();                                            // the tables; the window's first loads are in flight meanwhile
  // this lane's chunk of coefficient line 0, and DC 0, as plain 64-bit global addresses: the flush then forms each store address
  // with one multiply-add (as pointers, the compiler rebuilt them from the context inside the flush loop)
  const uint32_t chunk = lane & 7u, quarter = lane >> 3;
  const uint64_t a_line = (uint64_t)__cvta_generic_to_global(cx.coef + im.coef_off) + 16u * chunk;
  const uint64_t a_dc = (uint64_t)__cvta_generic_to_global(cx.dc + im.coef_off / 64);
  const uint32_t swz = 16u * chunk;                           // the lane's buffer swizzle, applied to a byte offset
  uint32_t tb12 = lds_u32(a_tbl + 4u * c);
  for (uint32_t it = 1; __any_sync(0xffffffffu, pos < lim); it++) {
    bool endb = false;
    uint32_t next_blk = blk;
    if (it & 1u) win.top_up();                                // warp-uniform, see StreamWindow
    if (pos < lim) {
      const uint32_t thr = pair_threshold(z, pos, hard_end);
      const uint32_t e_ac = lds_u32(a_lut + 4u * ((tb12 >> 16) + (win.hi >> (32 - kAcLutBits))));
      const bool is_dc = z == 0;
      uint32_t e = e_ac;
      if (is_dc) e = lds_u32(a_lut + 4u * ((tb12 & 0xFFFu) + (win.hi >> (32 - kDcLutBits))));
      if (__builtin_expect(e == 0, 0)) e = slow_lookup(slow, is_dc ? (tb12 & 0xFFFu) : (tb12 >> 16), win.hi, is_dc);
      // a pair needs the block open after its first symbol (z + adv1 < 64): blk and blk_limit are the same for both symbols.
      // Its second symbol starts before hard_end, so `lim` would have admitted it.
      const uint32_t st = huff_step(e, thr), one = e >> 16;
      const uint32_t tb = step_bits(st), adv = step_adv(st), s = step_size(st);
      const uint32_t tb1 = step_bits(one), s1 = step_size(one);
      if (tb != tb1 && s1) {                                  // a pair whose first symbol has a value: it lands before coefficient 63
        const uint32_t off = lds_u8(a_zig + (uint32_t)z + step_adv(one) - 1u);
        sts_u16(a_mybuf + (off ^ swz), (uint32_t)huff_extend(win.hi, tb1, s1));
      }
      if (s) {                                                // runs past coefficient 63 land on 63; a DC difference on 0
        const uint32_t off = lds_u8(a_zig + min((uint32_t)z + adv - 1u, 63u));
        sts_u16(a_mybuf + (off ^ swz), (uint32_t)huff_extend(win.hi, tb, s));
      }
      win.consume(st);
      pos += tb;
      z += (int)adv;
      if (is_dc) lim = hard_end;                              // a block once begun is decoded to its end
      endb = z >= 64;                                         // block finished (EOB, 64th coefficient, or garbage overrun)
      if (endb) {
        z = 0;
        tb12 = lds_u32(a_tbl + ((tb12 >> 10) & 0x3Cu));
        next_blk = (blk & ~kSkipBlock) + 1u;
        // the next block is ours if it starts inside the subsequence and inside the unit
        lim = next_blk < blk_limit ? end : 0u;
      }
    }
    // ---- flush the finished blocks of this warp, four per step: quarter q takes the q-th lowest one, one coalesced line each (the
    // entry's open block only clears its buffer)
    uint32_t m = __ballot_sync(0xffffffffu, endb);
    while (m) {
      const uint32_t m1 = m & (m - 1u), m2 = m1 & (m1 - 1u), m3 = m2 & (m2 - 1u);
      const uint32_t mq = quarter == 0 ? m : quarter == 1 ? m1 : quarter == 2 ? m2 : m3;
      m = m3 & (m3 - 1u);
      const uint32_t L = (__ffs(mq) - 1u) & 31u;
      const uint32_t fb = __shfl_sync(0xffffffffu, blk, L);
      if (mq) {
        const uint32_t a_src = a_wbuf + L * 128u + 16u * (chunk ^ (L & 7u));
        uint4 w = lds_v4(a_src);
        sts_v4(a_src, make_uint4(0u, 0u, 0u, 0u));
        if (fb < kSkipBlock) {
          if (chunk == 0) {                                   // natural position 0: the DC difference goes to the DC array
            stg_u16(a_dc + 2ull * fb, w.x);                   // every block has a DC term: the array needs no memset
            w.x &= 0xFFFF0000u;
          }
          stg_v4(a_line + 128ull * fb, w);
        }
      }
    }
    blk = next_blk;
    __syncwarp();
  }
}

// ============================================================================================
// D1: DC prediction on the compact per-block DC array (one int16 per block, MCU order).  One CTA per image; the blocks
// of each component are visited in scan order; restart intervals reset the predictor.
__global__ void __launch_bounds__(1024) dc_scan_kernel(const JpegImage *__restrict__ images, int16_t *__restrict__ dc_arena) {
  __shared__ int warp_tot[32];
  const JpegImage &im = images[blockIdx.x];
  int16_t *dc = dc_arena + im.coef_off / 64;
  const int nmcu = im.mcux * im.mcuy;
  const int ri = im.restart_interval > 0 ? im.restart_interval : nmcu;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  for (int comp = 0; comp < im.ncomp; comp++) {
    int nb = 0, bidx[kMaxBlocksPerMcu];
    for (int b = 0; b < im.bpm; b++) if (im.blk_comp[b] == comp) bidx[nb++] = b;
    const int total = nmcu * nb;
    if (ri >= nmcu) {
      // every warp owns a contiguous run of the component's blocks: pass 1 sums it (coalesced), the 32 run totals are
      // scanned once, pass 2 re-reads the run and writes the running predictor (two barriers per component)
      const int per = ((total + 31) / 32 + 31) / 32 * 32;
      const int i0 = wid * per, i1 = min(total, i0 + per);
      int sum = 0;
      for (int i = i0 + lane; i < i1; i += 32) sum += dc[(i / nb) * im.bpm + bidx[i % nb]];
      for (int o = 16; o; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
      __syncthreads();                                        // warp_tot of the previous component has been consumed
      if (lane == 0) warp_tot[wid] = sum;
      __syncthreads();
      int carry = 0;
      for (int w = 0; w < wid; w++) carry += warp_tot[w];
      for (int base = i0; base < i1; base += 32) {
        const int i = base + lane;
        int idx = 0, v = 0;
        if (i < i1) { idx = (i / nb) * im.bpm + bidx[i % nb]; v = dc[idx]; }
        int incl = v;
        for (int o = 1; o < 32; o <<= 1) { const int x = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += x; }
        if (i < i1) dc[idx] = (int16_t)(carry + incl);
        carry += __shfl_sync(0xffffffffu, incl, 31);
      }
    } else {
      const int nseg = (nmcu + ri - 1) / ri;
      for (int sgi = threadIdx.x; sgi < nseg; sgi += blockDim.x) {
        int pred = 0;
        const int m1 = min(nmcu, (sgi + 1) * ri);
        for (int m = sgi * ri; m < m1; m++)
          for (int k = 0; k < nb; k++) {
            const int idx = m * im.bpm + bidx[k];
            pred += dc[idx];
            dc[idx] = (int16_t)pred;
          }
      }
    }
  }
}

// Truncated / corrupt entropy-coded data: libjpeg stops decoding when the data runs out and leaves the remaining MCUs as all-zero
// coefficient blocks (jdhuff.c: insufficient_data -> the blocks keep the zeros of jzero_far, DC included), which decode to mid-gray.
// The blocks behind the last decoded one of every short unit get exactly that: zero coefficients and an ABSOLUTE DC of zero (this
// runs after the DC prediction).  One CTA per image; returns at once for intact images.
__global__ void __launch_bounds__(256) truncation_fixup_kernel(HuffCtx cx) {
  if (cx.status[blockIdx.x] == 0) return;
  const JpegImage &im = cx.images[blockIdx.x];
  uint4 *coef4 = reinterpret_cast<uint4 *>(cx.coef + im.coef_off);
  int16_t *dcv = cx.dc + im.coef_off / 64;
  for (int ui = im.unit_begin; ui < im.unit_end; ui++) {
    const JpegUnit &u = cx.units[ui];
    const int64_t b0 = (u.slot_base >> 6) + cx.unit_nblk[ui], b1 = (u.slot_base + u.nslots) >> 6;
    for (int64_t q = b0 * 8 + threadIdx.x; q < b1 * 8; q += blockDim.x) coef4[q] = make_uint4(0u, 0u, 0u, 0u);
    for (int64_t b = b0 + threadIdx.x; b < b1; b += blockDim.x) dcv[b] = 0;
  }
}

// ============================================================================================
// I1: dequantisation + islow IDCT (libjpeg jidctint: CONST_BITS 13, PASS1_BITS 2).  One thread per 8x8 block.  The arithmetic, and
// its relation to libjpeg-turbo's SIMD kernels, is in jpeg_idct_core.h.

// Dequantises and transforms block `gb` (index in MCU order over the arenas) with quantisation table q; rows[y] = the 8 output samples
// of row y, byte k = column k.
__device__ __forceinline__ void idct_block(const int16_t *__restrict__ coef_arena, const int16_t *__restrict__ dc_arena, int64_t gb,
                                           const uint16_t *__restrict__ q, uint2 *rows) {
  const int4 *src = reinterpret_cast<const int4 *>(coef_arena + gb * 64);
  const uint4 *q4 = reinterpret_cast<const uint4 *>(q);      // 8 x u16 per row in ONE 16-byte load (the table is 16-byte aligned)
  int w[32];
  uint32_t qw[32], rw[16];
#pragma unroll
  for (int r = 0; r < 8; r++) {
    const int4 v = __ldg(src + r);
    const uint4 qv = __ldg(q4 + r);
    w[4 * r] = v.x; w[4 * r + 1] = v.y; w[4 * r + 2] = v.z; w[4 * r + 3] = v.w;
    qw[4 * r] = qv.x; qw[4 * r + 1] = qv.y; qw[4 * r + 2] = qv.z; qw[4 * r + 3] = qv.w;
  }
  idct_block_words(w, qw, __ldg(dc_arena + gb), rw);
#pragma unroll
  for (int y = 0; y < 8; y++) rows[y] = make_uint2(rw[2 * y], rw[2 * y + 1]);
}

// Work list: the blocks of the MCUs [mcu_x0, +mcu_nx) x [mcu_y0, +mcu_ny) of every image (all MCUs unless a region of interest
// was requested) that idct_color_420 does not decode; first_work[i] = index of image i's first work block.
__global__ void __launch_bounds__(128) idct_kernel(const JpegImage *__restrict__ images, const int64_t *__restrict__ first_work, int nimages,
                                                   int64_t total_work, const int16_t *__restrict__ coef_arena,
                                                   const int16_t *__restrict__ dc_arena, const QuantSet *__restrict__ quants,
                                                   uint8_t *__restrict__ planes) {
  // contiguous range of blocks per CTA: the image is searched once and then only advanced
  __shared__ int s_first;
  const int64_t per_cta = ((total_work + gridDim.x - 1) / gridDim.x + 127) / 128 * 128;
  const int64_t b0 = (int64_t)blockIdx.x * per_cta, b1 = min(total_work, b0 + per_cta);
  if (b0 >= b1) return;
  if (threadIdx.x == 0) s_first = last_at_most(first_work, 0, nimages - 1, b0);
  __syncthreads();
  int ii = s_first;
  for (int64_t wb = b0 + threadIdx.x; wb < b1; wb += blockDim.x) {
    while (ii + 1 < nimages && first_work[ii + 1] <= wb) ii++;
    const JpegImage &im = images[ii];
    const int64_t lw = wb - first_work[ii];            // block index inside the window, MCU-row major
    // per-image counts fit 32 bits (the plan rejects images above 2^31 pixels): 32-bit divisions, a 64-bit one costs ~100 instructions
    const int wm = (int)((uint32_t)lw / (uint32_t)im.bpm), b = (int)((uint32_t)lw - (uint32_t)wm * (uint32_t)im.bpm);
    const int mx = im.mcu_x0 + wm % im.mcu_nx, my = im.mcu_y0 + wm / im.mcu_nx;
    const int64_t gb = im.coef_off / 64 + ((int64_t)my * im.mcux + mx) * im.bpm + b;     // block index in scan (MCU) order
    const int comp = im.blk_comp[b];
    const int bx = mx * im.hs[comp] + im.blk_x[b], by = my * im.vs[comp] + im.blk_y[b];
    uint2 rows[8];
    idct_block(coef_arena, dc_arena, gb, quants[im.quant_set].q[im.tq[comp]], rows);
    uint8_t *dst = planes + im.plane_off[comp] + ((int64_t)by * 8) * im.plane_w[comp] + bx * 8;
#pragma unroll
    for (int y = 0; y < 8; y++) *reinterpret_cast<uint2 *>(dst + (int64_t)y * im.plane_w[comp]) = rows[y];
  }
}

// ============================================================================================
// C1: chroma upsampling + colour conversion.  One thread per 4 output pixels of a row.
//
// libjpeg's fancy upsampling edge rules (jdsample.c), shared by every path below and by idct_color_420:
//   * vertical (v2): output row y blends chroma row y >> 1 (near, x 3) with the row above (y even) or below (y odd) (far), the far row
//     clamped to [0, dh - 1];
//   * horizontal h2v2: from the vertical sums cs = 3 * near + far, the outputs 2i and 2i + 1 of chroma column i are
//     (3 cs[i] + cs[i - 1] + 8) >> 4 and (3 cs[i] + cs[i + 1] + 7) >> 4, where the missing neighbour of the first column (i == 0) and of the
//     last one (i >= dw - 1, dw = the image's chroma width, not the padded plane's) is the column itself.
__device__ __forceinline__ int fancy_far_row(int y, int dh) { return min(max((y & 1) ? (y >> 1) + 1 : (y >> 1) - 1, 0), dh - 1); }
__device__ __forceinline__ int fancy_h2v2_even(int prev, int cur, int i) { return (cur * 3 + (i == 0 ? cur : prev) + 8) >> 4; }
__device__ __forceinline__ int fancy_h2v2_odd(int cur, int next, int i, int dw) { return (cur * 3 + (i >= dw - 1 ? cur : next) + 7) >> 4; }

__device__ __forceinline__ int up_sample(const uint8_t *__restrict__ pl, int pw, int dw, int dh, int hexp, int vexp, int fancy,
                                         int x, int y) {
  if (hexp == 1 && vexp == 1) return pl[(int64_t)y * pw + x];
  if (fancy && hexp == 2 && vexp == 1 && dw > 2) {                 // h2v1 fancy (jdsample.c h2v1_fancy_upsample)
    const uint8_t *r = pl + (int64_t)y * pw;
    const int i = x >> 1;
    if (x & 1) return i == dw - 1 ? r[i] : (r[i] * 3 + r[i + 1] + 2) >> 2;
    return i == 0 ? r[i] : (r[i] * 3 + r[i - 1] + 1) >> 2;
  }
  if (fancy && hexp == 2 && vexp == 2 && dw > 2) {                 // h2v2 fancy (triangle)
    const uint8_t *r0 = pl + (int64_t)(y >> 1) * pw, *r1 = pl + (int64_t)fancy_far_row(y, dh) * pw;
    const int i = x >> 1;
    const int cur = r0[i] * 3 + r1[i];
    if (x & 1) return fancy_h2v2_odd(cur, i >= dw - 1 ? 0 : r0[i + 1] * 3 + r1[i + 1], i, dw);
    return fancy_h2v2_even(i == 0 ? 0 : r0[i - 1] * 3 + r1[i - 1], cur, i);
  }
  if (fancy && hexp == 1 && vexp == 2) {                           // h1v2 fancy
    return (pl[(int64_t)(y >> 1) * pw + x] * 3 + pl[(int64_t)fancy_far_row(y, dh) * pw + x] + ((y & 1) ? 2 : 1)) >> 2;
  }
  return pl[(int64_t)(y / vexp) * pw + x / hexp];                  // box replication
}

__device__ __forceinline__ int clamp255(int v) { return min(max(v, 0), 255); }

__global__ void __launch_bounds__(256) color_kernel(const JpegImage *__restrict__ images, const int64_t *__restrict__ first_quad,
                                                    int nimages, int64_t total_quads, const uint8_t *__restrict__ planes) {
  for (int64_t gq = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; gq < total_quads; gq += (int64_t)gridDim.x * blockDim.x) {
    const int i = last_at_most(first_quad, 0, nimages - 1, gq);
    const JpegImage &im = images[i];
    if (im.fast_color) continue;
    const int64_t q = gq - first_quad[i];
    const int qpr = (im.win_w + 3) >> 2;
    const uint32_t qy = (uint32_t)q / (uint32_t)qpr;
    const int y = im.win_y0 + (int)qy, x0 = im.win_x0 + ((int)((uint32_t)q - qy * (uint32_t)qpr) << 2);
    const int W = im.width, H = im.height;
    const int nout = im.out_type == DALIB200_GRAY ? 1 : 3;
    uint8_t px[12];
    const int nx = min(4, im.win_x0 + im.win_w - x0);
    for (int k = 0; k < nx; k++) {
      const int x = x0 + k;
      int v[4];
      for (int c = 0; c < im.ncomp; c++) {
        const int hexp = im.hmax / im.hs[c], vexp = im.vmax / im.vs[c];
        const int dw = (W * im.hs[c] + im.hmax - 1) / im.hmax, dh = (H * im.vs[c] + im.vmax - 1) / im.vmax;
        v[c] = up_sample(planes + im.plane_off[c], im.plane_w[c], dw, dh, hexp, vexp, im.fancy, x, y);
      }
      const int cm = im.color;
      int r, g, b, yy, cb, cr;
      if (cm == kColorGray) { r = g = b = yy = v[0]; cb = cr = 128; }
      else if (cm == kColorRGB || cm == kColorCMYK) { r = v[0]; g = v[1]; b = v[2]; yy = cb = cr = 0; }
      else {
        yy = v[0]; cb = v[1]; cr = v[2];
        const int cbm = cb - 128, crm = cr - 128;                   // jdcolor.c, SCALEBITS = 16
        r = clamp255(yy + ((91881 * crm + 32768) >> 16));
        g = clamp255(yy + ((-22554 * cbm + 32768 - 46802 * crm) >> 16));
        b = clamp255(yy + ((116130 * cbm + 32768) >> 16));
      }
      if (cm >= kColorCMYK) {
        // C, M, Y: the samples (CMYK) or 255 - the YCbCr->RGB above (YCCK, jdcolor.c ycck_cmyk_convert); then OpenCV's
        // icvCvt_CMYK2BGR on these (inverted, Adobe-style) samples: R = K - ((255 - C) * K >> 8), and so on
        const int kk = v[3];
        const int ic = cm == kColorCMYK ? 255 - r : r, imy = cm == kColorCMYK ? 255 - g : g, iy = cm == kColorCMYK ? 255 - b : b;
        r = kk - ((ic * kk) >> 8); g = kk - ((imy * kk) >> 8); b = kk - ((iy * kk) >> 8);
      }
      if (im.out_type == DALIB200_RGB) { px[3 * k] = r; px[3 * k + 1] = g; px[3 * k + 2] = b; }
      else if (im.out_type == DALIB200_BGR) { px[3 * k] = b; px[3 * k + 1] = g; px[3 * k + 2] = r; }
      else if (im.out_type == DALIB200_YCbCr) { px[3 * k] = yy; px[3 * k + 1] = cb; px[3 * k + 2] = cr; }
      else if (cm == kColorRGB) px[k] = RgbJpegGray(r, g, b);
      else if (cm >= kColorCMYK) px[k] = (b * 1868 + g * 9617 + r * 4899 + 8192) >> 14;      // OpenCV icvCvt_CMYK2Gray
      else px[k] = yy;
    }
    uint8_t *o = im.out + ((int64_t)(y - im.win_y0) * im.win_w + (x0 - im.win_x0)) * nout;
    const int nb = nx * nout;
    if (nb == 12 && (reinterpret_cast<uintptr_t>(o) & 3) == 0) {
      uint32_t *o4 = reinterpret_cast<uint32_t *>(o);
      o4[0] = px[0] | (px[1] << 8) | (px[2] << 16) | ((uint32_t)px[3] << 24);
      o4[1] = px[4] | (px[5] << 8) | (px[6] << 16) | ((uint32_t)px[7] << 24);
      o4[2] = px[8] | (px[9] << 8) | (px[10] << 16) | ((uint32_t)px[11] << 24);
    } else {
      for (int k = 0; k < nb; k++) o[k] = px[k];
    }
  }
}


// ---------------------------------------------------------------------------------------------
// C1 fast path: 3-component YCbCr -> RGB/BGR.  One CTA = one output row segment of 1024 pixels of one image,
// one thread = 8 consecutive pixels: one 8-byte luma load, word loads of the two chroma rows, 24 output bytes.
constexpr int kColorSeg = 1024;

template <int HEXP, int VEXP>
__device__ __forceinline__ void chroma8(const uint8_t *__restrict__ pl, int pw, int dw, int dh, int fancy, int x0, int y, int *v) {
  if (HEXP == 1 && VEXP == 1) {
    const uint2 w = *reinterpret_cast<const uint2 *>(pl + (int64_t)y * pw + x0);
#pragma unroll
    for (int k = 0; k < 4; k++) { v[k] = (w.x >> (8 * k)) & 0xFF; v[4 + k] = (w.y >> (8 * k)) & 0xFF; }
    return;
  }
  if (HEXP == 2) {
    const int i0 = x0 >> 1;                       // 4 chroma samples i0..i0+3 (+ one neighbour each side)
    const bool fy = fancy && dw > 2;
    int cs[6];
    if (VEXP == 2) {
      const uint8_t *r0 = pl + (int64_t)(y >> 1) * pw, *r1 = pl + (int64_t)fancy_far_row(y, dh) * pw;
      const uint32_t a = *reinterpret_cast<const uint32_t *>(r0 + i0), b = *reinterpret_cast<const uint32_t *>(r1 + i0);
      if (!fy) {
#pragma unroll
        for (int k = 0; k < 4; k++) v[2 * k] = v[2 * k + 1] = (a >> (8 * k)) & 0xFF;
        return;
      }
#pragma unroll
      for (int k = 0; k < 4; k++) cs[1 + k] = 3 * (int)((a >> (8 * k)) & 0xFF) + (int)((b >> (8 * k)) & 0xFF);
      cs[0] = i0 > 0 ? 3 * r0[i0 - 1] + r1[i0 - 1] : 0;
      cs[5] = i0 + 4 < dw ? 3 * r0[i0 + 4] + r1[i0 + 4] : 0;
#pragma unroll
      for (int k = 0; k < 4; k++) {
        v[2 * k] = fancy_h2v2_even(cs[k], cs[1 + k], i0 + k);
        v[2 * k + 1] = fancy_h2v2_odd(cs[1 + k], cs[2 + k], i0 + k, dw);
      }
    } else {
      const uint8_t *r = pl + (int64_t)y * pw;
      const uint32_t a = *reinterpret_cast<const uint32_t *>(r + i0);
      if (!fy) {
#pragma unroll
        for (int k = 0; k < 4; k++) v[2 * k] = v[2 * k + 1] = (a >> (8 * k)) & 0xFF;
        return;
      }
#pragma unroll
      for (int k = 0; k < 4; k++) cs[1 + k] = (a >> (8 * k)) & 0xFF;
      cs[0] = i0 > 0 ? r[i0 - 1] : 0;
      cs[5] = i0 + 4 < dw ? r[i0 + 4] : 0;
#pragma unroll
      for (int k = 0; k < 4; k++) {
        const int i = i0 + k, cur = cs[1 + k];
        v[2 * k] = i == 0 ? cur : (cur * 3 + cs[k] + 1) >> 2;
        v[2 * k + 1] = i >= dw - 1 ? cur : (cur * 3 + cs[2 + k] + 2) >> 2;
      }
    }
    return;
  }
  // HEXP == 1, VEXP == 2 (4:4:0)
  {
    const uint2 a = *reinterpret_cast<const uint2 *>(pl + (int64_t)(y >> 1) * pw + x0);
    const uint2 b = *reinterpret_cast<const uint2 *>(pl + (int64_t)fancy_far_row(y, dh) * pw + x0);
    const int bias = (y & 1) ? 2 : 1;
#pragma unroll
    for (int k = 0; k < 8; k++) {
      const int p0 = ((k < 4 ? a.x : a.y) >> (8 * (k & 3))) & 0xFF, p1 = ((k < 4 ? b.x : b.y) >> (8 * (k & 3))) & 0xFF;
      v[k] = fancy ? (p0 * 3 + p1 + bias) >> 2 : p0;
    }
  }
}

template <int HEXP, int VEXP>
__device__ __forceinline__ void color_row8(const JpegImage &im, const uint8_t *__restrict__ planes, int x0, int y) {
  const int W = im.width, H = im.height;
  const uint2 yw = *reinterpret_cast<const uint2 *>(planes + im.plane_off[0] + (int64_t)y * im.plane_w[0] + x0);
  const int dw = (W + HEXP - 1) / HEXP, dh = (H + VEXP - 1) / VEXP;
  int cb[8], cr[8];
  chroma8<HEXP, VEXP>(planes + im.plane_off[1], im.plane_w[1], dw, dh, im.fancy, x0, y, cb);
  chroma8<HEXP, VEXP>(planes + im.plane_off[2], im.plane_w[2], dw, dh, im.fancy, x0, y, cr);
  uint32_t px[24];
  const bool bgr = im.out_type == DALIB200_BGR;
#pragma unroll
  for (int k = 0; k < 8; k++) {
    const int yy = ((k < 4 ? yw.x : yw.y) >> (8 * (k & 3))) & 0xFF;
    const int cbm = cb[k] - 128, crm = cr[k] - 128;
    const int r = clamp255(yy + ((91881 * crm + 32768) >> 16));
    const int g = clamp255(yy + ((-22554 * cbm + 32768 - 46802 * crm) >> 16));
    const int b = clamp255(yy + ((116130 * cbm + 32768) >> 16));
    px[3 * k] = (uint32_t)(bgr ? b : r); px[3 * k + 1] = (uint32_t)g; px[3 * k + 2] = (uint32_t)(bgr ? r : b);
  }
  uint8_t *o = im.out + ((int64_t)(y - im.win_y0) * im.win_w + (x0 - im.win_x0)) * 3;
  const int nx = min(8, im.win_x0 + im.win_w - x0);
  if (nx == 8 && (reinterpret_cast<uintptr_t>(o) & 7) == 0) {
    uint2 *o8 = reinterpret_cast<uint2 *>(o);
#pragma unroll
    for (int q = 0; q < 3; q++) {
      const uint32_t lo = px[8 * q] | (px[8 * q + 1] << 8) | (px[8 * q + 2] << 16) | (px[8 * q + 3] << 24);
      const uint32_t hi = px[8 * q + 4] | (px[8 * q + 5] << 8) | (px[8 * q + 6] << 16) | (px[8 * q + 7] << 24);
      o8[q] = make_uint2(lo, hi);
    }
  } else {
    for (int k = 0; k < 24; k++) if (k < nx * 3) o[k] = (uint8_t)px[k];
  }
}

// items: per image height * ceil(width / kColorSeg); images not eligible for this path (or decoded by idct_color_420) own zero items
__global__ void __launch_bounds__(128, 10) color_fast_kernel(const JpegImage *__restrict__ images, const int64_t *__restrict__ first_item,
                                                         int nimages, int64_t total_items, const uint8_t *__restrict__ planes) {
  // every CTA owns a contiguous range of items: the image is searched once (by one thread) and then only advanced -- the per-item,
  // per-thread binary search with its dependent global loads was a quarter of this kernel's stall samples
  __shared__ int s_first;
  const int64_t per_cta = (total_items + gridDim.x - 1) / gridDim.x;
  const int64_t it0 = (int64_t)blockIdx.x * per_cta, it1 = min(total_items, it0 + per_cta);
  if (it0 >= it1) return;
  if (threadIdx.x == 0) s_first = last_at_most(first_item, 0, nimages - 1, it0);
  __syncthreads();
  int lo = s_first;
  for (int64_t item = it0; item < it1; item++) {
    while (lo + 1 < nimages && first_item[lo + 1] <= item) lo++;
    const JpegImage &im = images[lo];
    const int64_t li = item - first_item[lo];
    const int segs = (im.win_w + kColorSeg - 1) / kColorSeg;
    const uint32_t lrow = (uint32_t)li / (uint32_t)segs, lseg = (uint32_t)li - lrow * (uint32_t)segs;     // 32-bit: see idct_kernel
    const int x0 = im.win_x0 + (int)lseg * kColorSeg + threadIdx.x * 8;
    if (x0 >= im.win_x0 + im.win_w) continue;
    const int hexp = im.hmax, vexp = im.vmax;     // chroma is 1x1 (checked on the host)
    const int y = im.win_y0 + (int)lrow;
    if (hexp == 2 && vexp == 2) color_row8<2, 2>(im, planes, x0, y);
    else if (hexp == 1 && vexp == 1) color_row8<1, 1>(im, planes, x0, y);
    else if (hexp == 2 && vexp == 1) color_row8<2, 1>(im, planes, x0, y);
    else color_row8<1, 2>(im, planes, x0, y);
  }
}

// ---------------------------------------------------------------------------------------------
// I1 + C1 fused for 4:2:0 YCbCr with fancy upsampling to RGB / BGR (fast_color == 2): dequantisation + IDCT into shared-memory tiles
// and the upsampling + colour conversion behind them, so the planes never reach HBM.
//
// Work item = a strip of kFusedMcus MCU columns of one image's window, walked down one MCU row ("band") at a time over a segment of at
// most kFusedMaxBands bands.  Band m emits the luma rows 16m - 1 .. 16m + 14 (the image's last band also 16m + 15): the two chroma rows
// of every such row (fancy_far_row) are then among chroma rows 8m - 1 .. 8m + 7, i.e. this band's and the last one of the band above.
// The IDCT of band m leaves its last luma and chroma rows in carry row m & 1 as well, where band m + 1 finds them while the IDCT of
// band m + 1 is already overwriting the band rows.  A segment that does not start at the top first transforms the band above it.  The
// horizontal halo is the edge column of the chroma blocks of the MCUs left and right of the strip.
//
// Warps 0-2 transform the luma and chroma blocks of the strip, one block per thread.  Warp 3 transforms the (up to) 4 halo blocks, of
// which one column each is needed, with 8 lanes per block (halo_pass1 / halo_pass2): a whole block per thread there would cost warp 3
// as many instructions as each of the others for 4 % of the work.  The colour unit (color_unit16) has no image-edge case: the thread
// that transforms the chroma block of the image's first or last chroma column also stores a copy of that column beside it.
static_assert(kFusedThreads == 128 && 6 * kFusedMcus <= 96, "idct_color_420: warps 0-2 take the strip's blocks, warp 3 the halo");

// items: per image fused_geo().nstrips * nseg, strips of one segment consecutive; one CTA per item
__global__ void __launch_bounds__(kFusedThreads, 5) idct_color_420(const JpegImage *__restrict__ images, const int64_t *__restrict__ first_item,
                                                                int nimages, const int16_t *__restrict__ coef_arena,
                                                                const int16_t *__restrict__ dc_arena, const QuantSet *__restrict__ quants) {
  __shared__ __align__(16) uint8_t s_y[18][16 * kFusedMcus];      // rows 0, 1: carry rows; 2 + r: luma row 16m + r of band m
  __shared__ __align__(16) uint8_t s_c[2][10][kFusedCPitch];      // Cb, Cr; rows 0, 1: carry rows; 2 + r: chroma row 8m + r
  __shared__ int s_hws[4][8][9];                                  // pass-1 workspace of the halo blocks (row y, column x)
  __shared__ int s_img;
  if (threadIdx.x == 0) s_img = last_at_most(first_item, 0, nimages - 1, (int64_t)blockIdx.x);
  __syncthreads();
  const int ii = s_img;
  const JpegImage &im = images[ii];
  const FusedGeo g = fused_geo(im);
  const int li = (int)(blockIdx.x - first_item[ii]);
  const int seg = li / g.nstrips, strip = li - seg * g.nstrips;
  const int mxa = g.mx0 + strip * kFusedMcus, nt = min(kFusedMcus, g.mx_end - mxa);
  const int b_lo = g.m0 + seg * g.seg_len, b_hi = min(g.m0 + g.nbands, b_lo + g.seg_len);
  if (b_lo >= b_hi) return;
  // this thread's block in every band: the luma blocks in tile order (the lanes of a warp store consecutive 8-byte runs of one row),
  // then Cb, Cr, then the chroma blocks of the MCUs left / right of the strip, of which only the edge column is kept
  const int j = threadIdx.x;
  const bool halo = j >= 96;
  int mx = 0, comp = 0, bx = 0, by = 0, col = 0;                  // col: tile byte of the block's column 0 (halo: of the kept column)
  bool active = true;
  if (j < 4 * nt) {
    by = j / (2 * nt);
    const int c8 = j - by * 2 * nt;
    mx = mxa + (c8 >> 1); bx = c8 & 1; col = 8 * c8;
  } else if (j < 6 * nt) {
    comp = 1 + (j - 4 * nt) / nt;
    const int u = (j - 4 * nt) % nt;
    mx = mxa + u; col = 8 + 8 * u;
  } else if (halo) {
    const int h = (j - 96) >> 3;
    comp = 1 + (h & 1);
    if (h < 2) { mx = mxa - 1; active = mxa > 0; col = 7; }
    else { mx = mxa + nt; active = mx < im.mcux; col = 8 + 8 * nt; }
  } else {
    active = false;
  }
  int b = 0;
  for (int k = 0; k < im.bpm; k++) if (im.blk_comp[k] == comp && im.blk_x[k] == bx && im.blk_y[k] == by) b = k;
  const uint16_t *q = quants[im.quant_set].q[im.tq[comp]];
  const int64_t blk0 = im.coef_off / 64;
  const int wx0 = im.win_x0, wx1 = im.win_x0 + im.win_w, wy0 = im.win_y0, wy1 = im.win_y0 + im.win_h;
  const int dw = (im.width + 1) >> 1, dh = (im.height + 1) >> 1;
  const ColorK ck = color_k(im.out_type == DALIB200_BGR);
  const int s0 = im.out_type == DALIB200_BGR ? 0 : 1;             // chroma of channel 0: Cr for RGB, Cb for BGR
  const int edge = dw - 1 - 8 * mx;                               // chroma block: column of the image's last chroma column if < 8
  for (int m = b_lo > 0 ? b_lo - 1 : b_lo; m < b_hi; m++) {
    if (halo) {
      // lane x: pass 1 on column x of block hb; then lane y: pass 2 on row y, the kept column only
      const int x = j & 7, hb = (j >> 3) & 3;
      int in[8] = { 0, 0, 0, 0, 0, 0, 0, 0 };
      uint32_t ac = 0;
      if (active) {
        const int64_t gb = blk0 + ((int64_t)m * im.mcux + mx) * im.bpm + b;
#pragma unroll
        for (int y = 0; y < 8; y++) {
          const int c = __ldg(coef_arena + gb * 64 + 8 * y + x);
          in[y] = wrap16(c * (int)__ldg(q + 8 * y + x));
          if (y) ac |= (uint32_t)c;
        }
        if (x == 0) in[0] = wrap16((int)__ldg(dc_arena + gb) * (int)__ldg(q));
      }
      ac |= __shfl_xor_sync(0xFFFFFFFFu, ac, 1);
      ac |= __shfl_xor_sync(0xFFFFFFFFu, ac, 2);
      ac |= __shfl_xor_sync(0xFFFFFFFFu, ac, 4);
      int wsc[8];
      halo_pass1(in, ac == 0, wsc);
#pragma unroll
      for (int y = 0; y < 8; y++) s_hws[hb][y][x] = wsc[y];
      __syncwarp();
      int wsr[8];
#pragma unroll
      for (int k = 0; k < 8; k++) wsr[k] = s_hws[hb][x][k];
      const uint8_t v = (uint8_t)halo_pass2(wsr, col == 7);
      if (active) {
        s_c[comp - 1][2 + x][col] = v;
        if (x == 7) s_c[comp - 1][m & 1][col] = v;
      }
    } else if (active) {
      uint2 rows[8];
      idct_block(coef_arena, dc_arena, blk0 + ((int64_t)m * im.mcux + mx) * im.bpm + b, q, rows);
      if (comp == 0) {
#pragma unroll
        for (int y = 0; y < 8; y++) *reinterpret_cast<uint2 *>(&s_y[2 + 8 * by + y][col]) = rows[y];
        if (by == 1) *reinterpret_cast<uint2 *>(&s_y[m & 1][col]) = rows[7];
      } else {
#pragma unroll
        for (int y = 0; y < 8; y++) *reinterpret_cast<uint2 *>(&s_c[comp - 1][2 + y][col]) = rows[y];
        *reinterpret_cast<uint2 *>(&s_c[comp - 1][m & 1][col]) = rows[7];
        if (mx == 0 || edge < 8) {      // libjpeg: the missing neighbour of the first / last chroma column is the column itself
#pragma unroll
          for (int y = 0; y < 9; y++) {
            uint8_t *t = s_c[comp - 1][y < 8 ? 2 + y : m & 1];
            const uint2 rv = rows[y < 8 ? y : 7];
            if (mx == 0) t[col - 1] = (uint8_t)rv.x;
            if (edge < 8) t[col + edge + 1] = (uint8_t)((edge < 4 ? rv.x : rv.y) >> (8 * (edge & 3)));
          }
        }
      }
    }
    __syncthreads();
    if (m >= b_lo) {
      const int carry = (m + 1) & 1;                          // = (m - 1) & 1: written by the band above
      const int ya = max(16 * m - 1, wy0), yb = min(16 * m + (m == im.mcuy - 1 ? 16 : 15), wy1);
      const int nunits = (yb - ya) * nt;                      // unit = 16 pixels of one row
      for (int e = threadIdx.x; e < nunits; e += kFusedThreads) {
        const int r = e / nt, u = e - r * nt;
        const int y = ya + r, x0 = 16 * (mxa + u);
        const int ly = y - 16 * m, cn = (y >> 1) - 8 * m, cf = fancy_far_row(y, dh) - 8 * m;
        const uint4 yv = *reinterpret_cast<const uint4 *>(&s_y[ly < 0 ? carry : 2 + ly][16 * u]);
        const int rn = cn < 0 ? carry : 2 + cn, rf = cf < 0 ? carry : 2 + cf;
        const uint32_t yw[4] = { yv.x, yv.y, yv.z, yv.w };
        uint32_t w[12];
        color_unit16(yw, s_c[s0][rn], s_c[s0][rf], s_c[1 - s0][rn], s_c[1 - s0][rf], 8 + 8 * u, ck, w);
        uint8_t *o = im.out + ((int64_t)(y - wy0) * im.win_w + (x0 - wx0)) * 3;     // clipped to the window below
        if (x0 >= wx0 && x0 + 16 <= wx1 && (reinterpret_cast<uintptr_t>(o) & 15) == 0) {
          uint4 *o16 = reinterpret_cast<uint4 *>(o);
#pragma unroll
          for (int t = 0; t < 3; t++) o16[t] = make_uint4(w[4 * t], w[4 * t + 1], w[4 * t + 2], w[4 * t + 3]);
          continue;
        }
#pragma unroll
        for (int h = 0; h < 2; h++) {
          const int xa = x0 + 8 * h;
          uint8_t *oh = o + 24 * h;
          if (xa >= wx0 && xa + 8 <= wx1 && (reinterpret_cast<uintptr_t>(oh) & 7) == 0) {
            uint2 *o8 = reinterpret_cast<uint2 *>(oh);
#pragma unroll
            for (int t = 0; t < 3; t++) o8[t] = make_uint2(w[6 * h + 2 * t], w[6 * h + 2 * t + 1]);
          } else {
#pragma unroll
            for (int n = 0; n < 24; n++)
              if (xa + n / 3 >= wx0 && xa + n / 3 < wx1) oh[n] = (uint8_t)(w[6 * h + n / 4] >> (8 * (n & 3)));
          }
        }
      }
    }
    __syncthreads();
  }
}

// ---------------------------------------------------------------------------------------------
// Post pass: orientation + region of interest + colour space + data type, one thread per output pixel.
// Colour formulas: kernels::color::itu_r_bt_601::rgb_to_ycbcr<Out, uint8_t> (color_space_conversion_impl.h:64-103), dtype
// conversion ConvertSatNorm<float>(uint8_t) = v * (1.0f / 255) (include/dali/core/convert.h:263-275).
template <typename Out> __device__ __forceinline__ Out post_cvt(uint32_t v);
template <> __device__ __forceinline__ uint8_t post_cvt<uint8_t>(uint32_t v) { return (uint8_t)v; }
template <> __device__ __forceinline__ float post_cvt<float>(uint32_t v) { return mul_rn((float)v, 1.0f / 255); }

__device__ __forceinline__ float post_dot3(float c0, float c1, float c2, float a, float b, float c) {
  return add_rn(add_rn(mul_rn(c0, a), mul_rn(c1, b)), mul_rn(c2, c));
}

template <typename Out>
__global__ void __launch_bounds__(256) jpeg_post_kernel(const JpegPost *__restrict__ posts, int n, int64_t total_px) {
  __shared__ int s_first;
  const int64_t per_cta = ((total_px + gridDim.x - 1) / gridDim.x + 255) / 256 * 256;
  const int64_t p0 = (int64_t)blockIdx.x * per_cta, p1 = min(total_px, p0 + per_cta);
  if (p0 >= p1) return;
  if (threadIdx.x == 0) {
    s_first = last_at_most(posts, 0, n - 1, p0, [](const JpegPost &p) { return p.first_px; });
  }
  __syncthreads();
  int ii = s_first;
  constexpr bool F = sizeof(Out) == 4;
  // coefficients of rgb_to_ycbcr<Out, uint8_t>: vec3 * scale_factor<uint8_t, Out>() (a float product per coefficient)
  const float sf = F ? (float)(1.0 / 255.0) : 1.0f;
  const float ky0 = mul_rn(0.25678823529f, sf), ky1 = mul_rn(0.50412941176f, sf), ky2 = mul_rn(0.09790588235f, sf);
  const float kb0 = mul_rn(-0.14822289945f, sf), kb1 = mul_rn(-0.29099278682f, sf), kb2 = mul_rn(0.43921568627f, sf);
  const float kr0 = mul_rn(0.43921568627f, sf), kr1 = mul_rn(-0.36778831435f, sf), kr2 = mul_rn(-0.07142737192f, sf);
  const float ybias = F ? 0.0625f : 16.0f, cbias = F ? 0.5f : 128.0f;
  for (int64_t gp = p0 + threadIdx.x; gp < p1; gp += blockDim.x) {
    while (ii + 1 < n && posts[ii + 1].first_px <= gp) ii++;
    const JpegPost &d = posts[ii];
    const int64_t lp = gp - d.first_px;
    const int oy = (int)((uint32_t)lp / (uint32_t)d.out_w), ox = (int)((uint32_t)lp - (uint32_t)oy * (uint32_t)d.out_w);
    const int fy = d.out_y0 + oy, fx = d.out_x0 + ox;           // oriented full-image coordinates
    int sy, sx;
    switch (d.orientation) {                                   // EXIF: where does the displayed pixel come from?
      case 2: sy = fy; sx = d.img_w - 1 - fx; break;
      case 3: sy = d.img_h - 1 - fy; sx = d.img_w - 1 - fx; break;
      case 4: sy = d.img_h - 1 - fy; sx = fx; break;
      case 5: sy = fx; sx = fy; break;
      case 6: sy = d.img_h - 1 - fx; sx = fy; break;
      case 7: sy = d.img_h - 1 - fx; sx = d.img_w - 1 - fy; break;
      case 8: sy = fx; sx = d.img_w - 1 - fy; break;
      default: sy = fy; sx = fx; break;
    }
    const uint8_t *sp = d.src + ((int64_t)(sy - d.win_y0) * d.src_w + (sx - d.win_x0)) * d.src_c;
    if (d.out_type == DALIB200_GRAY) {                         // the decoder produced the Y plane itself (src_c == 1)
      static_cast<Out *>(d.dst)[lp] = post_cvt<Out>(sp[0]);
      continue;
    }
    uint32_t r, g, b;
    if (d.src_c == 1) r = g = b = sp[0]; else { r = sp[0]; g = sp[1]; b = sp[2]; }
    Out *op = static_cast<Out *>(d.dst) + lp * 3;
    if (d.out_type == DALIB200_YCbCr) {
      const float fr = (float)r, fg = (float)g, fb = (float)b;
      const float yv = add_rn(post_dot3(ky0, ky1, ky2, fr, fg, fb), ybias);
      const float cb = add_rn(post_dot3(kb0, kb1, kb2, fr, fg, fb), cbias);
      const float cr = add_rn(post_dot3(kr0, kr1, kr2, fr, fg, fb), cbias);
      if (F) { op[0] = (Out)yv; op[1] = (Out)cb; op[2] = (Out)cr; }
      else { op[0] = (Out)sat_u8_half_away(yv); op[1] = (Out)sat_u8_half_away(cb); op[2] = (Out)sat_u8_half_away(cr); }
    } else if (d.out_type == DALIB200_BGR) {
      op[0] = post_cvt<Out>(b); op[1] = post_cvt<Out>(g); op[2] = post_cvt<Out>(r);
    } else {
      op[0] = post_cvt<Out>(r); op[1] = post_cvt<Out>(g); op[2] = post_cvt<Out>(b);
    }
  }
}

// ---------------------------------------------------------------------------------------------
// Reconstruct stage on the host: path choice, work lists, launches (jpeg_recon.h)
void ReconAddImage(JpegImage &im, bool fancy, bool planes_only, ReconTotals &t, int64_t *first_work, int64_t *first_fused,
                   int64_t *first_quad, int64_t *first_item) {
  im.fast_color = im.ncomp == 3 && im.color == kColorYCbCr && (im.out_type == DALIB200_RGB || im.out_type == DALIB200_BGR) &&
                  ((im.hmax == 2 && im.vmax <= 2) || (im.hmax == 1 && im.vmax <= 2));
  if (im.fast_color && fancy && im.hmax == 2 && im.vmax == 2 && (im.width + 1) / 2 > 2) im.fast_color = 2;    // idct_color_420
  if (planes_only) im.fast_color = 1;                                   // IDCT into the planes, no colour work items
  *first_work = t.work;
  *first_fused = t.fused;
  *first_quad = t.quads;
  *first_item = t.items;
  if (im.fast_color == 2) {
    const FusedGeo g = fused_geo(im);
    t.fused += (int64_t)g.nstrips * g.nseg;
    return;
  }
  t.work += (int64_t)im.mcu_nx * im.mcu_ny * im.bpm;
  if (planes_only) return;
  if (im.fast_color) t.items += (int64_t)((im.win_w + kColorSeg - 1) / kColorSeg) * im.win_h;
  else t.quads += (int64_t)((im.win_w + 3) / 4) * im.win_h;
}

int LaunchReconstruct(const ReconLaunch &a, cudaStream_t s) {
  const int sms = NumSMs();
  const int64_t total_blocks = a.totals.work;
  const int grid = (int)std::min<int64_t>((total_blocks + 127) / 128, (int64_t)sms * 32);
  if (total_blocks > 0)
    Launch("jpeg_idct", idct_kernel, grid, 128, 0, s, a.d_images, a.d_first_work, a.nimages, total_blocks, a.d_coef, a.d_dc, a.d_quants, a.d_planes);
  if (a.totals.fused > 0)
    Launch("jpeg_idct_color", idct_color_420, (int)a.totals.fused, kFusedThreads, 0, s, a.d_images, a.d_first_fused, a.nimages, a.d_coef, a.d_dc, a.d_quants);
  if (a.totals.quads > 0) {
    const int grid2 = (int)std::min<int64_t>((a.totals.quads + 255) / 256, (int64_t)sms * 32);
    Launch("jpeg_upsample_color_generic", color_kernel, grid2, 256, 0, s, a.d_images, a.d_first_quad, a.nimages, a.totals.quads, a.d_planes);
  }
  if (a.totals.items > 0) {
    const int grid3 = (int)std::min<int64_t>(a.totals.items, (int64_t)sms * 64);
    Launch("jpeg_upsample_color", color_fast_kernel, grid3, 128, 0, s, a.d_images, a.d_first_item, a.nimages, a.totals.items, a.d_planes);
  }
  return DALIB200_SUCCESS;
}

}  // namespace dalib200

// ============================================================================================
// host side
using namespace dalib200;  // NOLINT

namespace {

struct HostHuff { uint8_t bits[17]; uint8_t vals[256]; bool present = false; };
}  // namespace
// the decode stages of jpeg_prog.cu, png.cu, tiff.cu, webp.cu, bitmap.cu and ljpeg.cu (included here, behind the kernels, so that their
// line tables stay put); EXIF orientation
#include "jpeg_prog.h"
#include "png.h"
#include "tiff.h"
#include "webp.h"
#include "bitmap.h"
#include "ljpeg.h"
#include "exif.h"
namespace {

// The formats the plan takes, told apart by their signatures.  PNG, TIFF, WebP and BMP / PNM samples are planned and decoded by the
// stage of their format; everything else is parsed as JPEG.  A JPEG whose frame header is SOF3 becomes kLossless once parsed: the
// lossless stage plans and decodes it.
enum class Format { kJpeg, kPng, kTiff, kWebp, kBitmap, kLossless };

Format DetectFormat(const uint8_t *p, size_t n) {
  return IsPngStream(p, n) ? Format::kPng : IsTiffStream(p, n) ? Format::kTiff : IsWebpStream(p, n) ? Format::kWebp
       : IsBitmapStream(p, n) ? Format::kBitmap : Format::kJpeg;
}

struct ParsedJpeg {
  int width = 0, height = 0, ncomp = 0, precision = 8;
  int cid[4] = {0}, hs[4] = {0}, vs[4] = {0}, tq[4] = {0};
  int hmax = 0, vmax = 0;
  bool progressive = false, jfif = false, lossless = false;
  int ss = 0, se = 63, ah = 0, al = 0;   // spectral selection / predictor, successive approximation / point transform of the first scan
  Format format = Format::kJpeg;   // PNG, TIFF, WebP, BMP / PNM: width / height / ncomp / orientation / scan range and hs[0] / vs[0] only
  int adobe_transform = -1, orientation = 1, restart_interval = 0;
  uint16_t qt[4][64]; bool qt_present[4] = {false, false, false, false};
  HostHuff dc[4], ac[4];
  int scan_ncomp = 0, scan_comp[4] = {0}, td[4] = {0}, ta[4] = {0};
  size_t scan_begin = 0, scan_end = 0;
};

const uint8_t kZigzag[64] = {
   0,  1,  8, 16,  9,  2,  3, 10, 17, 24, 32, 25, 18, 11,  4,  5,
  12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13,  6,  7, 14, 21, 28,
  35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51,
  58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63 };

inline int rd16(const uint8_t *p) { return (p[0] << 8) | p[1]; }

// T.81 Annex B marker walk up to and including SOS.  Returns a DALIB200 status.
int ParseHeaders(const uint8_t *p, size_t n, ParsedJpeg &j, bool need_scan) {
  size_t pos = 2;
  if (n < 4 || p[0] != 0xFF || p[1] != 0xD8) { SetLastError("not a JPEG stream (missing SOI)"); return DALIB200_ERROR_BAD_DATA; }
  bool got_sof = false;
  while (pos + 4 <= n) {
    if (p[pos] != 0xFF) { SetLastError("JPEG: marker expected at offset %zu", pos); return DALIB200_ERROR_BAD_DATA; }
    while (pos < n && p[pos] == 0xFF) pos++;
    if (pos >= n) break;
    int m = p[pos++];
    if (m == 0xD8 || (m >= 0xD0 && m <= 0xD7) || m == 0x01) continue;
    if (m == 0xD9) break;
    if (pos + 2 > n) break;
    int L = rd16(p + pos);
    if (L < 2 || pos + L > n) { SetLastError("JPEG: truncated segment (marker 0x%02X)", m); return DALIB200_ERROR_BAD_DATA; }
    const uint8_t *s = p + pos + 2;
    int sl = L - 2;
    if (m == 0xDB) {
      int o = 0;
      while (o < sl) {
        int pq = s[o] >> 4, tq = s[o] & 15; o++;
        if (tq > 3 || o + (pq ? 128 : 64) > sl) { SetLastError("JPEG: bad DQT"); return DALIB200_ERROR_BAD_DATA; }
        for (int i = 0; i < 64; i++) { int v; if (pq) { v = rd16(s + o); o += 2; } else v = s[o++]; j.qt[tq][kZigzag[i]] = (uint16_t)v; }
        j.qt_present[tq] = true;
      }
    } else if (m == 0xC4) {
      int o = 0;
      while (o < sl) {
        if (o + 17 > sl) { SetLastError("JPEG: bad DHT"); return DALIB200_ERROR_BAD_DATA; }
        int tc = s[o] >> 4, th = s[o] & 15; o++;
        if (th > 3 || tc > 1) { SetLastError("JPEG: bad DHT id"); return DALIB200_ERROR_BAD_DATA; }
        HostHuff &h = tc ? j.ac[th] : j.dc[th];
        int cnt = 0; h.bits[0] = 0;
        for (int i = 1; i <= 16; i++) { h.bits[i] = s[o++]; cnt += h.bits[i]; }
        if (cnt > 256 || o + cnt > sl) { SetLastError("JPEG: bad DHT counts"); return DALIB200_ERROR_BAD_DATA; }
        memset(h.vals, 0, sizeof(h.vals));
        memcpy(h.vals, s + o, cnt); o += cnt;
        h.present = true;
      }
    } else if (m == 0xC0 || m == 0xC1 || m == 0xC2 || m == 0xC3) {
      if (sl < 6) { SetLastError("JPEG: bad SOF"); return DALIB200_ERROR_BAD_DATA; }
      j.progressive = m == 0xC2;
      j.lossless = m == 0xC3;
      j.precision = s[0]; j.height = rd16(s + 1); j.width = rd16(s + 3); j.ncomp = s[5];
      if (j.ncomp < 1 || j.ncomp > 4 || sl < 6 + 3 * j.ncomp) { SetLastError("JPEG: bad SOF component count"); return DALIB200_ERROR_BAD_DATA; }
      for (int c = 0; c < j.ncomp; c++) {
        j.cid[c] = s[6 + 3 * c]; j.hs[c] = s[7 + 3 * c] >> 4; j.vs[c] = s[7 + 3 * c] & 15; j.tq[c] = s[8 + 3 * c];
        if (j.hs[c] < 1 || j.hs[c] > 4 || j.vs[c] < 1 || j.vs[c] > 4 || j.tq[c] > 3) { SetLastError("JPEG: bad sampling factors"); return DALIB200_ERROR_BAD_DATA; }
        j.hmax = std::max(j.hmax, j.hs[c]); j.vmax = std::max(j.vmax, j.vs[c]);
      }
      got_sof = true;
    } else if (m >= 0xC5 && m <= 0xCF && m != 0xC8 && m != 0xCC) {
      SetLastError("JPEG: coding process 0x%02X (arithmetic / hierarchical) is not supported", m);
      return DALIB200_ERROR_UNSUPPORTED;
    } else if (m == 0xDD) {
      if (sl >= 2) j.restart_interval = rd16(s);
    } else if (m == 0xE0) {
      if (sl >= 5 && !memcmp(s, "JFIF\0", 5)) j.jfif = true;
    } else if (m == 0xE1) {
      if (sl >= 6 && !memcmp(s, "Exif\0\0", 6)) j.orientation = ParseExifOrientation(s + 6, sl - 6);
    } else if (m == 0xEE) {
      if (sl >= 12 && !memcmp(s, "Adobe", 5)) j.adobe_transform = s[11];
    } else if (m == 0xDA) {
      if (!got_sof) { SetLastError("JPEG: SOS before SOF"); return DALIB200_ERROR_BAD_DATA; }
      if (sl < 1) { SetLastError("JPEG: bad SOS"); return DALIB200_ERROR_BAD_DATA; }
      j.scan_ncomp = s[0];
      if (j.scan_ncomp < 1 || j.scan_ncomp > 4 || sl < 1 + 2 * j.scan_ncomp) { SetLastError("JPEG: bad SOS"); return DALIB200_ERROR_BAD_DATA; }
      for (int i = 0; i < j.scan_ncomp; i++) {
        int cs = s[1 + 2 * i], ci = -1;
        for (int c = 0; c < j.ncomp; c++) if (j.cid[c] == cs) ci = c;
        if (ci < 0) { SetLastError("JPEG: SOS references an unknown component"); return DALIB200_ERROR_BAD_DATA; }
        j.scan_comp[i] = ci; j.td[i] = s[2 + 2 * i] >> 4; j.ta[i] = s[2 + 2 * i] & 15;
      }
      if (sl >= 4 + 2 * j.scan_ncomp) {
        const uint8_t *t = s + 1 + 2 * j.scan_ncomp;
        j.ss = t[0]; j.se = t[1]; j.ah = t[2] >> 4; j.al = t[2] & 15;
      }
      j.scan_begin = pos + L;
      break;
    }
    pos += L;
    if (!need_scan && got_sof && m == 0xC0 + (j.progressive ? 2 : 0)) {
      // info-only callers may stop at SOF, but EXIF/Adobe can follow: keep walking until SOS (cheap)
    }
  }
  if (!got_sof) { SetLastError("JPEG: no frame header found"); return DALIB200_ERROR_BAD_DATA; }
  if (j.width == 0 || j.height == 0) { SetLastError("JPEG: zero image size"); return DALIB200_ERROR_BAD_DATA; }
  if (need_scan && !j.scan_begin) { SetLastError("JPEG: no scan found"); return DALIB200_ERROR_BAD_DATA; }
  return DALIB200_SUCCESS;
}

void FillInfo(const ParsedJpeg &j, dalib200JpegInfo *info) {
  info->width = j.width; info->height = j.height;
  info->components = j.ncomp;
  info->subsampling = (j.hs[0] << 4) | j.vs[0];
  info->restart_interval = j.restart_interval;
  info->orientation = j.orientation;
}

}  // namespace

struct JpegGeo { int orient = 1, rx0 = 0, ry0 = 0, rx1 = 0, ry1 = 0, out_c = 3; bool direct = true, planar_ok = false; };

struct dalib200JpegPlan {
  int max_batch = 0, n = 0;
  int output_type = DALIB200_RGB, fancy = 1, dtype = DALIB200_UINT8, adjust_orientation = 0;
  std::vector<JpegPost> posts;              // samples that need the post pass (indices in post_sample)
  std::vector<int> post_sample;
  std::vector<size_t> post_off;             // byte offset of each post sample's window inside d_post
  std::vector<int32_t> out_shape;           // n x 3 (H, W, C) of the operator output
  std::vector<uint8_t> planes_only;         // the sample's colour stage is skipped (the caller reads the planes)
  std::vector<JpegGeo> geo;                 // per-sample output geometry (orientation, region of interest, eligibility)
  std::vector<int64_t> first_work;          // IDCT work list prefix
  std::vector<int64_t> first_fused;         // idct_color_420 work list prefix
  int64_t total_work = 0, total_fused = 0, total_post_px = 0;
  size_t post_bytes = 0;
  uint8_t *d_post = nullptr; size_t d_post_cap = 0;
  JpegPost *d_posts = nullptr; size_t d_posts_cap = 0;
  std::vector<ParsedJpeg> parsed;
  std::vector<JpegImage> images;
  std::vector<JpegUnit> units;
  std::vector<TableSet> tables;
  std::vector<QuantSet> quants;
  std::vector<int64_t> first_quad, first_item;
  std::vector<int32_t> block_image;         // sync block -> image
  std::vector<int32_t> wblock_image;        // write block -> image
  std::vector<const uint8_t *> src_ptr;     // host pointers of the scan data (for staging; borrowed until JpegUpload returns)
  bool source_stable = false;               // JpegPlanSetSourceStable: page-locked sources are copied by the DMA engine directly
  int last_upload_direct = 0;
  std::vector<size_t> stage_off;            // offset of each sample's scan bytes inside the raw staging area
  size_t raw_bytes = 0, clean_bytes = 0, clean_alloc = 0;   // clean_alloc = clean_bytes + the read slack (clean_read_behind)
  uint32_t nchunks = 0;
  int64_t total_subseq = 0, total_coefs = 0, total_plane_bytes = 0, total_quads = 0, total_items = 0;
  int total_blocks_sync = 0, total_blocks_write = 0;
  int log2_sub = 10;
  // staging (pinned) and device buffers -- grow only
  dalib200::PinnedStage h_stage;            // descriptors and tables, then the scan bytes (JpegUpload): d_stage's layout
  uint8_t *d_stage = nullptr; size_t d_stage_cap = 0;
  size_t desc_bytes = 0, off_images = 0, off_units = 0, off_tables = 0, off_quants = 0, off_quads = 0, off_items = 0, off_work = 0, off_fused = 0, off_blkimg = 0, off_wblkimg = 0, off_raw = 0;
  uint8_t *d_clean = nullptr; size_t d_clean_cap = 0;
  uint32_t *d_chunk = nullptr; size_t d_chunk_cap = 0;
  uint32_t *d_unit_len = nullptr; size_t d_unit_cap = 0;
  uint64_t *d_state = nullptr; uint32_t *d_n = nullptr; size_t d_sub_cap = 0;
  uint4 *d_chain1 = nullptr, *d_chain2 = nullptr, *d_chain3 = nullptr;
  size_t d_chain1_cap = 0, d_chain2_cap = 0, d_chain3_cap = 0;
  uint32_t *d_chain_count = nullptr; size_t d_chain_count_cap = 0;
  int walk_max_grid = 0;
  int16_t *d_coef = nullptr; size_t d_coef_cap = 0;
  int16_t *d_dc = nullptr; size_t d_dc_cap = 0;
  uint8_t *d_planes = nullptr; size_t d_planes_cap = 0;
  int32_t *d_status = nullptr; size_t d_status_cap = 0;
  uint32_t *d_unit_nblk = nullptr; size_t d_unit_nblk_cap = 0;
  int32_t *h_status = nullptr; size_t h_status_cap = 0;        // pinned copy of d_status (JpegStatusAsync / JpegStatusFetch)
  dalib200::PinnedStage h_images;           // this launch's JpegImage and JpegPost descriptors (they carry the output pointers)
  bool staged = false, smem_opted = false;
  // the stages beside the baseline kernels (decode_stage.h).  The progressive stage writes coefficients for everything behind the entropy
  // stage; the PNG, TIFF, WebP and BMP / PNM stages decode whole streams into the same decode windows; the lossless samples' units join
  // U1 - U3 (in `units`, skipped by every DCT kernel) and their stage decodes the clean streams behind U3.  The post pass is shared.
  ProgStage prog;
  PngStage png;
  TiffStage tiff;
  WebpStage webp;
  BitmapStage bitmap;
  LjpegStage ljpeg;
  std::array<SideStage *, 6> stages() { return { &prog, &png, &tiff, &webp, &bitmap, &ljpeg }; }   // in launch order
  StreamStage &stage_of(Format f) {
    switch (f) {
      case Format::kPng: return png;
      case Format::kTiff: return tiff;
      case Format::kWebp: return webp;
      default: return bitmap;
    }
  }
};

namespace {
// Work lists that depend on the per-sample colour decision: post pass descriptors, colour work items, IDCT block ranges.  Run by
// PlanSetupEx and again by JpegPlanSetPlanesOnly (cheap: O(batch)).
void BuildWorkLists(dalib200JpegPlan *p) {
  const int n = p->n;
  p->posts.clear(); p->post_sample.clear(); p->post_off.clear();
  ReconTotals t;
  int64_t post_px = 0;
  size_t post_bytes = 0;
  for (int i = 0; i < n; i++) {
    JpegImage &im = p->images[i];
    const ParsedJpeg &j = p->parsed[i];
    const JpegGeo &ge = p->geo[i];
    const bool planes_only = p->planes_only[i] != 0;
    im.out_type = p->output_type;
    if (!ge.direct && !planes_only) {
      // the window is decoded to RGB (or to the Y plane for GRAY) into plan scratch; the post pass gathers / converts it
      im.out_type = p->output_type == DALIB200_GRAY ? DALIB200_GRAY : DALIB200_RGB;
      JpegPost po;
      memset(&po, 0, sizeof(po));
      po.src_w = im.win_w; po.src_c = ge.out_c == 1 ? 1 : 3;
      po.img_w = j.width; po.img_h = j.height; po.win_x0 = im.win_x0; po.win_y0 = im.win_y0;
      po.out_x0 = ge.rx0; po.out_y0 = ge.ry0; po.out_w = ge.rx1 - ge.rx0; po.out_h = ge.ry1 - ge.ry0;
      po.orientation = ge.orient; po.out_type = p->output_type; po.dtype = p->dtype;
      po.first_px = post_px;
      post_px += (int64_t)po.out_w * po.out_h;
      p->posts.push_back(po); p->post_sample.push_back(i); p->post_off.push_back(post_bytes);
      post_bytes += Align((size_t)im.win_w * im.win_h * po.src_c, 256);
    }
    if (j.format != Format::kJpeg) {   // decoded by png.cu / tiff.cu / webp.cu / bitmap.cu: no IDCT / colour work
      p->first_work[i] = t.work; p->first_fused[i] = t.fused; p->first_quad[i] = t.quads; p->first_item[i] = t.items;
      continue;
    }
    ReconAddImage(im, p->fancy != 0, planes_only, t, &p->first_work[i], &p->first_fused[i], &p->first_quad[i], &p->first_item[i]);
  }
  p->total_work = t.work; p->total_fused = t.fused; p->total_post_px = post_px; p->post_bytes = post_bytes; p->total_quads = t.quads;
  p->total_items = t.items;
}

// PNG, TIFF, WebP, BMP or PNM sample `sample` (format f): the stage of its format appends its descriptors, its staged bytes go to
// `raw_off` of the raw staging area, and `j` receives the fields the plan reads for every sample.  Returns a DALIB200 status.
int PlanSideSample(StreamStage &st, Format f, const uint8_t *data, size_t len, int sample, int64_t raw_off, ParsedJpeg &j) {
  StreamInfo info;
  std::string err;
  if (int rc = st.Plan(data, len, sample, raw_off, &info, &err)) { SetLastError("%s", err.c_str()); return rc; }
  j.format = f;
  j.width = info.width; j.height = info.height; j.ncomp = info.components; j.orientation = info.orientation;
  j.hs[0] = j.vs[0] = f == Format::kWebp ? 2 : 1;      // reported subsampling: WebP is 4:2:0 (VP8's only layout)
  j.scan_begin = info.stage_begin; j.scan_end = info.stage_end;
  return DALIB200_SUCCESS;
}

// The frame of a lossless JPEG (SOF3) sample as the lossless stage's planner (ljpeg_plan.h) reads it.
LjpegFrame LosslessFrame(const ParsedJpeg &j) {
  LjpegFrame f;
  f.width = j.width; f.height = j.height; f.ncomp = j.ncomp; f.precision = j.precision;
  for (int c = 0; c < 4; c++) { f.hs[c] = j.hs[c]; f.vs[c] = j.vs[c]; }
  f.scan_ncomp = j.scan_ncomp;
  f.scan_in_frame_order = true;
  for (int i = 0; i < j.scan_ncomp; i++) { f.td[j.scan_comp[i]] = j.td[i]; f.scan_in_frame_order &= j.scan_comp[i] == i; }
  f.pred = j.ss; f.se = j.se; f.ah = j.ah; f.pt = j.al;
  f.restart_interval = j.restart_interval; f.jfif = j.jfif; f.adobe_transform = j.adobe_transform;
  for (int t = 0; t < 4; t++) if (j.dc[t].present) { f.bits[t] = j.dc[t].bits; f.vals[t] = j.dc[t].vals; }
  return f;
}

// Output geometry of sample i: orientation, region of interest, decode window, post pass.  Returns a DALIB200 status.
int PlanGeometry(dalib200JpegPlan *p, int i, const dalib200JpegRoi *rois, const ParsedJpeg &j, JpegImage &im) {
  const int orient = p->adjust_orientation ? j.orientation : 1;
  const int W = j.width, H = j.height;
  const int OW = orient >= 5 ? H : W, OH = orient >= 5 ? W : H;          // oriented image size
  int rx0 = 0, ry0 = 0, rx1 = OW, ry1 = OH;                              // region of interest, oriented coordinates
  if (rois && rois[i].use_roi) {
    rx0 = rois[i].x0; ry0 = rois[i].y0; rx1 = rois[i].x1; ry1 = rois[i].y1;
    if (!(0 <= rx0 && rx0 < rx1 && rx1 <= OW && 0 <= ry0 && ry0 < ry1 && ry1 <= OH)) {
      SetLastError("decoders.image: sample %d: ROI [%d, %d) x [%d, %d) must be non-empty and fit within the image bounds (%d x %d)",
                   i, rx0, rx1, ry0, ry1, OW, OH);
      return DALIB200_ERROR_INVALID_ARGUMENT;
    }
  }
  // source rectangle of the region (the EXIF transforms map rectangles to rectangles)
  int sx0, sx1, sy0, sy1;
  {
    auto src_of = [&](int fy, int fx, int &sy, int &sx) {
      switch (orient) {
        case 2: sy = fy; sx = W - 1 - fx; break;
        case 3: sy = H - 1 - fy; sx = W - 1 - fx; break;
        case 4: sy = H - 1 - fy; sx = fx; break;
        case 5: sy = fx; sx = fy; break;
        case 6: sy = H - 1 - fx; sx = fy; break;
        case 7: sy = H - 1 - fx; sx = W - 1 - fy; break;
        case 8: sy = fx; sx = W - 1 - fy; break;
        default: sy = fy; sx = fx; break;
      }
    };
    int ay, ax, by_, bx_;
    src_of(ry0, rx0, ay, ax); src_of(ry1 - 1, rx1 - 1, by_, bx_);
    sy0 = std::min(ay, by_); sy1 = std::max(ay, by_) + 1; sx0 = std::min(ax, bx_); sx1 = std::max(ax, bx_) + 1;
  }
  const int output_type = p->output_type;
  const int out_c = output_type == DALIB200_GRAY ? 1 : 3;
  p->out_shape[3 * i] = ry1 - ry0; p->out_shape[3 * i + 1] = rx1 - rx0; p->out_shape[3 * i + 2] = out_c;
  if (j.format != Format::kJpeg) {   // any window: png_color / tiff_color / webp_color / bitmap_color produce pixels one by one
    im.win_x0 = sx0; im.win_w = sx1 - sx0;
  } else {
    im.win_x0 = sx0 & ~7; im.win_w = std::min(W, (sx1 + 7) & ~7) - im.win_x0;
  }
  im.win_y0 = sy0; im.win_h = sy1 - sy0;
  JpegGeo &ge = p->geo[i];
  ge.orient = orient; ge.rx0 = rx0; ge.ry0 = ry0; ge.rx1 = rx1; ge.ry1 = ry1; ge.out_c = out_c;
  ge.direct = orient == 1 && p->dtype == DALIB200_UINT8 && output_type != DALIB200_YCbCr && im.win_x0 == sx0 && im.win_x0 + im.win_w == sx1;
  // decode -> resize without the RGB image (the caller consumes the planes): 4:2:0 YCbCr, fancy upsampling, plain RGB u8 request
  ge.planar_ok = j.format == Format::kJpeg && j.ncomp == 3 && im.color == kColorYCbCr && j.hmax == 2 && j.vmax == 2 && p->fancy && orient == 1 && j.width > 4 &&
                 output_type == DALIB200_RGB && p->dtype == DALIB200_UINT8;
  const bool planes_only = rois && rois[i].planes_only;
  if (planes_only && !ge.planar_ok) {
    SetLastError("decoders.image: sample %d: planes_only needs a 3-component 4:2:0 YCbCr stream without orientation, RGB u8 output", i);
    return DALIB200_ERROR_UNSUPPORTED;
  }
  p->planes_only[i] = planes_only;
  return DALIB200_SUCCESS;
}
}  // namespace

extern "C" {

int dalib200JpegGetInfo(const uint8_t *data, size_t len, dalib200JpegInfo *info) try {
  DB_CHECK_ARG(data && info, "JpegGetInfo: null argument");
  ParsedJpeg j;
  const Format f = DetectFormat(data, len);
  // a PNG, TIFF, WebP, BMP or PNM stream is planned into a stage of its format of its own: no device resources
  auto plan_into = [&](auto &&st) { return PlanSideSample(st, f, data, len, 0, 0, j); };
  int rc = f == Format::kJpeg ? ParseHeaders(data, len, j, false)
         : f == Format::kPng  ? plan_into(PngStage())
         : f == Format::kTiff ? plan_into(TiffStage())
         : f == Format::kWebp ? plan_into(WebpStage())
                              : plan_into(BitmapStage());
  if (rc) return rc;
  FillInfo(j, info);
  return DALIB200_SUCCESS;
} DB_API_CATCH

int dalib200JpegPlanCreate(dalib200JpegPlan **plan, int max_batch) try {
  DB_CHECK_ARG(plan && max_batch > 0, "JpegPlanCreate: bad arguments");
  auto *p = new dalib200JpegPlan();
  p->max_batch = max_batch;
  for (SideStage *st : p->stages())
    if (!st->Create()) { SetLastError("JpegPlanCreate: cudaEventCreate failed"); delete p; return DALIB200_ERROR_CUDA; }
  *plan = p;
  return DALIB200_SUCCESS;
} DB_API_CATCH

int dalib200JpegPlanDestroy(dalib200JpegPlan *p) try {
  if (!p) return DALIB200_SUCCESS;
  for (SideStage *st : p->stages()) st->Destroy();
  p->h_stage.Free();
  p->h_images.Free();
  if (p->h_status) cudaFreeHost(p->h_status);
  void *bufs[] = { p->d_stage, p->d_clean, p->d_chunk, p->d_unit_len, p->d_state, p->d_n, p->d_coef, p->d_dc, p->d_planes, p->d_status,
                   p->d_chain1, p->d_chain2, p->d_chain3, p->d_chain_count, p->d_post, p->d_posts, p->d_unit_nblk };
  for (void *b : bufs) if (b) cudaFree(b);
  delete p;
  return DALIB200_SUCCESS;
} DB_API_CATCH

int dalib200JpegPlanGetInfo(const dalib200JpegPlan *p, int sample, dalib200JpegInfo *info) try {
  DB_CHECK_ARG(p && info && sample >= 0 && sample < p->n, "JpegPlanGetInfo: bad sample index");
  FillInfo(p->parsed[sample], info);
  return DALIB200_SUCCESS;
} DB_API_CATCH

size_t dalib200JpegPlanStagedBytes(const dalib200JpegPlan *p) { return p ? p->desc_bytes + p->raw_bytes : 0; }

int dalib200JpegPlanSetup(dalib200JpegPlan *p, int n, const uint8_t *const *streams, const size_t *lengths, int output_type,
                          int fancy_upsampling) try {
  dalib200JpegParams prm;
  prm.output_type = output_type; prm.fancy_upsampling = fancy_upsampling; prm.dtype = DALIB200_UINT8; prm.adjust_orientation = 0;
  return dalib200JpegPlanSetupEx(p, n, streams, lengths, &prm, nullptr);
} DB_API_CATCH

int dalib200JpegPlanSetPlanesOnly(dalib200JpegPlan *p, const uint8_t *want, uint8_t *granted) try {
  DB_CHECK_ARG(p && p->staged && want && granted, "JpegPlanSetPlanesOnly: call JpegPlanSetupEx first");
  for (int i = 0; i < p->n; i++) { granted[i] = want[i] && p->geo[i].planar_ok; p->planes_only[i] = granted[i]; }
  BuildWorkLists(p);
  uint8_t *h;
  if (int rc = p->h_stage.Stage(p->desc_bytes, &h)) return rc;
  memcpy(h + p->off_quads, p->first_quad.data(), sizeof(int64_t) * p->n);
  memcpy(h + p->off_items, p->first_item.data(), sizeof(int64_t) * p->n);
  memcpy(h + p->off_work, p->first_work.data(), sizeof(int64_t) * p->n);
  memcpy(h + p->off_fused, p->first_fused.data(), sizeof(int64_t) * p->n);
  return DALIB200_SUCCESS;
} DB_API_CATCH

int dalib200JpegPlanGetPlanes(const dalib200JpegPlan *p, int sample, dalib200PlanarImage *out) try {
  DB_CHECK_ARG(p && out && sample >= 0 && sample < p->n && p->d_planes, "JpegPlanGetPlanes: call JpegLaunch first");
  const JpegImage &im = p->images[sample];
  DB_CHECK_ARG(im.ncomp == 3, "JpegPlanGetPlanes: sample %d has %d components", sample, im.ncomp);
  out->y = p->d_planes + im.plane_off[0]; out->cb = p->d_planes + im.plane_off[1]; out->cr = p->d_planes + im.plane_off[2];
  out->pitch_y = im.plane_w[0]; out->pitch_c = im.plane_w[1];
  out->width = im.width; out->height = im.height;
  out->crop_x = 0; out->crop_y = 0;
  return DALIB200_SUCCESS;
} DB_API_CATCH

int dalib200JpegPlanGetOutputShape(const dalib200JpegPlan *p, int sample, int32_t *hwc) try {
  DB_CHECK_ARG(p && hwc && sample >= 0 && sample < p->n, "JpegPlanGetOutputShape: bad sample index");
  for (int d = 0; d < 3; d++) hwc[d] = p->out_shape[3 * sample + d];
  return DALIB200_SUCCESS;
} DB_API_CATCH

int dalib200JpegPlanSetupEx(dalib200JpegPlan *p, int n, const uint8_t *const *streams, const size_t *lengths,
                            const dalib200JpegParams *prm, const dalib200JpegRoi *rois) try {
  DB_CHECK_ARG(p && prm && (n == 0 || (streams && lengths)) && n >= 0, "JpegPlanSetup: null argument");
  DB_CHECK_ARG(n <= p->max_batch, "JpegPlanSetup: batch %d exceeds plan capacity %d", n, p->max_batch);
  const int output_type = prm->output_type, fancy_upsampling = prm->fancy_upsampling;
  DB_CHECK_ARG(output_type == DALIB200_RGB || output_type == DALIB200_BGR || output_type == DALIB200_GRAY || output_type == DALIB200_YCbCr,
               "decoders.image: output_type %d is not supported (RGB, BGR, GRAY, YCbCr)", output_type);
  DB_CHECK_ARG(prm->dtype == DALIB200_UINT8 || prm->dtype == DALIB200_FLOAT, "decoders.image: dtype %d is not supported (UINT8, FLOAT)", prm->dtype);
  p->staged = false;
  p->n = n; p->output_type = output_type; p->fancy = fancy_upsampling != 0;
  p->dtype = prm->dtype; p->adjust_orientation = prm->adjust_orientation != 0;
  p->posts.clear(); p->post_sample.clear(); p->post_off.clear();
  p->out_shape.assign((size_t)3 * n, 0);
  p->planes_only.assign(n, 0);
  p->geo.assign(n, JpegGeo());
  p->first_work.assign(n, 0);
  p->first_fused.assign(n, 0);

  p->parsed.assign(n, ParsedJpeg());
  p->images.assign(n, JpegImage());
  p->units.clear(); p->tables.clear(); p->quants.clear(); p->src_ptr.clear(); p->block_image.clear(); p->wblock_image.clear();
  p->first_quad.assign(n, 0);
  p->first_item.assign(n, 0);
  for (SideStage *st : p->stages()) st->Clear();
  std::map<std::string, int> table_cache, quant_cache;
  size_t raw = 0, clean = 0;
  uint32_t chunks = 0;
  int64_t subseq = 0, coefs = 0, planes = 0;
  int sync_blocks = 0, write_blocks = 0;
  // subsequence size: the longer, the fewer re-decodes until the chains lock onto the MCU phase; aim for >= ~200k
  // subsequences per batch (a full H100 holds 132 x 2048 = 270k threads), between 32 and 256 bytes
  size_t total_len = 0;
  for (int i = 0; i < n; i++) total_len += lengths[i];
  // DALIB200_JPEG_SUBSEQ_BYTES = 32 / 64 / 128 pins the size (rounded down to one of these), e.g. to test each size on small batches
  int log2_bytes = kMaxLog2Sub - 3;
  if (const char *ev = getenv("DALIB200_JPEG_SUBSEQ_BYTES")) {
    const int v = atoi(ev);
    log2_bytes = v >= 128 ? 7 : v >= 64 ? 6 : 5;
  } else {
    while (log2_bytes > 5 && (total_len >> log2_bytes) < 200000) log2_bytes--;
  }
  p->log2_sub = log2_bytes + 3;
  const size_t sub_bytes = (size_t)1 << log2_bytes;
  for (int i = 0; i < n; i++) {
    ParsedJpeg &j = p->parsed[i];
    DB_CHECK_ARG(streams[i] && lengths[i] > 0, "decoders.image: sample %d is empty", i);
    auto sample_error = [&](int rc, const std::string &what) { SetLastError("decoders.image: sample %d: %s", i, what.c_str()); return rc; };
    const Format f = DetectFormat(streams[i], lengths[i]);
    int rc = f != Format::kJpeg ? PlanSideSample(p->stage_of(f), f, streams[i], lengths[i], i, (int64_t)raw, j)
                                : ParseHeaders(streams[i], lengths[i], j, true);
    if (rc) return sample_error(rc, dalib200GetLastError());
    if (f != Format::kJpeg || j.lossless) {
      // PNG, TIFF, WebP, BMP, PNM: no units, subsequences or MCUs, so every JPEG kernel skips the sample; the stage of its format decodes
      // its staged range (the IDAT run, the span of the segments, the VP8 payload, the pixel array or raster) into the decode window.
      // Lossless JPEG: units for U1 - U3 only (the DCT kernels see no unit, subsequence or MCU of the sample); the lossless stage decodes
      // them.  The post pass behind is shared.
      JpegImage &im = p->images[i];
      memset(&im, 0, sizeof(im));
      im.width = j.width; im.height = j.height; im.out_type = output_type;
      im.unit_begin = im.unit_end = (int)p->units.size();
      im.subseq_begin = (int)subseq; im.block_begin = sync_blocks; im.wblock_begin = write_blocks; im.coef_off = coefs;
      if (j.lossless) {
        std::string err;
        rc = p->ljpeg.Plan(LosslessFrame(j), i, streams[i], lengths[i], j.scan_begin, raw, p->units, clean, chunks, &j.scan_end, &err);
        if (rc) return sample_error(rc, err);
        j.format = Format::kLossless;
      }
      if ((rc = PlanGeometry(p, i, rois, j, im))) return rc;
      p->src_ptr.push_back(streams[i] + j.scan_begin);
      raw += Align(j.scan_end - j.scan_begin, 16);
      continue;
    }
    auto unsupported = [&](const char *what) { return sample_error(DALIB200_ERROR_UNSUPPORTED, what); };
    // multi-scan streams -- progressive, or a sequential frame whose components come in separate scans -- take the scan-by-scan entropy
    // stage (jpeg_prog.cu); `prog` below means exactly that
    const bool prog = j.progressive || (j.ncomp > 1 && j.scan_ncomp != j.ncomp);
    if (prog) {
      // the frame layout comes from the frame header: the first scan of a progressive stream need not name every component, and its
      // Huffman tables are only the first of several snapshots (jpeg_prog_plan.h walks all scans below)
      j.scan_ncomp = j.ncomp;
      for (int c = 0; c < j.ncomp; c++) { j.scan_comp[c] = c; j.td[c] = j.ta[c] = 0; }
    }
    if ((int64_t)j.width * j.height >= (1ll << 31)) return unsupported("images of 2^31 pixels or more are not supported");
    if (j.precision != 8) return unsupported("only 8-bit baseline JPEG is supported");
    if (j.ncomp != 1 && j.ncomp != 3 && j.ncomp != 4) return unsupported("only 1-, 3- or 4-component JPEG is supported");
    if (j.scan_ncomp != j.ncomp) return unsupported("multi-scan (non-interleaved) baseline JPEG is not supported yet");
    if (j.ncomp == 3)
      for (int c = 1; c < j.ncomp; c++)
        if (j.hs[c] != 1 || j.vs[c] != 1) return unsupported("chroma sampling factors other than 1x1 are not supported");
    if (j.ncomp == 4)              // every component is upsampled by whole factors (CMYK / YCCK: each component may have its own)
      for (int c = 0; c < j.ncomp; c++)
        if (j.hmax % j.hs[c] || j.vmax % j.vs[c]) return unsupported("non-integral component sampling ratios are not supported");
    if (j.ncomp == 1) { j.hs[0] = j.vs[0] = 1; j.hmax = j.vmax = 1; }     // a single-component scan is never interleaved
    if (!(j.hmax == 1 || j.hmax == 2 || j.hmax == 4) || !(j.vmax == 1 || j.vmax == 2)) return unsupported("unsupported luma sampling factor");
    JpegImage &im = p->images[i];
    memset(&im, 0, sizeof(im));
    im.width = j.width; im.height = j.height; im.ncomp = j.ncomp;
    im.hmax = j.hmax; im.vmax = j.vmax;
    im.mcux = (j.width + 8 * j.hmax - 1) / (8 * j.hmax);
    im.mcuy = (j.height + 8 * j.vmax - 1) / (8 * j.vmax);
    im.restart_interval = prog ? 0 : j.restart_interval;      // progressive: the DC values arrive as one run of differences (jpeg_prog_core.h)
    im.out_type = output_type; im.fancy = p->fancy;
    if (j.ncomp == 1) im.color = kColorGray;
    else if (j.ncomp == 4) im.color = j.adobe_transform > 0 ? kColorYCCK : kColorCMYK;
    else im.color = j.adobe_transform == 0 || (j.adobe_transform < 0 && !j.jfif && j.cid[0] == 'R' && j.cid[1] == 'G' && j.cid[2] == 'B')
                    ? kColorRGB : kColorYCbCr;
    int bpm = 0;
    for (int si = 0; si < j.scan_ncomp; si++) {
      const int c = j.scan_comp[si];
      im.hs[c] = j.hs[c]; im.vs[c] = j.vs[c]; im.tq[c] = j.tq[c];
      // multi-scan: each component's table is the one defined when its first scan starts (the planner checks it below)
      if (!prog && !j.qt_present[j.tq[c]]) { SetLastError("decoders.image: sample %d: missing quantisation table", i); return DALIB200_ERROR_BAD_DATA; }
      if (j.td[si] > 1 || j.ta[si] > 1) return unsupported("Huffman table ids above 1 are not supported (baseline allows 0..1)");
      if (!prog && (!j.dc[j.td[si]].present || !j.ac[j.ta[si]].present)) { SetLastError("decoders.image: sample %d: missing Huffman table", i); return DALIB200_ERROR_BAD_DATA; }
      for (int v = 0; v < j.vs[c]; v++)
        for (int h = 0; h < j.hs[c]; h++) {
          if (bpm >= kMaxBlocksPerMcu) return unsupported("too many blocks per MCU");
          im.blk_comp[bpm] = c; im.blk_dc[bpm] = j.td[si]; im.blk_ac[bpm] = 2 + j.ta[si]; im.blk_x[bpm] = h; im.blk_y[bpm] = v;
          bpm++;
        }
    }
    im.bpm = bpm;
    // Huffman tables (dedup by content)
    {
      std::string key;
      if (prog) key = "progressive";            // never read by a kernel: the image has no units; one zeroed set keeps the index valid
      else
      for (int t = 0; t < 2; t++) { key.append(reinterpret_cast<const char *>(j.dc[t].bits), 17); key.append(reinterpret_cast<const char *>(j.dc[t].vals), 256); key.push_back(j.dc[t].present); }
      if (!prog)
      for (int t = 0; t < 2; t++) { key.append(reinterpret_cast<const char *>(j.ac[t].bits), 17); key.append(reinterpret_cast<const char *>(j.ac[t].vals), 256); key.push_back(j.ac[t].present); }
      auto it = table_cache.find(key);
      if (it == table_cache.end()) {
        TableSet ts;
        if (prog) memset(&ts, 0, sizeof(ts));
        else
        for (int t = 0; t < 2; t++) {
          BuildDeviceTable(j.dc[t].bits, j.dc[t].vals, ts.lut + LutOffset(t), ts.slow[t], true);
          BuildDeviceTable(j.ac[t].bits, j.ac[t].vals, ts.lut + LutOffset(2 + t), ts.slow[2 + t], false);
        }
        p->tables.push_back(ts);
        it = table_cache.emplace(key, (int)p->tables.size() - 1).first;
      }
      im.table_set = it->second;
    }
    auto set_quant = [&](const uint16_t (*qt)[64]) {         // quantisation tables, deduplicated by content
      std::string qk(reinterpret_cast<const char *>(qt), sizeof(QuantSet::q));
      auto qi = quant_cache.find(qk);
      if (qi == quant_cache.end()) {
        QuantSet qs; memcpy(qs.q, qt, sizeof(qs.q));
        p->quants.push_back(qs);
        qi = quant_cache.emplace(qk, (int)p->quants.size() - 1).first;
      }
      im.quant_set = qi->second;
    };
    if (!prog) set_quant(j.qt);                              // multi-scan samples: the tables the planner latches, below
    // entropy-coded segment(s)
    const uint8_t *d = streams[i];
    size_t sb = j.scan_begin, se = lengths[i];
    // trim at EOI if present at the very end (common case); otherwise the decoder stops on slot count
    if (se >= sb + 2 && d[se - 2] == 0xFF && d[se - 1] == 0xD9) se -= 2;
    j.scan_end = se;
    const int64_t nmcu = (int64_t)im.mcux * im.mcuy;
    im.unit_begin = (int)p->units.size();
    im.subseq_begin = (int)subseq;
    im.block_begin = sync_blocks;
    im.wblock_begin = write_blocks;
    int32_t local_sub = 0;
    auto add_unit = [&](size_t b, size_t e, int64_t mcu0, int64_t mcus) {
      JpegUnit u;
      memset(&u, 0, sizeof(u));
      u.raw_off = (uint32_t)(raw + (b - sb));
      u.raw_len = (uint32_t)(e - b);
      u.clean_off = (uint32_t)clean;
      u.first_chunk = chunks;
      u.image = i;
      u.first_subseq = local_sub;
      u.nsub_max = (int32_t)((u.raw_len + sub_bytes - 1) / sub_bytes);
      u.slot_base = mcu0 * bpm * 64;
      u.nslots = mcus * bpm * 64;
      clean += Align(u.raw_len + kCleanPad, 16);
      chunks += (u.raw_len + kChunkBytes - 1) / kChunkBytes;
      local_sub += u.nsub_max;
      p->units.push_back(u);
    };
    if (prog) {
      // no units: the scans are planned from the whole stream; their bytes are the staged range [scan_begin, scan_end) like a baseline
      // sample's, so JpegUpload needs no special case
      std::string err;
      uint16_t quant[4][64];
      if ((rc = p->prog.Plan(d, lengths[i], sb, se, i, (int64_t)raw, coefs, im, quant, &err))) return sample_error(rc, err);
      set_quant(quant);                                      // slot c of the set: the table component c latched
      for (int c = 0; c < j.ncomp; c++) im.tq[c] = c;
    } else if (j.restart_interval == 0) {
      add_unit(sb, se, 0, nmcu);
    } else {
      // split at RSTn markers (host scan; only images that carry DRI pay for it)
      size_t b = sb; int64_t mcu0 = 0;
      const uint8_t *q = d + sb, *end = d + se;
      while (true) {
        const uint8_t *f = q < end ? static_cast<const uint8_t *>(memchr(q, 0xFF, end - q)) : nullptr;
        if (!f || f + 1 >= end) break;
        if (f[1] >= 0xD0 && f[1] <= 0xD7) {
          const int64_t mcus = std::min<int64_t>(j.restart_interval, nmcu - mcu0);
          if (mcus > 0) add_unit(b, f - d, mcu0, mcus);
          mcu0 += mcus;
          b = (f - d) + 2; q = f + 2;
        } else {
          q = f + 1;
        }
      }
      if (mcu0 < nmcu) add_unit(b, se, mcu0, std::min<int64_t>(j.restart_interval, nmcu - mcu0));
    }
    im.unit_end = (int)p->units.size();
    im.nsub = local_sub;
    p->src_ptr.push_back(d + sb);
    raw += Align(se - sb, 16);
    subseq += local_sub;
    sync_blocks += (local_sub + kSyncThreads - 1) / kSyncThreads;
    p->block_image.resize(sync_blocks, i);
    write_blocks += (local_sub + kWriteThreads - 1) / kWriteThreads;
    p->wblock_image.resize(write_blocks, i);
    im.coef_off = coefs;
    coefs += nmcu * bpm * 64;
    for (int c = 0; c < j.ncomp; c++) {
      // pitch: a multiple of 16 bytes, so that every plane row can be the source of a TMA bulk copy (resample_planar_kernel)
      im.plane_w[c] = (int)Align((size_t)im.mcux * j.hs[c] * 8, 16); im.plane_h[c] = im.mcuy * j.vs[c] * 8;
      im.plane_off[c] = planes;
      planes += Align((size_t)im.plane_w[c] * im.plane_h[c], 16);
    }
    if ((rc = PlanGeometry(p, i, rois, j, im))) return rc;
    // MCUs the IDCT has to produce: the window plus the neighbours the (fancy) chroma upsampling reads
    {
      const int mw = 8 * j.hmax, mh = 8 * j.vmax, ex = 2 * j.hmax, ey = 2 * j.vmax;
      const int mx0 = std::max(0, im.win_x0 - ex) / mw, mx1 = std::min(im.mcux - 1, (im.win_x0 + im.win_w - 1 + ex) / mw);
      const int my0 = std::max(0, im.win_y0 - ey) / mh, my1 = std::min(im.mcuy - 1, (im.win_y0 + im.win_h - 1 + ey) / mh);
      im.mcu_x0 = mx0; im.mcu_y0 = my0; im.mcu_nx = mx1 - mx0 + 1; im.mcu_ny = my1 - my0 + 1;
    }
  }
  BuildWorkLists(p);
  p->prog.SortWaves();
  DB_CHECK_ARG(raw < (1ull << 32) && clean < (1ull << 32), "decoders.image: batch of encoded data exceeds 4 GiB");
  p->raw_bytes = raw; p->clean_bytes = clean; p->nchunks = chunks;
  DB_CHECK_ARG(p->tiff.segs.size() < (1ull << 31), "decoders.image: batch of more than 2^31 TIFF segments");
  p->clean_alloc = clean + (clean_read_behind(p->log2_sub) - kCleanPad);
  for (const JpegUnit &u : p->units)       // the clean length is at most raw_len: every load of the Huffman passes stays inside
    if ((size_t)u.clean_off + u.raw_len + clean_read_behind(p->log2_sub) > p->clean_alloc) {
      SetLastError("decoders.image: internal error (clean stream read bound)"); return DALIB200_ERROR_INTERNAL;
    }
  p->total_subseq = subseq; p->total_coefs = coefs; p->total_plane_bytes = planes;
  p->total_blocks_sync = sync_blocks; p->total_blocks_write = write_blocks;
  // ---- pack descriptors + raw scan bytes into pinned staging
  size_t off = 0;
  p->off_images = off; off += Align(sizeof(JpegImage) * n, 16);
  p->off_units = off; off += Align(sizeof(JpegUnit) * p->units.size(), 16);
  p->off_tables = off; off += Align(sizeof(TableSet) * p->tables.size(), 16);
  p->off_quants = off; off += Align(sizeof(QuantSet) * p->quants.size(), 16);
  p->off_quads = off; off += Align(sizeof(int64_t) * n, 16);
  p->off_items = off; off += Align(sizeof(int64_t) * n, 16);
  p->off_work = off; off += Align(sizeof(int64_t) * n, 16);
  p->off_fused = off; off += Align(sizeof(int64_t) * n, 16);
  p->off_blkimg = off; off += Align(sizeof(int32_t) * p->block_image.size(), 16);
  p->off_wblkimg = off; off += Align(sizeof(int32_t) * p->wblock_image.size(), 16);
  p->off_raw = off;
  p->desc_bytes = off;
  uint8_t *h;
  if (int rc = p->h_stage.Stage(off + raw + 64, &h)) return rc;
  memcpy(h + p->off_units, p->units.data(), sizeof(JpegUnit) * p->units.size());
  memcpy(h + p->off_tables, p->tables.data(), sizeof(TableSet) * p->tables.size());
  memcpy(h + p->off_quants, p->quants.data(), sizeof(QuantSet) * p->quants.size());
  memcpy(h + p->off_quads, p->first_quad.data(), sizeof(int64_t) * n);
  memcpy(h + p->off_items, p->first_item.data(), sizeof(int64_t) * n);
  memcpy(h + p->off_work, p->first_work.data(), sizeof(int64_t) * n);
  memcpy(h + p->off_fused, p->first_fused.data(), sizeof(int64_t) * n);
  memcpy(h + p->off_blkimg, p->block_image.data(), sizeof(int32_t) * p->block_image.size());
  memcpy(h + p->off_wblkimg, p->wblock_image.data(), sizeof(int32_t) * p->wblock_image.size());
  // the scan bytes themselves are staged by JpegUpload, chunk by chunk, so that the H2D copy starts while later samples
  // are still being copied into the pinned buffer
  p->stage_off.resize(n);
  {
    size_t o = 0;
    for (int i = 0; i < n; i++) { p->stage_off[i] = o; o += Align(p->parsed[i].scan_end - p->parsed[i].scan_begin, 16); }
  }
  p->staged = true;
  return DALIB200_SUCCESS;
} DB_API_CATCH

// test / debug accessor: quantised coefficients of one sample after DC prediction, MCU order, natural order in
// each block.  Synchronises the device.
int dalib200JpegDebugGetCoefficients(dalib200JpegPlan *p, int sample, int16_t *out, size_t count) try {
  DB_CHECK_ARG(p && out && sample >= 0 && sample < p->n && p->d_coef, "JpegDebugGetCoefficients: bad arguments");
  const JpegImage &im = p->images[sample];
  const size_t have = (size_t)im.mcux * im.mcuy * im.bpm * 64;
  DB_CHECK_ARG(count <= have, "JpegDebugGetCoefficients: sample has %zu coefficients", have);
  DB_CUDA(cudaDeviceSynchronize());
  DB_CUDA(cudaMemcpy(out, p->d_coef + im.coef_off, count * sizeof(int16_t), cudaMemcpyDeviceToHost));
  // the DC terms live in the compact per-block array
  std::vector<int16_t> dcs((count + 63) / 64);
  DB_CUDA(cudaMemcpy(dcs.data(), p->d_dc + im.coef_off / 64, dcs.size() * sizeof(int16_t), cudaMemcpyDeviceToHost));
  for (size_t b = 0; b * 64 < count; b++) out[b * 64] = dcs[b];
  return DALIB200_SUCCESS;
} DB_API_CATCH

// per-sample decode status written by the device (0 = ok, 1 = entropy-coded data ended early).  Synchronises.
int dalib200JpegGetStatus(dalib200JpegPlan *p, int32_t *status_out) try {
  DB_CHECK_ARG(p && status_out && p->d_status, "JpegGetStatus: bad arguments");
  DB_CUDA(cudaDeviceSynchronize());
  DB_CUDA(cudaMemcpy(status_out, p->d_status, sizeof(int32_t) * p->n, cudaMemcpyDeviceToHost));
  return DALIB200_SUCCESS;
} DB_API_CATCH

// Asynchronous variant: enqueues the copy of the per-sample status words into a pinned buffer of the plan; JpegStatusFetch reads
// that buffer without synchronising (valid once the stream has been synchronised by the caller, e.g. at Pipeline outputs()).
int dalib200JpegStatusAsync(dalib200JpegPlan *p, dalib200Stream_t stream) try {
  DB_CHECK_ARG(p && p->d_status, "JpegStatusAsync: nothing has been launched");
  if ((size_t)p->n > p->h_status_cap) {
    if (p->h_status) cudaFreeHost(p->h_status);
    p->h_status = nullptr; p->h_status_cap = 0;
    DB_CUDA(cudaMallocHost(reinterpret_cast<void **>(&p->h_status), sizeof(int32_t) * p->max_batch));
    p->h_status_cap = p->max_batch;
  }
  DB_CUDA(cudaMemcpyAsync(p->h_status, p->d_status, sizeof(int32_t) * p->n, cudaMemcpyDeviceToHost, stream));
  return DALIB200_SUCCESS;
} DB_API_CATCH

int dalib200JpegStatusFetch(const dalib200JpegPlan *p, int32_t *status_out, int n) try {
  DB_CHECK_ARG(p && status_out && p->h_status && n <= (int)p->h_status_cap, "JpegStatusFetch: call JpegStatusAsync first");
  for (int i = 0; i < n; i++) status_out[i] = p->h_status[i];
  return DALIB200_SUCCESS;
} DB_API_CATCH

int dalib200JpegPlanSetSourceStable(dalib200JpegPlan *p, int stable) try {
  DB_CHECK_ARG(p, "JpegPlanSetSourceStable: null plan");
  p->source_stable = stable != 0;
  return DALIB200_SUCCESS;
} DB_API_CATCH

int dalib200JpegPlanLastUploadDirect(const dalib200JpegPlan *p) { return p ? p->last_upload_direct : -1; }

int dalib200JpegUpload(dalib200JpegPlan *p, dalib200Stream_t stream) try {
  DB_CHECK_ARG(p && p->staged, "JpegUpload: call JpegPlanSetup first");
  if (p->n == 0) return DALIB200_SUCCESS;
  const size_t total = p->desc_bytes + p->raw_bytes;
  int rc = GrowDevice(p->d_stage, p->d_stage_cap, total + 64);
  if (rc) return rc;
  uint8_t *h;
  if ((rc = p->h_stage.Stage(total, &h))) return rc;
  // output pointers are patched at launch: images are uploaded there.  Descriptors and tables go first ...
  DB_CUDA(cudaMemcpyAsync(p->d_stage + p->off_units, h + p->off_units, p->off_raw - p->off_units, cudaMemcpyHostToDevice, stream));
  if ((rc = p->h_stage.Record(stream))) return rc;
  // Sources the caller declared stable (JpegPlanSetSourceStable) AND that are page-locked go to the device without the host
  // repack: one DMA per sample straight from the caller's buffer (no CPU memcpy, no bounce buffer -- with N ranks on one host
  // the repack of N x 100 MB per batch would otherwise saturate the host's memory system).  The kernels never read the padding
  // behind a sample (load_raw_word is bounded by raw_len), so it is left as it is.
  p->last_upload_direct = 0;
  if (p->source_stable) {
    bool pinned = true;
    for (int i = 0; i < p->n && pinned; i++) {
      cudaPointerAttributes a;
      if (cudaPointerGetAttributes(&a, p->src_ptr[i]) != cudaSuccess) { cudaGetLastError(); pinned = false; }
      else pinned = a.type == cudaMemoryTypeHost;
    }
    if (pinned) {
      // one batched submission for all samples (cudaMemcpyBatchAsync, CUDA 12.8+): 256 cudaMemcpyAsync calls cost milliseconds
      // of host time per batch; the per-sample loop below stays as the fallback when the driver rejects the batch call
      static bool batch_api_ok = getenv("DALIB200_NO_MEMCPY_BATCH") == nullptr;
      if (batch_api_ok && p->n > 1) {
        std::vector<void *> dsts(p->n), srcs(p->n);
        std::vector<size_t> sizes(p->n);
        for (int i = 0; i < p->n; i++) {
          dsts[i] = p->d_stage + p->off_raw + p->stage_off[i];
          srcs[i] = const_cast<uint8_t *>(p->src_ptr[i]);
          sizes[i] = p->parsed[i].scan_end - p->parsed[i].scan_begin;
        }
        cudaMemcpyAttributes attr;
        memset(&attr, 0, sizeof(attr));
        attr.srcAccessOrder = cudaMemcpySrcAccessOrderStream;
        size_t attr_idx = 0, fail_idx = 0;
        const cudaError_t e = cudaMemcpyBatchAsync(dsts.data(), srcs.data(), sizes.data(), (size_t)p->n, &attr, &attr_idx, 1, &fail_idx, stream);
        if (e == cudaSuccess) {
          p->last_upload_direct = 2;
          return DALIB200_SUCCESS;
        }
        cudaGetLastError();
        batch_api_ok = false;
      }
      for (int i = 0; i < p->n; i++) {
        const size_t len = p->parsed[i].scan_end - p->parsed[i].scan_begin;
        // neighbours in one arena (sample i + 1 starts where the device layout expects it): merged into one copy
        int j = i;
        size_t run = len;
        while (j + 1 < p->n && p->src_ptr[j + 1] == p->src_ptr[i] + (p->stage_off[j + 1] - p->stage_off[i])) {
          j++;
          run = (p->stage_off[j] - p->stage_off[i]) + (p->parsed[j].scan_end - p->parsed[j].scan_begin);
        }
        DB_CUDA(cudaMemcpyAsync(p->d_stage + p->off_raw + p->stage_off[i], p->src_ptr[i], run, cudaMemcpyHostToDevice, stream));
        i = j;
      }
      p->last_upload_direct = 1;
      return DALIB200_SUCCESS;
    }
  }
  // ... then the scan bytes in groups of ~8 MB: worker threads copy the samples into the pinned buffer in index order, the
  // calling thread issues the H2D copy of a group as soon as its last sample has landed (staging and PCIe transfer overlap).
  {
    const int n = p->n;
    std::vector<int> group_of(n);
    std::vector<int> group_cnt;
    std::vector<size_t> group_begin;
    size_t acc = 0;
    for (int i = 0; i < n; i++) {
      if (group_cnt.empty() || acc >= (8u << 20)) { group_cnt.push_back(0); group_begin.push_back(p->stage_off[i]); acc = 0; }
      group_of[i] = (int)group_cnt.size() - 1;
      group_cnt.back()++;
      acc += p->parsed[i].scan_end - p->parsed[i].scan_begin;
    }
    const int G = (int)group_cnt.size();
    std::vector<std::atomic<int>> done(G);
    for (auto &d : done) d.store(0);
    std::atomic<int> next{0};
    auto work = [&]() {
      for (int i; (i = next.fetch_add(1)) < n;) {
        const size_t len = p->parsed[i].scan_end - p->parsed[i].scan_begin;
        uint8_t *dstp = h + p->off_raw + p->stage_off[i];
        memcpy(dstp, p->src_ptr[i], len);
        memset(dstp + len, 0, Align(len, 16) - len);
        done[group_of[i]].fetch_add(1, std::memory_order_release);
      }
    };
    const int nthreads = std::max(1, std::min<int>({ (int)std::thread::hardware_concurrency() - 1, 12, n }));
    std::vector<std::thread> th;
    if (p->raw_bytes >= (1u << 20)) for (int t = 0; t < nthreads; t++) th.emplace_back(work);
    else work();
    cudaError_t err = cudaSuccess;
    for (int g = 0; g < G; g++) {
      while (done[g].load(std::memory_order_acquire) < group_cnt[g]) std::this_thread::yield();
      const size_t b0 = group_begin[g], b1 = g + 1 < G ? group_begin[g + 1] : p->raw_bytes;
      if (err == cudaSuccess && b1 > b0)
        err = cudaMemcpyAsync(p->d_stage + p->off_raw + b0, h + p->off_raw + b0, b1 - b0, cudaMemcpyHostToDevice, stream);
    }
    for (auto &t : th) t.join();
    if ((rc = p->h_stage.Record(stream))) return rc;      // behind the groups enqueued before a failed copy too
    DB_CUDA(err);
  }
  return DALIB200_SUCCESS;
} DB_API_CATCH

int dalib200JpegLaunch(dalib200JpegPlan *p, void *const *out_ptrs, dalib200Stream_t stream) try {
  DB_CHECK_ARG(p && p->staged && out_ptrs, "JpegLaunch: call JpegPlanSetup / JpegUpload first");
  if (p->n == 0) return DALIB200_SUCCESS;
  DB_CHECK_ARG(p->d_stage && p->d_stage_cap >= p->desc_bytes + p->raw_bytes, "JpegLaunch: JpegUpload has not been called for this batch");
  int rc;
  if ((rc = GrowDevice(p->d_clean, p->d_clean_cap, p->clean_alloc))) return rc;
  if ((rc = GrowDevice(p->d_chunk, p->d_chunk_cap, (size_t)p->nchunks + 1))) return rc;
  if ((rc = GrowDevice(p->d_unit_len, p->d_unit_cap, p->units.size() + 1))) return rc;
  {
    size_t cap2 = p->d_sub_cap;
    if ((rc = GrowDevice(p->d_state, p->d_sub_cap, (size_t)p->total_subseq + 1))) return rc;
    if ((rc = GrowDevice(p->d_n, cap2, (size_t)p->total_subseq + 1))) return rc;
  }
  if ((rc = GrowDevice(p->d_chain1, p->d_chain1_cap, (size_t)p->total_subseq + 1))) return rc;
  if ((rc = GrowDevice(p->d_chain2, p->d_chain2_cap, (size_t)p->total_subseq + 1))) return rc;
  if ((rc = GrowDevice(p->d_chain3, p->d_chain3_cap, (size_t)p->total_subseq + 1))) return rc;
  if ((rc = GrowDevice(p->d_chain_count, p->d_chain_count_cap, (size_t)8 + p->n))) return rc;     // chain counts, then chain_cut
  if ((rc = GrowDevice(p->d_coef, p->d_coef_cap, (size_t)p->total_coefs + 64))) return rc;
  if ((rc = GrowDevice(p->d_dc, p->d_dc_cap, (size_t)p->total_coefs / 64 + 64))) return rc;
  if ((rc = GrowDevice(p->d_planes, p->d_planes_cap, (size_t)p->total_plane_bytes + 64))) return rc;
  if ((rc = GrowDevice(p->d_status, p->d_status_cap, (size_t)p->n + 1))) return rc;
  if ((rc = GrowDevice(p->d_unit_nblk, p->d_unit_nblk_cap, p->units.size() + 1))) return rc;
  if (!p->posts.empty()) {
    if ((rc = GrowDevice(p->d_post, p->d_post_cap, p->post_bytes + 256))) return rc;
    if ((rc = GrowDevice(p->d_posts, p->d_posts_cap, p->posts.size()))) return rc;
  }
  // image descriptors carry the output pointers: small separate upload from their own pinned buffer (waiting on the event of
  // the big bit-stream copy here would stall the host for the whole H2D transfer)
  JpegImage *hi;                            // the output pointers of this launch
  {
    const size_t img_bytes = Align(sizeof(JpegImage) * p->n, 16);
    if ((rc = p->h_images.Stage(img_bytes + sizeof(JpegPost) * p->posts.size(), &hi))) return rc;
    for (int i = 0; i < p->n; i++) { hi[i] = p->images[i]; hi[i].out = static_cast<uint8_t *>(out_ptrs[i]); }
    JpegPost *hp = reinterpret_cast<JpegPost *>(reinterpret_cast<uint8_t *>(hi) + img_bytes);
    for (size_t k = 0; k < p->posts.size(); k++) {
      const int i = p->post_sample[k];
      hp[k] = p->posts[k];
      hp[k].src = p->d_post + p->post_off[k];
      hp[k].dst = out_ptrs[i];
      hi[i].out = p->d_post + p->post_off[k];              // the decoder writes the window into scratch
    }
    cudaError_t e = cudaMemcpyAsync(p->d_stage + p->off_images, hi, sizeof(JpegImage) * p->n, cudaMemcpyHostToDevice, stream);
    if (e == cudaSuccess && !p->posts.empty())
      e = cudaMemcpyAsync(p->d_posts, hp, sizeof(JpegPost) * p->posts.size(), cudaMemcpyHostToDevice, stream);
    if ((rc = p->h_images.Record(stream))) return rc;
    DB_CUDA(e);
  }
  const auto *d_images = reinterpret_cast<const JpegImage *>(p->d_stage + p->off_images);
  const auto *d_units = reinterpret_cast<const JpegUnit *>(p->d_stage + p->off_units);
  const auto *d_tables = reinterpret_cast<const TableSet *>(p->d_stage + p->off_tables);
  const auto *d_quants = reinterpret_cast<const QuantSet *>(p->d_stage + p->off_quants);
  const auto *d_quads = reinterpret_cast<const int64_t *>(p->d_stage + p->off_quads);
  const auto *d_items = reinterpret_cast<const int64_t *>(p->d_stage + p->off_items);
  const uint8_t *d_raw = p->d_stage + p->off_raw;
  const int nunits = (int)p->units.size();
  const int sms = NumSMs();
  cudaStream_t s = stream;
  // (the clean stream is zero-padded behind every unit by the scatter kernel itself: no memset of the 129 MB buffer)
  DB_CUDA(cudaMemsetAsync(p->d_status, 0, sizeof(int32_t) * p->n, s));
  DB_CUDA(cudaMemsetAsync(p->d_chain_count, 0, sizeof(uint32_t) * (8 + p->n), s));
  const StageInputs in{ hi, d_raw, p->d_status, p->d_coef, p->d_dc, p->d_clean, p->d_unit_len };
  if ((rc = p->prog.Run(in, s)) || (rc = p->png.Run(in, s)) || (rc = p->tiff.Run(in, s)) || (rc = p->webp.Run(in, s)) ||
      (rc = p->bitmap.Run(in, s)))
    return rc;
  // any_units: the batch has a baseline sample; lossless samples have units for U1 - U3 but nothing for the baseline entropy kernels
  const bool any_units = nunits > 0 && p->nchunks > 0 && p->total_blocks_sync > 0;
  if (nunits > 0 && p->nchunks > 0) {
    const int grid = (int)std::min<uint32_t>(p->nchunks, (uint32_t)sms * 16);
    Launch("jpeg_unstuff_count", unstuff_count_kernel, grid, 256, 0, s, d_raw, d_units, nunits, p->nchunks, p->d_chunk);
    Launch("jpeg_unstuff_scan", unstuff_scan_kernel, (nunits + 7) / 8, 256, 0, s, d_units, nunits, p->d_chunk, p->d_unit_len);
    Launch("jpeg_unstuff_scatter", unstuff_scatter_kernel, grid, 256, 0, s, d_raw, d_units, nunits, p->nchunks, p->d_chunk, p->d_clean);
  }
  if ((rc = p->ljpeg.Run(in, s))) return rc;            // forked behind U3, whose clean streams it reads
  HuffCtx cx;
  cx.images = d_images; cx.nimages = p->n; cx.block_image = reinterpret_cast<const int32_t *>(p->d_stage + p->off_blkimg);
  cx.wblock_image = reinterpret_cast<const int32_t *>(p->d_stage + p->off_wblkimg);
  cx.units = d_units; cx.unit_clean_len = p->d_unit_len; cx.tables = d_tables;
  cx.clean = p->d_clean; cx.s_state = p->d_state; cx.s_n = p->d_n; cx.coef = p->d_coef; cx.dc = p->d_dc; cx.log2_sub = p->log2_sub;
  cx.status = p->d_status; cx.unit_nblk = p->d_unit_nblk;
  cx.chains[0] = p->d_chain1; cx.chains[1] = p->d_chain2; cx.chains[2] = p->d_chain3; cx.chain_count = p->d_chain_count;
  cx.chain_cut = p->d_chain_count + 8;
  const size_t hsmem = sync_smem_bytes(p->log2_sub, false), wsmem = write_smem_bytes();
  const size_t walk_smem = kLutWords * 4 + 4 * sizeof(HuffSlow) + (size_t)(kTailColWords + kMaxBlocksPerMcu) * kTailThreads * 4;
  if (!p->smem_opted) {
    DB_CUDA(cudaFuncSetAttribute(huff_sync_intra_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sync_smem_bytes(kMaxLog2Sub, false)));
    DB_CUDA(cudaFuncSetAttribute(huff_write_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)wsmem));
    DB_CUDA(cudaFuncSetAttribute(huff_sync_walk_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)walk_smem));
    int per_sm = 0;
    DB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, huff_sync_walk_kernel, kTailThreads, walk_smem));
    p->walk_max_grid = std::max(1, per_sm) * sms * 4;
    p->smem_opted = true;
  }
  if (any_units) {
    Launch("jpeg_huff_sync_intra", huff_sync_intra_kernel, p->total_blocks_sync, kSyncThreads, hsmem, s, cx);
    // chain walk: grids sized for the expected list lengths (about 30 % / 8 % / 2.5 % of the subsequences carry a live chain
    // after 1 / 2 / 3 visits); CTAs beyond the actual length return at once, grid-stride loops cover longer lists
    auto walk_grid = [&](double frac) {
      const int64_t want = (int64_t)(p->total_subseq * frac) / kTailThreads + p->total_blocks_sync / kTailThreads + 1;
      return (int)std::max<int64_t>(1, std::min<int64_t>(p->walk_max_grid, want));
    };
    Launch("jpeg_huff_sync_walk1", huff_sync_walk_kernel, walk_grid(0.40), kTailThreads, walk_smem, s, cx, 0, 1, 1);
    Launch("jpeg_huff_sync_walk2", huff_sync_walk_kernel, walk_grid(0.14), kTailThreads, walk_smem, s, cx, 1, 2, 1);
    Launch("jpeg_huff_sync_walk3", huff_sync_walk_kernel, walk_grid(0.06), kTailThreads, walk_smem, s, cx, 2, 0, 1 << 30);
  }
  Launch("jpeg_huff_scan", huff_scan_kernel, p->n, 1024, 0, s, cx);
  if (any_units && p->total_blocks_write > 0) Launch("jpeg_huff_write", huff_write_kernel, p->total_blocks_write, kWriteThreads, wsmem, s, cx);
  if ((rc = p->prog.Join(s))) return rc;                // the progressive samples' coefficients and DC differences are in place
  Launch("jpeg_dc_scan", dc_scan_kernel, p->n, 1024, 0, s, d_images, p->d_dc);
  Launch("jpeg_truncation_fixup", truncation_fixup_kernel, p->n, 256, 0, s, cx);
  {
    ReconLaunch ra;
    ra.d_images = d_images; ra.nimages = p->n;
    ra.totals.work = p->total_work; ra.totals.fused = p->total_fused; ra.totals.quads = p->total_quads; ra.totals.items = p->total_items;
    ra.d_first_work = reinterpret_cast<const int64_t *>(p->d_stage + p->off_work);
    ra.d_first_fused = reinterpret_cast<const int64_t *>(p->d_stage + p->off_fused);
    ra.d_first_quad = d_quads; ra.d_first_item = d_items;
    ra.d_coef = p->d_coef; ra.d_dc = p->d_dc; ra.d_quants = d_quants; ra.d_planes = p->d_planes;
    if ((rc = LaunchReconstruct(ra, s))) return rc;
  }
  // the other stages' decode windows and status words are in place
  if ((rc = p->png.Join(s)) || (rc = p->tiff.Join(s)) || (rc = p->webp.Join(s)) || (rc = p->bitmap.Join(s)) || (rc = p->ljpeg.Join(s)))
    return rc;
  if (!p->posts.empty()) {
    const int grid = (int)std::max<int64_t>(1, std::min<int64_t>((p->total_post_px + 255) / 256, (int64_t)sms * 16));
    Launch("jpeg_post", p->dtype == DALIB200_FLOAT ? jpeg_post_kernel<float> : jpeg_post_kernel<uint8_t>, grid, 256, 0, s, p->d_posts, (int)p->posts.size(),
           p->total_post_px);
  }
  DB_CUDA(cudaGetLastError());
  return DALIB200_SUCCESS;
} DB_API_CATCH

}  // extern "C"
