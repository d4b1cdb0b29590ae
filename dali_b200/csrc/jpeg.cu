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
// The plan also takes PNG, TIFF and lossy WebP streams (detected by their signatures): png_plan.h walks their chunks, tiff_plan.h their
// IFD and webp_plan.h their RIFF chunks and VP8 headers at set-up, png.cu, tiff.cu and webp.cu decode them into the same decode windows
// on streams of their own, and the post pass below serves every format.  A PNG, TIFF or WebP sample has no units, subsequences or MCUs,
// so every kernel of this file skips it.
#include "common.cuh"
#include "jpeg_recon.h"
#include <algorithm>
#include <cstring>
#include <map>
#include <thread>

namespace dalib200 {

constexpr int kDcLutBits = 9, kAcLutBits = 11;   // first-level Huffman lookup widths (std DC codes are <= 9 bits)
constexpr int kDcLutSize = 1 << kDcLutBits, kAcLutSize = 1 << kAcLutBits;
constexpr int kLutWords = 2 * kDcLutSize + 2 * kAcLutSize;          // DC0 DC1 AC0 AC1 back to back: 20 KB
constexpr int kSyncThreads = 256;            // subsequences per synchronisation block
constexpr int kChunkBytes = 4096;            // un-stuffing chunk
constexpr uint32_t kCleanPad = 32;           // zero bytes behind the clean stream of every unit (at least: units are 16-byte aligned)
constexpr int kMaxLog2Sub = 10;              // largest subsequence: 2^10 bits = 128 bytes

// Huffman tables as the device sees them.  The first-level LUTs (one 32-bit entry per 10-bit prefix, see make_entry) are
// copied to shared memory by every sync block; the canonical tables for longer codes stay in global memory.
constexpr int kLongLut = 512;
struct HuffSlow {
  int32_t maxcode[18];        // T.81 F.2.2.3: maxcode[l] left-aligned to 16 bits (+1)
  int32_t valoff[18];         // valptr[l] - mincode[l]
  uint8_t vals[256];
  // canonical codes grow with their length, so the codes longer than the first-level LUT occupy the top [long_base, 65536) of the
  // left-aligned 16-bit code space -- 192 values for the standard tables.  When that range fits, ONE lookup indexed by
  // (window - long_base) replaces the length search (which ran on a single lane while the warp waited).  Entry = code length | symbol << 8, 0 = not a code.  long_n == 0: use the search.
  int32_t long_base, long_n;
  uint16_t long_lut[kLongLut];
};

struct TableSet {             // the 4 tables a baseline scan can reference: DC0, DC1, AC0, AC1
  uint32_t lut[kLutWords];    // 32-bit entries (make_entry): synchronisation passes
  uint16_t lut16[kLutWords];  // 16-bit entries (make_entry16): write pass (half the shared memory -> 3 x 8 warps more per SM)
  HuffSlow slow[4];
};
__host__ __device__ inline int LutOffset(int t) { return t < 2 ? t * kDcLutSize : 2 * kDcLutSize + (t - 2) * kAcLutSize; }

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

struct JpegUnit {
  uint32_t raw_off, raw_len;               // in the staged byte buffer
  uint32_t clean_off;                      // in the clean buffer (bytes, 16-aligned)
  uint32_t first_chunk;                    // global chunk index
  int32_t image;
  int32_t first_subseq;                    // image-local
  int32_t nsub_max;
  int64_t slot_base;                       // first coefficient slot of this unit (image-local)
  int64_t nslots;                          // expected number of slots (= MCUs * bpm * 64)
};

__constant__ uint8_t c_zigzag[64] = {
   0,  1,  8, 16,  9,  2,  3, 10, 17, 24, 32, 25, 18, 11,  4,  5,
  12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13,  6,  7, 14, 21, 28,
  35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51,
  58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63 };

// ============================================================================================
// U1..U3: byte un-stuffing
__device__ __forceinline__ int find_unit_by_chunk(const JpegUnit *u, int n, uint32_t chunk) {
  int lo = 0, hi = n - 1;
  while (lo < hi) {
    int mid = (lo + hi + 1) >> 1;
    if (u[mid].first_chunk <= chunk) lo = mid; else hi = mid - 1;
  }
  return lo;
}

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
  if (threadIdx.x == 0) s_ui = find_unit_by_chunk(units, nunits, ch0);
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
  if (threadIdx.x == 0) s_ui = find_unit_by_chunk(units, nunits, ch0);
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
constexpr uint64_t kStateMask = (1ull << 42) - 1;
constexpr uint32_t kMaxChainLen = 4095;
__device__ __forceinline__ uint64_t pack_state(uint32_t p, int c, int z, uint32_t cnt = 0, uint32_t t = 0) {
  return (uint64_t)p | ((uint64_t)(uint32_t)c << 32) | ((uint64_t)(uint32_t)z << 36) | ((uint64_t)min(cnt, 1023u) << 42) | ((uint64_t)t << 52);
}
__device__ __forceinline__ uint32_t state_count(uint64_t s) { return (uint32_t)(s >> 42) & 1023u; }

// LUT entry (host: MakeLutEntry): [4:0] bits consumed (code + magnitude, <= 31), [11:8] magnitude size s, [16:12] code
// length, [26:20] zig-zag advance (run + 1; 16 for ZRL; 64 for EOB; 1 for DC).  0 = code longer than the first-level width.
// The funnel shifts of the bit window take the entry register itself as the shift amount (shf.wrap masks it to 5 bits),
// which keeps the loop-carried dependency at LDS -> SHF -> SHF -> LEA -> LDS.
__device__ __forceinline__ uint32_t make_entry(uint32_t len, uint32_t sym, bool is_dc) {
  const uint32_t s = sym & 15u, r = sym >> 4;
  const uint32_t adv = is_dc ? 1u : (s == 0 ? (r == 15u ? 16u : 64u) : r + 1u);
  return (len + s) | (s << 8) | (len << 12) | (adv << 20);
}

// 16-bit entry of the write pass (host: MakeLutEntry16): [4:0] bits consumed, [8:5] magnitude size s, [15:9] zig-zag advance;
// code length = consumed - s.  0 = code longer than the first-level width.
__device__ __forceinline__ uint32_t make_entry16(uint32_t len, uint32_t sym, bool is_dc) {
  const uint32_t s = sym & 15u, r = sym >> 4;
  const uint32_t adv = is_dc ? 1u : (s == 0 ? (r == 15u ? 16u : 64u) : r + 1u);
  return (len + s) | (s << 5) | (adv << 9);
}

// codes longer than the first-level LUT (std tables: AC codes of 12..16 bits, < 1 % of the symbols): canonical search,
// T.81 F.2.2.3.  `toff` = LUT word offset of the table, which identifies it.  Returns code length | symbol << 8.
__device__ __noinline__ uint32_t slow_lookup(const HuffSlow *__restrict__ slow, uint32_t toff, uint32_t hi, bool is_dc) {
  const int tbl = toff < 2u * kDcLutSize ? (int)(toff / kDcLutSize) : 2 + (int)((toff - 2u * kDcLutSize) / kAcLutSize);
  const HuffSlow *sl = slow + tbl;
  const int32_t code16 = (int32_t)(hi >> 16);
  if (sl->long_n > 0) {
    const int idx = min(max(code16 - sl->long_base, 0), sl->long_n - 1);
    const uint32_t e = sl->long_lut[idx];
    return e ? e : 16u;                                      // corrupt / speculative: keep going deterministically (length 16, symbol 0)
  }
  uint32_t len = (is_dc ? kDcLutBits : kAcLutBits) + 1;
  while (len <= 16 && code16 >= sl->maxcode[len]) len++;
  uint32_t sym = 0;
  if (len > 16) len = 16;                                    // corrupt / speculative: keep going deterministically
  else sym = sl->vals[(sl->valoff[len] + (code16 >> (16 - len))) & 0xFF];
  return len | (sym << 8);
}
__device__ __forceinline__ uint32_t slow_symbol(const HuffSlow *__restrict__ slow, uint32_t toff, uint32_t hi, bool is_dc) {
  const uint32_t ls = slow_lookup(slow, toff, hi, is_dc);
  return make_entry(ls & 0xFFu, ls >> 8, is_dc);
}
__device__ __forceinline__ uint32_t slow_symbol16(const HuffSlow *__restrict__ slow, uint32_t toff, uint32_t hi, bool is_dc) {
  const uint32_t ls = slow_lookup(slow, toff, hi, is_dc);
  return make_entry16(ls & 0xFFu, ls >> 8, is_dc);
}

// Decodes the symbols that START before `end` (absolute bit positions inside the unit) without producing coefficients: the
// synchronisation only needs the state (pos, c, z) and `nb`, the number of completed blocks.  Branch-free apart from the loop
// and the rare long-code path.
template <class Win, class Lut, class Tbl>
__device__ __forceinline__ void decode_span(Win &win, const Lut &lut, const HuffSlow *__restrict__ slow,
                                            const Tbl &tbl, int bpm, uint32_t &pos, uint32_t end, int &c, int &z, uint32_t &nb) {
  uint32_t tb12 = tbl.load(c);                                // dc table offset | ac table offset << 16 (in LUT words)
  while (pos < end) {
    // the AC entry is fetched before z is known (it is the common case and sits on the loop-carried path); the DC entry only
    // by the lanes that start a block, so that its random-bank lookup costs one shared-memory wavefront instead of three
    const uint32_t e_ac = lut.load((tb12 >> 16) + (win.hi >> (32 - kAcLutBits)));
    const bool is_dc = z == 0;
    uint32_t e = e_ac;
    if (is_dc) e = lut.load((tb12 & 0xFFFFu) + (win.hi >> (32 - kDcLutBits)));
    if (__builtin_expect(e == 0, 0)) e = slow_symbol(slow, is_dc ? (tb12 & 0xFFFFu) : (tb12 >> 16), win.hi, is_dc);
    const uint32_t tb = e & 31u, adv = e >> 20;
    win.consume(e);
    pos += tb;
    z += (int)adv;
    const bool endb = z >= 64;                                // block finished (EOB, 64th coefficient, or garbage overrun)
    const int c1 = c + 1 == bpm ? 0 : c + 1;
    nb += endb ? 1u : 0u;
    c = endb ? c1 : c;
    z = endb ? 0 : z;
    if (endb) tb12 = tbl.load(c);
  }
}

__device__ __forceinline__ int find_unit_by_subseq(const JpegUnit *u, int ub, int ue, int j) {
  int lo = ub, hi = ue - 1;
  while (lo < hi) {
    int mid = (lo + hi + 1) >> 1;
    if (u[mid].first_subseq <= j) lo = mid; else hi = mid - 1;
  }
  return lo;
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
    sg.ui = im.unit_end - im.unit_begin == 1 ? im.unit_begin : find_unit_by_subseq(cx.units, im.unit_begin, im.unit_end, j);
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
  const int ui = im.unit_end - im.unit_begin == 1 ? im.unit_begin : find_unit_by_subseq(cx.units, im.unit_begin, im.unit_end, j);
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
    if (jl + 1 >= nsub_eff || t >= kMaxChainLen) break;       // end of the unit (or an absurdly long chain: corrupt data)
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

// H2b: one CTA per image: per-unit exclusive scan of the block counts (in place), status check.
__global__ void __launch_bounds__(1024) huff_scan_kernel(HuffCtx cx) {
  __shared__ uint32_t warp_tot[32];
  __shared__ uint32_t carry;
  const JpegImage &im = cx.images[blockIdx.x];
  const uint32_t sub_bits = 1u << cx.log2_sub;
  for (int ui = im.unit_begin; ui < im.unit_end; ui++) {
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
// (word j of lane l at l * 32 + (j ^ l): conflict free for the per-symbol 16-bit scatter of all lanes to the same j and for the
// flush) and the warp writes each finished block to HBM as ONE coalesced 128-byte line: no memset of the coefficient arena,
// no 2-byte read-modify-write traffic, ~12x fewer store wavefronts than a per-symbol scatter.
//
// The loop is a chain of dependent fixed-latency instructions (its stalls are fixed-latency waits and short scoreboards):
// throughput scales with resident warps.  The pass therefore runs its own block shape -- kWriteThreads subsequences per CTA,
// 16-bit LUT entries (10 KB instead of 20) and the stream read from global memory (StreamWindow), so that shared memory holds
// only the tables and the block buffers: 10.1 KB + 128 B per thread.
constexpr int kWriteThreads = 384;
constexpr int kWriteCtasPerSm = 3;       // 3 x (58.1 KB + 1 KB reserved) of the 228 KB per SM
struct WriteSmem {
  uint16_t *lut; uint32_t *tbl, *blkbuf; uint8_t *zig;
};
__host__ __device__ inline size_t write_smem_bytes() { return kLutWords * 2 + 16 * 4 /*tbl*/ + 64 /*zig*/ + (size_t)kWriteThreads * 128; }
__device__ __forceinline__ WriteSmem carve_write_smem(uint32_t *base) {
  WriteSmem s;
  s.lut = reinterpret_cast<uint16_t *>(base);
  s.tbl = base + kLutWords / 2;
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
    const uint4 *src = reinterpret_cast<const uint4 *>(cx.tables[im.table_set].lut16);
    uint4 *dst = reinterpret_cast<uint4 *>(sm.lut);
    for (int i = threadIdx.x; i < kLutWords * 2 / 16; i += blockDim.x) dst[i] = __ldg(src + i);
    if (threadIdx.x < kMaxBlocksPerMcu) sm.tbl[threadIdx.x] = tbl_word(im, threadIdx.x);
    if (threadIdx.x < 64) sm.zig[threadIdx.x] = c_zigzag[threadIdx.x];
  }
  SubGeom sg;
  {
    const int j = (blockIdx.x - im.wblock_begin) * kWriteThreads + threadIdx.x;     // image-local subsequence
    sg.valid = j < im.nsub;
    sg.ui = 0; sg.jl = 0; sg.nsub_eff = 0; sg.clean_bits = 0;
    sg.g = (int64_t)im.subseq_begin + j;
    if (sg.valid) {
      sg.ui = im.unit_end - im.unit_begin == 1 ? im.unit_begin : find_unit_by_subseq(cx.units, im.unit_begin, im.unit_end, j);
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
  uint32_t pos = 0, nb = 0, end = 0, hard_end = 0, blk0 = 0, blk_limit = 0;
  int c = 0, z = 0;
  bool active = sg.valid;
  if (active) {
    const JpegUnit &u = cx.units[sg.ui];
    if (sg.jl > 0) {
      const uint64_t prev = cx.s_state[sg.g - 1];
      pos = (uint32_t)prev; c = (int)((prev >> 32) & 15u); z = (int)((prev >> 36) & 63u);
    }
    end = min((sg.jl + 1) << cx.log2_sub, sg.clean_bits);
    hard_end = sg.clean_bits;
    const uint32_t ublk = (uint32_t)(u.slot_base >> 6);
    blk0 = ublk + cx.s_n[sg.g];
    blk_limit = ublk + (uint32_t)(u.nslots >> 6);
    active = pos < end && blk0 < blk_limit;                  // pad bits behind the last block of a unit are not symbols
  }
  bool own = z == 0;                                          // a block starts exactly at the entry: it is ours
  StreamWindow win;
  win.clear();
  if (active) win.init(cx.clean + cx.units[sg.ui].clean_off, pos);
  __syncthreads();                                            // the tables; the window's first loads are in flight meanwhile
  int16_t *coef = cx.coef + im.coef_off;
  int16_t *dcv = cx.dc + im.coef_off / 64;
  const int bpm = im.bpm;
  uint32_t tb12 = lds_u32(a_tbl + 4u * c);
  for (uint32_t it = 1; __any_sync(0xffffffffu, active); it++) {
    bool flush = false;
    const uint32_t blk = blk0 + nb;
    if (it & 1u) win.top_up();                                // warp-uniform, see StreamWindow
    if (active) {
      const uint32_t e_ac = lds_u16(a_lut + 2u * ((tb12 >> 16) + (win.hi >> (32 - kAcLutBits))));
      const bool is_dc = z == 0;
      uint32_t e = e_ac;
      if (is_dc) e = lds_u16(a_lut + 2u * ((tb12 & 0xFFFFu) + (win.hi >> (32 - kDcLutBits))));
      if (__builtin_expect(e == 0, 0)) e = slow_symbol16(slow, is_dc ? (tb12 & 0xFFFFu) : (tb12 >> 16), win.hi, is_dc);
      const uint32_t tb = e & 31u, adv = e >> 9, s = (e >> 5) & 15u;
      {
        // magnitude bits (EXTEND, T.81 F.2.2.1), computed by every lane: s == 0 gives v == 0
        const uint32_t len = tb - s;
        const uint32_t bits = (uint32_t)(((uint64_t)(win.hi << len)) >> (32u - s));      // 64-bit shift: s == 0 -> 0
        // (measured: a funnel-shift + sign-mask formulation of EXTEND is 3 instructions shorter but made this kernel slower)
        const int v = (int)bits - ((s == 0 || ((bits >> (s - 1u)) & 1u)) ? 0 : (int)((1u << s) - 1u));
        if (own) {
          if (is_dc) {
            dcv[blk] = (int16_t)v;                            // every block has a DC term: the compact array needs no memset
          } else if (s) {
            const uint32_t nat = lds_u8(a_zig + min((uint32_t)z + adv - 1u, 63u));
            sts_u16(a_mybuf + 4u * ((nat >> 1) ^ lane) + 2u * (nat & 1u), (uint32_t)v);
          }
        }
      }
      win.consume(e);
      pos += tb;
      z += (int)adv;
      const bool endb = z >= 64;                              // block finished (EOB, 64th coefficient, or garbage overrun)
      const int c1 = c + 1 == bpm ? 0 : c + 1;
      flush = endb && own;
      nb += endb ? 1u : 0u;
      own = own || endb;                                      // the open block of the entry is over: what follows is ours
      c = endb ? c1 : c;
      z = endb ? 0 : z;
      if (endb) tb12 = lds_u32(a_tbl + 4u * c);
      // keep going while symbols start inside the subsequence, then until the last own block is complete
      active = blk0 + nb < blk_limit && (pos < end || (z != 0 && pos < hard_end));
    }
    // ---- flush the finished blocks of this warp, one coalesced line each
    uint32_t m = __ballot_sync(0xffffffffu, flush);
    while (m) {
      const uint32_t L = __ffs(m) - 1u;
      m &= m - 1u;
      const uint32_t fb = __shfl_sync(0xffffffffu, blk, L);
      const uint32_t a_src = a_wbuf + L * 128u + 4u * (lane ^ L);
      const uint32_t w = lds_u32(a_src);
      sts_u32(a_src, 0u);
      reinterpret_cast<uint32_t *>(coef + (size_t)fb * 64)[lane] = w;
    }
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
// I1: dequantisation + islow IDCT (libjpeg jidctint: CONST_BITS 13, PASS1_BITS 2).  One thread per 8x8 block.
#define FIX_0_298631336 2446
#define FIX_0_390180644 3196
#define FIX_0_541196100 4433
#define FIX_0_765366865 6270
#define FIX_0_899976223 7373
#define FIX_1_175875602 9633
#define FIX_1_501321110 12299
#define FIX_1_847759065 15137
#define FIX_1_961570560 16069
#define FIX_2_053119869 16819
#define FIX_2_562915447 20995
#define FIX_3_072711026 25172

template <int SHIFT>
__device__ __forceinline__ void idct8(int i0, int i1, int i2, int i3, int i4, int i5, int i6, int i7, int *o) {
  int z1, z2, z3, z4, z5, tmp0, tmp1, tmp2, tmp3, tmp10, tmp11, tmp12, tmp13;
  z2 = i2; z3 = i6;
  z1 = (z2 + z3) * FIX_0_541196100;
  tmp2 = z1 + z3 * (-FIX_1_847759065);
  tmp3 = z1 + z2 * FIX_0_765366865;
  z2 = i0; z3 = i4;
  tmp0 = (int)((unsigned)(z2 + z3) << 13);
  tmp1 = (int)((unsigned)(z2 - z3) << 13);
  tmp10 = tmp0 + tmp3; tmp13 = tmp0 - tmp3; tmp11 = tmp1 + tmp2; tmp12 = tmp1 - tmp2;
  tmp0 = i7; tmp1 = i5; tmp2 = i3; tmp3 = i1;
  z1 = tmp0 + tmp3; z2 = tmp1 + tmp2; z3 = tmp0 + tmp2; z4 = tmp1 + tmp3;
  z5 = (z3 + z4) * FIX_1_175875602;
  tmp0 *= FIX_0_298631336; tmp1 *= FIX_2_053119869; tmp2 *= FIX_3_072711026; tmp3 *= FIX_1_501321110;
  z1 *= -FIX_0_899976223; z2 *= -FIX_2_562915447; z3 *= -FIX_1_961570560; z4 *= -FIX_0_390180644;
  z3 += z5; z4 += z5;
  tmp0 += z1 + z3; tmp1 += z2 + z4; tmp2 += z2 + z3; tmp3 += z1 + z4;
  const int r = 1 << (SHIFT - 1);
  o[0] = (tmp10 + tmp3 + r) >> SHIFT; o[7] = (tmp10 - tmp3 + r) >> SHIFT;
  o[1] = (tmp11 + tmp2 + r) >> SHIFT; o[6] = (tmp11 - tmp2 + r) >> SHIFT;
  o[2] = (tmp12 + tmp1 + r) >> SHIFT; o[5] = (tmp12 - tmp1 + r) >> SHIFT;
  o[3] = (tmp13 + tmp0 + r) >> SHIFT; o[4] = (tmp13 - tmp0 + r) >> SHIFT;
}

__device__ __forceinline__ uint32_t range_limit(int x) {     // libjpeg range_limit[(x) & RANGE_MASK], table centred on 128
  // idx = x & 1023: [0,128) -> idx + 128, [128,512) -> 255, [512,896) -> 0, [896,1024) -> idx - 896.  With y = (x + 128) & 1023
  // this is: y < 256 -> y, y < 640 -> 255, else 0.
  const uint32_t y = (uint32_t)(x + 128) & 1023u;
  return y < 640u ? min(y, 255u) : 0u;
}

__device__ __forceinline__ int find_by_prefix(const int64_t *first, int n, int64_t v) {
  int lo = 0, hi = n - 1;
  while (lo < hi) {
    int mid = (lo + hi + 1) >> 1;
    if (first[mid] <= v) lo = mid; else hi = mid - 1;
  }
  return lo;
}

// Dequantises and transforms block `gb` (index in MCU order over the arenas) with quantisation table q; rows[y] = the 8 output samples
// of row y, byte k = column k.
__device__ __forceinline__ void idct_block(const int16_t *__restrict__ coef_arena, const int16_t *__restrict__ dc_arena, int64_t gb,
                                           const uint16_t *__restrict__ q, uint2 *rows) {
  const int4 *src = reinterpret_cast<const int4 *>(coef_arena + gb * 64);
  int ws[64];
  {
    int in[64];
    const uint4 *q4 = reinterpret_cast<const uint4 *>(q);      // 8 x u16 per row in ONE 16-byte load (the table is 16-byte aligned)
    uint32_t q00 = 0;
#pragma unroll
    for (int r = 0; r < 8; r++) {
      const int4 v = __ldg(src + r);
      const uint4 qv = __ldg(q4 + r);
      const int w[4] = { v.x, v.y, v.z, v.w };
      const uint32_t qw[4] = { qv.x, qv.y, qv.z, qv.w };
      if (r == 0) q00 = qv.x & 0xFFFFu;
#pragma unroll
      for (int k = 0; k < 4; k++) {
        in[r * 8 + 2 * k] = (int)(int16_t)(w[k] & 0xFFFF) * (int)(qw[k] & 0xFFFFu);
        in[r * 8 + 2 * k + 1] = (w[k] >> 16) * (int)(qw[k] >> 16);
      }
    }
    in[0] = (int)__ldg(dc_arena + gb) * (int)q00;         // DC lives in the compact array (after prediction)
#pragma unroll
    for (int x = 0; x < 8; x++) {       // pass 1: columns
      int o[8];
      idct8<11>(in[x], in[8 + x], in[16 + x], in[24 + x], in[32 + x], in[40 + x], in[48 + x], in[56 + x], o);
#pragma unroll
      for (int y = 0; y < 8; y++) ws[y * 8 + x] = o[y];
    }
  }
#pragma unroll
  for (int y = 0; y < 8; y++) {         // pass 2: rows
    int o[8];
    idct8<18>(ws[y * 8], ws[y * 8 + 1], ws[y * 8 + 2], ws[y * 8 + 3], ws[y * 8 + 4], ws[y * 8 + 5], ws[y * 8 + 6], ws[y * 8 + 7], o);
    rows[y].x = range_limit(o[0]) | (range_limit(o[1]) << 8) | (range_limit(o[2]) << 16) | (range_limit(o[3]) << 24);
    rows[y].y = range_limit(o[4]) | (range_limit(o[5]) << 8) | (range_limit(o[6]) << 16) | (range_limit(o[7]) << 24);
  }
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
  if (threadIdx.x == 0) s_first = find_by_prefix(first_work, nimages, b0);
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
    int lo = 0, hi = nimages - 1;
    while (lo < hi) { int mid = (lo + hi + 1) >> 1; if (first_quad[mid] <= gq) lo = mid; else hi = mid - 1; }
    const JpegImage &im = images[lo];
    if (im.fast_color) continue;
    const int64_t q = gq - first_quad[lo];
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
      else if (cm == kColorRGB) px[k] = (r * 19595 + g * 38470 + b * 7471 + 32768) >> 16;
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

// four ints -> four saturated bytes of one word (byte 0 = p0): two cvt.pack.sat instead of eight min/max and three merges
__device__ __forceinline__ uint32_t pack4_sat_u8(int p0, int p1, int p2, int p3) {
  uint32_t hi, w;
  asm("cvt.pack.sat.u8.s32.b32 %0, %1, %2, %3;" : "=r"(hi) : "r"(p3), "r"(p2), "r"(0));
  asm("cvt.pack.sat.u8.s32.b32 %0, %1, %2, %3;" : "=r"(w) : "r"(p1), "r"(p0), "r"(hi));
  return w;
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
  if (threadIdx.x == 0) s_first = find_by_prefix(first_item, nimages, it0);
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
// the 16 upsampled chroma samples of luma columns 2 * i0 .. 2 * i0 + 15 from the near / far chroma tile rows; c = tile byte of column i0
__device__ __forceinline__ void fancy_row16(const uint8_t *near, const uint8_t *far, int c, int i0, int dw, int *v) {
  const uint2 a = *reinterpret_cast<const uint2 *>(near + c), b = *reinterpret_cast<const uint2 *>(far + c);
  int cs[10];
  cs[0] = 3 * near[c - 1] + far[c - 1];                    // read, but unused, at the image's left / right edge
  cs[9] = 3 * near[c + 8] + far[c + 8];
#pragma unroll
  for (int k = 0; k < 8; k++) cs[1 + k] = 3 * (int)(((k < 4 ? a.x : a.y) >> (8 * (k & 3))) & 0xFFu) + (int)(((k < 4 ? b.x : b.y) >> (8 * (k & 3))) & 0xFFu);
#pragma unroll
  for (int k = 0; k < 8; k++) {
    v[2 * k] = fancy_h2v2_even(cs[k], cs[1 + k], i0 + k);
    v[2 * k + 1] = fancy_h2v2_odd(cs[1 + k], cs[2 + k], i0 + k, dw);
  }
}

// items: per image fused_geo().nstrips * nseg, strips of one segment consecutive; one CTA per item
__global__ void __launch_bounds__(kFusedThreads, 5) idct_color_420(const JpegImage *__restrict__ images, const int64_t *__restrict__ first_item,
                                                                int nimages, const int16_t *__restrict__ coef_arena,
                                                                const int16_t *__restrict__ dc_arena, const QuantSet *__restrict__ quants) {
  __shared__ __align__(16) uint8_t s_y[18][16 * kFusedMcus];      // rows 0, 1: carry rows; 2 + r: luma row 16m + r of band m
  __shared__ __align__(16) uint8_t s_c[2][10][kFusedCPitch];      // Cb, Cr; rows 0, 1: carry rows; 2 + r: chroma row 8m + r
  __shared__ int s_img;
  if (threadIdx.x == 0) s_img = find_by_prefix(first_item, nimages, blockIdx.x);
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
  } else if (j < 6 * nt + 4) {
    const int h = j - 6 * nt;
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
  const bool bgr = im.out_type == DALIB200_BGR;
  for (int m = b_lo > 0 ? b_lo - 1 : b_lo; m < b_hi; m++) {
    if (active) {
      uint2 rows[8];
      idct_block(coef_arena, dc_arena, blk0 + ((int64_t)m * im.mcux + mx) * im.bpm + b, q, rows);
      if (comp == 0) {
#pragma unroll
        for (int y = 0; y < 8; y++) *reinterpret_cast<uint2 *>(&s_y[2 + 8 * by + y][col]) = rows[y];
        if (by == 1) *reinterpret_cast<uint2 *>(&s_y[m & 1][col]) = rows[7];
      } else if (j < 6 * nt) {
#pragma unroll
        for (int y = 0; y < 8; y++) *reinterpret_cast<uint2 *>(&s_c[comp - 1][2 + y][col]) = rows[y];
        *reinterpret_cast<uint2 *>(&s_c[comp - 1][m & 1][col]) = rows[7];
      } else {
        const bool left = col == 7;                           // left neighbour: its column 7; right neighbour: its column 0
#pragma unroll
        for (int y = 0; y < 8; y++) s_c[comp - 1][2 + y][col] = (uint8_t)(left ? rows[y].y >> 24 : rows[y].x);
        s_c[comp - 1][m & 1][col] = (uint8_t)(left ? rows[7].y >> 24 : rows[7].x);
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
        int cb[16], cr[16];
        fancy_row16(s_c[0][rn], s_c[0][rf], 8 + 8 * u, 8 * (mxa + u), dw, cb);
        fancy_row16(s_c[1][rn], s_c[1][rf], 8 + 8 * u, 8 * (mxa + u), dw, cr);
        const uint32_t yw[4] = { yv.x, yv.y, yv.z, yv.w };
        uint32_t w[12];
#pragma unroll
        for (int h = 0; h < 2; h++) {
          int px[24];
#pragma unroll
          for (int k = 0; k < 8; k++) {
            const int yy = (int)((yw[2 * h + (k >> 2)] >> (8 * (k & 3))) & 0xFFu);
            const int cbm = cb[8 * h + k] - 128, crm = cr[8 * h + k] - 128;
            const int rr = yy + ((91881 * crm + 32768) >> 16);    // jdcolor.c, SCALEBITS 16; saturated by the pack (range_limit)
            const int gg = yy + ((-22554 * cbm + 32768 - 46802 * crm) >> 16);
            const int bb = yy + ((116130 * cbm + 32768) >> 16);
            px[3 * k] = bgr ? bb : rr; px[3 * k + 1] = gg; px[3 * k + 2] = bgr ? rr : bb;
          }
#pragma unroll
          for (int t = 0; t < 6; t++) w[6 * h + t] = pack4_sat_u8(px[4 * t], px[4 * t + 1], px[4 * t + 2], px[4 * t + 3]);
        }
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
    int lo = 0, hi = n - 1;
    while (lo < hi) { int mid = (lo + hi + 1) >> 1; if (posts[mid].first_px <= p0) lo = mid; else hi = mid - 1; }
    s_first = lo;
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
  if (total_blocks > 0) {
    ProfScope ps_("jpeg_idct", s);
    idct_kernel<<<grid, 128, 0, s>>>(a.d_images, a.d_first_work, a.nimages, total_blocks, a.d_coef, a.d_dc, a.d_quants, a.d_planes);
  }
  if (a.totals.fused > 0) {
    { ProfScope ps_("jpeg_idct_color", s); idct_color_420<<<(int)a.totals.fused, kFusedThreads, 0, s>>>(a.d_images, a.d_first_fused, a.nimages, a.d_coef, a.d_dc, a.d_quants); }
    CountLaunch();
  }
  if (a.totals.quads > 0) {
    const int grid2 = (int)std::min<int64_t>((a.totals.quads + 255) / 256, (int64_t)sms * 32);
    { ProfScope ps_("jpeg_upsample_color_generic", s); color_kernel<<<grid2, 256, 0, s>>>(a.d_images, a.d_first_quad, a.nimages, a.totals.quads, a.d_planes); }
    CountLaunch();
  }
  if (a.totals.items > 0) {
    const int grid3 = (int)std::min<int64_t>(a.totals.items, (int64_t)sms * 64);
    { ProfScope ps_("jpeg_upsample_color", s); color_fast_kernel<<<grid3, 128, 0, s>>>(a.d_images, a.d_first_item, a.nimages, a.totals.items, a.d_planes); }
    CountLaunch();
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
// progressive streams: planner + launch interface of jpeg_prog.cu (included here, behind the kernels, so that their line tables stay put)
#include "jpeg_prog.h"
#include "jpeg_prog_plan.h"
// EXIF orientation (shared with the PNG and WebP planners); PNG, TIFF and WebP streams: planners + launch interfaces of png.cu, tiff.cu
// and webp.cu
#include "exif.h"
#include "png.h"
#include "png_plan.h"
#include "tiff.h"
#include "tiff_plan.h"
#include "webp.h"
#include "webp_plan.h"
namespace {

struct ParsedJpeg {
  int width = 0, height = 0, ncomp = 0, precision = 8;
  int cid[4] = {0}, hs[4] = {0}, vs[4] = {0}, tq[4] = {0};
  int hmax = 0, vmax = 0;
  bool progressive = false, jfif = false;
  bool png = false;           // a PNG stream (png_plan.h): width / height / ncomp / orientation / scan range only
  bool tiff = false;          // a TIFF stream (tiff_plan.h): the same fields
  bool webp = false;          // a lossy WebP stream (webp_plan.h): the same fields
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
    } else if (m == 0xC0 || m == 0xC1 || m == 0xC2) {
      if (sl < 6) { SetLastError("JPEG: bad SOF"); return DALIB200_ERROR_BAD_DATA; }
      j.progressive = m == 0xC2;
      j.precision = s[0]; j.height = rd16(s + 1); j.width = rd16(s + 3); j.ncomp = s[5];
      if (j.ncomp < 1 || j.ncomp > 4 || sl < 6 + 3 * j.ncomp) { SetLastError("JPEG: bad SOF component count"); return DALIB200_ERROR_BAD_DATA; }
      for (int c = 0; c < j.ncomp; c++) {
        j.cid[c] = s[6 + 3 * c]; j.hs[c] = s[7 + 3 * c] >> 4; j.vs[c] = s[7 + 3 * c] & 15; j.tq[c] = s[8 + 3 * c];
        if (j.hs[c] < 1 || j.hs[c] > 4 || j.vs[c] < 1 || j.vs[c] > 4 || j.tq[c] > 3) { SetLastError("JPEG: bad sampling factors"); return DALIB200_ERROR_BAD_DATA; }
        j.hmax = std::max(j.hmax, j.hs[c]); j.vmax = std::max(j.vmax, j.vs[c]);
      }
      got_sof = true;
    } else if (m >= 0xC3 && m <= 0xCF && m != 0xC4 && m != 0xC8 && m != 0xCC) {
      SetLastError("JPEG: coding process 0x%02X (lossless / arithmetic / hierarchical) is not supported", m);
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

// PNG stream (png_plan.h): fills the fields of `j` the plan reads for every sample (size, components, orientation, staged byte
// range); `im` / `chunks`, when given, receive the device descriptors of batch image `image`.  Returns a DALIB200 status.
int ParsePng(const uint8_t *p, size_t n, ParsedJpeg &j, PngImage *im, std::vector<PngChunk> *chunks, int image) {
  PngImage tmp;
  std::vector<PngChunk> tmpc;
  PngInfo info;
  std::string err;
  const int rc = PlanPng(p, n, image, im ? im : &tmp, chunks ? *chunks : tmpc, &info, &err);
  if (rc) { SetLastError("%s", err.c_str()); return rc; }
  j.png = true;
  j.width = info.width; j.height = info.height; j.ncomp = info.components; j.orientation = info.orientation;
  j.hs[0] = j.vs[0] = 1;
  j.scan_begin = info.stage_begin; j.scan_end = info.stage_end;
  return DALIB200_SUCCESS;
}

// TIFF stream (tiff_plan.h), as ParsePng; `dec_base` / `dec_bytes`: the image's range of the decoded-segment scratch
int ParseTiff(const uint8_t *p, size_t n, ParsedJpeg &j, TiffImage *im, std::vector<TiffSeg> *segs, int image, int64_t dec_base,
              int64_t *dec_bytes) {
  TiffImage tmp;
  std::vector<TiffSeg> tmps;
  TiffInfo info;
  int64_t tmpd;
  std::string err;
  const int rc = PlanTiff(p, n, image, im ? im : &tmp, segs ? *segs : tmps, dec_base, dec_bytes ? dec_bytes : &tmpd, &info, &err);
  if (rc) { SetLastError("%s", err.c_str()); return rc; }
  j.tiff = true;
  j.width = info.width; j.height = info.height; j.ncomp = info.components; j.orientation = info.orientation;
  j.hs[0] = j.vs[0] = 1;
  j.scan_begin = info.stage_begin; j.scan_end = info.stage_end;
  return DALIB200_SUCCESS;
}

// lossy WebP stream (webp_plan.h), as ParsePng; `scratch_base` / `scratch_bytes`: the image's range of the WebP scratch.  The
// subsampling reported is 4:2:0 (VP8's only layout).
int ParseWebp(const uint8_t *p, size_t n, ParsedJpeg &j, WebpImage *im, int image, int64_t scratch_base, int64_t *scratch_bytes) {
  WebpImage tmp;
  WebpInfo info;
  int64_t tmpb;
  std::string err;
  const int rc = PlanWebp(p, n, image, im ? im : &tmp, scratch_base, scratch_bytes ? scratch_bytes : &tmpb, &info, &err);
  if (rc) { SetLastError("%s", err.c_str()); return rc; }
  j.webp = true;
  j.width = info.width; j.height = info.height; j.ncomp = info.components; j.orientation = info.orientation;
  j.hs[0] = j.vs[0] = 2;
  j.scan_begin = info.stage_begin; j.scan_end = info.stage_end;
  return DALIB200_SUCCESS;
}

void FillInfo(const ParsedJpeg &j, dalib200JpegInfo *info) {
  info->width = j.width; info->height = j.height;
  info->components = j.ncomp;
  info->subsampling = (j.hs[0] << 4) | j.vs[0];
  info->restart_interval = j.restart_interval;
  info->orientation = j.orientation;
}

uint32_t MakeLutEntry(int len, int sym, bool is_dc) {       // keep in sync with make_entry (device)
  const uint32_t s = sym & 15, r = (uint32_t)sym >> 4;
  const uint32_t adv = is_dc ? 1u : (s == 0 ? (r == 15u ? 16u : 64u) : r + 1u);
  return ((uint32_t)len + s) | (s << 8) | ((uint32_t)len << 12) | (adv << 20);
}

uint16_t MakeLutEntry16(int len, int sym, bool is_dc) {     // keep in sync with make_entry16 (device)
  const uint32_t s = sym & 15, r = (uint32_t)sym >> 4;
  const uint32_t adv = is_dc ? 1u : (s == 0 ? (r == 15u ? 16u : 64u) : r + 1u);
  return (uint16_t)(((uint32_t)len + s) | (s << 5) | (adv << 9));
}

void BuildDeviceTable(const HostHuff &h, uint32_t *lut, uint16_t *lut16, HuffSlow &t, bool is_dc) {
  const int kLutBits = is_dc ? kDcLutBits : kAcLutBits, kLutSize = 1 << kLutBits;
  memset(&t, 0, sizeof(t));
  memset(lut, 0, sizeof(uint32_t) * kLutSize);
  memset(lut16, 0, sizeof(uint16_t) * kLutSize);
  int code = 0, k = 0;
  for (int l = 1; l <= 16; l++) {
    const int mincode = code;
    t.valoff[l] = k - mincode;
    for (int i = 0; i < h.bits[l]; i++, k++, code++) {
      if (l <= kLutBits) {
        const int lo = code << (kLutBits - l), cnt = 1 << (kLutBits - l);
        for (int e = 0; e < cnt && lo + e < kLutSize; e++) {
          lut[lo + e] = MakeLutEntry(l, h.vals[k & 255], is_dc);
          lut16[lo + e] = MakeLutEntry16(l, h.vals[k & 255], is_dc);
        }
      }
    }
    // a 16-bit window belongs to length l iff it is < maxcode[l] (exclusive bound, left-aligned) and matched
    // no shorter length; for an empty length the bound equals the previous one, so nothing matches
    t.maxcode[l] = code << (16 - l);
    code <<= 1;
  }
  t.maxcode[17] = 0x7fffffff;
  memcpy(t.vals, h.vals, 256);
  // direct table for the codes behind the first level (see HuffSlow)
  t.long_base = t.maxcode[kLutBits];
  const int range = 65536 - t.long_base;
  t.long_n = 0;
  if (range > 0 && range <= kLongLut) {
    t.long_n = range;
    int c2 = 0, k2 = 0;
    for (int l = 1; l <= 16; l++) {
      for (int i = 0; i < h.bits[l]; i++, k2++, c2++) {
        if (l > kLutBits) {
          const int lo = (c2 << (16 - l)) - t.long_base, cnt = 1 << (16 - l);
          for (int e = 0; e < cnt; e++)
            if (lo + e >= 0 && lo + e < range) t.long_lut[lo + e] = (uint16_t)(l | (h.vals[k2 & 255] << 8));
        }
      }
      c2 <<= 1;
    }
  }
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
  uint8_t *h_stage = nullptr; size_t h_stage_cap = 0;
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
  cudaEvent_t uploaded = nullptr, img_uploaded = nullptr;
  uint8_t *h_images = nullptr; size_t h_images_cap = 0;
  bool pending = false, img_pending = false, staged = false, smem_opted = false;
  // progressive (SOF2) samples: their entropy stage runs in jpeg_prog.cu, everything behind it is shared
  std::vector<dalib200::ProgImage> prog_images;
  std::vector<dalib200::ProgScan> prog_scans;     // sorted by wave
  std::vector<dalib200::ProgHuff> prog_huff;
  std::vector<int> prog_wave_begin;
  std::vector<int64_t> prog_first_blk;
  int64_t prog_total_blocks = 0;
  dalib200::DescArena prog_arena;
  cudaEvent_t prog_uploaded = nullptr, prog_fork = nullptr, prog_join = nullptr;
  cudaStream_t prog_stream = nullptr;      // the scans are serial chains on one warp each: they run beside the baseline entropy stage
  bool prog_pending = false;
  // PNG samples: decoded by png.cu on a stream of their own into the same decode windows; the post pass is shared
  std::vector<dalib200::PngImage> png_images;
  std::vector<dalib200::PngChunk> png_chunks;
  int64_t png_scan_bytes = 0;
  uint8_t *d_png_scan = nullptr; size_t d_png_scan_cap = 0;   // filtered scanlines (grow only)
  dalib200::DescArena png_arena;
  cudaEvent_t png_uploaded = nullptr, png_fork = nullptr, png_join = nullptr;
  cudaStream_t png_stream = nullptr;
  bool png_pending = false;
  // TIFF samples: decoded by tiff.cu on a stream of their own, like the PNG samples
  std::vector<dalib200::TiffImage> tiff_images;
  std::vector<dalib200::TiffSeg> tiff_segs;
  int64_t tiff_dec_bytes = 0;
  uint8_t *d_tiff_dec = nullptr; size_t d_tiff_dec_cap = 0;    // decoded segments (grow only)
  uint8_t *d_tiff_slots = nullptr; size_t d_tiff_slots_cap = 0; // segment working memory (grow only)
  dalib200::DescArena tiff_arena;
  cudaEvent_t tiff_uploaded = nullptr, tiff_fork = nullptr, tiff_join = nullptr;
  cudaStream_t tiff_stream = nullptr;
  bool tiff_pending = false;
  // WebP samples: decoded by webp.cu on a stream of their own, like the PNG and TIFF samples
  std::vector<dalib200::WebpImage> webp_images;
  int64_t webp_scratch_bytes = 0;
  uint8_t *d_webp_scratch = nullptr; size_t d_webp_scratch_cap = 0;   // coefficients, macroblocks, planes (grow only)
  dalib200::DescArena webp_arena;
  cudaEvent_t webp_uploaded = nullptr, webp_fork = nullptr, webp_join = nullptr;
  cudaStream_t webp_stream = nullptr;
  bool webp_pending = false;
};

namespace {

template <typename T>
int GrowDevice(T *&ptr, size_t &cap, size_t need) {
  if (need <= cap) return DALIB200_SUCCESS;
  size_t ncap = std::max(need + need / 4, (size_t)4096);
  if (ptr) cudaFree(ptr);
  ptr = nullptr; cap = 0;
  DB_CUDA(cudaMalloc(reinterpret_cast<void **>(&ptr), ncap * sizeof(T)));
  cap = ncap;
  return DALIB200_SUCCESS;
}

inline size_t Align(size_t v, size_t a) { return (v + a - 1) / a * a; }

}  // namespace

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
    if (j.png || j.tiff || j.webp) {   // decoded by png.cu / tiff.cu / webp.cu: no IDCT / colour work
      p->first_work[i] = t.work; p->first_fused[i] = t.fused; p->first_quad[i] = t.quads; p->first_item[i] = t.items;
      continue;
    }
    ReconAddImage(im, p->fancy != 0, planes_only, t, &p->first_work[i], &p->first_fused[i], &p->first_quad[i], &p->first_item[i]);
  }
  p->total_work = t.work; p->total_fused = t.fused; p->total_post_px = post_px; p->post_bytes = post_bytes; p->total_quads = t.quads;
  p->total_items = t.items;
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
  if (j.png || j.tiff || j.webp) {   // any window: png_color / tiff_color / webp_color produce pixels one by one
    im.win_x0 = sx0; im.win_w = sx1 - sx0;
  } else {
    im.win_x0 = sx0 & ~7; im.win_w = std::min(W, (sx1 + 7) & ~7) - im.win_x0;
  }
  im.win_y0 = sy0; im.win_h = sy1 - sy0;
  JpegGeo &ge = p->geo[i];
  ge.orient = orient; ge.rx0 = rx0; ge.ry0 = ry0; ge.rx1 = rx1; ge.ry1 = ry1; ge.out_c = out_c;
  ge.direct = orient == 1 && p->dtype == DALIB200_UINT8 && output_type != DALIB200_YCbCr && im.win_x0 == sx0 && im.win_x0 + im.win_w == sx1;
  // decode -> resize without the RGB image (the caller consumes the planes): 4:2:0 YCbCr, fancy upsampling, plain RGB u8 request
  ge.planar_ok = !j.png && !j.tiff && !j.webp && j.ncomp == 3 && im.color == kColorYCbCr && j.hmax == 2 && j.vmax == 2 && p->fancy && orient == 1 && j.width > 4 &&
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
  int rc = IsPngStream(data, len) ? ParsePng(data, len, j, nullptr, nullptr, 0)
           : IsTiffStream(data, len) ? ParseTiff(data, len, j, nullptr, nullptr, 0, 0, nullptr)
           : IsWebpStream(data, len) ? ParseWebp(data, len, j, nullptr, 0, 0, nullptr) : ParseHeaders(data, len, j, false);
  if (rc) return rc;
  FillInfo(j, info);
  return DALIB200_SUCCESS;
} DB_API_CATCH

int dalib200JpegPlanCreate(dalib200JpegPlan **plan, int max_batch) try {
  DB_CHECK_ARG(plan && max_batch > 0, "JpegPlanCreate: bad arguments");
  auto *p = new dalib200JpegPlan();
  p->max_batch = max_batch;
  if (cudaEventCreateWithFlags(&p->uploaded, cudaEventDisableTiming) != cudaSuccess ||
      cudaEventCreateWithFlags(&p->img_uploaded, cudaEventDisableTiming) != cudaSuccess ||
      cudaEventCreateWithFlags(&p->prog_uploaded, cudaEventDisableTiming) != cudaSuccess ||
      cudaEventCreateWithFlags(&p->prog_fork, cudaEventDisableTiming) != cudaSuccess ||
      cudaEventCreateWithFlags(&p->prog_join, cudaEventDisableTiming) != cudaSuccess ||
      cudaEventCreateWithFlags(&p->png_uploaded, cudaEventDisableTiming) != cudaSuccess ||
      cudaEventCreateWithFlags(&p->png_fork, cudaEventDisableTiming) != cudaSuccess ||
      cudaEventCreateWithFlags(&p->png_join, cudaEventDisableTiming) != cudaSuccess ||
      cudaEventCreateWithFlags(&p->tiff_uploaded, cudaEventDisableTiming) != cudaSuccess ||
      cudaEventCreateWithFlags(&p->tiff_fork, cudaEventDisableTiming) != cudaSuccess ||
      cudaEventCreateWithFlags(&p->tiff_join, cudaEventDisableTiming) != cudaSuccess ||
      cudaEventCreateWithFlags(&p->webp_uploaded, cudaEventDisableTiming) != cudaSuccess ||
      cudaEventCreateWithFlags(&p->webp_fork, cudaEventDisableTiming) != cudaSuccess ||
      cudaEventCreateWithFlags(&p->webp_join, cudaEventDisableTiming) != cudaSuccess) {
    SetLastError("JpegPlanCreate: cudaEventCreate failed"); delete p; return DALIB200_ERROR_CUDA;
  }
  *plan = p;
  return DALIB200_SUCCESS;
} DB_API_CATCH

int dalib200JpegPlanDestroy(dalib200JpegPlan *p) try {
  if (!p) return DALIB200_SUCCESS;
  if (p->uploaded) { cudaEventSynchronize(p->uploaded); cudaEventDestroy(p->uploaded); }
  if (p->img_uploaded) { cudaEventSynchronize(p->img_uploaded); cudaEventDestroy(p->img_uploaded); }
  if (p->prog_stream) { cudaStreamSynchronize(p->prog_stream); cudaStreamDestroy(p->prog_stream); }
  if (p->prog_uploaded) { cudaEventSynchronize(p->prog_uploaded); cudaEventDestroy(p->prog_uploaded); }
  if (p->prog_fork) cudaEventDestroy(p->prog_fork);
  if (p->prog_join) cudaEventDestroy(p->prog_join);
  p->prog_arena.Free();
  if (p->png_stream) { cudaStreamSynchronize(p->png_stream); cudaStreamDestroy(p->png_stream); }
  if (p->png_uploaded) { cudaEventSynchronize(p->png_uploaded); cudaEventDestroy(p->png_uploaded); }
  if (p->png_fork) cudaEventDestroy(p->png_fork);
  if (p->png_join) cudaEventDestroy(p->png_join);
  p->png_arena.Free();
  if (p->d_png_scan) cudaFree(p->d_png_scan);
  if (p->tiff_stream) { cudaStreamSynchronize(p->tiff_stream); cudaStreamDestroy(p->tiff_stream); }
  if (p->tiff_uploaded) { cudaEventSynchronize(p->tiff_uploaded); cudaEventDestroy(p->tiff_uploaded); }
  if (p->tiff_fork) cudaEventDestroy(p->tiff_fork);
  if (p->tiff_join) cudaEventDestroy(p->tiff_join);
  p->tiff_arena.Free();
  if (p->d_tiff_dec) cudaFree(p->d_tiff_dec);
  if (p->d_tiff_slots) cudaFree(p->d_tiff_slots);
  if (p->webp_stream) { cudaStreamSynchronize(p->webp_stream); cudaStreamDestroy(p->webp_stream); }
  if (p->webp_uploaded) { cudaEventSynchronize(p->webp_uploaded); cudaEventDestroy(p->webp_uploaded); }
  if (p->webp_fork) cudaEventDestroy(p->webp_fork);
  if (p->webp_join) cudaEventDestroy(p->webp_join);
  p->webp_arena.Free();
  if (p->d_webp_scratch) cudaFree(p->d_webp_scratch);
  if (p->h_stage) cudaFreeHost(p->h_stage);
  if (p->h_images) cudaFreeHost(p->h_images);
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
  memcpy(p->h_stage + p->off_quads, p->first_quad.data(), sizeof(int64_t) * p->n);
  memcpy(p->h_stage + p->off_items, p->first_item.data(), sizeof(int64_t) * p->n);
  memcpy(p->h_stage + p->off_work, p->first_work.data(), sizeof(int64_t) * p->n);
  memcpy(p->h_stage + p->off_fused, p->first_fused.data(), sizeof(int64_t) * p->n);
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
  p->prog_images.clear(); p->prog_scans.clear(); p->prog_huff.clear(); p->prog_wave_begin.clear(); p->prog_first_blk.clear();
  p->prog_total_blocks = 0;
  p->png_images.clear(); p->png_chunks.clear();
  int64_t png_scan = 0;
  p->tiff_images.clear(); p->tiff_segs.clear();
  int64_t tiff_dec = 0;
  p->webp_images.clear();
  int64_t webp_scratch = 0;
  std::map<std::string, int> table_cache, quant_cache, prog_table_cache;
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
    if (IsPngStream(streams[i], lengths[i])) {
      // PNG: no units, subsequences or MCUs, so every JPEG kernel skips the sample; png.cu decodes its IDAT run (the staged range)
      // into the decode window, and the post pass behind it is shared
      dalib200::PngImage pim;
      int rc = ParsePng(streams[i], lengths[i], j, &pim, &p->png_chunks, (int)p->png_images.size());
      if (rc) { std::string m = dalib200GetLastError(); SetLastError("decoders.image: sample %d: %s", i, m.c_str()); return rc; }
      JpegImage &im = p->images[i];
      memset(&im, 0, sizeof(im));
      im.width = j.width; im.height = j.height; im.out_type = output_type;
      im.unit_begin = im.unit_end = (int)p->units.size();
      im.subseq_begin = (int)subseq; im.block_begin = sync_blocks; im.wblock_begin = write_blocks; im.coef_off = coefs;
      if ((rc = PlanGeometry(p, i, rois, j, im))) return rc;
      pim.sample = i;
      pim.raw_off = (int64_t)raw;
      pim.scan_off = png_scan;
      png_scan += (int64_t)Align((size_t)pim.scan_bytes, 16);
      p->png_images.push_back(pim);
      p->src_ptr.push_back(streams[i] + j.scan_begin);
      raw += Align(j.scan_end - j.scan_begin, 16);
      continue;
    }
    if (IsTiffStream(streams[i], lengths[i])) {
      // TIFF: as PNG; tiff.cu decodes its segments (the staged range is their span) into the decode window
      dalib200::TiffImage tim;
      int64_t dec_bytes = 0;
      int rc = ParseTiff(streams[i], lengths[i], j, &tim, &p->tiff_segs, (int)p->tiff_images.size(), tiff_dec, &dec_bytes);
      if (rc) { std::string m = dalib200GetLastError(); SetLastError("decoders.image: sample %d: %s", i, m.c_str()); return rc; }
      JpegImage &im = p->images[i];
      memset(&im, 0, sizeof(im));
      im.width = j.width; im.height = j.height; im.out_type = output_type;
      im.unit_begin = im.unit_end = (int)p->units.size();
      im.subseq_begin = (int)subseq; im.block_begin = sync_blocks; im.wblock_begin = write_blocks; im.coef_off = coefs;
      if ((rc = PlanGeometry(p, i, rois, j, im))) return rc;
      tim.sample = i;
      tim.raw_off = (int64_t)raw;
      tiff_dec += dec_bytes;
      p->tiff_images.push_back(tim);
      p->src_ptr.push_back(streams[i] + j.scan_begin);
      raw += Align(j.scan_end - j.scan_begin, 16);
      continue;
    }
    if (IsWebpStream(streams[i], lengths[i])) {
      // WebP: as PNG; webp.cu decodes its VP8 payload (the staged range) into the decode window
      dalib200::WebpImage wim;
      int64_t bytes = 0;
      int rc = ParseWebp(streams[i], lengths[i], j, &wim, (int)p->webp_images.size(), webp_scratch, &bytes);
      if (rc) { std::string m = dalib200GetLastError(); SetLastError("decoders.image: sample %d: %s", i, m.c_str()); return rc; }
      JpegImage &im = p->images[i];
      memset(&im, 0, sizeof(im));
      im.width = j.width; im.height = j.height; im.out_type = output_type;
      im.unit_begin = im.unit_end = (int)p->units.size();
      im.subseq_begin = (int)subseq; im.block_begin = sync_blocks; im.wblock_begin = write_blocks; im.coef_off = coefs;
      if ((rc = PlanGeometry(p, i, rois, j, im))) return rc;
      wim.sample = i;
      wim.raw_off = (int64_t)raw;
      webp_scratch += bytes;
      p->webp_images.push_back(wim);
      p->src_ptr.push_back(streams[i] + j.scan_begin);
      raw += Align(j.scan_end - j.scan_begin, 16);
      continue;
    }
    int rc = ParseHeaders(streams[i], lengths[i], j, true);
    if (rc) { std::string m = dalib200GetLastError(); SetLastError("decoders.image: sample %d: %s", i, m.c_str()); return rc; }
    auto unsupported = [&](const char *what) { SetLastError("decoders.image: sample %d: %s", i, what); return DALIB200_ERROR_UNSUPPORTED; };
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
      if (!j.qt_present[j.tq[c]]) { SetLastError("decoders.image: sample %d: missing quantisation table", i); return DALIB200_ERROR_BAD_DATA; }
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
          BuildDeviceTable(j.dc[t], ts.lut + LutOffset(t), ts.lut16 + LutOffset(t), ts.slow[t], true);
          BuildDeviceTable(j.ac[t], ts.lut + LutOffset(2 + t), ts.lut16 + LutOffset(2 + t), ts.slow[2 + t], false);
        }
        p->tables.push_back(ts);
        it = table_cache.emplace(key, (int)p->tables.size() - 1).first;
      }
      im.table_set = it->second;
      std::string qk(reinterpret_cast<const char *>(j.qt), sizeof(j.qt));
      auto qi = quant_cache.find(qk);
      if (qi == quant_cache.end()) {
        QuantSet qs; memcpy(qs.q, j.qt, sizeof(j.qt));
        p->quants.push_back(qs);
        qi = quant_cache.emplace(qk, (int)p->quants.size() - 1).first;
      }
      im.quant_set = qi->second;
    }
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
      dalib200::ProgImage pim;
      memset(&pim, 0, sizeof(pim));
      std::string perr;
      const size_t first_new = p->prog_scans.size();
      rc = dalib200::PlanProgressive(d, lengths[i], sb, (int)p->prog_images.size(), &pim, p->prog_scans, p->prog_huff, prog_table_cache, &perr);
      if (rc) { SetLastError("decoders.image: sample %d: %s", i, perr.c_str()); return rc; }
      for (size_t k = first_new; k < p->prog_scans.size(); k++)
        if ((size_t)p->prog_scans[k].data_off + p->prog_scans[k].data_len > se - sb) {
          // a scan that runs into the trimmed end-of-image marker ends in front of it
          auto &sc = p->prog_scans[k];
          sc.data_len = sc.data_off >= se - sb ? 0 : (uint32_t)(se - sb - sc.data_off);
        }
      if (pim.ncomp != im.ncomp || pim.mcux != im.mcux || pim.mcuy != im.mcuy || pim.bpm != bpm) {
        SetLastError("decoders.image: sample %d: internal error (progressive frame layout)", i); return DALIB200_ERROR_INTERNAL;
      }
      pim.sample = i;
      pim.raw_off = (int64_t)raw;
      pim.coef_off = coefs;
      p->prog_first_blk.push_back(p->prog_total_blocks);
      p->prog_total_blocks += nmcu * bpm;
      p->prog_images.push_back(pim);
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
  if (!p->prog_scans.empty()) {
    std::stable_sort(p->prog_scans.begin(), p->prog_scans.end(), [](const dalib200::ProgScan &a, const dalib200::ProgScan &b) { return a.wave < b.wave; });
    const int nw = p->prog_scans.back().wave + 1;
    p->prog_wave_begin.assign(nw + 1, 0);
    for (const auto &sc : p->prog_scans) p->prog_wave_begin[sc.wave + 1]++;
    for (int w = 0; w < nw; w++) p->prog_wave_begin[w + 1] += p->prog_wave_begin[w];
  }
  DB_CHECK_ARG(raw < (1ull << 32) && clean < (1ull << 32), "decoders.image: batch of encoded data exceeds 4 GiB");
  p->raw_bytes = raw; p->clean_bytes = clean; p->nchunks = chunks;
  p->png_scan_bytes = png_scan;
  p->tiff_dec_bytes = tiff_dec;
  p->webp_scratch_bytes = webp_scratch;
  DB_CHECK_ARG(p->tiff_segs.size() < (1ull << 31), "decoders.image: batch of more than 2^31 TIFF segments");
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
  const size_t total = off + raw + 64;
  if (p->pending) { DB_CUDA(cudaEventSynchronize(p->uploaded)); p->pending = false; }
  if (total > p->h_stage_cap) {
    if (p->h_stage) cudaFreeHost(p->h_stage);
    p->h_stage = nullptr; p->h_stage_cap = 0;
    size_t ncap = total + total / 4;
    DB_CUDA(cudaMallocHost(reinterpret_cast<void **>(&p->h_stage), ncap));
    p->h_stage_cap = ncap;
  }
  memcpy(p->h_stage + p->off_units, p->units.data(), sizeof(JpegUnit) * p->units.size());
  memcpy(p->h_stage + p->off_tables, p->tables.data(), sizeof(TableSet) * p->tables.size());
  memcpy(p->h_stage + p->off_quants, p->quants.data(), sizeof(QuantSet) * p->quants.size());
  memcpy(p->h_stage + p->off_quads, p->first_quad.data(), sizeof(int64_t) * n);
  memcpy(p->h_stage + p->off_items, p->first_item.data(), sizeof(int64_t) * n);
  memcpy(p->h_stage + p->off_work, p->first_work.data(), sizeof(int64_t) * n);
  memcpy(p->h_stage + p->off_fused, p->first_fused.data(), sizeof(int64_t) * n);
  memcpy(p->h_stage + p->off_blkimg, p->block_image.data(), sizeof(int32_t) * p->block_image.size());
  memcpy(p->h_stage + p->off_wblkimg, p->wblock_image.data(), sizeof(int32_t) * p->wblock_image.size());
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
  // output pointers are patched at launch: images are uploaded there.  Descriptors and tables go first ...
  DB_CUDA(cudaMemcpyAsync(p->d_stage + p->off_units, p->h_stage + p->off_units, p->off_raw - p->off_units, cudaMemcpyHostToDevice, stream));
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
          DB_CUDA(cudaEventRecord(p->uploaded, stream));
          p->pending = true;
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
      DB_CUDA(cudaEventRecord(p->uploaded, stream));
      p->pending = true;
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
        uint8_t *dstp = p->h_stage + p->off_raw + p->stage_off[i];
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
        err = cudaMemcpyAsync(p->d_stage + p->off_raw + b0, p->h_stage + p->off_raw + b0, b1 - b0, cudaMemcpyHostToDevice, stream);
    }
    for (auto &t : th) t.join();
    DB_CUDA(err);
  }
  DB_CUDA(cudaEventRecord(p->uploaded, stream));
  p->pending = true;
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
  if ((rc = GrowDevice(p->d_chain_count, p->d_chain_count_cap, (size_t)8))) return rc;
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
  {
    if (p->img_pending) { DB_CUDA(cudaEventSynchronize(p->img_uploaded)); p->img_pending = false; }
    const size_t img_bytes = Align(sizeof(JpegImage) * p->n, 16);
    const size_t need = img_bytes + sizeof(JpegPost) * p->posts.size();
    if (need > p->h_images_cap) {
      if (p->h_images) cudaFreeHost(p->h_images);
      p->h_images = nullptr; p->h_images_cap = 0;
      DB_CUDA(cudaMallocHost(reinterpret_cast<void **>(&p->h_images), need * 2));
      p->h_images_cap = need * 2;
    }
    JpegImage *hi = reinterpret_cast<JpegImage *>(p->h_images);
    for (int i = 0; i < p->n; i++) { hi[i] = p->images[i]; hi[i].out = static_cast<uint8_t *>(out_ptrs[i]); }
    JpegPost *hp = reinterpret_cast<JpegPost *>(p->h_images + img_bytes);
    for (size_t k = 0; k < p->posts.size(); k++) {
      const int i = p->post_sample[k];
      hp[k] = p->posts[k];
      hp[k].src = p->d_post + p->post_off[k];
      hp[k].dst = out_ptrs[i];
      hi[i].out = p->d_post + p->post_off[k];              // the decoder writes the window into scratch
    }
    DB_CUDA(cudaMemcpyAsync(p->d_stage + p->off_images, hi, sizeof(JpegImage) * p->n, cudaMemcpyHostToDevice, stream));
    if (!p->posts.empty())
      DB_CUDA(cudaMemcpyAsync(p->d_posts, hp, sizeof(JpegPost) * p->posts.size(), cudaMemcpyHostToDevice, stream));
    DB_CUDA(cudaEventRecord(p->img_uploaded, stream));
    p->img_pending = true;
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
  DB_CUDA(cudaMemsetAsync(p->d_chain_count, 0, sizeof(uint32_t) * 8, s));
  if (!p->prog_images.empty()) {
    // progressive samples: scans wave by wave into the same coefficient arena, DC left as differences for dc_scan (jpeg_prog.cu).
    // A scan is a serial chain on ONE warp (milliseconds for a large image) that leaves the GPU empty: the stage is forked onto a
    // stream of its own here, behind the upload and the status clear, runs beside the baseline samples' entropy kernels and is joined
    // in front of dc_scan.  It touches only the progressive samples' ranges of the coefficient / DC arenas and their status words.
    using namespace dalib200;
    if (!p->prog_stream) DB_CUDA(cudaStreamCreateWithFlags(&p->prog_stream, cudaStreamNonBlocking));
    cudaStream_t ps = p->prog_stream;
    DB_CUDA(cudaEventRecord(p->prog_fork, s));
    DB_CUDA(cudaStreamWaitEvent(ps, p->prog_fork, 0));
    if (p->prog_pending) { DB_CUDA(cudaEventSynchronize(p->prog_uploaded)); p->prog_pending = false; }
    const size_t npi = p->prog_images.size(), nsc = p->prog_scans.size(), nh = p->prog_huff.size();
    const size_t o_img = 0, o_scan = Align(o_img + sizeof(ProgImage) * npi, 16), o_huff = Align(o_scan + sizeof(ProgScan) * nsc, 16),
                 o_blk = Align(o_huff + sizeof(ProgHuff) * nh, 16), pbytes = Align(o_blk + sizeof(int64_t) * npi, 16);
    if ((rc = p->prog_arena.Reserve(pbytes))) return rc;
    memcpy(p->prog_arena.host + o_img, p->prog_images.data(), sizeof(ProgImage) * npi);
    memcpy(p->prog_arena.host + o_scan, p->prog_scans.data(), sizeof(ProgScan) * nsc);
    memcpy(p->prog_arena.host + o_huff, p->prog_huff.data(), sizeof(ProgHuff) * nh);
    memcpy(p->prog_arena.host + o_blk, p->prog_first_blk.data(), sizeof(int64_t) * npi);
    if ((rc = p->prog_arena.Upload(pbytes, ps))) return rc;
    DB_CUDA(cudaEventRecord(p->prog_uploaded, ps));
    p->prog_pending = true;
    ProgLaunch a;
    a.d_images = reinterpret_cast<const ProgImage *>(p->prog_arena.dev + o_img); a.nimages = (int)npi;
    a.d_scans = reinterpret_cast<const ProgScan *>(p->prog_arena.dev + o_scan);
    a.d_huff = reinterpret_cast<const ProgHuff *>(p->prog_arena.dev + o_huff);
    a.d_first_blk = reinterpret_cast<const int64_t *>(p->prog_arena.dev + o_blk);
    a.total_blocks = p->prog_total_blocks;
    a.wave_begin = &p->prog_wave_begin; a.h_images = &p->prog_images;
    a.d_raw = d_raw; a.d_coef = p->d_coef; a.d_dc = p->d_dc; a.d_status = p->d_status;
    if ((rc = LaunchProgressive(a, ps))) return rc;
    DB_CUDA(cudaEventRecord(p->prog_join, ps));
  }
  if (!p->png_images.empty()) {
    // PNG samples (png.cu): the inflate is a serial chain per image, so the stage is forked onto a stream of its own behind the upload
    // and the status clear, runs beside the JPEG samples' kernels and is joined in front of the post pass.  It writes only the PNG
    // samples' decode windows, its scanline scratch and their status words.
    using namespace dalib200;
    if ((rc = GrowDevice(p->d_png_scan, p->d_png_scan_cap, (size_t)p->png_scan_bytes + 16))) return rc;
    if (!p->png_stream) DB_CUDA(cudaStreamCreateWithFlags(&p->png_stream, cudaStreamNonBlocking));
    cudaStream_t ps = p->png_stream;
    DB_CUDA(cudaEventRecord(p->png_fork, s));
    DB_CUDA(cudaStreamWaitEvent(ps, p->png_fork, 0));
    if (p->png_pending) { DB_CUDA(cudaEventSynchronize(p->png_uploaded)); p->png_pending = false; }
    const JpegImage *hi = reinterpret_cast<const JpegImage *>(p->h_images);    // the output pointers of this launch
    int64_t px = 0;
    for (PngImage &pi : p->png_images) {
      const JpegImage &im = hi[pi.sample];
      pi.out = im.out; pi.out_type = im.out_type;
      pi.win_x0 = im.win_x0; pi.win_y0 = im.win_y0; pi.win_w = im.win_w; pi.win_h = im.win_h;
      pi.first_px = px;
      px += (int64_t)im.win_w * im.win_h;
    }
    const size_t npi = p->png_images.size(), nch = p->png_chunks.size();
    const size_t o_chunk = Align(sizeof(PngImage) * npi, 16), pbytes = Align(o_chunk + sizeof(PngChunk) * nch, 16);
    if ((rc = p->png_arena.Reserve(pbytes))) return rc;
    memcpy(p->png_arena.host, p->png_images.data(), sizeof(PngImage) * npi);
    memcpy(p->png_arena.host + o_chunk, p->png_chunks.data(), sizeof(PngChunk) * nch);
    if ((rc = p->png_arena.Upload(pbytes, ps))) return rc;
    DB_CUDA(cudaEventRecord(p->png_uploaded, ps));
    p->png_pending = true;
    PngLaunch a;
    a.d_images = reinterpret_cast<const PngImage *>(p->png_arena.dev); a.nimages = (int)npi;
    a.d_chunks = reinterpret_cast<const PngChunk *>(p->png_arena.dev + o_chunk); a.nchunks = (int)nch;
    a.total_px = px;
    a.d_raw = d_raw; a.d_scan = p->d_png_scan; a.d_status = p->d_status;
    if ((rc = LaunchPng(a, ps))) return rc;
    DB_CUDA(cudaEventRecord(p->png_join, ps));
  }
  if (!p->tiff_images.empty()) {
    // TIFF samples (tiff.cu): forked onto a stream of their own as the PNG samples are, so that a TIFF written as one big strip (a serial
    // chain) runs beside the JPEG kernels.  It writes only the TIFF samples' decode windows, its scratch and their status words.
    using namespace dalib200;
    const int nseg = (int)p->tiff_segs.size();
    if ((rc = GrowDevice(p->d_tiff_dec, p->d_tiff_dec_cap, (size_t)p->tiff_dec_bytes + 16))) return rc;
    if ((rc = GrowDevice(p->d_tiff_slots, p->d_tiff_slots_cap, (size_t)TiffSlotCount(nseg) * kTiffSlotBytes))) return rc;
    if (!p->tiff_stream) DB_CUDA(cudaStreamCreateWithFlags(&p->tiff_stream, cudaStreamNonBlocking));
    cudaStream_t ts = p->tiff_stream;
    DB_CUDA(cudaEventRecord(p->tiff_fork, s));
    DB_CUDA(cudaStreamWaitEvent(ts, p->tiff_fork, 0));
    if (p->tiff_pending) { DB_CUDA(cudaEventSynchronize(p->tiff_uploaded)); p->tiff_pending = false; }
    const JpegImage *hi = reinterpret_cast<const JpegImage *>(p->h_images);    // the output pointers of this launch
    int64_t px = 0;
    for (TiffImage &ti : p->tiff_images) {
      const JpegImage &im = hi[ti.sample];
      ti.out = im.out; ti.out_type = im.out_type;
      ti.win_x0 = im.win_x0; ti.win_y0 = im.win_y0; ti.win_w = im.win_w; ti.win_h = im.win_h;
      ti.first_px = px;
      px += (int64_t)im.win_w * im.win_h;
    }
    const size_t nti = p->tiff_images.size();
    const size_t o_seg = Align(sizeof(TiffImage) * nti, 16), tbytes = Align(o_seg + sizeof(TiffSeg) * nseg, 16);
    if ((rc = p->tiff_arena.Reserve(tbytes))) return rc;
    memcpy(p->tiff_arena.host, p->tiff_images.data(), sizeof(TiffImage) * nti);
    memcpy(p->tiff_arena.host + o_seg, p->tiff_segs.data(), sizeof(TiffSeg) * nseg);
    if ((rc = p->tiff_arena.Upload(tbytes, ts))) return rc;
    DB_CUDA(cudaEventRecord(p->tiff_uploaded, ts));
    p->tiff_pending = true;
    TiffLaunch a;
    a.d_images = reinterpret_cast<const TiffImage *>(p->tiff_arena.dev); a.nimages = (int)nti;
    a.d_segs = reinterpret_cast<const TiffSeg *>(p->tiff_arena.dev + o_seg); a.nsegs = nseg;
    a.total_px = px;
    a.d_raw = d_raw; a.d_dec = p->d_tiff_dec; a.d_slots = p->d_tiff_slots; a.d_status = p->d_status;
    if ((rc = LaunchTiff(a, ts))) return rc;
    DB_CUDA(cudaEventRecord(p->tiff_join, ts));
  }
  if (!p->webp_images.empty()) {
    // WebP samples (webp.cu): forked onto a stream of their own as the PNG and TIFF samples are; the entropy decode of an image is a
    // serial chain.  It writes only the WebP samples' decode windows, its scratch and their status words.
    using namespace dalib200;
    if ((rc = GrowDevice(p->d_webp_scratch, p->d_webp_scratch_cap, (size_t)p->webp_scratch_bytes + 16))) return rc;
    if (!p->webp_stream) DB_CUDA(cudaStreamCreateWithFlags(&p->webp_stream, cudaStreamNonBlocking));
    cudaStream_t ws = p->webp_stream;
    DB_CUDA(cudaEventRecord(p->webp_fork, s));
    DB_CUDA(cudaStreamWaitEvent(ws, p->webp_fork, 0));
    if (p->webp_pending) { DB_CUDA(cudaEventSynchronize(p->webp_uploaded)); p->webp_pending = false; }
    const JpegImage *hi = reinterpret_cast<const JpegImage *>(p->h_images);    // the output pointers of this launch
    int64_t px = 0;
    for (WebpImage &wi : p->webp_images) {
      const JpegImage &im = hi[wi.sample];
      wi.out = im.out; wi.out_type = im.out_type;
      wi.win_x0 = im.win_x0; wi.win_y0 = im.win_y0; wi.win_w = im.win_w; wi.win_h = im.win_h;
      wi.first_px = px;
      px += (int64_t)im.win_w * im.win_h;
    }
    const size_t nwi = p->webp_images.size(), wbytes = Align(sizeof(WebpImage) * nwi, 16);
    if ((rc = p->webp_arena.Reserve(wbytes))) return rc;
    memcpy(p->webp_arena.host, p->webp_images.data(), sizeof(WebpImage) * nwi);
    if ((rc = p->webp_arena.Upload(wbytes, ws))) return rc;
    DB_CUDA(cudaEventRecord(p->webp_uploaded, ws));
    p->webp_pending = true;
    WebpLaunch a;
    a.d_images = reinterpret_cast<const WebpImage *>(p->webp_arena.dev); a.nimages = (int)nwi;
    a.total_px = px;
    a.d_raw = d_raw; a.d_scratch = p->d_webp_scratch; a.d_status = p->d_status;
    if ((rc = LaunchWebp(a, ws))) return rc;
    DB_CUDA(cudaEventRecord(p->webp_join, ws));
  }
  const bool any_units = nunits > 0 && p->nchunks > 0 && p->total_blocks_sync > 0;      // false: every sample of the batch is progressive
  if (any_units) {
    const int grid = (int)std::min<uint32_t>(p->nchunks, (uint32_t)sms * 16);
    { ProfScope ps_("jpeg_unstuff_count", s); unstuff_count_kernel<<<grid, 256, 0, s>>>(d_raw, d_units, nunits, p->nchunks, p->d_chunk); }
    { ProfScope ps_("jpeg_unstuff_scan", s); unstuff_scan_kernel<<<(nunits + 7) / 8, 256, 0, s>>>(d_units, nunits, p->d_chunk, p->d_unit_len); }
    { ProfScope ps_("jpeg_unstuff_scatter", s); unstuff_scatter_kernel<<<grid, 256, 0, s>>>(d_raw, d_units, nunits, p->nchunks, p->d_chunk, p->d_clean); }
    CountLaunch(3);
  }
  HuffCtx cx;
  cx.images = d_images; cx.nimages = p->n; cx.block_image = reinterpret_cast<const int32_t *>(p->d_stage + p->off_blkimg);
  cx.wblock_image = reinterpret_cast<const int32_t *>(p->d_stage + p->off_wblkimg);
  cx.units = d_units; cx.unit_clean_len = p->d_unit_len; cx.tables = d_tables;
  cx.clean = p->d_clean; cx.s_state = p->d_state; cx.s_n = p->d_n; cx.coef = p->d_coef; cx.dc = p->d_dc; cx.log2_sub = p->log2_sub;
  cx.status = p->d_status; cx.unit_nblk = p->d_unit_nblk;
  cx.chains[0] = p->d_chain1; cx.chains[1] = p->d_chain2; cx.chains[2] = p->d_chain3; cx.chain_count = p->d_chain_count;
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
  if (any_units) { ProfScope ps_("jpeg_huff_sync_intra", s); huff_sync_intra_kernel<<<p->total_blocks_sync, kSyncThreads, hsmem, s>>>(cx); }
  if (any_units) {
    // chain walk: grids sized for the expected list lengths (about 30 % / 8 % / 2.5 % of the subsequences carry a live chain
    // after 1 / 2 / 3 visits); CTAs beyond the actual length return at once, grid-stride loops cover longer lists
    auto walk_grid = [&](double frac) {
      const int64_t want = (int64_t)(p->total_subseq * frac) / kTailThreads + p->total_blocks_sync / kTailThreads + 1;
      return (int)std::max<int64_t>(1, std::min<int64_t>(p->walk_max_grid, want));
    };
    { ProfScope ps_("jpeg_huff_sync_walk1", s); huff_sync_walk_kernel<<<walk_grid(0.40), kTailThreads, walk_smem, s>>>(cx, 0, 1, 1); }
    { ProfScope ps_("jpeg_huff_sync_walk2", s); huff_sync_walk_kernel<<<walk_grid(0.14), kTailThreads, walk_smem, s>>>(cx, 1, 2, 1); }
    { ProfScope ps_("jpeg_huff_sync_walk3", s); huff_sync_walk_kernel<<<walk_grid(0.06), kTailThreads, walk_smem, s>>>(cx, 2, 0, 1 << 30); }
    CountLaunch(2);
  }
  { ProfScope ps_("jpeg_huff_scan", s); huff_scan_kernel<<<p->n, 1024, 0, s>>>(cx); }
  CountLaunch();
  if (any_units && p->total_blocks_write > 0) { ProfScope ps_("jpeg_huff_write", s); huff_write_kernel<<<p->total_blocks_write, kWriteThreads, wsmem, s>>>(cx); }
  if (!p->prog_images.empty()) DB_CUDA(cudaStreamWaitEvent(s, p->prog_join, 0));      // the progressive samples' coefficients and DC differences are in place
  { ProfScope ps_("jpeg_dc_scan", s); dc_scan_kernel<<<p->n, 1024, 0, s>>>(d_images, p->d_dc); }
  { ProfScope ps_("jpeg_truncation_fixup", s); truncation_fixup_kernel<<<p->n, 256, 0, s>>>(cx); }
  CountLaunch();
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
  if (!p->png_images.empty()) DB_CUDA(cudaStreamWaitEvent(s, p->png_join, 0));       // the PNG samples' windows and status are in place
  if (!p->tiff_images.empty()) DB_CUDA(cudaStreamWaitEvent(s, p->tiff_join, 0));     // the TIFF samples' windows and status are in place
  if (!p->webp_images.empty()) DB_CUDA(cudaStreamWaitEvent(s, p->webp_join, 0));     // the WebP samples' windows and status are in place
  if (!p->posts.empty()) {
    const int grid = (int)std::max<int64_t>(1, std::min<int64_t>((p->total_post_px + 255) / 256, (int64_t)sms * 16));
    ProfScope ps_("jpeg_post", s);
    if (p->dtype == DALIB200_FLOAT) jpeg_post_kernel<float><<<grid, 256, 0, s>>>(p->d_posts, (int)p->posts.size(), p->total_post_px);
    else jpeg_post_kernel<uint8_t><<<grid, 256, 0, s>>>(p->d_posts, (int)p->posts.size(), p->total_post_px);
    CountLaunch();
  }
  CountLaunch(5);
  DB_CUDA(cudaGetLastError());
  return DALIB200_SUCCESS;
} DB_API_CATCH

}  // extern "C"
