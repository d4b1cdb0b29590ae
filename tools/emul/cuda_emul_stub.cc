// tools/emul/cuda_emul_stub.cc -- TEST INFRASTRUCTURE.  LD_PRELOAD replacement of the CUDA runtime calls the library makes, like
// tools/fuzz/cuda_stub.c, with two differences: "device" memory is host memory whose copies and memsets really happen, and the launches
// of the 3-D resize, progressive JPEG, PNG, TIFF, WebP, BMP / PNM, lossless JPEG, audio decode, arithmetic-expression, reduction, equalize, filter, erase and paste kernels (and U2 / U3, which feed the
// lossless JPEG stage) are
// EXECUTED on the host -- their bodies are single
// host/device functions (dali_b200/csrc/resample3d_core.h, jpeg_prog_core.h, png_core.h, tiff_core.h, webp_core.h, bitmap_core.h, arith_core.h ...), so a
// launch is a loop over blocks and threads around
// the same function the device runs.  All other kernels are no-ops.  With this preloaded, the real launch path of the library runs
// end to end without a GPU -- descriptor upload, temporaries, stage order, grid-stride loops, wave ranges, arena offsets -- and
// tests/test_launch_emul_cpu.py compares what lands in "device" memory with the oracle.
//
// DALIB200_EMUL_TRACE=<file> also writes the stream-ordering calls to <file>, one line each, in host call order: event creation,
// record, stream wait, synchronisation and destruction, stream creation, synchronisation and destruction, cudaMemsetAsync, H2D
// cudaMemcpyAsync and every kernel launch (by its demangled name).  Events and streams are renumbered by first appearance (e0, e1, ...,
// s0, s1, ...; a destroyed handle's number is not reused), so two runs of one batch give the same text, and
// tests/test_decoder_stage_order_emul_cpu.py can check the order of the decoder's side stages from it.  An H2D copy names its source:
// p<k> for the k-th cudaMallocHost allocation (counted from 0 in allocation order), "-" for any other host memory; with that,
// tests/test_pinned_reuse_emul_cpu.py checks that every plan waits for the last copy out of a pinned buffer before it reuses it.
//   g++ -std=c++17 -O2 -ffp-contract=off -shared -fPIC -I/usr/local/cuda/include tools/emul/cuda_emul_stub.cc -ldl
#ifndef _GNU_SOURCE
#define _GNU_SOURCE
#endif
#include <cxxabi.h>
#include <dlfcn.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <algorithm>
#include <map>
#include <mutex>
#include <string>
#include <vector>
#include "../../include/dali_b200.h"
#include "../../dali_b200/csrc/resample3d_core.h"
#include "../../dali_b200/csrc/jpeg_prog_core.h"
#include "../../dali_b200/csrc/png_core.h"
#include "../../dali_b200/csrc/tiff_core.h"
#include "../../dali_b200/csrc/webp_core.h"
#include "../../dali_b200/csrc/bitmap_core.h"
#include "../../dali_b200/csrc/jpeg_recon.h"
#include "../../dali_b200/csrc/ljpeg_core.h"
#include "../../dali_b200/csrc/audio_decode_core.h"
#include "../../dali_b200/csrc/arith_plan.h"
#include "../../dali_b200/csrc/reduce_plan.h"
#include "../../dali_b200/csrc/equalize_core.h"
#include "../../dali_b200/csrc/filter_plan.h"
#include "../../dali_b200/csrc/erase_plan.h"
#include "../../dali_b200/csrc/paste_plan.h"

using namespace dalib200;
typedef int cudaError_t;
struct Dim3 { unsigned x, y, z; };

// ---- call trace (DALIB200_EMUL_TRACE)
static FILE *trace_file() {
  static FILE *f = [] { const char *p = getenv("DALIB200_EMUL_TRACE"); return p && *p ? fopen(p, "w") : nullptr; }();
  return f;
}
static std::mutex g_trace_mu;
static std::map<const void *, int> g_events, g_streams;
static int g_nevents = 0, g_nstreams = 0;
static int ev(const void *e) { auto it = g_events.find(e); return it != g_events.end() ? it->second : (g_events[e] = g_nevents++); }
static int st(const void *s) { auto it = g_streams.find(s); return it != g_streams.end() ? it->second : (g_streams[s] = g_nstreams++); }
static int forget(std::map<const void *, int> &m, int id, const void *h) { m.erase(h); return id; }   // the allocator may reuse h
// cudaMallocHost allocations (base -> size, number in allocation order) while they live, to name the source of an H2D copy
static std::mutex g_pinned_mu;
static std::map<const void *, std::pair<size_t, int>> g_pinned;
static int g_npinned = 0;
static int pinned_of(const void *p) {           // the allocation holding p, or -1
  std::lock_guard<std::mutex> l(g_pinned_mu);
  auto it = g_pinned.upper_bound(p);
  if (it == g_pinned.begin()) return -1;
  --it;
  return static_cast<const char *>(p) < static_cast<const char *>(it->first) + it->second.first ? it->second.second : -1;
}
#define TRACE(...)                                                                                            \
  do {                                                                                                        \
    if (FILE *f_ = trace_file()) {                                                                            \
      std::lock_guard<std::mutex> l_(g_trace_mu);                                                             \
      fprintf(f_, __VA_ARGS__); fputc('\n', f_); fflush(f_);                                                  \
    }                                                                                                         \
  } while (0)
// "dalib200::jpeg_post_kernel<float>" of "_ZN8dalib20016jpeg_post_kernelIfEEvPKNS_8JpegPostEil": no return type, no parameters
static std::string kernel_name(const char *mangled) {
  int rc = 0;
  char *d = abi::__cxa_demangle(mangled, nullptr, nullptr, &rc);
  std::string s = rc == 0 && d ? d : *mangled ? mangled : "?";
  free(d);
  s = s.substr(0, s.find('('));
  if (!s.compare(0, 5, "void ")) s = s.substr(5);
  return s;
}

extern "C" {
cudaError_t cudaEventCreateWithFlags(void **e, unsigned) { *e = malloc(8); TRACE("event_create e%d", ev(*e)); return 0; }
cudaError_t cudaEventCreate(void **e) { *e = malloc(8); TRACE("event_create e%d", ev(*e)); return 0; }
cudaError_t cudaEventDestroy(void *e) { TRACE("event_destroy e%d", forget(g_events, ev(e), e)); free(e); return 0; }
cudaError_t cudaEventSynchronize(void *e) { TRACE("event_sync e%d", ev(e)); return 0; }
cudaError_t cudaEventRecord(void *e, void *s) { TRACE("record e%d s%d", ev(e), st(s)); return 0; }
cudaError_t cudaEventQuery(void *) { return 0; }
cudaError_t cudaHostAlloc(void **p, size_t n, unsigned) { *p = calloc(n ? n : 1, 1); return *p ? 0 : 2; }
cudaError_t cudaMallocHost(void **p, size_t n) {
  *p = calloc(n ? n : 1, 1);
  if (!*p) return 2;
  std::lock_guard<std::mutex> l(g_pinned_mu);
  g_pinned[*p] = { n, g_npinned++ };
  return 0;
}
cudaError_t cudaFreeHost(void *p) {
  { std::lock_guard<std::mutex> l(g_pinned_mu); g_pinned.erase(p); }
  free(p);
  return 0;
}
// fresh "device" memory is filled with a pattern: a kernel that relies on zeroed memory it never cleared shows up
cudaError_t cudaMalloc(void **p, size_t n) { *p = malloc(n ? n : 1); if (*p) memset(*p, 0xA5, n ? n : 1); return *p ? 0 : 2; }
cudaError_t cudaFree(void *p) { free(p); return 0; }
cudaError_t cudaGetDevice(int *d) { *d = 0; return 0; }
cudaError_t cudaSetDevice(int) { return 0; }
cudaError_t cudaGetDeviceCount(int *n) { *n = 1; return 0; }
cudaError_t cudaDeviceGetAttribute(int *v, int, int) { *v = 132; return 0; }
static int g_last_error = 0;                    // sticky like the runtime's: a launch with an empty grid must surface at the next check
cudaError_t cudaGetLastError(void) { const int e = g_last_error; g_last_error = 0; return e; }
cudaError_t cudaPeekAtLastError(void) { return g_last_error; }
const char *cudaGetErrorName(cudaError_t e) { return e == 9 ? "cudaErrorInvalidConfiguration" : e ? "cudaErrorUnknown" : "cudaSuccess"; }
const char *cudaGetErrorString(cudaError_t e) { return e == 9 ? "invalid configuration argument (emulated launch)" : e ? "error" : "no error"; }
cudaError_t cudaStreamSynchronize(void *s) { TRACE("stream_sync s%d", st(s)); return 0; }
cudaError_t cudaMemsetAsync(void *p, int v, size_t n, void *s) { TRACE("memset s%d %zu", st(s), n); memset(p, v, n); return 0; }
cudaError_t cudaMemcpyAsync(void *d, const void *s, size_t n, int kind, void *stream) {
  if (kind == 1) {                                              // cudaMemcpyHostToDevice
    const int h = pinned_of(s);
    if (h >= 0) TRACE("h2d s%d %zu p%d", st(stream), n, h);
    else TRACE("h2d s%d %zu -", st(stream), n);
  }
  memmove(d, s, n);
  return 0;
}
cudaError_t cudaMemcpy(void *d, const void *s, size_t n, int) { memmove(d, s, n); return 0; }
cudaError_t cudaMemset(void *p, int v, size_t n) { memset(p, v, n); return 0; }
cudaError_t cudaDeviceSynchronize(void) { return 0; }
cudaError_t cudaMemcpyBatchAsync(void **d, void **s, size_t *sz, size_t cnt, void *, size_t *, size_t, size_t *, void *) {
  for (size_t i = 0; i < cnt; i++) memmove(d[i], s[i], sz[i]);
  return 0;
}
struct stubPtrAttr { int type; int device; void *devp; void *hostp; };
cudaError_t cudaPointerGetAttributes(stubPtrAttr *a, const void *p) { a->type = 0; a->device = 0; a->devp = 0; a->hostp = (void *)p; return 0; }
cudaError_t cudaGetDriverEntryPoint(const char *, void **fn, unsigned long long, int *status) { *fn = 0; if (status) *status = 1; return 0; }
cudaError_t cudaEventElapsedTime(float *ms, void *, void *) { *ms = 0; return 0; }
cudaError_t cudaStreamCreateWithFlags(void **s, unsigned) { *s = malloc(8); TRACE("stream_create s%d", st(*s)); return 0; }
cudaError_t cudaStreamCreate(void **s) { *s = malloc(8); TRACE("stream_create s%d", st(*s)); return 0; }
cudaError_t cudaStreamDestroy(void *s) { TRACE("stream_destroy s%d", forget(g_streams, st(s), s)); free(s); return 0; }
cudaError_t cudaStreamWaitEvent(void *s, void *e, unsigned) { TRACE("wait s%d e%d", st(s), ev(e)); return 0; }
cudaError_t cudaFuncSetAttribute(const void *, int, int) { return 0; }
cudaError_t cudaOccupancyMaxActiveBlocksPerMultiprocessor(int *n, const void *, int, size_t) { *n = 2; return 0; }
cudaError_t cudaOccupancyMaxActiveBlocksPerMultiprocessorWithFlags(int *n, const void *, int, size_t, unsigned) { *n = 2; return 0; }

static long g_emulated[35];
long emul_launch_count(int which) { return g_emulated[which]; }
void emul_trace_mark(const char *text) { TRACE("# %s", text); }    // a section header in the trace, written by the test

// kernels of dali_b200/csrc/resample3d.cu, jpeg_prog.cu, png.cu, tiff.cu, webp.cu and bitmap.cu, thread by thread
static void run_resample3d_pass(Dim3 g, Dim3 b, void **args) {
  const R3Pass *passes = *static_cast<const R3Pass **>(args[0]);
  const int32_t *tab = *static_cast<const int32_t **>(args[1]);
  const int stride = *static_cast<int *>(args[2]);
  for (unsigned by = 0; by < g.y; by++) {
    const R3Pass p = passes[(int64_t)by * stride];
    const int64_t step = (int64_t)g.x * b.x;
    for (unsigned bx = 0; bx < g.x; bx++)
      for (unsigned tx = 0; tx < b.x; tx++)
        for (int64_t e = (int64_t)bx * b.x + tx; e < p.total; e += step) r3_element(p, tab, e);
  }
}
static void run_prog_scan(Dim3 g, Dim3, void **args) {
  const ProgScan *scans = *static_cast<const ProgScan **>(args[0]);
  const int first = *static_cast<int *>(args[1]);
  const ProgImage *images = *static_cast<const ProgImage **>(args[2]);
  const ProgHuff *huff = *static_cast<const ProgHuff **>(args[3]);
  const uint8_t *raw = *static_cast<const uint8_t **>(args[4]);
  int16_t *coef = *static_cast<int16_t **>(args[5]);
  int32_t *status = *static_cast<int32_t **>(args[6]);
  for (int bx = (int)g.x - 1; bx >= 0; bx--) {             // blocks of a launch run in no particular order: take the reverse one
    const ProgScan s = scans[first + bx];
    const ProgImage im = images[s.image];
    if (prog_decode_scan(s, im, huff, raw, coef)) status[im.sample] = 1;
  }
}
static void run_prog_dc(Dim3 g, Dim3 b, void **args) {
  const ProgImage *images = *static_cast<const ProgImage **>(args[0]);
  const int64_t *first_blk = *static_cast<const int64_t **>(args[1]);
  const int nimages = *static_cast<int *>(args[2]);
  const int64_t total = *static_cast<int64_t *>(args[3]);
  const int16_t *coef = *static_cast<const int16_t **>(args[4]);
  int16_t *dc = *static_cast<int16_t **>(args[5]);
  int32_t *status = *static_cast<int32_t **>(args[6]);
  const int64_t step = (int64_t)g.x * b.x;
  for (unsigned bx = 0; bx < g.x; bx++)
    for (unsigned tx = 0; tx < b.x; tx++)
      for (int64_t e = (int64_t)bx * b.x + tx; e < total; e += step) {
        const int i = last_at_most(first_blk, 0, nimages - 1, e);
        prog_dc_difference(images[i], coef, dc, e - first_blk[i]);
        if (e == first_blk[i] && images[i].incomplete) status[images[i].sample] = 1;
      }
}

static void run_png_crc(Dim3 g, Dim3 b, void **args) {
  const PngChunk *chunks = *static_cast<const PngChunk **>(args[0]);
  const int nchunks = *static_cast<int *>(args[1]);
  const PngImage *images = *static_cast<const PngImage **>(args[2]);
  const uint8_t *raw = *static_cast<const uint8_t **>(args[3]);
  int32_t *status = *static_cast<int32_t **>(args[4]);
  uint32_t table[256];
  for (uint32_t i = 0; i < 256; i++) table[i] = png_crc_table_entry(i);
  for (int k = 0; k < (int)(g.x * b.x) && k < nchunks; k++) {
    const PngImage &im = images[chunks[k].image];
    if (!png_chunk_crc_ok(raw + im.raw_off + chunks[k].off - 4, chunks[k].len, table)) status[im.sample] = 1;
  }
}
static void run_png_inflate(Dim3 g, Dim3, void **args) {
  const PngImage *images = *static_cast<const PngImage **>(args[0]);
  const PngChunk *chunks = *static_cast<const PngChunk **>(args[1]);
  const uint8_t *raw = *static_cast<const uint8_t **>(args[2]);
  uint8_t *scan = *static_cast<uint8_t **>(args[3]);
  int32_t *status = *static_cast<int32_t **>(args[4]);
  InflateWork *w = new InflateWork;
  for (int bx = (int)g.x - 1; bx >= 0; bx--) {             // one working thread per block, blocks in no particular order
    const PngImage &im = images[bx];
    if (status[im.sample]) continue;
    if (png_inflate_unfilter(im, chunks, raw, scan + im.scan_off, *w)) status[im.sample] = 1;
  }
  delete w;
}
static void run_png_color(Dim3 g, Dim3 b, void **args) {
  const PngImage *images = *static_cast<const PngImage **>(args[0]);
  const int nimages = *static_cast<int *>(args[1]);
  const int64_t total = *static_cast<int64_t *>(args[2]);
  const uint8_t *scan = *static_cast<const uint8_t **>(args[3]);
  const int64_t step = (int64_t)g.x * b.x;
  for (unsigned bx = 0; bx < g.x; bx++)
    for (unsigned tx = 0; tx < b.x; tx++)
      for (int64_t e = (int64_t)bx * b.x + tx; e < total; e += step) {
        const PngImage &im = images[last_at_most(images, 0, nimages - 1, e, [](const PngImage &m) { return m.first_px; })];
        const int64_t lp = e - im.first_px;
        const int ly = (int)(lp / im.win_w), lx = (int)(lp - (int64_t)ly * im.win_w);
        png_pixel(im, scan + im.scan_off, lx, ly);
      }
}

static void run_tiff_segment(Dim3 g, Dim3 b, void **args) {
  const TiffImage *images = *static_cast<const TiffImage **>(args[0]);
  const TiffSeg *segs = *static_cast<const TiffSeg **>(args[1]);
  const int nsegs = *static_cast<int *>(args[2]);
  const int lanes = *static_cast<int *>(args[3]);
  const uint8_t *raw = *static_cast<const uint8_t **>(args[4]);
  uint8_t *dec = *static_cast<uint8_t **>(args[5]);
  uint8_t *slots = *static_cast<uint8_t **>(args[6]);
  int32_t *status = *static_cast<int32_t **>(args[7]);
  for (int bx = (int)g.x - 1; bx >= 0; bx--)                 // blocks of a launch run in no particular order: take the reverse one
    for (int tx = 0; tx < (int)b.x && tx < lanes; tx++) {
      const int w = bx * lanes + tx;
      for (int k = w; k < nsegs; k += (int)g.x * lanes) {
        const TiffImage &im = images[segs[k].image];
        if (status[im.sample]) continue;
        if (tiff_decode_segment(im, segs[k], raw, dec + segs[k].dec_off, slots + (size_t)w * kTiffSlotBytes)) status[im.sample] = 1;
      }
    }
}
static void run_tiff_color(Dim3 g, Dim3 b, void **args) {
  const TiffImage *images = *static_cast<const TiffImage **>(args[0]);
  const int nimages = *static_cast<int *>(args[1]);
  const int64_t total = *static_cast<int64_t *>(args[2]);
  const TiffSeg *segs = *static_cast<const TiffSeg **>(args[3]);
  const uint8_t *dec = *static_cast<const uint8_t **>(args[4]);
  const int64_t step = (int64_t)g.x * b.x;
  for (unsigned bx = 0; bx < g.x; bx++)
    for (unsigned tx = 0; tx < b.x; tx++)
      for (int64_t e = (int64_t)bx * b.x + tx; e < total; e += step) {
        const TiffImage &im = images[last_at_most(images, 0, nimages - 1, e, [](const TiffImage &m) { return m.first_px; })];
        const int64_t lp = e - im.first_px;
        const int ly = (int)(lp / im.win_w), lx = (int)(lp - (int64_t)ly * im.win_w);
        tiff_pixel(im, segs, dec, lx, ly);
      }
}

static void run_webp_entropy(Dim3 g, Dim3 b, void **args) {
  const WebpImage *images = *static_cast<const WebpImage **>(args[0]);
  const int nimages = *static_cast<int *>(args[1]);
  const int lanes = *static_cast<int *>(args[2]);
  const uint8_t *raw = *static_cast<const uint8_t **>(args[3]);
  uint8_t *scratch = *static_cast<uint8_t **>(args[4]);
  int32_t *status = *static_cast<int32_t **>(args[5]);
  for (int bx = (int)g.x - 1; bx >= 0; bx--)                 // blocks of a launch run in no particular order: take the reverse one
    for (int tx = 0; tx < (int)b.x && tx < lanes; tx++)
      for (int k = bx * lanes + tx; k < nimages; k += (int)g.x * lanes) {
        const WebpImage &im = images[k];
        if (webp_entropy(im, raw, reinterpret_cast<WebpMb *>(scratch + im.mb_off), reinterpret_cast<int16_t *>(scratch + im.coef_off),
                         reinterpret_cast<uint32_t *>(scratch + im.ctx_off)))
          status[im.sample] = 1;
      }
}
// webp_wave_kernel<false / true>: one block per image; the macroblocks of each diagonal run in REVERSE thread order, so that a
// dependency between two macroblocks of one diagonal shows up as a mismatch
static void run_webp_wave(Dim3 g, Dim3 b, void **args, bool filter) {
  const WebpImage *images = *static_cast<const WebpImage **>(args[0]);
  uint8_t *scratch = *static_cast<uint8_t **>(args[1]);
  const int32_t *status = *static_cast<const int32_t **>(args[2]);
  for (int bx = (int)g.x - 1; bx >= 0; bx--) {
    const WebpImage &im = images[bx];
    if (status[im.sample] || (filter && im.filter_type == 0)) continue;
    const WebpMb *mbs = reinterpret_cast<const WebpMb *>(scratch + im.mb_off);
    const int16_t *coef = reinterpret_cast<const int16_t *>(scratch + im.coef_off);
    for (int d = 0; d < im.mb_w + 2 * (im.mb_h - 1); d++) {
      const int y_lo = std::max(0, (d - im.mb_w + 2) / 2), y_hi = std::min(im.mb_h - 1, d / 2);
      for (int tx = (int)b.x - 1; tx >= 0; tx--)
        for (int y = y_lo + tx; y <= y_hi; y += (int)b.x) {
          if (filter) webp_filter_mb(im, mbs, scratch, d - 2 * y, y);
          else webp_recon_mb(im, mbs, coef, scratch, d - 2 * y, y);
        }
    }
  }
}
static void run_webp_color(Dim3 g, Dim3 b, void **args) {
  const WebpImage *images = *static_cast<const WebpImage **>(args[0]);
  const int nimages = *static_cast<int *>(args[1]);
  const int64_t total = *static_cast<int64_t *>(args[2]);
  uint8_t *scratch = *static_cast<uint8_t **>(args[3]);
  const int64_t step = (int64_t)g.x * b.x;
  for (unsigned bx = 0; bx < g.x; bx++)
    for (unsigned tx = 0; tx < b.x; tx++)
      for (int64_t e = (int64_t)bx * b.x + tx; e < total; e += step) {
        const WebpImage &im = images[last_at_most(images, 0, nimages - 1, e, [](const WebpImage &m) { return m.first_px; })];
        const int64_t lp = e - im.first_px;
        const int ly = (int)(lp / im.win_w), lx = (int)(lp - (int64_t)ly * im.win_w);
        webp_pixel(im, scratch, lx, ly);
      }
}

static void run_bitmap_unpack(Dim3 g, Dim3 b, void **args) {
  const BitmapImage *images = *static_cast<const BitmapImage **>(args[0]);
  const int32_t *list = *static_cast<const int32_t **>(args[1]);
  const int nlist = *static_cast<int *>(args[2]);
  const int lanes = *static_cast<int *>(args[3]);
  const uint8_t *raw = *static_cast<const uint8_t **>(args[4]);
  uint8_t *scratch = *static_cast<uint8_t **>(args[5]);
  int32_t *status = *static_cast<int32_t **>(args[6]);
  for (int bx = (int)g.x - 1; bx >= 0; bx--)                 // blocks of a launch run in no particular order: take the reverse one
    for (int tx = 0; tx < (int)b.x && tx < lanes; tx++)
      for (int k = bx * lanes + tx; k < nlist; k += (int)g.x * lanes) {
        const BitmapImage &im = images[list[k]];
        if (bitmap_unpack(im, raw + im.raw_off, scratch + im.plane_off)) status[im.sample] = 1;
      }
}
static void run_bitmap_color(Dim3 g, Dim3 b, void **args) {
  const BitmapImage *images = *static_cast<const BitmapImage **>(args[0]);
  const int nimages = *static_cast<int *>(args[1]);
  const int64_t total = *static_cast<int64_t *>(args[2]);
  const uint8_t *raw = *static_cast<const uint8_t **>(args[3]);
  const uint8_t *scratch = *static_cast<const uint8_t **>(args[4]);
  const int64_t step = (int64_t)g.x * b.x;
  for (unsigned bx = 0; bx < g.x; bx++)
    for (unsigned tx = 0; tx < b.x; tx++)
      for (int64_t e = (int64_t)bx * b.x + tx; e < total; e += step) {
        const BitmapImage &im = images[last_at_most(images, 0, nimages - 1, e, [](const BitmapImage &m) { return m.first_grp; })];
        bitmap_group(im, im.unpack == kBitmapDirect ? raw + im.raw_off : scratch + im.plane_off, e - im.first_grp);
      }
}

// U2 / U3 of jpeg.cu as their result: each unit's clean length, and its clean stream (FF 00 -> FF, word-swapped, zero pad behind it).
// They serve the lossless JPEG stage here; the baseline kernels that read the clean streams are not emulated.
static uint32_t unstuff_unit(const uint8_t *raw, const JpegUnit &u, uint8_t *clean) {
  uint32_t q = 0;
  for (uint32_t i = 0; i < u.raw_len; i++) {
    const uint8_t *p = raw + u.raw_off + i;
    if (i > 0 && p[0] == 0 && p[-1] == 0xFF) continue;
    if (clean) clean[(u.clean_off + q) ^ 3u] = p[0];
    q++;
  }
  if (clean)
    for (uint32_t e = u.clean_off + q; e < u.clean_off + ((u.raw_len + 32u + 15u) & ~15u); e++) clean[e ^ 3u] = 0;
  return q;
}
static const uint8_t *g_unstuff_raw;                 // the raw buffer of the last unstuff_count launch (the scan launch has none)
static void run_unstuff_count(void **args) { g_unstuff_raw = *static_cast<const uint8_t **>(args[0]); }
static void run_unstuff_scan(void **args) {
  const JpegUnit *units = *static_cast<const JpegUnit **>(args[0]);
  const int n = *static_cast<int *>(args[1]);
  uint32_t *len = *static_cast<uint32_t **>(args[3]);
  for (int k = n - 1; k >= 0; k--) len[k] = unstuff_unit(g_unstuff_raw, units[k], nullptr);
}
static void run_unstuff_scatter(void **args) {
  const uint8_t *raw = *static_cast<const uint8_t **>(args[0]);
  const JpegUnit *units = *static_cast<const JpegUnit **>(args[1]);
  const int n = *static_cast<int *>(args[2]);
  uint8_t *clean = *static_cast<uint8_t **>(args[5]);
  for (int k = n - 1; k >= 0; k--) unstuff_unit(raw, units[k], clean);
}

// ljpeg.cu.  ljpeg_sync and ljpeg_write take the subsequences in REVERSE order, so that a chain always meets the records of the chains
// that started to its right first; ljpeg_recon walks each band in raster order, which keeps every dependency of the wavefront.
static int ljpeg_unit_of(const LjpegLaunch &a, int64_t g) {
  int k = a.nunits - 1;
  while (a.d_units[k].first_sub > g) k--;
  return k;
}
static void run_ljpeg_sync(void **args) {
  const LjpegLaunch &a = *static_cast<const LjpegLaunch *>(args[0]);
  auto amax = [](uint64_t *p, uint64_t v) { const uint64_t o = *p; if (v > o) *p = v; return o; };
  for (int64_t g = a.total_sub - 1; g >= 0; g--) {
    const LjpegUnit &u = a.d_units[ljpeg_unit_of(a, g)];
    ljpeg_walk(a.d_images[u.image], u, g, a.d_clean, a.d_unit_clean_len, a.d_tables, a.d_rec, amax);
  }
}
static void run_ljpeg_scan(void **args) {
  const LjpegLaunch &a = *static_cast<const LjpegLaunch *>(args[0]);
  for (int k = a.nunits - 1; k >= 0; k--) {
    const LjpegUnit &u = a.d_units[k];
    const LjpegImage &im = a.d_images[u.image];
    const uint32_t nsub = (a.d_unit_clean_len[u.junit] * 8u + (1u << kLjpegLog2Sub) - 1) >> kLjpegLog2Sub;
    uint32_t run = 0;
    for (uint32_t i = 0; i < nsub; i++) { a.d_first[u.first_sub + i] = run; run += ljpeg_count(a.d_rec[u.first_sub + i]); }
    if ((int64_t)run < u.nsym || im.bad_rst) a.d_status[im.sample] = 1;
    for (int64_t s = run; s < u.nsym; s++) a.d_diff[u.sym_off + s] = 0;
  }
}
static void run_ljpeg_write(void **args) {
  const LjpegLaunch &a = *static_cast<const LjpegLaunch *>(args[0]);
  for (int64_t g = a.total_sub - 1; g >= 0; g--) {
    const LjpegUnit &u = a.d_units[ljpeg_unit_of(a, g)];
    const LjpegImage &im = a.d_images[u.image];
    if (ljpeg_write(im, u, g, a.d_clean, a.d_unit_clean_len, a.d_tables, a.d_rec, a.d_first[g], a.d_diff)) a.d_status[im.sample] = 1;
  }
}
static void run_ljpeg_recon(Dim3 g, void **args) {
  const LjpegImage *images = *static_cast<const LjpegImage **>(args[0]);
  const LjpegBand *bands = *static_cast<const LjpegBand **>(args[1]);
  int16_t *diff = *static_cast<int16_t **>(args[2]);
  for (int bx = (int)g.x - 1; bx >= 0; bx--) {
    const LjpegBand bd = bands[bx];
    const LjpegImage &im = images[bd.image];
    const int W = im.width, C = im.ncomp;
    const int32_t init = 1 << (im.precision - im.pt - 1);
    auto at = [&](int y, int x) -> int16_t & { return diff[im.diff_off + ((int64_t)y * W + x) * C + bd.comp]; };
    for (int y = bd.y0; y < bd.y1; y++)
      for (int x = 0; x < W; x++) {
        const bool fl = y == bd.y0;
        const int32_t Ra = x ? (uint16_t)at(y, x - 1) : 0, Rb = fl ? 0 : (uint16_t)at(y - 1, x), Rc = fl || !x ? 0 : (uint16_t)at(y - 1, x - 1);
        at(y, x) = (int16_t)((at(y, x) + ljpeg_predict(im.pred, fl, x, init, Ra, Rb, Rc)) & 0xFFFF);
      }
  }
}
static void run_ljpeg_color(void **args) {
  const LjpegImage *images = *static_cast<const LjpegImage **>(args[0]);
  const int n = *static_cast<int *>(args[1]);
  const int64_t total = *static_cast<int64_t *>(args[2]);
  const int16_t *diff = *static_cast<const int16_t **>(args[3]);
  for (int64_t e = total - 1; e >= 0; e--) {
    int i = n - 1;
    while (images[i].first_px > e) i--;
    ljpeg_pixel(images[i], diff, e - images[i].first_px, [](int r, int gg, int b) { return RgbJpegGray(r, gg, b); });
  }
}

// audio_decode.cu: every pass over its whole index space in REVERSE order (the sync pass's atomic add is a plain one here, so the
// candidates land in reverse byte order), with the descriptor searches the kernels make.
static void run_flac_sync(void **args) {
  const AudioLaunch &a = *static_cast<const AudioLaunch *>(args[0]);
  auto add = [](uint32_t *p, uint32_t v) { const uint32_t o = *p; *p = o + v; return o; };
  for (int64_t g = a.flac_bytes - 1; g >= 0; g--) {
    const int f = last_at_most(a.flac, 0, a.nf - 1, g, [](const FlacDesc &d) { return d.first_byte; });
    flac_sync_at(a.flac[f], f, a.raw, g - a.flac[f].first_byte, a.fend, a.cand, a.ccount, add);
  }
}
static void run_flac_frame(void **args) {
  const AudioLaunch &a = *static_cast<const AudioLaunch *>(args[0]);
  for (int64_t k = a.cand_slots - 1; k >= 0; k--) {
    const int f = last_at_most(a.flac, 0, a.nf - 1, k, [](const FlacDesc &d) { return d.cand_base; });
    flac_candidate(a.flac[f], f, a.raw, k - a.flac[f].cand_base, a.cand, a.ccount, a.fend);
  }
}
static void run_flac_chain(void **args) {
  const AudioLaunch &a = *static_cast<const AudioLaunch *>(args[0]);
  for (int f = a.nf - 1; f >= 0; f--)
    if (!flac_chain(a.flac[f], f, a.raw, a.fend, a.ccount, a.frames, a.nframes)) a.status[a.flac[f].sample] = 1;
}
static void run_flac_decode(void **args) {
  const AudioLaunch &a = *static_cast<const AudioLaunch *>(args[0]);
  for (int64_t k = a.frame_slots - 1; k >= 0; k--) {
    const int f = last_at_most(a.flac, 0, a.nf - 1, k, [](const FlacDesc &d) { return d.frame_base; });
    if (!flac_decode(a.flac[f], f, a.raw, k - a.flac[f].frame_base, a.frames, a.nframes, a.pcm)) a.status[a.flac[f].sample] = 1;
  }
}
static void run_audio_convert(void **args) {
  const AudioLaunch &a = *static_cast<const AudioLaunch *>(args[0]);
  for (int i = a.n - 1; i >= 0; i--) *a.descs[i].rate_out = a.descs[i].rate;
  for (int64_t e = a.total_elems - 1; e >= 0; e--) {
    const AudioDesc &d = a.descs[last_at_most(a.descs, 0, a.n - 1, e, [](const AudioDesc &p) { return p.first_elem; })];
    audio_convert(d, a.raw, a.pcm, e - d.first_elem, [](float x, float y) { return x * y; }, [](float x, float y) { return x + y; });
  }
}
// audio_resample_kernel (audio_tail.cu) is not a host/device function: its launches are recorded, not run.  For each sample of the last
// launch the stub keeps the descriptor's lengths and channels and a copy of its input, so that a test can check what decoders.audio hands
// to the resampler.  The layout restates audio_tail.cu's ArDesc.
struct EmulArDesc { const float *in; float *out; int64_t n_in, n_out, first_item; double scale; int32_t channels; };
static std::vector<std::vector<float>> g_res_in;
static std::vector<EmulArDesc> g_res_desc;
static void run_audio_resample_record(void **args) {
  const EmulArDesc *d = *static_cast<const EmulArDesc **>(args[0]);
  const int n = *static_cast<int *>(args[1]);
  g_res_desc.assign(d, d + n);
  g_res_in.assign(n, {});
  for (int i = 0; i < n; i++) g_res_in[i].assign(d[i].in, d[i].in + d[i].n_in * d[i].channels);
}
int emul_resample_count(void) { return (int)g_res_desc.size(); }
// info: { n_in, n_out, channels }; copies the input (n_in * channels floats) to dst when dst is not NULL
void emul_resample_sample(int i, int64_t *info, float *dst) {
  info[0] = g_res_desc[i].n_in; info[1] = g_res_desc[i].n_out; info[2] = g_res_desc[i].channels;
  if (dst) memcpy(dst, g_res_in[i].data(), g_res_in[i].size() * sizeof(float));
}

// arith.cu: the work items of the launch in REVERSE order, the threads of each block in reverse order
static void run_arith(Dim3 g, Dim3 b, void **args, bool wide) {
  const ArithProgram &p = *static_cast<const ArithProgram *>(args[0]);
  const ArithSample *samples = *static_cast<const ArithSample **>(args[1]);
  const int n = *static_cast<int *>(args[2]);
  const int64_t total = *static_cast<int64_t *>(args[3]);
  (void)g;
  for (int64_t item = total - 1; item >= 0; item--) {
    int s = n - 1;
    while (samples[s].first_item > item) s--;
    const ArithSample &d = samples[s];
    const int64_t e0 = (item - d.first_item) * kArithItem, e1 = std::min(d.n, e0 + kArithItem);
    for (int64_t base = e0; base < e1; base += (int64_t)kArithEpt * b.x)
      for (int tx = (int)b.x - 1; tx >= 0; tx--) {
        if (wide) arith_elements<true>(p, d, base, e1, tx);
        else arith_elements<false>(p, d, base, e1, tx);
      }
  }
}

// reduce.cu: the template arguments come from the demangled name ("dalib200::reduce_pass_kernel<unsigned char, unsigned long, 2>");
// the work items of the launch run in REVERSE order, the threads of each block in reverse order
static int red_type_code(const std::string &t) {
  static const char *const names[] = { "unsigned char", "unsigned short", "unsigned int", "unsigned long", "signed char", "short", "int",
                                       "long", "dalib200::RedHalf", "float", "double" };
  for (int k = 0; k < 11; k++)
    if (t == names[k]) return k;
  return -1;
}
static std::vector<std::string> red_template_args(const std::string &name) {
  std::vector<std::string> a;
  const size_t lt = name.find('<'), gt = name.rfind('>');
  std::string cur;
  for (size_t k = lt + 1; k < gt; k++) {
    if (name[k] == ',') { a.push_back(cur); cur.clear(); continue; }
    if (!(cur.empty() && name[k] == ' ')) cur += name[k];
  }
  a.push_back(cur);
  return a;
}
static void run_reduce(const std::string &name, void **args, bool combine) {
  const RedPass *descs = *static_cast<const RedPass **>(args[0]);
  const int n = *static_cast<int *>(args[1]);
  const int64_t total = *static_cast<int64_t *>(args[2]);
  const RedFinal f = *static_cast<const RedFinal *>(args[3]);
  const std::vector<std::string> ta = red_template_args(name);
  const int tc = red_type_code(ta[0]), ac = red_type_code(combine ? ta[0] : ta[1]);
  const int e = atoi((combine ? ta[1] : ta[2]).c_str());
  const int32_t acc = ac == kRedI64 ? kAccI64 : ac == kRedU64 ? kAccU64 : ac == kRedF32 ? kAccF32 : kAccF64;
  alignas(16) static uint8_t smem[kRedSmemBytes];
  const auto body = [&](auto t, auto a, auto el) {
    typedef decltype(t) T;
    typedef decltype(a) A;
    constexpr int E = decltype(el)::value;
    A *sm = reinterpret_cast<A *>(smem), *sm2 = reinterpret_cast<A *>(smem + kRedThreads * 16 * 8);
    for (int64_t item = total - 1; item >= 0; item--) {
      const RedPass &d = descs[last_at_most(descs, 0, n - 1, item, [&](const RedPass &p) { return combine ? p.cfirst : p.first_item; })];
      if (combine) {
        for (int tx = kRedThreads - 1; tx >= 0; tx--) red_combine<A, E>(d, f, item - d.cfirst, tx);
        continue;
      }
      const int64_t local = item - d.first_item;
      if (d.path == kRedPathColumns) {
        for (int tx = kRedThreads - 1; tx >= 0; tx--) red_columns<T, A, E>(d, f, local, tx);
        continue;
      }
      const RedRun u = red_run<T>(d, local);
      for (int tx = kRedThreads - 1; tx >= 0; tx--) red_inner_fold<T, A, E>(d, u, sm, tx);
      for (int tx = kRedThreads - 1; tx >= 0; tx--) red_inner_slices<T, A, E>(d, u, sm, sm2, tx);
      for (int i = (int)d.I - 1; i >= 0; i--) {
        A v[32];
        for (int l = 31; l >= 0; l--) v[l] = red_inner_lane<A, E>(d, sm2, i, l);
        red_store(d, f, u.ch, u.o * d.I + i, red_tree32<A, E>(v));
      }
    }
  };
  red_dispatch(tc, acc, e, body);
}

// equalize.cu: the work items of the launch run in REVERSE order, the threads of each block in reverse order; the apply kernel's
// per-plane warp scan runs lane by lane (eq_lut_plane)
static void run_equalize(void **args, bool apply) {
  const EqSample *descs = *static_cast<const EqSample **>(args[0]);
  const int n = *static_cast<int *>(args[1]);
  const int64_t total = *static_cast<int64_t *>(args[2]);
  uint32_t *hist = *static_cast<uint32_t **>(args[3]);
  static uint32_t sh[kEqSmemWords];
  static uint8_t lut[kEqMaxChannels * 256];
  for (int64_t item = total - 1; item >= 0; item--) {
    const EqSample &d = descs[last_at_most(descs, 0, n - 1, item, [](const EqSample &e) { return e.first_item; })];
    const int64_t local = item - d.first_item;
    if (apply) {
      const int64_t frame = eq_item(d, local).frame;
      for (int c = d.C - 1; c >= 0; c--) eq_lut_plane(hist + d.hist_off + (frame * d.C + c) * 256, d.plane, lut + c * 256);
      for (int t = kEqThreads - 1; t >= 0; t--) eq_apply_thread(d, local, lut, t);
      continue;
    }
    memset(sh, 0, sizeof(sh));
    for (int t = kEqThreads - 1; t >= 0; t--) eq_hist_thread(d, local, sh + ((t >> 5) % d.nsub) * d.C * 256, t);
    for (int t = kEqThreads - 1; t >= 0; t--) eq_hist_flush(d, local, sh, hist, t);
  }
}

cudaError_t cudaLaunchKernel(const void *func, Dim3 grid, Dim3 block, void **args, size_t, void *stream) {
  // the library is usually loaded with RTLD_LOCAL (ctypes): identify the kernel by the name of the host stub `func` points at
  Dl_info di;
  const char *name = func && dladdr(func, &di) && di.dli_sname && di.dli_saddr == func ? di.dli_sname : "";
  TRACE("launch %s s%d", kernel_name(name).c_str(), st(stream));
  const bool is_r3 = !strcmp(name, "_ZN8dalib20022resample3d_pass_kernelEPKNS_6R3PassEPKii");
  const bool is_scan = !strcmp(name, "_ZN8dalib20016prog_scan_kernelEPKNS_8ProgScanEiPKNS_9ProgImageEPKNS_8ProgHuffEPKhPsPi");
  const bool is_dc = !strcmp(name, "_ZN8dalib20014prog_dc_kernelEPKNS_9ProgImageEPKlilPKsPsPi");
  const bool is_png_crc = !strcmp(name, "_ZN8dalib20014png_crc_kernelEPKNS_8PngChunkEiPKNS_8PngImageEPKhPi");
  const bool is_png_inflate = !strcmp(name, "_ZN8dalib20018png_inflate_kernelEPKNS_8PngImageEPKNS_8PngChunkEPKhPhPi");
  const bool is_png_color = !strcmp(name, "_ZN8dalib20016png_color_kernelEPKNS_8PngImageEilPKh");
  const bool is_tiff_segment = !strcmp(name, "_ZN8dalib20019tiff_segment_kernelEPKNS_9TiffImageEPKNS_7TiffSegEiiPKhPhS8_Pi");
  const bool is_tiff_color = !strcmp(name, "_ZN8dalib20017tiff_color_kernelEPKNS_9TiffImageEilPKNS_7TiffSegEPKh");
  const bool is_webp_entropy = !strcmp(name, "_ZN8dalib20019webp_entropy_kernelEPKNS_9WebpImageEiiPKhPhPi");
  const bool is_webp_recon = !strcmp(name, "_ZN8dalib20016webp_wave_kernelILb0EEEvPKNS_9WebpImageEPhPKi");
  const bool is_webp_filter = !strcmp(name, "_ZN8dalib20016webp_wave_kernelILb1EEEvPKNS_9WebpImageEPhPKi");
  const bool is_webp_color = !strcmp(name, "_ZN8dalib20017webp_color_kernelEPKNS_9WebpImageEilPh");
  const bool is_bitmap_unpack = !strcmp(name, "_ZN8dalib20020bitmap_unpack_kernelEPKNS_11BitmapImageEPKiiiPKhPhPi");
  const bool is_bitmap_color = !strcmp(name, "_ZN8dalib20019bitmap_color_kernelEPKNS_11BitmapImageEilPKhS4_");
  const bool is_unstuff_count = !strcmp(name, "_ZN8dalib20020unstuff_count_kernelEPKhPKNS_8JpegUnitEijPj");
  const bool is_unstuff_scan = !strcmp(name, "_ZN8dalib20019unstuff_scan_kernelEPKNS_8JpegUnitEiPjS3_");
  const bool is_unstuff_scatter = !strcmp(name, "_ZN8dalib20022unstuff_scatter_kernelEPKhPKNS_8JpegUnitEijPKjPh");
  const bool is_ljpeg_sync = !strcmp(name, "_ZN8dalib20017ljpeg_sync_kernelENS_11LjpegLaunchE");
  const bool is_ljpeg_scan = !strcmp(name, "_ZN8dalib20017ljpeg_scan_kernelENS_11LjpegLaunchE");
  const bool is_ljpeg_write = !strcmp(name, "_ZN8dalib20018ljpeg_write_kernelENS_11LjpegLaunchE");
  const bool is_ljpeg_recon = !strcmp(name, "_ZN8dalib20018ljpeg_recon_kernelEPKNS_10LjpegImageEPKNS_9LjpegBandEPs");
  const bool is_ljpeg_color = !strcmp(name, "_ZN8dalib20018ljpeg_color_kernelEPKNS_10LjpegImageEilPKs");
  const bool is_flac_sync = !strcmp(name, "_ZN8dalib20016flac_sync_kernelENS_11AudioLaunchE");
  const bool is_flac_frame = !strcmp(name, "_ZN8dalib20017flac_frame_kernelENS_11AudioLaunchEi");
  const bool is_flac_chain = !strcmp(name, "_ZN8dalib20017flac_chain_kernelENS_11AudioLaunchE");
  const bool is_flac_decode = !strcmp(name, "_ZN8dalib20018flac_decode_kernelENS_11AudioLaunchEi");
  const bool is_audio_convert = !strcmp(name, "_ZN8dalib20020audio_convert_kernelENS_11AudioLaunchE");
  const bool is_audio_resample = !strcmp(name, "_ZN8dalib20021audio_resample_kernelEPKNS_6ArDescEilNS_8ArWindowE");
  const bool is_arith_wide = !strcmp(name, "_ZN8dalib20012arith_kernelILb1EEEvNS_12ArithProgramEPKNS_11ArithSampleEil");
  const bool is_arith = is_arith_wide || !strcmp(name, "_ZN8dalib20012arith_kernelILb0EEEvNS_12ArithProgramEPKNS_11ArithSampleEil");
  const std::string kname = kernel_name(name);
  const bool is_reduce_pass = !kname.compare(0, 29, "dalib200::reduce_pass_kernel<");
  const bool is_reduce_combine = !kname.compare(0, 32, "dalib200::reduce_combine_kernel<");
  const bool is_eq_hist = !strcmp(name, "_ZN8dalib20020equalize_hist_kernelEPKNS_8EqSampleEilPj");
  const bool is_eq_apply = !strcmp(name, "_ZN8dalib20021equalize_apply_kernelEPKNS_8EqSampleEilPKj");
  const bool is_filter = !kname.compare(0, 24, "dalib200::filter_kernel<");
  const bool is_erase = !kname.compare(0, 23, "dalib200::erase_kernel<");
  const bool is_paste = !kname.compare(0, 23, "dalib200::paste_kernel<");
  if (grid.x == 0 || grid.y == 0 || grid.z == 0 || block.x == 0 || grid.y > 65535 || block.x > 1024) {
    g_last_error = 9;                              // cudaErrorInvalidConfiguration
    return 9;
  }
  if (is_r3) { run_resample3d_pass(grid, block, args); g_emulated[0]++; }
  else if (is_scan) { run_prog_scan(grid, block, args); g_emulated[1]++; }
  else if (is_dc) { run_prog_dc(grid, block, args); g_emulated[2]++; }
  else if (is_png_crc) { run_png_crc(grid, block, args); g_emulated[3]++; }
  else if (is_png_inflate) { run_png_inflate(grid, block, args); g_emulated[4]++; }
  else if (is_png_color) { run_png_color(grid, block, args); g_emulated[5]++; }
  else if (is_tiff_segment) { run_tiff_segment(grid, block, args); g_emulated[6]++; }
  else if (is_tiff_color) { run_tiff_color(grid, block, args); g_emulated[7]++; }
  else if (is_webp_entropy) { run_webp_entropy(grid, block, args); g_emulated[8]++; }
  else if (is_webp_recon) { run_webp_wave(grid, block, args, false); g_emulated[9]++; }
  else if (is_webp_filter) { run_webp_wave(grid, block, args, true); g_emulated[10]++; }
  else if (is_webp_color) { run_webp_color(grid, block, args); g_emulated[11]++; }
  else if (is_bitmap_unpack) { run_bitmap_unpack(grid, block, args); g_emulated[12]++; }
  else if (is_bitmap_color) { run_bitmap_color(grid, block, args); g_emulated[13]++; }
  else if (is_unstuff_count) { run_unstuff_count(args); g_emulated[14]++; }
  else if (is_unstuff_scan) { run_unstuff_scan(args); g_emulated[14]++; }
  else if (is_unstuff_scatter) { run_unstuff_scatter(args); g_emulated[14]++; }
  else if (is_ljpeg_sync) { run_ljpeg_sync(args); g_emulated[15]++; }
  else if (is_ljpeg_scan) { run_ljpeg_scan(args); g_emulated[16]++; }
  else if (is_ljpeg_write) { run_ljpeg_write(args); g_emulated[17]++; }
  else if (is_ljpeg_recon) { run_ljpeg_recon(grid, args); g_emulated[18]++; }
  else if (is_ljpeg_color) { run_ljpeg_color(args); g_emulated[19]++; }
  else if (is_flac_sync) { run_flac_sync(args); g_emulated[21]++; }
  else if (is_flac_frame) { run_flac_frame(args); g_emulated[22]++; }
  else if (is_flac_chain) { run_flac_chain(args); g_emulated[23]++; }
  else if (is_flac_decode) { run_flac_decode(args); g_emulated[24]++; }
  else if (is_audio_convert) { run_audio_convert(args); g_emulated[25]++; }
  else if (is_audio_resample) { run_audio_resample_record(args); g_emulated[26]++; }
  else if (is_arith) { run_arith(grid, block, args, is_arith_wide); g_emulated[27]++; }
  else if (is_reduce_pass) { run_reduce(kname, args, false); g_emulated[28]++; }
  else if (is_reduce_combine) { run_reduce(kname, args, true); g_emulated[29]++; }
  else if (is_eq_hist) { run_equalize(args, false); g_emulated[30]++; }
  else if (is_eq_apply) { run_equalize(args, true); g_emulated[31]++; }
  else if (is_filter) {                            // filter.cu: FltRunOnHost, the types from the descriptors
    FltRunOnHost(*static_cast<const FltSample **>(args[0]), *static_cast<int *>(args[1]), *static_cast<int64_t *>(args[2]),
                 *static_cast<int *>(args[3]), *static_cast<int *>(args[4]));
    g_emulated[32]++;
  }
  else if (is_erase) {                             // erase.cu: ErRunOnHost, the element size from the descriptors
    ErRunOnHost(*static_cast<const ErSample **>(args[0]), *static_cast<int *>(args[1]), *static_cast<int64_t *>(args[2]),
                *static_cast<const uint8_t **>(args[3]), *static_cast<int *>(args[4]));
    g_emulated[33]++;
  }
  else if (is_paste) {                             // paste.cu: PsRunOnHost, the element size and conversion from the batch
    PsRunOnHost(*static_cast<const PsSample **>(args[0]), *static_cast<int *>(args[1]), *static_cast<int64_t *>(args[2]),
                *static_cast<const PsBatch *>(args[3]));
    g_emulated[34]++;
  }
  return 0;
}
}  // extern "C"
