// dali_b200/csrc/ljpeg.cu -- lossless JPEG (SOF3) decoding inside decoders.image.
//
// The planner (ljpeg_plan.h) checks the frame and splits the scan into restart intervals on the host; their bytes are un-stuffed by the
// JPEG path's U1 - U3 with every other unit of the batch.  Behind that, on the stream that ran U3:
//   L1 + L2a  ljpeg_sync     one thread per 128-byte subsequence: speculative decode from its first bit, then the chain that carries its
//                            exit state to the right until it agrees with the record (ljpeg_walk, ljpeg_core.h)
//   L2b       ljpeg_scan     one CTA per unit: exclusive scan of the symbol counts, status of a short unit or a bad restart sequence
//   L3        ljpeg_write    one thread per subsequence: decode from the true entry state, int16 differences into the arena
//   L4        ljpeg_recon    one CTA per (image, component, restart band): the prediction as a wavefront over the diagonals x + y,
//                            one thread per line, reconstructed in place
//   L5        ljpeg_color    one thread per window pixel: << Pt, colour rules, into the decode window
// Orientation, region of interest, YCbCr and float output are the JPEG path's post pass over that window (jpeg.cu jpeg_post_kernel).
#include "common.cuh"
#include "jpeg_recon.h"
#include "ljpeg.h"
#include <algorithm>

namespace dalib200 {

constexpr int kLjpegRecThreads = 512;

__global__ void __launch_bounds__(256) ljpeg_sync_kernel(LjpegLaunch a) {
  const int64_t step = (int64_t)gridDim.x * blockDim.x;
  for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g < a.total_sub; g += step) {
    const LjpegUnit &u = a.d_units[last_at_most(a.d_units, 0, a.nunits - 1, g, [](const LjpegUnit &p) { return p.first_sub; })];
    ljpeg_walk(a.d_images[u.image], u, g, a.d_clean, a.d_unit_clean_len, a.d_tables, a.d_rec,
               [](uint64_t *p, uint64_t v) { return (uint64_t)atomicMax(reinterpret_cast<unsigned long long *>(p), (unsigned long long)v); });
  }
}

__global__ void __launch_bounds__(256) ljpeg_scan_kernel(LjpegLaunch a) {
  __shared__ uint32_t warp_tot[8];
  __shared__ uint32_t carry;
  const LjpegUnit &u = a.d_units[blockIdx.x];
  const LjpegImage &im = a.d_images[u.image];
  const uint32_t clean_bits = a.d_unit_clean_len[u.junit] * 8u;
  const uint32_t nsub = (clean_bits + (1u << kLjpegLog2Sub) - 1) >> kLjpegLog2Sub;
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  for (uint32_t base = 0; base < nsub; base += blockDim.x) {
    const uint32_t i = base + threadIdx.x;
    const uint32_t v = i < nsub ? ljpeg_count(a.d_rec[u.first_sub + i]) : 0u;
    uint32_t incl = v;
    for (int o = 1; o < 32; o <<= 1) { const uint32_t x = __shfl_up_sync(0xffffffffu, incl, o); if ((threadIdx.x & 31) >= (uint32_t)o) incl += x; }
    if ((threadIdx.x & 31) == 31) warp_tot[threadIdx.x >> 5] = incl;
    __syncthreads();
    uint32_t woff = 0, tot = 0;
    for (int w = 0; w < (int)(blockDim.x >> 5); w++) { if (w < (int)(threadIdx.x >> 5)) woff += warp_tot[w]; tot += warp_tot[w]; }
    if (i < nsub) a.d_first[u.first_sub + i] = carry + woff + incl - v;
    __syncthreads();
    if (threadIdx.x == 0) carry += tot;
    __syncthreads();
  }
  // the pad bits behind the data may decode into a few more symbols, so only a SHORT count is an error; the samples it lacks are 0
  const int64_t have = carry;
  if (threadIdx.x == 0 && (have < u.nsym || im.bad_rst)) a.d_status[im.sample] = 1;
  for (int64_t k = have + threadIdx.x; k < u.nsym; k += blockDim.x) a.d_diff[u.sym_off + k] = 0;
}

__global__ void __launch_bounds__(256) ljpeg_write_kernel(LjpegLaunch a) {
  const int64_t step = (int64_t)gridDim.x * blockDim.x;
  for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g < a.total_sub; g += step) {
    const LjpegUnit &u = a.d_units[last_at_most(a.d_units, 0, a.nunits - 1, g, [](const LjpegUnit &p) { return p.first_sub; })];
    const LjpegImage &im = a.d_images[u.image];
    if (ljpeg_write(im, u, g, a.d_clean, a.d_unit_clean_len, a.d_tables, a.d_rec, a.d_first[g], a.d_diff)) a.d_status[im.sample] = 1;
  }
}

// Thread t owns line y0 + t of a strip of blockDim.x lines and reaches column x at step x + t: (x - 1, y) is its own previous sample,
// (x, y - 1) and (x - 1, y - 1) are the samples of thread t - 1 at the previous two steps (exchanged through shared memory, one barrier
// per step).  Thread 0 of a later strip reads the line above from the arena, where the previous strip left it.
__global__ void __launch_bounds__(kLjpegRecThreads) ljpeg_recon_kernel(const LjpegImage *__restrict__ images, const LjpegBand *__restrict__ bands,
                                                                       int16_t *diff) {
  __shared__ int32_t up[2][kLjpegRecThreads];
  const LjpegBand bd = bands[blockIdx.x];
  const LjpegImage &im = images[bd.image];
  const int W = im.width, C = im.ncomp, t = threadIdx.x, pred = im.pred;
  const int32_t init = 1 << (im.precision - im.pt - 1);
  int16_t *base = diff + im.diff_off + bd.comp;
  for (int r0 = bd.y0; r0 < bd.y1; r0 += blockDim.x) {
    const int rows = min((int)blockDim.x, bd.y1 - r0), y = r0 + t;
    const bool own = t < rows, first_line = y == bd.y0;
    int16_t *row = base + (int64_t)y * W * C;
    const int16_t *above = row - (int64_t)W * C;
    int32_t Ra = 0, Rb = 0, Rc = 0;
    int32_t nxt = own ? row[0] : 0;
    for (int d = 0; d < W + rows - 1; d++) {
      const int x = d - t;
      if (own && x >= 0 && x < W) {
        Rc = Rb;
        if (!first_line) Rb = t == 0 ? (int32_t)(uint16_t)above[(int64_t)x * C] : up[(d - 1) & 1][t - 1];
        const int32_t v = (nxt + ljpeg_predict(pred, first_line, x, init, Ra, Rb, Rc)) & 0xFFFF;
        if (x + 1 < W) nxt = row[(int64_t)(x + 1) * C];
        row[(int64_t)x * C] = (int16_t)v;
        Ra = v;
        up[d & 1][t] = v;
      }
      __syncthreads();
    }
  }
}

__global__ void __launch_bounds__(256) ljpeg_color_kernel(const LjpegImage *__restrict__ images, int nimages, int64_t total,
                                                          const int16_t *__restrict__ diff) {
  const int64_t step = (int64_t)gridDim.x * blockDim.x;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += step) {
    const int i = last_at_most(images, 0, nimages - 1, e, [](const LjpegImage &im) { return im.first_px; });
    ljpeg_pixel(images[i], diff, e - images[i].first_px, [](int r, int g, int b) { return RgbJpegGray(r, g, b); });
  }
}

int LjpegStage::Plan(const LjpegFrame &f, int sample, const uint8_t *d, size_t len, size_t sb, size_t raw, std::vector<JpegUnit> &junits,
                     size_t &clean, uint32_t &chunks, size_t *scan_end, std::string *err) {
  LjpegImage im;
  if (int rc = PlanLjpegFrame(f, &im, tables, err)) return rc;
  if ((int64_t)f.width * f.height >= (1ll << 31)) {
    *err = "images of 2^31 pixels or more are not supported";
    return DALIB200_ERROR_UNSUPPORTED;
  }
  size_t se = len;
  if (se >= sb + 2 && d[se - 2] == 0xFF && d[se - 1] == 0xD9) se -= 2;
  *scan_end = se;
  const int W = f.width, H = f.height, C = f.ncomp;
  const int lines = f.restart_interval ? f.restart_interval / W : H;
  const int nunits = (H + lines - 1) / lines;
  std::vector<std::pair<size_t, size_t>> segs;
  im.bad_rst = SplitLjpegUnits(d, sb, se, nunits, segs);
  for (const auto &sg : segs)
    if (sg.second - sg.first > kLjpegMaxUnitBytes) {
      *err = "lossless JPEG: an entropy-coded segment above " + std::to_string(kLjpegMaxUnitBytes) +
             " bytes is not supported (use restart intervals)";
      return DALIB200_ERROR_UNSUPPORTED;
    }
  im.sample = sample;
  im.diff_off = diff_elems;
  diff_elems += (int64_t)Align((size_t)W * H * C, 8);
  const int li = (int)images.size();
  for (int k = 0; k < nunits; k++) {
    JpegUnit u;
    memset(&u, 0, sizeof(u));
    u.raw_off = (uint32_t)(raw + (segs[k].first - sb));
    u.raw_len = (uint32_t)(segs[k].second - segs[k].first);
    u.clean_off = (uint32_t)clean;
    u.first_chunk = chunks;
    u.image = sample;
    LjpegUnit lu;
    lu.junit = (int32_t)junits.size(); lu.image = li;
    lu.first_sub = total_sub;
    lu.nsub = (int32_t)((u.raw_len + (1u << (kLjpegLog2Sub - 3)) - 1) >> (kLjpegLog2Sub - 3));
    lu.clean_off = u.clean_off;
    const int y0 = k * lines, y1 = std::min(H, y0 + lines);
    lu.nsym = (int64_t)(y1 - y0) * W * C;
    lu.sym_off = im.diff_off + (int64_t)y0 * W * C;
    for (int c = 0; c < C; c++) bands.push_back(LjpegBand{ li, c, y0, y1 });
    total_sub += lu.nsub;
    clean += Align(u.raw_len + kCleanPad, 16);
    chunks += (u.raw_len + kChunkBytes - 1) / kChunkBytes;
    junits.push_back(u);
    units.push_back(lu);
  }
  images.push_back(im);
  return DALIB200_SUCCESS;
}

int LjpegStage::Reserve() {
  int rc;
  if ((rc = GrowDevice(d_diff, d_diff_cap, (size_t)diff_elems + 8))) return rc;
  if ((rc = GrowDevice(d_rec, d_rec_cap, (size_t)total_sub + 1))) return rc;
  return GrowDevice(d_first, d_first_cap, (size_t)total_sub + 1);
}

int LjpegStage::Enqueue(const StageInputs &in, cudaStream_t s) {
  LjpegLaunch a;
  a.total_px = FillWindows(images, in.images);
  if (int rc = arena.Pack(s, std::tie(a.d_images, a.d_units, a.d_tables, a.d_bands), images, units, tables, bands)) return rc;
  a.nimages = (int)images.size(); a.nunits = (int)units.size(); a.nbands = (int)bands.size();
  a.total_sub = total_sub;
  a.d_clean = in.d_clean; a.d_unit_clean_len = in.d_unit_clean_len;
  a.d_rec = d_rec; a.d_first = d_first; a.d_diff = d_diff; a.d_status = in.d_status;
  const int sms = NumSMs();
  auto grid_of = [&](int64_t n) { return (int)std::max<int64_t>(1, std::min<int64_t>((n + 255) / 256, (int64_t)sms * 16)); };
  if (a.total_sub > 0) {
    DB_CUDA(cudaMemsetAsync(a.d_rec, 0, sizeof(uint64_t) * a.total_sub, s));
    Launch("ljpeg_sync", ljpeg_sync_kernel, grid_of(a.total_sub), 256, 0, s, a);
  }
  Launch("ljpeg_scan", ljpeg_scan_kernel, a.nunits, 256, 0, s, a);
  if (a.total_sub > 0) Launch("ljpeg_write", ljpeg_write_kernel, grid_of(a.total_sub), 256, 0, s, a);
  Launch("ljpeg_recon", ljpeg_recon_kernel, a.nbands, kLjpegRecThreads, 0, s, a.d_images, a.d_bands, a.d_diff);
  Launch("ljpeg_color", ljpeg_color_kernel, grid_of(a.total_px), 256, 0, s, a.d_images, a.nimages, a.total_px, a.d_diff);
  DB_CUDA(cudaGetLastError());
  return DALIB200_SUCCESS;
}

}  // namespace dalib200
