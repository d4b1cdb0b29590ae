// tools/emul/paste_emul.cc -- TEST INFRASTRUCTURE.  The planner of fn.multi_paste / fn.paste (dali_b200/csrc/paste_plan.h) and the
// kernel's per-thread bodies (paste_core.h) compiled for the host, so that tests/test_paste_cpu.py runs them without a GPU:
//   g++ -std=c++17 -O2 -shared -fPIC tools/emul/paste_emul.cc -o paste_emul.so                  (ctypes: emul_paste, emul_paste_canvas)
//   g++ -std=c++17 -O1 -g -fsanitize=address,undefined -DPASTE_EMUL_MAIN tools/emul/paste_emul.cc -o ps_fuzz
// The second form plans and runs random types, channel counts, batches, regions (in_ids and multi-input forms, every argument form),
// output sizes and byte offsets, checks every output bit for bit against a direct statement (each element from the last region that
// covers it) and the bytes around it, and prints "ok <cases>"; under the sanitizers it checks that no plan reaches memory it must not.
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>
#include "../../dali_b200/csrc/paste_plan.h"

using namespace dalib200;

static int run_plan(PsPlanData &p, const void *const *ins, void *const *outs, int64_t *out_shapes, int64_t *items, int64_t *bands) {
  for (size_t k = 0; out_shapes && k < p.out_shapes.size(); k++) out_shapes[k] = p.out_shapes[k];
  for (int i = 0; items && i < p.n; i++) items[i] = p.samples[i].items;
  for (int i = 0; bands && i < p.n; i++) bands[i] = p.samples[i].items ? p.samples[i].nbands : 0;
  if (!outs) return 0;
  std::vector<PsSample> d = p.samples;
  // the fill table at a 16-byte boundary, as in the arena
  std::vector<uint8_t> fmem(p.fill.size() + 16);
  uint8_t *const ft = fmem.data() + ((16 - ((uintptr_t)fmem.data() & 15)) & 15);
  memcpy(ft, p.fill.data(), p.fill.size());
  for (int i = 0; i < p.n; i++) {
    if (!d[i].items) continue;
    d[i].out = outs[i];
    d[i].bands = p.bands.data() + p.band_off[i];
    d[i].segs = p.segs.data() + p.seg_off[i];
  }
  PsBatch B = { ins, ft, p.nfill, p.in_type, p.out_type, 0 };
  PsRunOnHost(d.data(), p.n, p.items, B);
  return 0;
}

// multi_paste: plans, and when outs is not NULL runs the kernel on the host.  Arguments as dalib200PasteSetup.  Returns 0, or 1 with
// the planner's message in err.  items / bands (may be NULL) receive the work items and the bands of each output.
extern "C" int emul_paste(int in_type, int out_type, int ninputs, int n, const int *ndims, const char *const *layouts, const int64_t *in_shapes,
                          const int32_t *in_ids, const int64_t *in_id_counts, const double *const *args, const int64_t *const *counts,
                          const int64_t *out_sizes, const float *fill, int nfill, const void *const *ins, void *const *outs,
                          int64_t *out_shapes, int64_t *items, int64_t *bands, char *err, int errcap) {
  PsPlanData p;
  std::string e;
  if (!PsSetup(&p, in_type, out_type, ninputs, n, ndims, layouts, in_shapes, in_ids, in_id_counts, args, counts, out_sizes, fill, nfill, &e)) {
    snprintf(err, errcap, "%s", e.c_str());
    return 1;
  }
  return run_plan(p, ins, outs, out_shapes, items, bands);
}

// paste: as dalib200PasteCanvasSetup.
extern "C" int emul_paste_canvas(int in_type, int n, int ndim, const char *layout, const int64_t *in_shapes, int n_channels, const float *ratio,
                                 const float *paste_x, const float *paste_y, const float *min_canvas, const float *fill, int nfill,
                                 const void *const *ins, void *const *outs, int64_t *out_shapes, char *err, int errcap) {
  PsPlanData p;
  std::string e;
  if (!PsCanvasSetup(&p, in_type, n, ndim, layout, in_shapes, n_channels, ratio, paste_x, paste_y, min_canvas, fill, nfill, &e)) {
    snprintf(err, errcap, "%s", e.c_str());
    return 1;
  }
  return run_plan(p, ins, outs, out_shapes, nullptr, nullptr);
}

#ifdef PASTE_EMUL_MAIN
int main(int argc, char **argv) {
  const int cases = argc > 1 ? atoi(argv[1]) : 300;
  srand(argc > 2 ? atoi(argv[2]) : 1);
  char err[512];
  for (int c = 0; c < cases; c++) {
    const int it = rand() % 12, ot = rand() % 3 ? it : rand() % 12, isz = arith_size(it), osz = arith_size(ot);
    const int C = 1 + rand() % 5, n = 1 + rand() % 4;
    const bool ids = rand() % 2;
    const int ninputs = ids ? 1 : 1 + rand() % 4;
    std::vector<int64_t> shapes((size_t)ninputs * n * 3);
    for (int s = 0; s < ninputs * n; s++) {
      shapes[(size_t)s * 3] = rand() % 8 == 0 ? 0 : 1 + rand() % 30;
      shapes[(size_t)s * 3 + 1] = 1 + rand() % 40;
      shapes[(size_t)s * 3 + 2] = C;
    }
    std::vector<int64_t> osz_hw((size_t)n * 2);
    for (auto &v : osz_hw) v = rand() % 10 == 0 ? 0 : 1 + rand() % 50;
    // regions: pixel rectangles drawn inside their source and the output, given in absolute form
    std::vector<int32_t> idv;
    std::vector<int64_t> idc(n), cnt(n);
    std::vector<double> ia, sh, oa;
    std::vector<PsRegion> all;
    std::vector<int64_t> nreg(n);
    for (int i = 0; i < n; i++) {
      const int K = ids ? (rand() % 6 == 0 ? 0 : rand() % 5 == 0 ? 20 + rand() % 40 : 1 + rand() % 4) : ninputs;
      idc[i] = K;
      cnt[i] = 2 * K;
      nreg[i] = K;
      for (int k = 0; k < K; k++) {
        const int src = ids ? rand() % n : k * n + i;
        if (ids) idv.push_back(src);
        const int64_t Hs = shapes[(size_t)src * 3], Ws = shapes[(size_t)src * 3 + 1], H = osz_hw[2 * i], W = osz_hw[2 * i + 1];
        const int64_t h = rand() % 7 == 0 ? 0 : rand() % (std::min(Hs, H) + 1), w = rand() % 7 == 0 ? 0 : rand() % (std::min(Ws, W) + 1);
        const int64_t iy = rand() % (Hs - h + 1), ix = rand() % (Ws - w + 1), oy = rand() % (H - h + 1), ox = rand() % (W - w + 1);
        ia.push_back((double)iy), ia.push_back((double)ix);
        sh.push_back((double)h), sh.push_back((double)w);
        oa.push_back((double)oy), oa.push_back((double)ox);
        all.push_back(PsRegion{ src, iy, ix, h, w, oy, ox });
      }
    }
    ia.push_back(0), sh.push_back(0), oa.push_back(0);
    const double *args[6] = { ia.data(), nullptr, sh.data(), nullptr, oa.data(), nullptr };
    const int64_t *counts[6] = { cnt.data(), nullptr, cnt.data(), nullptr, cnt.data(), nullptr };
    std::vector<int> ndims(ninputs, 3);
    std::vector<const char *> lays(ninputs, "HWC");
    const int nfill = 1;
    const float fill = 0.0f;
    std::vector<std::vector<uint8_t>> in(ninputs * n), out(n);
    std::vector<const void *> ip(ninputs * n);
    std::vector<void *> op(n);
    for (int s = 0; s < ninputs * n; s++) {
      const int64_t vol = shapes[(size_t)s * 3] * shapes[(size_t)s * 3 + 1] * C;
      in[s].resize(vol * isz + 32);
      for (auto &x : in[s]) x = it == kABool ? (uint8_t)(rand() % 2) : (uint8_t)rand();
      ip[s] = in[s].data() + 16 + isz * (rand() % (16 / isz));
    }
    std::vector<int64_t> ovol(n);
    for (int i = 0; i < n; i++) {
      ovol[i] = osz_hw[2 * i] * osz_hw[2 * i + 1] * C;
      out[i].assign(ovol[i] * osz + 64, 0xA5);
      op[i] = out[i].data() + 16 + osz * (rand() % (16 / osz));
    }
    int64_t oshapes[3 * 8];
    if (emul_paste(it, ot, ninputs, n, ndims.data(), lays.data(), shapes.data(), ids ? (idv.empty() ? (const int32_t *)&nfill : idv.data()) : nullptr,
                   ids ? idc.data() : nullptr, args, counts, osz_hw.data(), &fill, nfill, ip.data(), op.data(), oshapes, nullptr, nullptr, err,
                   sizeof(err))) {
      fprintf(stderr, "case %d refused: %s\n", c, err);
      return 1;
    }
    size_t r0 = 0;
    for (int i = 0; i < n; i++) {
      const int64_t H = osz_hw[2 * i], W = osz_hw[2 * i + 1];
      std::vector<uint8_t> want(ovol[i] * osz, 0);
      for (int64_t y = 0; y < H; y++)
        for (int64_t x = 0; x < W; x++) {
          const PsRegion *top = nullptr;
          for (int64_t k = 0; k < nreg[i]; k++) {
            const PsRegion &r = all[r0 + k];
            if (r.h && r.w && y >= r.oy && y < r.oy + r.h && x >= r.ox && x < r.ox + r.w) top = &r;
          }
          if (!top) continue;
          const int64_t Ws = shapes[(size_t)top->src * 3 + 1];
          for (int ch = 0; ch < C; ch++) {
            const int64_t se = ((y - top->oy + top->iy) * Ws + (x - top->ox + top->ix)) * C + ch, oe = (y * W + x) * C + ch;
            const uint64_t v = arith_load(ip[top->src], se, it);
            const uint64_t b = it == ot ? (uint64_t)0 : arith_to_bits(arith_cast(v, it, ot), ot);
            if (it == ot) memcpy(want.data() + oe * osz, static_cast<const uint8_t *>(ip[top->src]) + se * isz, isz);
            else memcpy(want.data() + oe * osz, &b, osz);
          }
        }
      r0 += nreg[i];
      const int64_t pre = static_cast<const uint8_t *>(op[i]) - out[i].data();
      for (int64_t k = 0; k < (int64_t)out[i].size(); k++) {
        const bool in_out = k >= pre && k < pre + ovol[i] * osz;
        if (!in_out && out[i][k] != 0xA5) { fprintf(stderr, "case %d: a write outside the output\n", c); return 1; }
        if (in_out && out[i][k] != want[k - pre]) {
          fprintf(stderr, "case %d (types %d -> %d, C %d, sample %d of %d, %d inputs) differs at byte %lld\n", c, it, ot, C, i, n, ninputs,
                  (long long)(k - pre));
          return 1;
        }
      }
    }
  }
  printf("ok %d\n", cases);
  return 0;
}
#endif
