// tools/emul/filter_emul.cc -- TEST INFRASTRUCTURE.  The planner of fn.experimental.filter (dali_b200/csrc/filter_plan.h) and the
// kernel's per-thread bodies (filter_core.h) compiled for the host, so that tests/test_filter_cpu.py runs them without a GPU:
//   g++ -std=c++17 -O2 -ffp-contract=off -shared -fPIC tools/emul/filter_emul.cc -o filter_emul.so          (ctypes: emul_filter)
//   g++ -std=c++17 -O1 -g -ffp-contract=off -fsanitize=address,undefined -DFILTER_EMUL_MAIN tools/emul/filter_emul.cc -o flt_fuzz
// The second form plans and runs random types, layouts, shapes, filters, anchors, borders, modes, fill values and byte offsets,
// checks every output bit for bit against a direct statement (one fmaf per tap, filter rows outer) and the bytes around it, and prints
// "ok <cases>"; under the sanitizers it checks that no plan reaches memory it must not.
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>
#include "../../dali_b200/csrc/filter_plan.h"

using namespace dalib200;

// Plans, and when outs is not NULL runs the kernel on the host.  Filters and fill values are host pointers (fills NULL: none).
// Returns 0, or 1 with the planner's message in err.
extern "C" int emul_filter(int in_type, int out_type, int n, int ndim, const int64_t *in_shapes, const char *layout, const int64_t *filter_shapes,
                           const int32_t *anchors, int border, int mode, int fill_type, const int64_t *fill_counts, int64_t *out_shapes,
                           const void *const *ins, const void *const *filters, const void *const *fills, void *const *outs, int64_t *items,
                           char *err, int errcap) {
  FltPlanData p;
  std::string e;
  if (!FltSetup(&p, in_type, out_type, n, ndim, in_shapes, layout, kAF32, 2, filter_shapes, anchors, border, mode, fill_type, fill_counts,
                out_shapes, &e)) {
    snprintf(err, errcap, "%s", e.c_str());
    return 1;
  }
  for (int i = 0; items && i < n; i++) items[i] = p.samples[i].items;
  if (!outs) return 0;
  std::vector<FltSample> d = p.samples;
  for (int i = 0; i < n; i++) {
    if (!d[i].items) continue;
    d[i].in = ins[i];
    d[i].out = outs[i];
    d[i].filter = static_cast<const float *>(filters[i]);
    d[i].fill = p.has_fill ? fills[i] : nullptr;
  }
  FltRunOnHost(d.data(), n, p.items, p.row_floats, p.chunk);
  return 0;
}

#ifdef FILTER_EMUL_MAIN
static int64_t ref_index(int64_t i, int64_t n, int border) {   // the border rules, stated by walking instead of by period
  if (border == kFltConstant) return i >= 0 && i < n ? i : -1;
  if (border == kFltClamp) return i < 0 ? 0 : i >= n ? n - 1 : i;
  if (border == kFltWrap) return ((i % n) + n) % n;
  while (i < 0 || i >= n) {
    if (n == 1) return 0;
    if (border == kFltReflect101) i = i < 0 ? -i : 2 * (n - 1) - i;
    else i = i < 0 ? -i - 1 : 2 * n - 1 - i;
  }
  return i;
}

template <typename T> static float to_f(const void *p, int64_t k) { return flt_to_float(static_cast<const T *>(p)[k]); }

int main(int argc, char **argv) {
  const int cases = argc > 1 ? atoi(argv[1]) : 300;
  srand(argc > 2 ? atoi(argv[2]) : 1);
  const int types[] = { kAU8, kAI8, kAU16, kAI16, kAF16, kAF32 };
  char err[512];
  for (int c = 0; c < cases; c++) {
    const int in_type = types[rand() % 6], out_type = rand() % 3 ? in_type : kAF32, esz = FltTypeSize(in_type),
              osz = FltTypeSize(out_type);
    const int li = rand() % 5;                               // 4: the empty layout
    const char *layout = li < 4 ? kFltLayouts[li] : "";
    const int ndim = li < 4 ? (int)strlen(layout) : 2 + rand() % 2 * (1 + rand() % 2);
    const char *lay = li < 4 ? layout : ndim == 2 ? "HW" : ndim == 3 ? "HWC" : "FHWC";
    const int border = rand() % 5, mode = rand() % 4 == 0 ? kFltValid : kFltSame;
    const bool fill = rand() % 2;
    const int n = 1 + rand() % 3;
    std::vector<int64_t> shapes((size_t)n * ndim), fshapes(2 * (size_t)n), outs_shape((size_t)n * ndim), fcount(n);
    std::vector<int32_t> anchors(2 * (size_t)n);
    std::vector<std::vector<float>> filt(n);
    for (int i = 0; i < n; i++) {
      int64_t *s = shapes.data() + (size_t)i * ndim;
      for (int a = 0; a < ndim; a++) {
        const char ax = lay[a];
        s[a] = ax == 'C' ? 1 + rand() % (rand() % 4 ? 4 : kFltMaxChannels) : ax == 'F' ? rand() % 3
             : rand() % 12 == 0 ? 0 : 1 + rand() % (rand() % 4 ? 20 : 300);
      }
      const int64_t H = s[lay[0] == 'F'], W = s[(lay[0] == 'F') + 1];
      fshapes[2 * i] = 1 + rand() % (rand() % 4 ? 7 : 40);
      fshapes[2 * i + 1] = 1 + rand() % (rand() % 4 ? 7 : 40);
      if (mode == kFltValid) {
        fshapes[2 * i] = 1 + rand() % (H > 0 ? (H < 30 ? H : 30) : 1);
        fshapes[2 * i + 1] = 1 + rand() % (W > 0 ? (W < 30 ? W : 30) : 1);
        if (H == 0 || W == 0) s[lay[0] == 'F'] = s[(lay[0] == 'F') + 1] = 3, fshapes[2 * i] = fshapes[2 * i + 1] = 1;
      }
      anchors[2 * i] = rand() % 3 ? -1 : rand() % fshapes[2 * i];
      anchors[2 * i + 1] = rand() % 3 ? -1 : rand() % fshapes[2 * i + 1];
      filt[i].resize(fshapes[2 * i] * fshapes[2 * i + 1]);
      for (auto &v : filt[i]) v = (float)(rand() % 2001 - 1000) / 256.0f;
      fcount[i] = lay[0] == 'F' && rand() % 2 ? s[0] : 1;
    }
    std::vector<std::vector<uint8_t>> in(n), out(n), fills(n);
    std::vector<const void *> ip(n), fp(n), vp(n);
    std::vector<void *> op(n);
    std::vector<int64_t> vol(n, 1), ovol(n, 1), items(n);
    if (emul_filter(in_type, out_type, n, ndim, shapes.data(), layout, fshapes.data(), anchors.data(), border, mode, fill ? in_type : -1,
                    fcount.data(), outs_shape.data(), nullptr, nullptr, nullptr, nullptr, items.data(), err, sizeof(err))) {
      fprintf(stderr, "case %d refused: %s\n", c, err);
      return 1;
    }
    for (int i = 0; i < n; i++) {
      for (int a = 0; a < ndim; a++) vol[i] *= shapes[(size_t)i * ndim + a], ovol[i] *= outs_shape[(size_t)i * ndim + a];
      in[i].resize(vol[i] * esz + 32);
      for (auto &x : in[i]) x = (uint8_t)rand();
      if (in_type == kAF16 || in_type == kAF32)                // finite values of a moderate range
        for (int64_t k = 0; k < vol[i]; k++) {
          const float v = (float)(rand() % 20001 - 10000) / 64.0f;
          if (in_type == kAF32) memcpy(in[i].data() + 16 + k * 4, &v, 4);
          else { const uint16_t h = (uint16_t)arith_to_bits(arith_uf(arith_half_rne(v)), kAF16); memcpy(in[i].data() + 16 + k * 2, &h, 2); }
        }
      ip[i] = in[i].data() + 16 - (in_type == kAU8 || in_type == kAI8 ? rand() % 16 : 0);
      out[i].assign(ovol[i] * osz + 64, 0xA5);
      op[i] = out[i].data() + 16 + (osz == 1 ? rand() % 16 : osz * (rand() % 4));
      fp[i] = filt[i].data();
      fills[i].resize(fcount[i] * esz + 1);
      for (auto &x : fills[i]) x = (uint8_t)(rand() % 7);
      vp[i] = fills[i].data();
    }
    if (emul_filter(in_type, out_type, n, ndim, shapes.data(), layout, fshapes.data(), anchors.data(), border, mode, fill ? in_type : -1,
                    fcount.data(), outs_shape.data(), ip.data(), fp.data(), vp.data(), op.data(), items.data(), err, sizeof(err))) {
      fprintf(stderr, "case %d refused: %s\n", c, err);
      return 1;
    }
    for (int i = 0; i < n; i++) {
      const int64_t *s = shapes.data() + (size_t)i * ndim, *os = outs_shape.data() + (size_t)i * ndim;
      const int ah = lay[0] == 'F';
      const int64_t F = ah ? s[0] : 1, H = s[ah], W = s[ah + 1], C = lay[strlen(lay) - 1] == 'C' ? s[ah + 2] : 1, Ho = os[ah], Wo = os[ah + 1];
      const int fh = (int)fshapes[2 * i], fw = (int)fshapes[2 * i + 1];
      const int ar = mode == kFltValid ? 0 : anchors[2 * i] < 0 ? fh / 2 : anchors[2 * i];
      const int ac = mode == kFltValid ? 0 : anchors[2 * i + 1] < 0 ? fw / 2 : anchors[2 * i + 1];
      std::vector<uint8_t> want(ovol[i] * osz);
      for (int64_t f = 0; f < F; f++) {
        float fv = 0;
        if (fill) flt_dispatch(in_type, in_type, [&](auto t, auto) { fv = to_f<decltype(t)>(fills[i].data(), fcount[i] > 1 ? f : 0); });
        for (int64_t y = 0; y < Ho; y++)
          for (int64_t x = 0; x < Wo; x++)
            for (int64_t ch = 0; ch < C; ch++) {
              float acc = 0.0f;
              for (int r = 0; r < fh; r++)
                for (int q = 0; q < fw; q++) {
                  const int64_t iy = ref_index(y + r - ar, H, border), ix = ref_index(x + q - ac, W, border);
                  float v = fv;
                  if (iy >= 0 && ix >= 0)
                    flt_dispatch(in_type, in_type, [&](auto t, auto) { v = to_f<decltype(t)>(ip[i], ((f * H + iy) * W + ix) * C + ch); });
                  acc = fmaf(filt[i][r * fw + q], v, acc);
                }
              const int64_t k = ((f * Ho + y) * Wo + x) * C + ch;
              flt_dispatch(in_type, out_type, [&](auto, auto to) {
                const auto o = flt_from_float<decltype(to)>(acc);
                memcpy(want.data() + k * osz, &o, osz);
              });
            }
      }
      const uint8_t *got = static_cast<const uint8_t *>(op[i]);
      const int64_t pre = got - out[i].data();
      for (int64_t k = 0; k < (int64_t)out[i].size(); k++) {
        const bool inside = k >= pre && k < pre + ovol[i] * osz;
        if (!inside && out[i][k] != 0xA5) { fprintf(stderr, "case %d: a write outside the output\n", c); return 1; }
        if (inside && out[i][k] != want[k - pre]) {
          fprintf(stderr, "case %d (layout %s, type %d -> %d, border %d, mode %d, sample %d) differs at byte %lld\n", c, lay, in_type,
                  out_type, border, mode, i, (long long)(k - pre));
          return 1;
        }
      }
    }
  }
  printf("ok %d\n", cases);
  return 0;
}
#endif
