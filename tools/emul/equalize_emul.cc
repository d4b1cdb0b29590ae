// tools/emul/equalize_emul.cc -- TEST INFRASTRUCTURE.  The planner of fn.experimental.equalize (dali_b200/csrc/equalize_plan.h) and
// the kernels' per-thread bodies (equalize_core.h) compiled for the host, so that tests/test_equalize_cpu.py runs them without a GPU:
//   g++ -std=c++17 -O2 -ffp-contract=off -shared -fPIC tools/emul/equalize_emul.cc -o equalize_emul.so          (ctypes: emul_equalize)
//   g++ -std=c++17 -O1 -g -ffp-contract=off -fsanitize=address,undefined -DEQUALIZE_EMUL_MAIN tools/emul/equalize_emul.cc -o eq_fuzz
// The second form plans and runs random layouts, shapes and byte offsets, checks every output against a direct statement of
// cv2.equalizeHist per plane and prints "ok <cases>"; under the sanitizers it checks that no plan reaches memory it must not.
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>
#include "../../dali_b200/csrc/equalize_plan.h"

using namespace dalib200;

// Both kernels as the device runs them, work items and threads in reverse order.
static void run_equalize(const std::vector<EqSample> &d, int64_t items, uint32_t *hist) {
  static uint32_t sh[kEqSmemWords];
  static uint8_t lut[kEqMaxChannels * 256];
  for (int64_t item = items - 1; item >= 0; item--) {
    const EqSample &s = d[last_at_most(d.data(), 0, (int)d.size() - 1, item, [](const EqSample &e) { return e.first_item; })];
    memset(sh, 0, sizeof(sh));
    for (int t = kEqThreads - 1; t >= 0; t--) eq_hist_thread(s, item - s.first_item, sh + ((t >> 5) % s.nsub) * s.C * 256, t);
    for (int t = kEqThreads - 1; t >= 0; t--) eq_hist_flush(s, item - s.first_item, sh, hist, t);
  }
  for (int64_t item = items - 1; item >= 0; item--) {
    const EqSample &s = d[last_at_most(d.data(), 0, (int)d.size() - 1, item, [](const EqSample &e) { return e.first_item; })];
    const int64_t frame = eq_item(s, item - s.first_item).frame;
    for (int c = s.C - 1; c >= 0; c--) eq_lut_plane(hist + s.hist_off + (frame * s.C + c) * 256, s.plane, lut + c * 256);
    for (int t = kEqThreads - 1; t >= 0; t--) eq_apply_thread(s, item - s.first_item, lut, t);
  }
}

// Plans, and when outs is not NULL runs both kernels.  geom (NULL or n x 4): frames' items per frame, channels, stride and the
// sample's items.  Returns 0, or 1 with the planner's message in err.
extern "C" int emul_equalize(int in_type, int n, int ndim, const int64_t *in_shapes, const char *layout, const void *const *ins,
                             void *const *outs, int64_t *geom, char *err, int errcap) {
  EqPlanData p;
  std::string e;
  if (!EqSetup(&p, in_type, n, ndim, in_shapes, layout, &e)) {
    snprintf(err, errcap, "%s", e.c_str());
    return 1;
  }
  for (int i = 0; geom && i < n; i++) {
    const EqSample &s = p.samples[i];
    geom[4 * i] = s.ipf; geom[4 * i + 1] = s.C; geom[4 * i + 2] = s.stride; geom[4 * i + 3] = s.items;
  }
  if (!outs) return 0;
  std::vector<EqSample> d = p.samples;
  for (int i = 0; i < n; i++)
    if (d[i].items) EqBind(d[i], ins[i], outs[i]);
  std::vector<uint32_t> hist((size_t)p.hist_words, 0);
  run_equalize(d, p.items, hist.data());
  return 0;
}

#ifdef EQUALIZE_EMUL_MAIN
// cv2.equalizeHist of one plane of `total` pixels, read at p[k * step]: the direct statement, in double where it is exact
static void reference_plane(const uint8_t *p, int64_t total, int64_t step, uint8_t *q) {
  int64_t h[256] = {0};
  for (int64_t k = 0; k < total; k++) h[p[k * step]]++;
  int i = 0;
  while (!h[i]) i++;
  uint8_t lut[256];
  if (h[i] == total) {
    for (int k = 0; k < 256; k++) lut[k] = (uint8_t)k;
  } else {
    const float scale = 255.0f / (float)(total - h[i]);
    int64_t sum = 0;
    for (int k = 0; k < 256; k++) {
      if (k > i) sum += h[k];
      const float v = (float)sum * scale;
      const long r = lrintf(v);
      lut[k] = k <= i ? 0 : (uint8_t)(r < 0 ? 0 : r > 255 ? 255 : r);
    }
  }
  for (int64_t k = 0; k < total; k++) q[k * step] = lut[p[k * step]];
}

int main(int argc, char **argv) {
  const int cases = argc > 1 ? atoi(argv[1]) : 300;
  srand(argc > 2 ? atoi(argv[2]) : 1);
  char err[512];
  for (int c = 0; c < cases; c++) {
    const int li = rand() % 7;                               // 6: the empty layout
    const char *layout = li < 6 ? kEqLayouts[li] : "";
    const int ndim = li < 6 ? (int)strlen(layout) : 2 + rand() % 3;
    const char *lay = li < 6 ? layout : ndim == 2 ? "HW" : ndim == 3 ? "HWC" : "FHWC";
    const int n = 1 + rand() % 4;
    std::vector<int64_t> shapes((size_t)n * ndim);
    for (int i = 0; i < n; i++)
      for (int a = 0; a < ndim; a++) {
        const char ax = lay[a];
        int64_t &e = shapes[(size_t)i * ndim + a];
        e = ax == 'C' ? 1 + rand() % kEqMaxChannels : ax == 'F' ? rand() % 4 : rand() % 9 == 0 ? 0 : 1 + rand() % (rand() % 4 ? 40 : 400);
      }
    std::vector<std::vector<uint8_t>> in(n), out(n);
    std::vector<const void *> ip(n);
    std::vector<void *> op(n);
    std::vector<int64_t> vol(n, 1);
    for (int i = 0; i < n; i++) {
      for (int a = 0; a < ndim; a++) vol[i] *= shapes[(size_t)i * ndim + a];
      in[i].resize(vol[i] + 32);
      const int kind = rand() % 3, lo = rand() % 256, span = 1 + rand() % 256;
      for (auto &x : in[i]) x = (uint8_t)(kind == 0 ? rand() : kind == 1 ? lo : (lo + rand() % span) % 256);
      out[i].assign(vol[i] + 64, 0xA5);
      ip[i] = in[i].data() + rand() % 16;
      op[i] = out[i].data() + 16 + rand() % 16;
    }
    if (emul_equalize(0, n, ndim, shapes.data(), layout, ip.data(), op.data(), nullptr, err, sizeof(err))) {
      fprintf(stderr, "case %d refused: %s\n", c, err);
      return 1;
    }
    const char *hp = strchr(lay, 'H'), *cp = strchr(lay, 'C');
    for (int i = 0; i < n; i++) {
      const int64_t *s = shapes.data() + (size_t)i * ndim;
      const int64_t F = lay[0] == 'F' ? s[0] : 1, H = s[hp - lay], W = s[hp - lay + 1], C = cp ? s[cp - lay] : 1;
      const bool chw = cp && cp < hp;
      std::vector<uint8_t> want(vol[i]);
      for (int64_t f = 0; f < F; f++)
        for (int64_t ch = 0; ch < C && H * W > 0; ch++) {
          const int64_t base = f * H * W * C + (chw ? ch * H * W : ch);
          reference_plane(static_cast<const uint8_t *>(ip[i]) + base, H * W, chw ? 1 : C, want.data() + base);
        }
      const uint8_t *got = static_cast<const uint8_t *>(op[i]);
      const int64_t pre = got - out[i].data();
      for (int64_t k = 0; k < (int64_t)out[i].size(); k++) {
        const bool inside = k >= pre && k < pre + vol[i];
        if (!inside && out[i][k] != 0xA5) { fprintf(stderr, "case %d: a write outside the output\n", c); return 1; }
        if (inside && out[i][k] != want[k - pre]) {
          fprintf(stderr, "case %d (layout %s, sample %d) differs at %lld\n", c, lay, i, (long long)(k - pre));
          return 1;
        }
      }
    }
  }
  printf("ok %d\n", cases);
  return 0;
}
#endif
