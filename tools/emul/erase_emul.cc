// tools/emul/erase_emul.cc -- TEST INFRASTRUCTURE.  The planner of fn.erase (dali_b200/csrc/erase_plan.h) and the kernel's
// per-thread bodies (erase_core.h) compiled for the host, so that tests/test_erase_cpu.py runs them without a GPU:
//   g++ -std=c++17 -O2 -shared -fPIC tools/emul/erase_emul.cc -o erase_emul.so                           (ctypes: emul_erase)
//   g++ -std=c++17 -O1 -g -fsanitize=address,undefined -DERASE_EMUL_MAIN tools/emul/erase_emul.cc -o er_fuzz
// The second form plans and runs random types, layouts, shapes, erased axes, regions, coordinate flags, fills and byte offsets,
// checks every output bit for bit against a direct statement (a per-element test against every clipped region) and the bytes
// around it, and prints "ok <cases>"; under the sanitizers it checks that no plan reaches memory it must not.
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>
#include "../../dali_b200/csrc/erase_plan.h"

using namespace dalib200;

// Plans, and when outs is not NULL runs the kernel on the host.  axis_names NULL: axes.  Returns 0, or 1 with the planner's message in
// err.  items (may be NULL) receives the work items of each sample, bands the number of bands of each sample.
extern "C" int emul_erase(int type, int n, int ndim, const int64_t *shapes, const char *layout, const char *axis_names, const int32_t *axes,
                          int naxes, const float *anchors, const int64_t *anchor_counts, const float *region_shapes,
                          const int64_t *shape_counts, int norm_anchor, int norm_shape, int centered, const float *fill, int nfill,
                          const void *const *ins, void *const *outs, int64_t *items, int64_t *bands, char *err, int errcap) {
  ErPlanData p;
  std::string e;
  if (!ErSetup(&p, type, n, ndim, shapes, layout, axis_names, axes, naxes, anchors, anchor_counts, region_shapes, shape_counts, norm_anchor,
               norm_shape, centered, fill, nfill, &e)) {
    snprintf(err, errcap, "%s", e.c_str());
    return 1;
  }
  for (int i = 0; items && i < n; i++) items[i] = p.samples[i].items;
  for (int i = 0; bands && i < n; i++) bands[i] = p.samples[i].items ? p.samples[i].nbands : 0;
  if (!outs) return 0;
  std::vector<ErSample> d = p.samples;
  // the fill table at a 16-byte boundary, as in the arena
  std::vector<uint8_t> fmem(p.fill.size() + 16);
  uint8_t *const ft = fmem.data() + ((16 - ((uintptr_t)fmem.data() & 15)) & 15);
  memcpy(ft, p.fill.data(), p.fill.size());
  for (int i = 0; i < n; i++) {
    if (!d[i].items) continue;
    d[i].in = ins[i];
    d[i].out = outs[i];
    d[i].bands = p.bands.data() + p.band_off[i];
    d[i].ivals = p.ivals.data() + p.ival_off[i];
  }
  ErRunOnHost(d.data(), n, p.items, ft, p.nfill);
  return 0;
}

#ifdef ERASE_EMUL_MAIN
static int64_t llround_ref(double x) { return std::llround(x); }

int main(int argc, char **argv) {
  const int cases = argc > 1 ? atoi(argv[1]) : 300;
  srand(argc > 2 ? atoi(argv[2]) : 1);
  const char *layouts[] = { "T", "TC", "ft", "HW", "HWC", "CHW", "FHWC", "FCHW", "DHWC", "FDHWC", "" };
  char err[512];
  for (int c = 0; c < cases; c++) {
    const int type = rand() % 12, esz = arith_size(type);
    const char *layout = layouts[rand() % 11];
    const int ndim = *layout ? (int)strlen(layout) : 1 + rand() % 6;
    // erased axes: a random non-empty subset in a random order
    std::vector<int32_t> axes;
    for (int a = 0; a < ndim; a++)
      if (rand() % 2) axes.push_back(a);
    if (axes.empty()) axes.push_back(rand() % ndim);
    for (size_t k = axes.size(); k > 1; k--) std::swap(axes[k - 1], axes[rand() % k]);
    const int nax = (int)axes.size();
    std::string names;
    const bool by_name = *layout && rand() % 2;
    for (int a : axes) names += layout[*layout ? a : 0];
    const int cdim = *layout && strchr(layout, 'C') ? (int)(strchr(layout, 'C') - layout) : -1;
    bool c_erased = false;
    for (int a : axes) c_erased |= a == cdim;
    const int n = 1 + rand() % 3;
    std::vector<int64_t> shapes((size_t)n * ndim);
    const int64_t cext = 1 + rand() % 5;
    for (int i = 0; i < n; i++)
      for (int a = 0; a < ndim; a++)
        shapes[(size_t)i * ndim + a] = a == cdim ? cext : rand() % 10 == 0 ? 0 : 1 + rand() % (ndim > 3 ? 6 : ndim > 1 ? 20 : 200);
    const int nfill = cdim >= 0 && !c_erased && rand() % 2 ? (int)cext : 1;
    std::vector<float> fill(nfill);
    for (auto &f : fill) f = (float)(rand() % 1000 - 300) / (rand() % 2 ? 1.0f : 7.0f);
    const int na = rand() % 3, ns = rand() % 3, cen = rand() % 3 == 0;
    std::vector<int64_t> counts(n);
    std::vector<float> anc, shp;
    for (int i = 0; i < n; i++) {
      const int regions = rand() % 5 == 0 ? 0 : rand() % 4 == 0 ? 20 + rand() % 50 : 1 + rand() % 3;
      counts[i] = (int64_t)regions * nax;
      for (int r = 0; r < regions; r++)
        for (int k = 0; k < nax; k++) {
          const int64_t ext = shapes[(size_t)i * ndim + axes[k]];
          if (na) anc.push_back((float)(rand() % 1000) / 800.0f - 0.1f);
          else anc.push_back((float)(rand() % (int)(ext + 6)) - 3.0f + (rand() % 2 ? 0.5f : 0.0f));
          if (ns) shp.push_back((float)(rand() % 1000) / 1000.0f);
          else shp.push_back((float)(rand() % (int)(ext + 4)) + (rand() % 2 ? 0.5f : 0.0f));
        }
    }
    std::vector<std::vector<uint8_t>> in(n), out(n);
    std::vector<const void *> ip(n);
    std::vector<void *> op(n);
    std::vector<int64_t> vol(n, 1);
    for (int i = 0; i < n; i++) {
      for (int a = 0; a < ndim; a++) vol[i] *= shapes[(size_t)i * ndim + a];
      in[i].resize(vol[i] * esz + 32);
      for (auto &x : in[i]) x = (uint8_t)rand();
      ip[i] = in[i].data() + 16 + esz * (rand() % (16 / esz));
      out[i].assign(vol[i] * esz + 64, 0xA5);
      op[i] = out[i].data() + 16 + esz * (rand() % (16 / esz));
    }
    if (emul_erase(type, n, ndim, shapes.data(), layout, by_name ? names.c_str() : nullptr, axes.data(), nax, anc.data(), counts.data(),
                   shp.data(), counts.data(), na != 0, ns != 0, cen, fill.data(), nfill, ip.data(), op.data(), nullptr, nullptr, err,
                   sizeof(err))) {
      fprintf(stderr, "case %d refused: %s\n", c, err);
      return 1;
    }
    std::vector<uint8_t> fbits((size_t)nfill * 8);
    for (int k = 0; k < nfill; k++) {
      const uint64_t b = arith_to_bits(arith_cast(arith_uf(fill[k]), kAF32, type), type);
      memcpy(fbits.data() + (size_t)k * esz, &b, esz);
    }
    int64_t vpos = 0;
    for (int i = 0; i < n; i++) {
      const int64_t *s = shapes.data() + (size_t)i * ndim;
      // the clipped boxes, stated directly
      std::vector<std::vector<int64_t>> bs, es;
      for (int64_t r = 0; r < counts[i] / nax; r++) {
        std::vector<int64_t> b(ndim, 0), e(s, s + ndim);
        for (int k = 0; k < nax; k++) {
          const int a = axes[k];
          double x = anc[vpos + r * nax + k], w = shp[vpos + r * nax + k];
          if (na) x *= (double)s[a];
          if (ns) w *= (double)s[a];
          if (cen) x -= w / 2;
          b[a] = std::min(std::max(llround_ref(x), (int64_t)0), s[a]);
          e[a] = std::min(std::max(llround_ref(x + w), (int64_t)0), s[a]);
        }
        bs.push_back(b), es.push_back(e);
      }
      vpos += counts[i];
      std::vector<uint8_t> want(vol[i] * esz);
      for (int64_t k = 0; k < vol[i]; k++) {
        int64_t coord[kErMaxDim], rest = k;
        for (int a = ndim - 1; a >= 0; a--) coord[a] = rest % s[a], rest /= s[a];
        bool inside = false;
        for (size_t r = 0; r < bs.size() && !inside; r++) {
          bool all = true;
          for (int a = 0; a < ndim; a++) all &= coord[a] >= bs[r][a] && coord[a] < es[r][a];
          inside = all;
        }
        const int ch = nfill > 1 ? (int)coord[cdim] : 0;
        memcpy(want.data() + k * esz, inside ? fbits.data() + (size_t)ch * esz : static_cast<const uint8_t *>(ip[i]) + k * esz, esz);
      }
      const int64_t pre = static_cast<const uint8_t *>(op[i]) - out[i].data();
      for (int64_t k = 0; k < (int64_t)out[i].size(); k++) {
        const bool in_out = k >= pre && k < pre + vol[i] * esz;
        if (!in_out && out[i][k] != 0xA5) { fprintf(stderr, "case %d: a write outside the output\n", c); return 1; }
        if (in_out && out[i][k] != want[k - pre]) {
          fprintf(stderr, "case %d (layout \"%s\", ndim %d, type %d, sample %d) differs at byte %lld\n", c, layout, ndim, type, i,
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
