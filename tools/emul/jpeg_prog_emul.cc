// tools/emul/jpeg_prog_emul.cc -- TEST INFRASTRUCTURE.  Runs the progressive-JPEG scan decoder of the product on the host.
//
// The device kernels prog_scan_kernel / prog_dc_kernel (dali_b200/csrc/jpeg_prog.cu) are thin wrappers around prog_decode_scan() and
// prog_dc_difference() (dali_b200/csrc/jpeg_prog_core.h); the planner (jpeg_prog_plan.h) is plain C++.  This file compiles them with
// the host compiler and runs the scans wave by wave like the launches do, then applies the prefix sum of the shared dc_scan stage, so
// that tests/test_jpeg_prog_cpu.py can compare the quantised coefficients with those of the baseline twin of the same image (same
// DCT + quantisation, different entropy coding) and the decoded pixels with libjpeg-turbo's, on a machine without a GPU.
//   g++ -O2 -shared -fPIC -I/usr/local/cuda/include tools/emul/jpeg_prog_emul.cc
#include <cstdlib>
#include <map>
#include <string>
#include <vector>
#include "../../include/dali_b200.h"
#include "../../dali_b200/csrc/jpeg_prog_plan.h"

using namespace dalib200;

// coef: [mcuy * mcux * bpm][64] int16 (MCU order, natural order per block, absolute DC in slot 0 on return).
// info: { ncomp, mcux, mcuy, bpm, nscans, nwaves, truncated }.  Call with coef == NULL to query the sizes only.
extern "C" int emul_jpeg_progressive(const uint8_t *data, size_t len, int16_t *coef, int *info) {
  std::vector<ProgScan> scans;
  std::vector<ProgHuff> huff;
  std::map<std::string, int> cache;
  std::string err;
  ProgImage im;
  memset(&im, 0, sizeof(im));
  uint16_t quant[4][64];
  int rc = PlanProgressive(data, len, 0, 0, &im, scans, huff, cache, quant, &err);
  if (rc) return rc;
  int nwaves = 0;
  for (auto &s : scans) nwaves = std::max(nwaves, s.wave + 1);
  info[0] = im.ncomp; info[1] = im.mcux; info[2] = im.mcuy; info[3] = im.bpm; info[4] = (int)scans.size(); info[5] = nwaves; info[6] = im.incomplete;
  if (!coef) return 0;
  const int64_t nblk = (int64_t)im.mcux * im.mcuy * im.bpm;
  memset(coef, 0, sizeof(int16_t) * 64 * nblk);
  for (int w = 0; w < nwaves; w++)
    for (int k = (int)scans.size() - 1; k >= 0; k--)          // within a wave the order must not matter: run it backwards
      if (scans[k].wave == w) info[6] |= prog_decode_scan(scans[k], im, huff.data(), data, coef);
  // the shared stage: differences -> dc_scan's prefix sum per component in MCU order (jpeg.cu dc_scan_kernel)
  std::vector<int16_t> dc(nblk);
  for (int64_t b = 0; b < nblk; b++) prog_dc_difference(im, coef, dc.data(), b);
  for (int c = 0; c < im.ncomp; c++) {
    int pred = 0;
    const int nb = im.hs[c] * im.vs[c];
    for (int64_t m = 0; m < (int64_t)im.mcux * im.mcuy; m++)
      for (int k = 0; k < nb; k++) { const int64_t b = m * im.bpm + im.blk0[c] + k; pred += dc[b]; coef[b * 64] = (int16_t)pred; }
  }
  return 0;
}

// qt: [4][64] uint16, the quantisation table each component latched at its first scan (natural order).  Returns the planner's status.
extern "C" int emul_jpeg_prog_quant(const uint8_t *data, size_t len, uint16_t *qt) {
  std::vector<ProgScan> scans;
  std::vector<ProgHuff> huff;
  std::map<std::string, int> cache;
  std::string err;
  ProgImage im;
  memset(&im, 0, sizeof(im));
  return PlanProgressive(data, len, 0, 0, &im, scans, huff, cache, reinterpret_cast<uint16_t (*)[64]>(qt), &err);
}
