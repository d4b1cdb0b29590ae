// tools/emul/resample3d_emul.cc -- TEST INFRASTRUCTURE.  Runs the 3-D resampler's plan through its per-element function on the host.
//
// The device kernel resample3d_pass_kernel (dali_b200/csrc/resample3d.cu) is a grid-stride loop around r3_element()
// (dali_b200/csrc/resample3d_core.h), one output element per thread, no cooperation between threads; the planner
// (resample3d_plan.h) is plain C++.  This file compiles both with the host compiler and executes every pass element by element on host
// memory, so that tests/test_resample3d_emul_cpu.py can compare planner + arithmetic with the reference's SeparableResampleCPU<.., 3>
// bit for bit on a machine without a GPU.  What it cannot cover is the launch itself (descriptor upload, grid shape): that is the
// `-m gpu` test's job.  Built by the test:  g++ -O2 -ffp-contract=off -shared -fPIC ...
#include <cstdlib>
#include <string>
#include <vector>
#include "../../dali_b200/csrc/resample3d_plan.h"

using namespace dalib200;

extern "C" int emul_resample3d(const dalib200Resample3DSample *s, int in_dtype, int out_dtype, const void *in, void *out, int *order) {
  std::vector<int32_t> tables;
  R3SamplePlan sp;
  std::string err;
  int rc = PlanResample3D(*s, in_dtype, out_dtype, tables, &sp, &err);
  if (rc) return rc;
  if (order) for (int k = 0; k < 3; k++) order[k] = sp.order[k];
  std::vector<float> t0((size_t)sp.tmp_floats[0] + 4), t1((size_t)sp.tmp_floats[1] + 4);
  for (int k = 0; k < sp.npass; k++) {
    R3Pass p = sp.pass[k];
    p.in = k == 0 ? in : k == 1 ? static_cast<const void *>(t0.data()) : static_cast<const void *>(t1.data());
    p.out = k == sp.npass - 1 ? out : k == 0 ? static_cast<void *>(t0.data()) : static_cast<void *>(t1.data());
    for (int64_t e = 0; e < p.total; e++) r3_element(p, tables.data(), e);
  }
  return 0;
}
