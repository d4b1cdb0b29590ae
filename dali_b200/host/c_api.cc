// dali_b200/host/c_api.cc -- C interface of the host layer (pipeline construction / run / outputs), bound from Python
// with ctypes (dali_b200/backend.py).  Style follows the reference's C API (include/dali/dali.h:43-164,428-1250:
// opaque handles, integer status, thread-local last error); only what the Python layer needs is exposed.
#include <algorithm>
#include <cstring>
#include <stdexcept>
#include <string>
#include "dali.h"
#include "../../include/dali_b200.h"
#include "../csrc/equalize_plan.h"

using namespace dali;  // NOLINT

static thread_local std::string g_err;

#define API_BEGIN try {
#define API_END                                       \
  }                                                   \
  catch (const std::exception &e) { g_err = e.what(); return 1; } \
  catch (...) { g_err = "unknown error"; return 1; }  \
  return 0;

template <typename TL>
static void FillInfo(const TL *tl, int *n, int *ndim, int *dtype, char *layout, int *contiguous) {
  DALI_ENFORCE(tl, "output not available");
  *n = tl->num_samples(); *ndim = tl->sample_dim(); *dtype = tl->type();
  snprintf(layout, 16, "%s", tl->GetLayout().str().c_str());
  *contiguous = tl->IsContiguous();
}

extern "C" {

const char *dalihLastError() { return g_err.c_str(); }

// ---- OpSpec
int dalihOpSpecCreate(void **spec, const char *schema) { API_BEGIN *spec = new OpSpec(schema); API_END }
int dalihOpSpecDestroy(void *spec) { API_BEGIN delete static_cast<OpSpec *>(spec); API_END }
int dalihOpSpecAddArgInt(void *s, const char *n, int64_t v) { API_BEGIN static_cast<OpSpec *>(s)->AddArg(n, MakeArg(v)); API_END }
int dalihOpSpecAddArgFloat(void *s, const char *n, double v) { API_BEGIN static_cast<OpSpec *>(s)->AddArg(n, MakeArg(v)); API_END }
int dalihOpSpecAddArgBool(void *s, const char *n, int v) { API_BEGIN static_cast<OpSpec *>(s)->AddArg(n, MakeArg(v != 0)); API_END }
int dalihOpSpecAddArgString(void *s, const char *n, const char *v) { API_BEGIN static_cast<OpSpec *>(s)->AddArg(n, MakeArg(std::string(v))); API_END }
int dalihOpSpecAddArgFloatVec(void *s, const char *n, const float *v, int cnt) {
  API_BEGIN static_cast<OpSpec *>(s)->AddArg(n, MakeArg(std::vector<float>(v, v + cnt))); API_END
}
int dalihOpSpecAddArgDoubleVec(void *s, const char *n, const double *v, int cnt) {
  API_BEGIN
  ArgValue a = MakeArg(std::vector<float>(v, v + cnt));
  a.dv.assign(v, v + cnt);
  static_cast<OpSpec *>(s)->AddArg(n, a);
  API_END
}
int dalihOpSpecAddArgIntVec(void *s, const char *n, const int64_t *v, int cnt) {
  API_BEGIN static_cast<OpSpec *>(s)->AddArg(n, MakeArg(std::vector<int64_t>(v, v + cnt))); API_END
}
int dalihOpSpecAddInput(void *s, const char *name, const char *device) { API_BEGIN static_cast<OpSpec *>(s)->AddInput(name, device); API_END }
int dalihOpSpecAddOutput(void *s, const char *name, const char *device) { API_BEGIN static_cast<OpSpec *>(s)->AddOutput(name, device); API_END }
int dalihOpSpecAddArgumentInput(void *s, const char *arg, const char *input) { API_BEGIN static_cast<OpSpec *>(s)->AddArgumentInput(arg, input); API_END }

// ---- schema introspection (drives the generation of fn.* wrappers, like ops/__init__.py:553-715 in the reference)
int dalihNumSchemas() { return static_cast<int>(SchemaRegistry::Names().size()); }
int dalihSchemaName(int i, char *out, int cap) {
  API_BEGIN
  auto names = SchemaRegistry::Names();
  DALI_ENFORCE(i >= 0 && i < static_cast<int>(names.size()), "schema index out of range");
  snprintf(out, cap, "%s", names[i].c_str());
  API_END
}
// writes a '\n'-separated list: "name|tensor_ok(0/1)|required(0/1)"
int dalihSchemaArgs(const char *schema, char *out, int cap) {
  API_BEGIN
  const auto &s = SchemaRegistry::GetSchema(schema);
  std::string r;
  for (auto &n : s.ArgNames()) {
    const bool req = std::find(s.Required().begin(), s.Required().end(), n) != s.Required().end();
    r += n + "|" + (s.TensorArgAllowed(n) ? "1" : "0") + "|" + (req ? "1" : "0") + "\n";
  }
  DALI_ENFORCE(static_cast<int>(r.size()) < cap, "buffer too small");
  snprintf(out, cap, "%s", r.c_str());
  API_END
}
int dalihSchemaInfo(const char *schema, int *min_in, int *max_in, int *num_out, char *doc, int cap) {
  API_BEGIN
  const auto &s = SchemaRegistry::GetSchema(schema);
  *min_in = s.MinNumInput(); *max_in = s.MaxNumInput(); *num_out = s.NumOutput();
  if (doc) snprintf(doc, cap, "%s", s.doc().c_str());
  API_END
}
int dalihOperatorRegistered(const char *schema, const char *backend) {
  return OperatorRegistry::Registry(backend).count(schema) ? 1 : 0;
}

// ---- Pipeline
int dalihPipelineCreate(void **pipe, int max_batch, int num_threads, int device_id) {
  API_BEGIN *pipe = new Pipeline(max_batch, num_threads, device_id); API_END
}
int dalihPipelineDestroy(void *p) { API_BEGIN delete static_cast<Pipeline *>(p); API_END }
int dalihPipelineAddExternalInput(void *p, const char *name, const char *device, const char *layout) {
  API_BEGIN static_cast<Pipeline *>(p)->AddExternalInput(name, device, layout ? layout : ""); API_END
}
int dalihPipelineAddOperator(void *p, void *spec, const char *inst_name) {
  API_BEGIN static_cast<Pipeline *>(p)->AddOperator(*static_cast<OpSpec *>(spec), inst_name); API_END
}
int dalihPipelineSetOutputs(void *p, int n, const char *const *names, const char *const *devices) {
  API_BEGIN
  std::vector<std::pair<std::string, std::string>> o;
  for (int i = 0; i < n; i++) o.emplace_back(names[i], devices[i]);
  static_cast<Pipeline *>(p)->SetOutputDescs(o);
  API_END
}
int dalihPipelineBuild(void *p) { API_BEGIN static_cast<Pipeline *>(p)->Build(); API_END }
int dalihPipelineFeedInput(void *p, const char *name, int n, const void *const *ptrs, const int64_t *shapes, int ndim, int dtype,
                           const char *layout) {
  API_BEGIN
  TensorListShape sh(n, ndim);
  for (int i = 0; i < n; i++) sh.set_tensor_shape(i, TensorShape(shapes + static_cast<size_t>(i) * ndim, shapes + static_cast<size_t>(i + 1) * ndim));
  static_cast<Pipeline *>(p)->SetExternalInput(name, std::vector<const void *>(ptrs, ptrs + n), sh, static_cast<DALIDataType>(dtype),
                                               layout ? layout : "");
  API_END
}
// no_copy != 0: the caller keeps the buffers valid AND unmodified until the iteration has completed (external_source(no_copy=True))
int dalihPipelineFeedInputEx(void *p, const char *name, int n, const void *const *ptrs, const int64_t *shapes, int ndim, int dtype,
                             const char *layout, int no_copy) {
  API_BEGIN
  TensorListShape sh(n, ndim);
  for (int i = 0; i < n; i++) sh.set_tensor_shape(i, TensorShape(shapes + static_cast<size_t>(i) * ndim, shapes + static_cast<size_t>(i + 1) * ndim));
  static_cast<Pipeline *>(p)->SetExternalInput(name, std::vector<const void *>(ptrs, ptrs + n), sh, static_cast<DALIDataType>(dtype),
                                               layout ? layout : "", no_copy != 0);
  API_END
}
int dalihPipelineRun(void *p) { API_BEGIN static_cast<Pipeline *>(p)->Run(); API_END }
int dalihPipelineWait(void *p) { API_BEGIN static_cast<Pipeline *>(p)->WaitOutputs(); API_END }
int dalihPipelineNumOutputs(void *p) { return static_cast<Pipeline *>(p)->NumOutputs(); }
int dalihPipelineStream(void *p, void **stream) { API_BEGIN *stream = static_cast<Pipeline *>(p)->stream(); API_END }

int dalihPipelineOutputInfo(void *p, int i, int *is_gpu, int *n, int *ndim, int *dtype, char *layout, int *contiguous) {
  API_BEGIN
  auto *pp = static_cast<Pipeline *>(p);
  *is_gpu = pp->OutputIsGPU(i);
  if (*is_gpu) FillInfo(pp->OutputGPU(i), n, ndim, dtype, layout, contiguous); else FillInfo(pp->OutputCPU(i), n, ndim, dtype, layout, contiguous);
  API_END
}
int dalihPipelineOutputData(void *p, int i, int64_t *shapes, void **ptrs) {
  API_BEGIN
  auto *pp = static_cast<Pipeline *>(p);
  auto fill = [&](const auto *tl) {
    DALI_ENFORCE(tl, "output not available");
    const int nd = tl->sample_dim();
    for (int s = 0; s < tl->num_samples(); s++) {
      for (int d = 0; d < nd; d++) shapes[static_cast<size_t>(s) * nd + d] = tl->tensor_shape_span(s)[d];
      ptrs[s] = const_cast<void *>(tl->raw_tensor(s));
    }
  };
  if (pp->OutputIsGPU(i)) fill(pp->OutputGPU(i)); else fill(pp->OutputCPU(i));
  API_END
}


// Test hook (CPU): Pad's output-shape rule and argument checks without a device.  naxes < 0: no `axes`; axis_names NULL: none;
// nalign 0: no `align`; nshape 0: no `shape` (else the same nshape values for every sample).  out_shapes: n x ndim.
int dalihTestPadShape(int n, int ndim, const int64_t *in_shapes, const char *layout, const int64_t *axes, int naxes, const char *axis_names,
                      const int64_t *align, int nalign, const int64_t *shape, int nshape, float fill_value, int dtype, int64_t *out_shapes) {
  API_BEGIN
  OpSpec spec("Pad");
  if (naxes >= 0) spec.AddArg("axes", MakeArg(std::vector<int64_t>(axes, axes + naxes)));
  if (axis_names) spec.AddArg("axis_names", MakeArg(std::string(axis_names)));
  if (nalign > 0) spec.AddArg("align", MakeArg(std::vector<int64_t>(align, align + nalign)));
  const PadArgs a = PadResolveArgs(spec, ndim, layout ? layout : "");
  std::vector<std::vector<int64_t>> shp;
  if (nshape > 0) shp.assign(n, std::vector<int64_t>(shape, shape + nshape));
  PadOutputShapes(a, n, ndim, in_shapes, shp, out_shapes);
  PadFillBits(fill_value, static_cast<DALIDataType>(dtype));
  API_END
}

// Test hooks (CPU): Transpose's and Cat's / Stack's argument, layout and shape rules without a device -- the operators' own argument
// resolution followed by the plan set-up of the kernel library.  nperm < 0: no `perm`; output_layout NULL: none; axis_name NULL: none;
// has_axis 0: `axis` left at its default.  out_shapes: n x output ndim; out_layout: the output layout (cap bytes).
static void PermuteSetupOrThrow(int rc) {
  if (rc != DALIB200_SUCCESS) throw std::runtime_error(dalib200GetLastError());
}

int dalihTestTranspose(int n, int ndim, const int64_t *in_shapes, const char *layout, const int64_t *perm, int nperm, int transpose_layout,
                       const char *output_layout, int elem_size, int64_t *out_shapes, char *out_layout, int cap) {
  API_BEGIN
  OpSpec spec("Transpose");
  if (nperm >= 0) spec.AddArg("perm", MakeArg(std::vector<int64_t>(perm, perm + nperm)));
  spec.AddArg("transpose_layout", MakeArg(transpose_layout != 0));
  if (output_layout) spec.AddArg("output_layout", MakeArg(std::string(output_layout)));
  const TransposeArgs a = TransposeResolveArgs(spec, ndim, layout ? layout : "");
  std::vector<int32_t> p(a.perm.begin(), a.perm.end());
  dalib200PermutePlan *plan = nullptr;
  PermuteSetupOrThrow(dalib200PermutePlanCreate(&plan, std::max(n, 1)));
  const int rc = dalib200TransposeSetup(plan, n, ndim, elem_size, in_shapes, p.data(), out_shapes);
  dalib200PermutePlanDestroy(plan);
  PermuteSetupOrThrow(rc);
  snprintf(out_layout, cap, "%s", a.layout.c_str());
  API_END
}

int dalihTestJoin(int stack, int n, int nin, int ndim, const int64_t *in_shapes, const char *const *layouts, int has_axis, int axis,
                  const char *axis_name, int elem_size, int64_t *out_shapes, char *out_layout, int cap) {
  API_BEGIN
  OpSpec spec(stack ? "Stack" : "Cat");
  if (has_axis) spec.AddArg("axis", MakeArg(axis));
  if (axis_name) spec.AddArg("axis_name", MakeArg(std::string(axis_name)));
  std::vector<std::string> ls;
  for (int k = 0; k < nin; k++) ls.push_back(layouts && layouts[k] ? layouts[k] : "");
  const JoinArgs a = JoinResolveArgs(spec, stack != 0, ndim, ls);
  dalib200PermutePlan *plan = nullptr;
  PermuteSetupOrThrow(dalib200PermutePlanCreate(&plan, std::max(n * nin, 1)));
  const int rc = dalib200JoinSetup(plan, n, nin, ndim, elem_size, in_shapes, a.axis, stack, out_shapes);
  dalib200PermutePlanDestroy(plan);
  PermuteSetupOrThrow(rc);
  snprintf(out_layout, cap, "%s", a.layout.c_str());
  API_END
}

// Test hook (CPU): fn.reductions.*'s argument, type and shape rules without a device -- the operator's own argument resolution and
// mean check, then the plan set-up of the kernel library.  op: DALIB200_REDUCE_*; naxes < 0: no `axes`; axis_names NULL: none;
// dtype < 0: none; mean_shapes NULL: no mean input (else n x mean_ndim).  out_shapes: n x output ndim (written to *out_ndim);
// *out_type: the output type; out_layout: the output layout (cap bytes).
int dalihTestReduce(int op, int in_type, int n, int ndim, const int64_t *in_shapes, const char *layout, const int64_t *axes, int naxes,
                    const char *axis_names, int keep_dims, int dtype, int ddof, const int64_t *mean_shapes, int mean_ndim,
                    int64_t *out_shapes, int *out_ndim, int *out_type, char *out_layout, int cap) {
  API_BEGIN
  static const char *const schemas[] = { "reductions__Min", "reductions__Max", "reductions__Sum", "reductions__Mean",
                                         "reductions__MeanSquare", "reductions__RMS", "reductions__StdDev", "reductions__Variance" };
  if (op < 0 || op > 7) throw std::runtime_error("unknown reduction");
  OpSpec spec(schemas[op]);
  if (naxes >= 0) spec.AddArg("axes", MakeArg(std::vector<int64_t>(axes, axes + naxes)));
  if (axis_names) spec.AddArg("axis_names", MakeArg(std::string(axis_names)));
  spec.AddArg("keep_dims", MakeArg(keep_dims != 0));
  const ReduceArgs a = ReduceResolveArgs(spec, ndim, layout ? layout : "");
  const std::string name = std::string("reductions.") + (schemas[op] + strlen("reductions__"));
  if (mean_shapes)
    for (int i = 0; i < n; i++) ReduceCheckMean(name.c_str(), i, mean_shapes + (size_t)i * mean_ndim, mean_ndim, in_shapes + (size_t)i * ndim, ndim, a.mask);
  dalib200ReducePlan *plan = nullptr;
  PermuteSetupOrThrow(dalib200ReducePlanCreate(&plan, std::max(n, 1)));
  int32_t t = dtype;
  const int rc = dalib200ReduceSetup(plan, op, in_type, &t, n, ndim, in_shapes, a.mask, a.keep_dims, ddof, out_shapes);
  dalib200ReducePlanDestroy(plan);
  PermuteSetupOrThrow(rc);
  int ond = 0;
  for (int k = 0; k < ndim; k++) ond += a.keep_dims || !((a.mask >> k) & 1);
  *out_ndim = ond;
  *out_type = t;
  snprintf(out_layout, cap, "%s", a.layout.c_str());
  API_END
}

// Test hook (CPU): fn.experimental.equalize's type, layout and shape rules without a device -- the plan set-up the operator makes.
// resolved: the layout the planner reads the input with (cap bytes; the output keeps the input's own layout).
int dalihTestEqualize(int in_type, int n, int ndim, const int64_t *in_shapes, const char *layout, char *resolved, int cap) {
  API_BEGIN
  dalib200EqualizePlan *plan = nullptr;
  PermuteSetupOrThrow(dalib200EqualizePlanCreate(&plan, std::max(n, 1)));
  const int rc = dalib200EqualizeSetup(plan, in_type, n, ndim, in_shapes, layout);
  dalib200EqualizePlanDestroy(plan);
  PermuteSetupOrThrow(rc);
  std::string err;
  snprintf(resolved, cap, "%s", dalib200::kEqLayouts[dalib200::EqResolveLayout(layout, ndim, &err)]);
  API_END
}

// Test hook (CPU): fn.experimental.filter's argument, type, layout and shape rules without a device -- the argument resolution and the
// plan set-up the operator makes.  anchors: n x nanchor values of `anchor` per sample; dtype -1: none; fill_type -1: no input 2.
// out_shapes: n x ndim.
int dalihTestFilter(int in_type, int dtype, int n, int ndim, const int64_t *in_shapes, const char *layout, int filter_type, int filter_ndim,
                    const int64_t *filter_shapes, const int32_t *anchors, int nanchor, const char *border, const char *mode, int fill_type,
                    const int64_t *fill_counts, int64_t *out_shapes) {
  API_BEGIN
  OpSpec spec("experimental__Filter");
  spec.AddArg("border", MakeArg(std::string(border))).AddArg("mode", MakeArg(std::string(mode)));
  const FilterArgs a = FilterResolveArgs(spec);
  std::vector<int32_t> rc2((size_t)n * 2);
  for (int i = 0; i < n; i++) FilterAnchor(i, std::vector<int>(anchors + (size_t)i * nanchor, anchors + (size_t)(i + 1) * nanchor), rc2.data() + 2 * i);
  dalib200FilterPlan *plan = nullptr;
  PermuteSetupOrThrow(dalib200FilterPlanCreate(&plan, std::max(n, 1)));
  const int rc = dalib200FilterSetup(plan, in_type, dtype, n, ndim, in_shapes, layout, filter_type, filter_ndim, filter_shapes, rc2.data(),
                                     a.border, a.mode, fill_type, fill_counts, out_shapes);
  dalib200FilterPlanDestroy(plan);
  PermuteSetupOrThrow(rc);
  API_END
}

// Test hook (CPU): fn.erase's argument, type, layout, region and fill rules without a device -- the argument resolution and the plan
// set-up the operator makes.  Arguments left unset: axis_names NULL, naxes -1, normalized* -1, nfill -1.  anchors / region_shapes:
// every sample's values back to back, anchor_counts / shape_counts per sample.
int dalihTestErase(int type, int n, int ndim, const int64_t *shapes, const char *layout, const char *axis_names, const int32_t *axes, int naxes,
                   const float *anchors, const int64_t *anchor_counts, const float *region_shapes, const int64_t *shape_counts, int normalized,
                   int normalized_anchor, int normalized_shape, int centered_anchor, const float *fill, int nfill) {
  API_BEGIN
  OpSpec spec("Erase");
  if (axis_names) spec.AddArg("axis_names", MakeArg(std::string(axis_names)));
  if (naxes >= 0) spec.AddArg("axes", MakeArg(std::vector<int>(axes, axes + naxes)));
  if (normalized >= 0) spec.AddArg("normalized", MakeArg(normalized != 0));
  if (normalized_anchor >= 0) spec.AddArg("normalized_anchor", MakeArg(normalized_anchor != 0));
  if (normalized_shape >= 0) spec.AddArg("normalized_shape", MakeArg(normalized_shape != 0));
  spec.AddArg("centered_anchor", MakeArg(centered_anchor != 0));
  if (nfill >= 0) spec.AddArg("fill_value", MakeArg(std::vector<float>(fill, fill + nfill)));
  const EraseArgs a = EraseResolveArgs(spec, layout ? layout : "");
  dalib200ErasePlan *plan = nullptr;
  PermuteSetupOrThrow(dalib200ErasePlanCreate(&plan, std::max(n, 1)));
  const int rc = dalib200EraseSetup(plan, type, n, ndim, shapes, layout, a.by_name ? a.axis_names.c_str() : nullptr, a.axes.data(),
                                    (int)a.axes.size(), anchors, anchor_counts, region_shapes, shape_counts, a.norm_anchor, a.norm_shape,
                                    a.centered, a.fill.data(), (int)a.fill.size());
  dalib200ErasePlanDestroy(plan);
  PermuteSetupOrThrow(rc);
  API_END
}

// Test hook (CPU): fn.multi_paste's argument reading, type, layout, shape and region rules without a device -- the argument resolution
// and the plan set-up the operator makes, every argument given as a list (the same for every sample).  NULL in_ids, region_args[a]
// or output_size: not given; dtype -1: not given.  out_shapes: n x 3, written.
int dalihTestMultiPaste(int in_type, int dtype, int ninputs, int n, const int *ndims, const char *const *layouts, const int64_t *in_shapes,
                        const int64_t *in_ids, int nids, const double *const *region_args, const int *region_nvals, const int64_t *output_size,
                        int64_t *out_shapes) {
  API_BEGIN
  static const char *const names[kMultiPasteRegionArgs] = { "in_anchors", "in_anchors_rel", "shapes", "shapes_rel", "out_anchors",
                                                            "out_anchors_rel" };
  OpSpec spec("MultiPaste");
  if (dtype >= 0) spec.AddArg("dtype", MakeArg(dtype));
  if (in_ids) spec.AddArg("in_ids", MakeArg(std::vector<int64_t>(in_ids, in_ids + nids)));
  for (int r = 0; r < kMultiPasteRegionArgs; r++) {
    if (!region_args[r]) continue;
    ArgValue a = MakeArg(std::vector<float>(region_args[r], region_args[r] + region_nvals[r]));
    a.dv.assign(region_args[r], region_args[r] + region_nvals[r]);
    spec.AddArg(names[r], a);
  }
  if (output_size) spec.AddArg("output_size", MakeArg(std::vector<int64_t>(output_size, output_size + 2)));
  const MultiPasteArgs a = MultiPasteResolveArgs(spec, nullptr, n);
  dalib200PastePlan *plan = nullptr;
  PermuteSetupOrThrow(dalib200PastePlanCreate(&plan, std::max(n, 1)));
  const int rc = MultiPasteSetup(plan, a, in_type, ninputs, n, ndims, layouts, in_shapes, out_shapes);
  dalib200PastePlanDestroy(plan);
  PermuteSetupOrThrow(rc);
  API_END
}

}  // extern "C"
