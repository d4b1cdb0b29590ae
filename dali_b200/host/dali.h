// dali_b200/host/dali.h -- an API-compatible subset of the reference's operator boundary, compiled from our own
// sources (the reference itself cannot be built or installed here, SURVEY.md section 7).
//
// Same names and meaning as the reference so that operator sources read the same on both sides:
//   OperatorBase / Operator<Backend>          dali/pipeline/operator/operator.h:76-319
//   DALI_REGISTER_OPERATOR, registries        operator.h:327-333, operator_factory.h:37-139
//   OpSchema / DALI_SCHEMA                    dali/pipeline/operator/op_schema.h:154,1096-1109
//   OpSpec                                    dali/pipeline/operator/op_spec.h:323-393
//   Workspace / OutputDesc                    dali/pipeline/workspace/workspace.h:41-44,138
//   TensorList<Backend>                       dali/pipeline/data/tensor_list.h:75-640
//   Pipeline                                  dali/pipeline/pipeline.h:62-465
// Only what the hot-path operators need is present; there is NO CPU implementation of the hot-path ops --
// instantiating them for the CPU backend throws.
#ifndef DALI_B200_HOST_DALI_H_
#define DALI_B200_HOST_DALI_H_

#include <cuda_runtime.h>
#include <cstdint>
#include <cstring>
#include <functional>
#include <map>
#include <memory>
#include <sstream>
#include <stdexcept>
#include <string>
#include <utility>
#include <vector>

struct dalib200PastePlan;   // include/dali_b200.h

namespace dali {

// ---------------------------------------------------------------------------------------------- errors
struct DALIException : std::runtime_error { using std::runtime_error::runtime_error; };

template <typename... Args>
std::string make_string(const Args &...args) {
  std::ostringstream ss;
  (void)std::initializer_list<int>{ (ss << args, 0)... };
  return ss.str();
}
#define DALI_FAIL(msg) throw ::dali::DALIException(::dali::make_string(msg))
#define DALI_ENFORCE(cond, ...) \
  do { if (!(cond)) throw ::dali::DALIException(::dali::make_string("Assert on \"" #cond "\" failed: ", ##__VA_ARGS__)); } while (0)
#define CUDA_CALL(call) \
  do { cudaError_t e__ = (call); if (e__ != cudaSuccess) throw ::dali::DALIException(::dali::make_string( \
       "CUDA error ", cudaGetErrorName(e__), ": ", cudaGetErrorString(e__), " (", #call, ")")); } while (0)

// ---------------------------------------------------------------------------------------------- types
enum DALIDataType : int {
  DALI_NO_TYPE = -1, DALI_UINT8 = 0, DALI_UINT16 = 1, DALI_UINT32 = 2, DALI_UINT64 = 3, DALI_INT8 = 4, DALI_INT16 = 5,
  DALI_INT32 = 6, DALI_INT64 = 7, DALI_FLOAT16 = 8, DALI_FLOAT = 9, DALI_FLOAT64 = 10, DALI_BOOL = 11
};
enum DALIInterpType : int { DALI_INTERP_NN = 0, DALI_INTERP_LINEAR = 1, DALI_INTERP_CUBIC = 2, DALI_INTERP_LANCZOS3 = 3,
                            DALI_INTERP_TRIANGULAR = 4, DALI_INTERP_GAUSSIAN = 5 };
enum DALIImageType : int { DALI_RGB = 0, DALI_BGR = 1, DALI_GRAY = 2, DALI_YCbCr = 3, DALI_ANY_DATA = 4 };

inline size_t TypeSize(DALIDataType t) {
  switch (t) {
    case DALI_UINT8: case DALI_INT8: case DALI_BOOL: return 1;
    case DALI_UINT16: case DALI_INT16: case DALI_FLOAT16: return 2;
    case DALI_UINT32: case DALI_INT32: case DALI_FLOAT: return 4;
    case DALI_UINT64: case DALI_INT64: case DALI_FLOAT64: return 8;
    default: return 0;
  }
}

struct CPUBackend {};
struct GPUBackend {};
struct MixedBackend {};

using TensorShape = std::vector<int64_t>;
inline int64_t volume(const TensorShape &s) { int64_t v = 1; for (auto e : s) v *= e; return v; }

class TensorLayout {
 public:
  TensorLayout() = default;
  TensorLayout(const char *s) : s_(s) {}            // NOLINT
  TensorLayout(const std::string &s) : s_(s) {}     // NOLINT
  int ndim() const { return static_cast<int>(s_.size()); }
  bool empty() const { return s_.empty(); }
  int find(char c) const { auto p = s_.find(c); return p == std::string::npos ? -1 : static_cast<int>(p); }
  char operator[](int i) const { return s_[i]; }
  const std::string &str() const { return s_; }
  bool operator==(const TensorLayout &o) const { return s_ == o.s_; }
  bool operator!=(const TensorLayout &o) const { return s_ != o.s_; }
 private:
  std::string s_;
};

class TensorListShape {
 public:
  TensorListShape() = default;
  TensorListShape(int num_samples, int ndim) { resize(num_samples, ndim); }
  void resize(int num_samples, int ndim) { n_ = num_samples; ndim_ = ndim; data_.assign(static_cast<size_t>(n_) * ndim_, 0); }
  int num_samples() const { return n_; }
  int sample_dim() const { return ndim_; }
  const int64_t *tensor_shape_span(int i) const { return data_.data() + static_cast<size_t>(i) * ndim_; }
  TensorShape tensor_shape(int i) const { return TensorShape(tensor_shape_span(i), tensor_shape_span(i) + ndim_); }
  TensorShape operator[](int i) const { return tensor_shape(i); }
  void set_tensor_shape(int i, const TensorShape &s) {
    DALI_ENFORCE(static_cast<int>(s.size()) == ndim_, "shape dimensionality mismatch");
    std::copy(s.begin(), s.end(), data_.begin() + static_cast<size_t>(i) * ndim_);
  }
  int64_t tensor_size(int i) const { int64_t v = 1; for (int d = 0; d < ndim_; d++) v *= tensor_shape_span(i)[d]; return v; }
  int64_t num_elements() const { int64_t v = 0; for (int i = 0; i < n_; i++) v += tensor_size(i); return v; }
  bool operator==(const TensorListShape &o) const { return n_ == o.n_ && ndim_ == o.ndim_ && data_ == o.data_; }
 private:
  int n_ = 0, ndim_ = 0;
  std::vector<int64_t> data_;
};

struct OutputDesc {
  TensorListShape shape;
  DALIDataType type = DALI_NO_TYPE;
};

// ---------------------------------------------------------------------------------------------- TensorList
// Per-sample pointers over either one owned contiguous allocation (Resize) or borrowed memory (ShareData).
template <typename Backend>
class TensorList {
 public:
  TensorList() = default;
  TensorList(const TensorList &) = delete;
  TensorList &operator=(const TensorList &) = delete;
  ~TensorList() { Free(); }

  int num_samples() const { return shape_.num_samples(); }
  const TensorListShape &shape() const { return shape_; }
  TensorShape tensor_shape(int i) const { return shape_.tensor_shape(i); }
  const int64_t *tensor_shape_span(int i) const { return shape_.tensor_shape_span(i); }
  DALIDataType type() const { return type_; }
  const TensorLayout &GetLayout() const { return layout_; }
  void SetLayout(const TensorLayout &l) { layout_ = l; }
  int sample_dim() const { return shape_.sample_dim(); }

  const void *raw_tensor(int i) const { return ptrs_[i]; }
  void *raw_mutable_tensor(int i) { return ptrs_[i]; }
  template <typename T> const T *tensor(int i) const { return static_cast<const T *>(ptrs_[i]); }
  template <typename T> T *mutable_tensor(int i) { return static_cast<T *>(ptrs_[i]); }
  bool IsContiguous() const { return owned_; }
  const void *contiguous_data() const { return owned_ ? data_ : nullptr; }
  size_t nbytes() const { return static_cast<size_t>(shape_.num_elements()) * TypeSize(type_); }

  // executor-side allocation (exec_node_task.cc:296-307: output.Resize(desc.shape, desc.type))
  void Resize(const TensorListShape &shape, DALIDataType type);
  // borrow external per-sample memory (ExternalSource no_copy, decoder input)
  void ShareData(const std::vector<void *> &ptrs, const TensorListShape &shape, DALIDataType type) {
    shape_ = shape; type_ = type; ptrs_ = ptrs; owned_ = false; stable_ = false;
  }
  // borrowed memory the producer promised to keep valid and unmodified until the iteration has completed
  // (external_source(no_copy=True), reader-owned buffers): consumers may read it asynchronously
  void set_stable(bool v) { stable_ = v; }
  bool stable() const { return stable_; }

 private:
  void Free();
  TensorListShape shape_;
  DALIDataType type_ = DALI_NO_TYPE;
  TensorLayout layout_;
  std::vector<void *> ptrs_;
  void *data_ = nullptr;
  size_t capacity_ = 0;
  bool owned_ = false, stable_ = false;
};

// ---------------------------------------------------------------------------------------------- OpSpec
struct ArgValue {
  enum Kind { NONE, INT, FLOAT, BOOL, STRING, INT_VEC, FLOAT_VEC, STRING_VEC } kind = NONE;
  int64_t i = 0;
  double f = 0;
  std::string s;
  std::vector<int64_t> iv;
  std::vector<float> fv;
  std::vector<double> dv;           // FLOAT_VEC given in double precision (fv holds the same values rounded to float)
  std::vector<std::string> sv;
};

class Workspace;

class OpSpec {
 public:
  OpSpec() = default;
  explicit OpSpec(const std::string &schema_name) : name_(schema_name) {}
  const std::string &SchemaName() const { return name_; }
  const std::string &name() const { return name_; }

  OpSpec &AddArg(const std::string &n, const ArgValue &v) { args_[n] = v; return *this; }
  OpSpec &AddInput(const std::string &name, const std::string &device) { inputs_.push_back({name, device}); return *this; }
  OpSpec &AddOutput(const std::string &name, const std::string &device) { outputs_.push_back({name, device}); return *this; }
  OpSpec &AddArgumentInput(const std::string &arg, const std::string &input_name) { arg_inputs_[arg] = input_name; return *this; }

  int NumInput() const { return static_cast<int>(inputs_.size()); }        // regular inputs
  int NumOutput() const { return static_cast<int>(outputs_.size()); }
  const std::pair<std::string, std::string> &Input(int i) const { return inputs_[i]; }
  const std::pair<std::string, std::string> &Output(int i) const { return outputs_[i]; }
  const std::map<std::string, std::string> &ArgumentInputs() const { return arg_inputs_; }

  bool HasArgument(const std::string &n) const { return args_.count(n) != 0; }           // explicitly given, scalar
  bool HasTensorArgument(const std::string &n) const { return arg_inputs_.count(n) != 0; }
  bool ArgumentDefined(const std::string &n) const { return HasArgument(n) || HasTensorArgument(n); }

  // scalar access; falls back to the schema default.  With (ws, idx) a tensor argument is read per sample.
  template <typename T> T GetArgument(const std::string &n, const Workspace *ws = nullptr, int idx = 0) const;
  template <typename T> bool TryGetArgument(T &out, const std::string &n) const;
  template <typename T> std::vector<T> GetRepeatedArgument(const std::string &n) const;
  // per-sample vector argument (tensor argument rows or a broadcast repeated argument)
  std::vector<float> GetFloatVecArgument(const std::string &n, const Workspace *ws, int idx, int expected = -1) const;

  const ArgValue *FindArg(const std::string &n) const;   // explicit or schema default; nullptr if neither

 private:
  std::string name_;
  std::map<std::string, ArgValue> args_;
  std::vector<std::pair<std::string, std::string>> inputs_, outputs_;
  std::map<std::string, std::string> arg_inputs_;
};


// explicit specialisations (defined in pipeline.cc)
#define DALI_DECL_GETARG(T) template <> T OpSpec::GetArgument<T>(const std::string &n, const Workspace *ws, int idx) const;
DALI_DECL_GETARG(double) DALI_DECL_GETARG(float) DALI_DECL_GETARG(int) DALI_DECL_GETARG(int64_t) DALI_DECL_GETARG(bool)
DALI_DECL_GETARG(DALIDataType) DALI_DECL_GETARG(DALIInterpType) DALI_DECL_GETARG(DALIImageType) DALI_DECL_GETARG(std::string)
DALI_DECL_GETARG(TensorLayout)
#undef DALI_DECL_GETARG
template <> bool OpSpec::TryGetArgument<float>(float &, const std::string &) const;
template <> bool OpSpec::TryGetArgument<int>(int &, const std::string &) const;
template <> bool OpSpec::TryGetArgument<bool>(bool &, const std::string &) const;
template <> bool OpSpec::TryGetArgument<std::string>(std::string &, const std::string &) const;
template <> bool OpSpec::TryGetArgument<DALIDataType>(DALIDataType &, const std::string &) const;
template <> bool OpSpec::TryGetArgument<std::vector<float>>(std::vector<float> &, const std::string &) const;
template <> std::vector<float> OpSpec::GetRepeatedArgument<float>(const std::string &) const;
template <> std::vector<int> OpSpec::GetRepeatedArgument<int>(const std::string &) const;

// ---------------------------------------------------------------------------------------------- OpSchema
class OpSchema {
 public:
  explicit OpSchema(const std::string &name) : name_(name) {}
  OpSchema &DocStr(const std::string &d) { doc_ = d; return *this; }
  OpSchema &NumInput(int n) { min_in_ = max_in_ = n; return *this; }
  OpSchema &NumInput(int lo, int hi) { min_in_ = lo; max_in_ = hi; return *this; }
  OpSchema &NumOutput(int n) { num_out_ = n; return *this; }
  OpSchema &AllowSequences() { allow_sequences_ = true; return *this; }
  OpSchema &InputLayout(int, const std::vector<std::string> &layouts) { layouts_ = layouts; return *this; }
  OpSchema &AddArg(const std::string &n, const std::string &doc, bool tensor_ok = false) {
    required_.push_back(n); docs_[n] = doc; tensor_ok_[n] = tensor_ok; return *this;
  }
  template <typename T> OpSchema &AddOptionalArg(const std::string &n, const std::string &doc, const T &def, bool tensor_ok = false);
  OpSchema &AddOptionalArgNoDefault(const std::string &n, const std::string &doc, bool tensor_ok = false) {
    optional_nodefault_.push_back(n); docs_[n] = doc; tensor_ok_[n] = tensor_ok; return *this;
  }
  const std::string &name() const { return name_; }
  const std::string &doc() const { return doc_; }
  int MinNumInput() const { return min_in_; }
  int MaxNumInput() const { return max_in_; }
  int NumOutput() const { return num_out_; }
  bool AllowsSequences() const { return allow_sequences_; }
  const std::map<std::string, ArgValue> &Defaults() const { return defaults_; }
  bool HasArgument(const std::string &n) const { return docs_.count(n) != 0; }
  bool TensorArgAllowed(const std::string &n) const { auto it = tensor_ok_.find(n); return it != tensor_ok_.end() && it->second; }
  const std::vector<std::string> &Required() const { return required_; }
  std::vector<std::string> ArgNames() const { std::vector<std::string> r; for (auto &kv : docs_) r.push_back(kv.first); return r; }
  void CheckArgs(const OpSpec &spec) const;
 private:
  std::string name_, doc_;
  int min_in_ = 0, max_in_ = 0, num_out_ = 1;
  bool allow_sequences_ = false;
  std::vector<std::string> layouts_, required_, optional_nodefault_;
  std::map<std::string, std::string> docs_;
  std::map<std::string, bool> tensor_ok_;
  std::map<std::string, ArgValue> defaults_;
};

class SchemaRegistry {
 public:
  static OpSchema &RegisterSchema(const std::string &name);
  static const OpSchema &GetSchema(const std::string &name);
  static const OpSchema *TryGetSchema(const std::string &name);
  static std::vector<std::string> Names();
};

#define DALI_SCHEMA_CONCAT_(a, b) a##b
#define DALI_SCHEMA_CONCAT(a, b) DALI_SCHEMA_CONCAT_(a, b)
#define DALI_SCHEMA(OpName) \
  static ::dali::OpSchema &DALI_SCHEMA_CONCAT(schema_reg_##OpName##_, __LINE__) = ::dali::SchemaRegistry::RegisterSchema(#OpName)

inline ArgValue MakeArg(int64_t v) { ArgValue a; a.kind = ArgValue::INT; a.i = v; return a; }
inline ArgValue MakeArg(int v) { return MakeArg(static_cast<int64_t>(v)); }
inline ArgValue MakeArg(double v) { ArgValue a; a.kind = ArgValue::FLOAT; a.f = v; return a; }
inline ArgValue MakeArg(float v) { return MakeArg(static_cast<double>(v)); }
inline ArgValue MakeArg(bool v) { ArgValue a; a.kind = ArgValue::BOOL; a.i = v; return a; }
inline ArgValue MakeArg(const std::string &v) { ArgValue a; a.kind = ArgValue::STRING; a.s = v; return a; }
inline ArgValue MakeArg(const char *v) { return MakeArg(std::string(v)); }
inline ArgValue MakeArg(const std::vector<float> &v) { ArgValue a; a.kind = ArgValue::FLOAT_VEC; a.fv = v; return a; }
inline ArgValue MakeArg(const std::vector<int64_t> &v) { ArgValue a; a.kind = ArgValue::INT_VEC; a.iv = v; return a; }
inline ArgValue MakeArg(const std::vector<int> &v) { ArgValue a; a.kind = ArgValue::INT_VEC; a.iv.assign(v.begin(), v.end()); return a; }
inline ArgValue MakeArg(DALIDataType v) { return MakeArg(static_cast<int64_t>(v)); }
inline ArgValue MakeArg(DALIInterpType v) { return MakeArg(static_cast<int64_t>(v)); }
inline ArgValue MakeArg(DALIImageType v) { return MakeArg(static_cast<int64_t>(v)); }

template <typename T>
OpSchema &OpSchema::AddOptionalArg(const std::string &n, const std::string &doc, const T &def, bool tensor_ok) {
  defaults_[n] = MakeArg(def); docs_[n] = doc; tensor_ok_[n] = tensor_ok;
  return *this;
}

// ---------------------------------------------------------------------------------------------- Workspace
class Workspace {
 public:
  template <typename Backend> const TensorList<Backend> &Input(int i) const;
  template <typename Backend> TensorList<Backend> &Output(int i) const;
  bool InputIsType(int i, bool gpu) const { return inputs_[i].gpu != nullptr ? gpu : !gpu; }
  const TensorList<CPUBackend> &ArgumentInput(const std::string &name) const {
    auto it = arg_inputs_.find(name);
    DALI_ENFORCE(it != arg_inputs_.end(), "Argument input \"", name, "\" not found in the workspace");
    return *it->second;
  }
  bool HasArgumentInput(const std::string &name) const { return arg_inputs_.count(name) != 0; }
  int NumInput() const { return static_cast<int>(inputs_.size()); }
  int NumOutput() const { return static_cast<int>(outputs_.size()); }
  int GetInputBatchSize(int i) const;
  cudaStream_t stream() const { return stream_; }
  bool has_stream() const { return true; }

  // executor side
  struct Slot { TensorList<CPUBackend> *cpu = nullptr; TensorList<GPUBackend> *gpu = nullptr; };
  void AddInput(TensorList<CPUBackend> *t) { inputs_.push_back({t, nullptr}); }
  void AddInput(TensorList<GPUBackend> *t) { inputs_.push_back({nullptr, t}); }
  void AddOutput(TensorList<CPUBackend> *t) { outputs_.push_back({t, nullptr}); }
  void AddOutput(TensorList<GPUBackend> *t) { outputs_.push_back({nullptr, t}); }
  void AddArgumentInput(const std::string &n, const TensorList<CPUBackend> *t) { arg_inputs_[n] = t; }
  void set_stream(cudaStream_t s) { stream_ = s; }
  const std::vector<Slot> &outputs() const { return outputs_; }
 private:
  std::vector<Slot> inputs_, outputs_;
  std::map<std::string, const TensorList<CPUBackend> *> arg_inputs_;
  cudaStream_t stream_ = nullptr;
};

template <> inline const TensorList<CPUBackend> &Workspace::Input<CPUBackend>(int i) const {
  DALI_ENFORCE(inputs_.at(i).cpu, "Input ", i, " is not a CPU TensorList"); return *inputs_[i].cpu; }
template <> inline const TensorList<GPUBackend> &Workspace::Input<GPUBackend>(int i) const {
  DALI_ENFORCE(inputs_.at(i).gpu, "Input ", i, " is not a GPU TensorList"); return *inputs_[i].gpu; }
template <> inline TensorList<CPUBackend> &Workspace::Output<CPUBackend>(int i) const {
  DALI_ENFORCE(outputs_.at(i).cpu, "Output ", i, " is not a CPU TensorList"); return *outputs_[i].cpu; }
template <> inline TensorList<GPUBackend> &Workspace::Output<GPUBackend>(int i) const {
  DALI_ENFORCE(outputs_.at(i).gpu, "Output ", i, " is not a GPU TensorList"); return *outputs_[i].gpu; }
inline int Workspace::GetInputBatchSize(int i) const {
  return inputs_.at(i).cpu ? inputs_[i].cpu->num_samples() : inputs_[i].gpu->num_samples();
}

// ---------------------------------------------------------------------------------------------- Operator
class OperatorBase {
 public:
  explicit OperatorBase(const OpSpec &spec)
      : spec_(spec), num_threads_(spec.GetArgument<int>("num_threads")), max_batch_size_(spec.GetArgument<int>("max_batch_size")) {}
  virtual ~OperatorBase() = default;
  // operator.h:88-105
  bool Setup(std::vector<OutputDesc> &output_desc, const Workspace &ws) { return SetupImpl(output_desc, ws); }
  void Run(Workspace &ws) { RunImpl(ws); }
  virtual bool HasContiguousOutputs() const { return true; }
  // called by the executor once the iteration's stream has been synchronised (where the reference's executor rethrows the
  // errors captured during the run, exec_node_task.cc): operators with device-side status words check them here
  virtual void CheckCompletion() {}
  const OpSpec &GetSpec() const { return spec_; }
 protected:
  virtual bool SetupImpl(std::vector<OutputDesc> &output_desc, const Workspace &ws) = 0;
  virtual void RunImpl(Workspace &ws) = 0;
  const OpSpec spec_;
  int num_threads_;
  int max_batch_size_;
};

// Executor-level fusion of an image decoder with the Resize that consumes it (SURVEY.md 8f rank 1): when the decoded image has no
// other consumer the pipeline links the two operators; the decoder then defers its launch to the Resize, which asks it for the
// component planes of the samples its planar kernel can take and resizes them without the RGB image ever being written.
struct PlanarSource {            // mirrors dalib200PlanarImage (include/dali_b200.h)
  const uint8_t *y, *cb, *cr;
  int32_t pitch_y, pitch_c, width, height, crop_x, crop_y;
};
class PlanarProducer {
 public:
  virtual ~PlanarProducer() = default;
  virtual void EnableDeferredRun() = 0;                                      // build time: a fused consumer exists
  virtual void SelectPlanar(const std::vector<uint8_t> &want, std::vector<uint8_t> &granted) = 0;   // per iteration, from the consumer's Setup
  virtual void RunDeferred(cudaStream_t stream) = 0;                          // upload + decode (planes only where granted)
  virtual void GetPlanarSource(int sample, PlanarSource *out) = 0;            // after RunDeferred
};
class PlanarConsumer {
 public:
  virtual ~PlanarConsumer() = default;
  virtual void AttachProducer(PlanarProducer *p) = 0;
};

// Spectrogram -> MelFilterBank fusion (one kernel, the spectrogram is not materialised): same linking scheme
class SpectrumProducer {
 public:
  virtual ~SpectrumProducer() = default;
  virtual void EnableDeferredRun() = 0;                            // build time: the only consumer is a MelFilterBank
  virtual bool Deferred() const = 0;                               // this iteration's launch was left to the consumer
  virtual void *SpectrogramPlan() = 0;                             // dalib200SpectrogramPlan *
  virtual const std::vector<const void *> &DeferredInputs() const = 0;
};
class SpectrumConsumer {
 public:
  virtual ~SpectrumConsumer() = default;
  virtual void AttachProducer(SpectrumProducer *p) = 0;
};

// PreemphasisFilter -> Spectrogram fusion (the spectrogram's framing applies the filter, the filtered signal is not
// materialised): same linking scheme
class PreemphasisProducer {
 public:
  virtual ~PreemphasisProducer() = default;
  virtual void EnableDeferredRun() = 0;                            // build time: the only consumer is a Spectrogram
  virtual bool Deferred() const = 0;                               // this iteration's filter was left to the consumer
  virtual const std::vector<const void *> &DeferredInputs() const = 0;   // the unfiltered f32 signals
  virtual const std::vector<float> &Coefficients() const = 0;      // per sample
  virtual int Border() const = 0;                                  // DALIB200_BORDER_*
};
class PreemphasisConsumer {
 public:
  virtual ~PreemphasisConsumer() = default;
  virtual void AttachProducer(PreemphasisProducer *p) = 0;
};

// Pad's output extents (dali/operators/generic/pad.h): for every padded axis the batch maximum (shape absent or negative) or
// max(shape, the sample's extent), rounded up to a multiple of align; other axes keep their extent.  in / out: n x ndim.
// shapes: per-sample requested extents (one per padded axis) or empty.  Throws on bad arguments.
struct PadArgs {
  std::vector<int> axes;                   // padded axes, resolved from axes / axis_names (all axes by default)
  std::vector<int64_t> align;              // one per padded axis
};
PadArgs PadResolveArgs(const OpSpec &spec, int ndim, const std::string &layout);
void PadOutputShapes(const PadArgs &a, int n, int ndim, const int64_t *in, const std::vector<std::vector<int64_t>> &shapes, int64_t *out);
// fill_value as the bits of one element of `type`; throws when the value is not exactly representable in it
uint32_t PadFillBits(float fill, DALIDataType type);

// Transpose's permutation (the dimensions reversed when `perm` is absent) and output layout (output_layout, else the input layout
// permuted when transpose_layout, else the input layout).  Throws on bad arguments.
struct TransposeArgs {
  std::vector<int> perm;
  std::string layout;
};
TransposeArgs TransposeResolveArgs(const OpSpec &spec, int ndim, const std::string &layout);
// Cat's / Stack's axis (negative values counted from the back of the input, for Stack of the output) and output layout; layouts:
// one per input.  Throws on bad arguments.
struct JoinArgs {
  int axis = 0;
  std::string layout;
};
JoinArgs JoinResolveArgs(const OpSpec &spec, bool stack, int ndim, const std::vector<std::string> &layouts);

// fn.reductions.*: the reduced axes as a mask (`axes`, negative counted from the back, or `axis_names` against the layout; all axes
// when neither is given) and the output layout.  Throws on bad arguments.
struct ReduceArgs {
  uint32_t mask = 0;
  bool keep_dims = false;
  std::string layout;
};
ReduceArgs ReduceResolveArgs(const OpSpec &spec, int ndim, const std::string &layout);
// DALIB200_REDUCE_* of a reductions__* schema name
int ReduceOpOf(const std::string &schema);
// StdDev / Variance: the mean of sample i must have the output's shape, with or without the reduced axes as unit axes
void ReduceCheckMean(const char *name, int i, const int64_t *mean_shape, int mean_ndim, const int64_t *in_shape, int ndim, uint32_t mask);

// fn.experimental.filter: `border` and `mode` as DALIB200_FILTER_* codes; FilterAnchor: the (row, column) anchor of sample i from
// the values of `anchor` (one per filter axis, or [-1]).  Throw on bad arguments.
struct FilterArgs {
  int border = 0, mode = 0;
};
FilterArgs FilterResolveArgs(const OpSpec &spec);
void FilterAnchor(int i, const std::vector<int> &vals, int32_t *row_col);

// fn.erase: the erased axes -- axis_names when given, else axes when given, else "HW" for an input with a layout and axes' default
// [1, 0] for one without -- the coordinate flags (normalized_anchor / normalized_shape override normalized) and the fill values.
struct EraseArgs {
  bool by_name = false;
  std::string axis_names;
  std::vector<int32_t> axes;
  int norm_anchor = 0, norm_shape = 0, centered = 0;
  std::vector<float> fill;
};
EraseArgs EraseResolveArgs(const OpSpec &spec, const std::string &layout);

// fn.multi_paste: in_ids and the six region arguments (in_anchors, in_anchors_rel, shapes, shapes_rel, out_anchors, out_anchors_rel)
// of every sample back to back with their per-sample counts -- a per-sample CPU tensor input read with its shape ([K] for in_ids,
// [K, 2] for the others), or a list used for every sample -- output_size per sample, and dtype (-1: the input's type).
constexpr int kMultiPasteRegionArgs = 6;
struct MultiPasteArgs {
  bool has_ids = false, has_size = false;
  bool has[kMultiPasteRegionArgs] = {};
  std::vector<int32_t> ids;
  std::vector<int64_t> id_counts, sizes;
  std::vector<double> vals[kMultiPasteRegionArgs];
  std::vector<int64_t> counts[kMultiPasteRegionArgs];
  int dtype = -1;
};
MultiPasteArgs MultiPasteResolveArgs(const OpSpec &spec, const Workspace *ws, int n);
// dalib200PasteSetup with the resolved arguments (fill 0); returns its status.
int MultiPasteSetup(::dalib200PastePlan *plan, const MultiPasteArgs &a, int in_type, int ninputs, int n, const int *ndims,
                    const char *const *layouts, const int64_t *in_shapes, int64_t *out_shapes);

template <typename Backend>
class Operator : public OperatorBase {
 public:
  explicit Operator(const OpSpec &spec) : OperatorBase(spec) {}
};

#define USE_OPERATOR_MEMBERS() using OperatorBase::spec_; using OperatorBase::num_threads_; using OperatorBase::max_batch_size_

using OperatorCreator = std::function<std::unique_ptr<OperatorBase>(const OpSpec &)>;

class OperatorRegistry {
 public:
  static std::map<std::string, OperatorCreator> &Registry(const std::string &backend);   // "cpu" | "gpu" | "mixed"
  static void Register(const std::string &backend, const std::string &name, OperatorCreator c);
  static std::vector<std::string> RegisteredNames(const std::string &backend);
};

struct OperatorRegisterer {
  OperatorRegisterer(const char *backend, const char *name, OperatorCreator c) { OperatorRegistry::Register(backend, name, std::move(c)); }
};

#define DALI_OP_BACKEND_CPU "cpu"
#define DALI_OP_BACKEND_GPU "gpu"
#define DALI_OP_BACKEND_Mixed "mixed"
#define DALI_REGISTER_OPERATOR(OpName, OpType, device)                                                              \
  static ::dali::OperatorRegisterer DALI_SCHEMA_CONCAT(op_reg_##OpName##_##device##_, __LINE__)(                    \
      DALI_OP_BACKEND_##device, #OpName,                                                                            \
      [](const ::dali::OpSpec &spec) -> std::unique_ptr<::dali::OperatorBase> { return std::make_unique<OpType>(spec); })

// operator.cc:157-170
std::unique_ptr<OperatorBase> InstantiateOperator(const OpSpec &spec);

// ---------------------------------------------------------------------------------------------- Pipeline
class Pipeline {
 public:
  Pipeline(int max_batch_size, int num_threads, int device_id);
  ~Pipeline();
  int max_batch_size() const { return max_batch_size_; }
  int device_id() const { return device_id_; }
  cudaStream_t stream() const { return stream_; }

  void AddExternalInput(const std::string &name, const std::string &device, const std::string &layout);
  void AddOperator(const OpSpec &spec, const std::string &inst_name);
  void SetOutputDescs(const std::vector<std::pair<std::string, std::string>> &outs);   // (name, device)
  void Build();
  // External data: host pointers, one per sample.  For device == "gpu" the samples are copied H2D on the pipeline stream.
  void SetExternalInput(const std::string &name, const std::vector<const void *> &ptrs, const TensorListShape &shape,
                        DALIDataType type, const std::string &layout, bool no_copy = false);
  void Run();
  // Synchronises the pipeline stream.  Returned pointers stay valid until the next Run().
  int NumOutputs() const { return static_cast<int>(output_names_.size()); }
  bool OutputIsGPU(int i) const;
  const TensorList<CPUBackend> *OutputCPU(int i) const;
  const TensorList<GPUBackend> *OutputGPU(int i) const;
  void WaitOutputs();

 private:
  struct Edge {
    std::string device;
    std::unique_ptr<TensorList<CPUBackend>> cpu;
    std::unique_ptr<TensorList<GPUBackend>> gpu;
    std::vector<uint8_t> host_copy;      // keeps external CPU data alive when it was copied
    bool external = false;
    std::string layout;
  };
  struct Node {
    OpSpec spec;
    std::string name;
    std::unique_ptr<OperatorBase> op;
  };
  Edge &GetEdge(const std::string &name, const std::string &device);
  // Links every Consumer operator to the Producer of its first input when that input feeds nothing else and is not a pipeline
  // output: the producer then defers its launch to the consumer (pipeline.cc)
  template <typename Producer, typename Consumer> void LinkSoleConsumers();
  int max_batch_size_, num_threads_, device_id_;
  cudaStream_t stream_ = nullptr;
  std::map<std::string, Edge> edges_;       // key: name + "/" + device
  std::vector<Node> nodes_;
  std::vector<std::pair<std::string, std::string>> output_names_;
  bool built_ = false;
};

}  // namespace dali
#endif  // DALI_B200_HOST_DALI_H_
