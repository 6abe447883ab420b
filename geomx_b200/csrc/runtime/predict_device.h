// The planned predictor on an H100 (GXPredCreate* with dev_type 2): predict.h's graph, shape inference and liveness-planned arena, run as
// sm_90a kernels (kernels/predict_dev.cu).  On the device the planner also takes the general executor's other operators (namespace
// extended below), so every graph the host serves, on either engine, runs here.
//
// libgeomx_capi.so links no CUDA: the kernels library is dlopen'ed from the directory this library was loaded from, on the first device
// request, and reached through its `gx_pred_*` entry points only.  Parameters go to the device once, at create, together with what is
// derived from them (BatchNorm's per-channel scale and shift, convolution weights padded to TMA-aligned rows); clones share them.  Each
// handle owns one device allocation (arena | input slots | convolution workspace) and a non-blocking stream.  Forward records every
// operator into a CUDA graph on its first call and replays it afterwards; PartialForward launches one operator.  Every call makes the
// handle's device current and gives the caller's back (DeviceGuard).  Every operator's arguments are checked here, before anything is
// launched.
#pragma once
#include <dlfcn.h>

#include <limits>
#include <mutex>
#include <type_traits>

#include "graph.h"
#include "predict.h"

namespace gxrt {
namespace predict {

struct DeviceApi {
  int (*device_count)(int*);
  int (*device_cc)(int, int*, int*);
  int (*get_device)(int*, int*);
  int (*set_device)(int);
  const char* (*error_string)(int);
  int (*malloc)(void**, size_t);
  int (*free)(void*);
  int (*h2d)(void*, const void*, size_t, void*);
  int (*d2h)(void*, const void*, size_t, void*);
  int (*memset)(void*, size_t, void*);
  int (*stream_create)(void**);
  int (*stream_destroy)(void*);
  int (*stream_sync)(void*);
  int (*capture_begin)(void*);
  int (*capture_end)(void*, void**);
  int (*graph_launch)(void*, void*);
  int (*graph_destroy)(void*);
  int (*map)(int, const float*, float*, long long, void*);
  int (*pointwise)(int, const float*, float*, long long, float, float, void*);
  int (*affine)(const float*, float*, long long, long long, long long, const float*, const float*, void*);
  int (*binary)(int, const float*, const float*, float*, long long, int, const long long*, const long long*, const long long*, void*);
  int (*transpose)(const float*, float*, long long, int, const long long*, const long long*, void*);
  int (*add_n)(const float* const*, int, float*, long long, void*);
  int (*concat_part)(const float*, float*, long long, long long, long long, long long, void*);
  int (*softmax)(const float*, float*, long long, long long, long long, int, void*);
  int (*embedding)(const float*, const float*, float*, long long, long long, long long, void*);
  int (*pool)(const float*, float*, long long, int, int, int, int, int, int, int, int, int, int, int, int, void*);
  int (*fc)(const float*, const float*, const float*, float*, int, int, int, void*);
  long long (*conv_workspace)(int, int, int, int, int, int, int, int);
  int (*conv)(const float*, const float*, long long, const float*, float*, float*, long long, int, int, int, int, int, int, int, int, int, int, int, int,
              int, int, int, int, void*);
  int (*gather)(const float*, float*, long long, int, const long long*, int, float, void*);
  int (*take)(const float*, const float*, float*, long long, long long, long long, long long, void*);
  int (*one_hot)(const float*, float*, long long, long long, float, float, void*);
  int (*where)(const float*, const float*, const float*, float*, long long, void*);
  int (*arg)(const float*, float*, long long, long long, long long, int, void*);
  int (*reduce)(int, const float*, float*, long long, int, const long long*, int, const long long*, float, void*);
  int (*norm)(int, const float*, const float*, const float*, float*, long long, long long, long long, float, void*);
  int (*lrn)(const float*, float*, long long, long long, long long, long long, float, float, float, void*);
  int (*softmax_ce)(const float*, const float*, float*, long long, long long, void*);
  int (*dot)(const float*, const float*, float*, int, int, int, int, int, void*);
  long long (*deconv_workspace)(int, int, int, int, int, int, int, int);
  int (*deconv)(const float*, const float*, const float*, float*, float*, long long, int, int, int, int, int, int, int, int, int, int, int, int, int, int,
                int, int, void*);

  void Check(int rc, const std::string& what) const { if (rc != 0) throw std::runtime_error(what + " failed: " + error_string(rc)); }

  // the entry points of libgeomx_kernels.so next to this library; throws (every time) when it cannot be loaded
  static const DeviceApi& Get() {
    static std::once_flag once;
    static DeviceApi api;
    static std::string error;
    std::call_once(once, [] { error = Load(&api); });
    if (!error.empty()) throw std::runtime_error(error);
    return api;
  }

 private:
  static std::string Load(DeviceApi* a) {
    Dl_info info;
    if (dladdr(reinterpret_cast<void*>(&DeviceApi::Load), &info) == 0 || info.dli_fname == nullptr) return "cannot locate the loaded C library";
    std::string dir = info.dli_fname;
    const size_t slash = dir.rfind('/');
    dir = slash == std::string::npos ? "." : dir.substr(0, slash);
    const std::string path = dir + "/libgeomx_kernels.so";
    void* lib = dlopen(path.c_str(), RTLD_NOW | RTLD_LOCAL);
    if (lib == nullptr) { const char* e = dlerror(); return "cannot load the device kernels " + path + ": " + (e ? e : "unknown error"); }
    std::string missing;
    auto sym = [&](auto& fn, const char* name) {
      void* p = dlsym(lib, name);
      if (p == nullptr && missing.empty()) missing = name;
      fn = reinterpret_cast<std::remove_reference_t<decltype(fn)>>(p);
    };
    sym(a->device_count, "gx_pred_device_count"); sym(a->device_cc, "gx_pred_device_cc"); sym(a->get_device, "gx_pred_get_device");
    sym(a->set_device, "gx_pred_set_device"); sym(a->error_string, "gx_pred_error_string"); sym(a->malloc, "gx_pred_malloc"); sym(a->free, "gx_pred_free");
    sym(a->h2d, "gx_pred_h2d"); sym(a->d2h, "gx_pred_d2h"); sym(a->memset, "gx_pred_memset"); sym(a->stream_create, "gx_pred_stream_create");
    sym(a->stream_destroy, "gx_pred_stream_destroy"); sym(a->stream_sync, "gx_pred_stream_sync"); sym(a->capture_begin, "gx_pred_capture_begin");
    sym(a->capture_end, "gx_pred_capture_end"); sym(a->graph_launch, "gx_pred_graph_launch"); sym(a->graph_destroy, "gx_pred_graph_destroy");
    sym(a->map, "gx_pred_map"); sym(a->pointwise, "gx_pred_pointwise"); sym(a->affine, "gx_pred_affine"); sym(a->binary, "gx_pred_binary");
    sym(a->transpose, "gx_pred_transpose"); sym(a->add_n, "gx_pred_add_n"); sym(a->concat_part, "gx_pred_concat_part"); sym(a->softmax, "gx_pred_softmax");
    sym(a->embedding, "gx_pred_embedding"); sym(a->pool, "gx_pred_pool"); sym(a->fc, "gx_pred_fc"); sym(a->conv_workspace, "gx_pred_conv_workspace");
    sym(a->conv, "gx_pred_conv"); sym(a->gather, "gx_pred_gather"); sym(a->take, "gx_pred_take"); sym(a->one_hot, "gx_pred_one_hot");
    sym(a->where, "gx_pred_where"); sym(a->arg, "gx_pred_arg"); sym(a->reduce, "gx_pred_reduce"); sym(a->norm, "gx_pred_norm"); sym(a->lrn, "gx_pred_lrn");
    sym(a->softmax_ce, "gx_pred_softmax_ce"); sym(a->dot, "gx_pred_dot"); sym(a->deconv_workspace, "gx_pred_deconv_workspace");
    sym(a->deconv, "gx_pred_deconv");
    if (!missing.empty()) return path + " has no entry point " + missing + " (an older build?)";
    return "";
  }
};

// ------------------------------------------------------------------------------------------------ the device-only operator set
// Every operator of the general executor (train_exec.h Executor::Run) that the planned set lacks.  Its nodes are planned with the general
// executor's canonical names, string attributes and shape rules (graph.h), so the device reads a graph exactly as the general executor does.
namespace extended {

// the node as the general executor's graph sees it; inputs carry only their names (InferNode's messages)
inline graph::Node GraphNode(const Node& nd, const std::vector<const Node*>& in = {}) {
  graph::Node g;
  g.op = graph::CanonicalOp(nd.op); g.name = nd.name; g.attrs = nd.sattrs;
  for (const Node* i : in) { auto v = std::make_shared<graph::Node>(); v->name = i->name; g.inputs.push_back(graph::Entry{v, 0}); }
  return g;
}
inline std::map<std::string, std::string> StringAttrs(const Node& nd) {
  std::map<std::string, std::string> m;
  const JValue* o = nd.attrs.Object();
  if (o == nullptr || o->kind != JValue::kObj) return m;
  for (auto& kv : o->obj) {
    if (kv.first == "__attr__" && kv.second.kind == JValue::kObj) { for (auto& u : kv.second.obj) m[u.first] = graph::JAttrToString(u.second); continue; }
    if (kv.second.kind != JValue::kNull) m[kv.first] = graph::JAttrToString(kv.second);
  }
  return m;
}
inline int NumOutputs(const Node& nd) {
  if (graph::CanonicalOp(nd.op) != "SliceChannel") return 1;
  Node t = nd; t.sattrs = StringAttrs(nd);
  return graph::NumOutputs(GraphNode(t));
}
inline bool Has(const std::string& op) { return graph::FindOp(op) != nullptr; }
// graph.h FromJSON's checks first: a variadic operator's count attribute defaults to its inputs, and the input count must be the operator's
inline void Infer(Node& nd, const std::vector<const Node*>& in) {
  nd.sattrs = StringAttrs(nd);
  const graph::OpDef& d = graph::GetOp(nd.op);
  if (*d.key_var_num_args && !graph::AttrView(nd.sattrs).Has(d.key_var_num_args)) nd.sattrs[d.key_var_num_args] = std::to_string(in.size());
  const size_t want = d.inputs(graph::AttrView(nd.sattrs)).size();
  if (in.size() != want)
    throw std::runtime_error(nd.name + " (" + d.name + "): " + std::to_string(in.size()) + " inputs in the file, the operator takes " + std::to_string(want));
  const graph::Node g = GraphNode(nd, in);
  std::vector<const Shape*> shapes;
  for (const Node* i : in) shapes.push_back(&i->shape);
  Shape out;
  if (!graph::InferNode(g, shapes, [](size_t, const Shape&) {}, &out)) throw std::runtime_error(nd.name + " (" + g.op + "): the output shape cannot be inferred");
  nd.op = g.op; nd.extended = true; nd.num_out = graph::NumOutputs(g); nd.shape = out;
}
inline const ExtendedOps* Ops() { static const ExtendedOps ops{&Has, &NumOutputs, &Infer}; return &ops; }

// the general executor's unary kinds that the planned set lacks, in the order of train_exec.h Un() (device kinds 11..30)
inline int UnaryKind(const std::string& op) {
  static const char* names[] = {"sin", "cos", "tan", "arcsin", "arccos", "arctan", "sinh", "cosh", "log1p", "expm1", "log2", "log10", "rsqrt", "reciprocal",
                                "cbrt", "erf", "floor", "ceil", "round", "sign"};
  for (int i = 0; i < 20; ++i) if (op == names[i]) return 11 + i;
  return -1;
}
// binary power and comparisons (device kinds 6..12), scalar power / max / min (pointwise modes 9..12)
inline int BinaryKind(const std::string& op) {
  static const char* names[] = {"broadcast_power", "broadcast_equal", "broadcast_not_equal", "broadcast_greater", "broadcast_greater_equal", "broadcast_lesser",
                                "broadcast_lesser_equal"};
  for (int i = 0; i < 7; ++i) if (op == names[i]) return 6 + i;
  return -1;
}
inline int ScalarMode(const std::string& op) {
  static const char* names[] = {"_power_scalar", "_rpower_scalar", "_maximum_scalar", "_minimum_scalar"};
  for (int i = 0; i < 4; ++i) if (op == names[i]) return 9 + i;
  return -1;
}
inline bool IsGather(const std::string& op) {
  static const char* names[] = {"slice_axis", "slice", "SwapAxis", "tile", "repeat", "Pad", "reverse", "broadcast_to", "broadcast_axis", "UpSampling", "SliceChannel"};
  for (auto n : names) if (op == n) return true;
  return false;
}
inline bool IsReduce(const std::string& op) { return op == "sum" || op == "mean" || op == "max" || op == "min" || op == "prod" || op == "norm"; }
inline void SplitAxis(const Shape& s, int64_t ax, int64_t* outer, int64_t* c, int64_t* inner) {
  *outer = 1; *inner = 1; *c = s[ax];
  for (int64_t i = 0; i < ax; ++i) *outer *= s[i];
  for (size_t i = ax + 1; i < s.size(); ++i) *inner *= s[i];
}

}  // namespace extended

// makes `dev` current for its lifetime and gives the caller's device back.  A thread that had no current CUDA context keeps `dev`:
// "restoring" the device 0 that cudaGetDevice reports for such a thread would create a context on a GPU the caller never used.
class DeviceGuard {
 public:
  DeviceGuard(const DeviceApi& api, int dev) : api_(api) {
    int had_context = 0;
    api.Check(api.get_device(&prev_, &had_context), "cudaGetDevice");
    if (prev_ != dev) { api.Check(api.set_device(dev), "cudaSetDevice"); switched_ = had_context != 0; }
  }
  ~DeviceGuard() { if (switched_) api_.set_device(prev_); }
  DeviceGuard(const DeviceGuard&) = delete;
  DeviceGuard& operator=(const DeviceGuard&) = delete;
 private:
  const DeviceApi& api_;
  int prev_ = 0;
  bool switched_ = false;
};

// parameters on the device, shared by a handle, its MultiThread siblings and its Reshape clones
struct DeviceParams {
  const DeviceApi* api = nullptr;
  int dev = 0;
  void* buf = nullptr;
  std::map<std::string, float*> by_name;
  std::map<int, std::pair<float*, float*>> bn;          // BatchNorm node -> scale, shift
  std::map<int, std::pair<float*, int64_t>> conv_w;     // Convolution node -> weight with rows padded to a multiple of 4, row stride
  DeviceParams() = default;
  DeviceParams(const DeviceParams&) = delete;
  DeviceParams& operator=(const DeviceParams&) = delete;
  ~DeviceParams() {
    if (buf == nullptr) return;
    try { DeviceGuard g(*api, dev); api->free(buf); } catch (...) {}
  }
};

class DevicePredictor {
 public:
  // checks the device, uploads the parameters and binds the plan; `plan` was built without a host arena
  static std::unique_ptr<DevicePredictor> Create(std::unique_ptr<Predictor> plan, int dev_id) {
    const DeviceApi& api = DeviceApi::Get();
    int count = 0;
    const int rc = api.device_count(&count);
    if (rc != 0 || count == 0) throw std::runtime_error(std::string("no CUDA device is visible") + (rc ? std::string(" (") + api.error_string(rc) + ")" : ""));
    if (dev_id < 0 || dev_id >= count) throw std::runtime_error("dev_id " + std::to_string(dev_id) + " is out of range: " + std::to_string(count) + " CUDA device(s) visible");
    int major = 0, minor = 0;
    api.Check(api.device_cc(dev_id, &major, &minor), "cudaDeviceGetAttribute");
    if (major != 9 || minor != 0)
      throw std::runtime_error("device " + std::to_string(dev_id) + " is sm_" + std::to_string(major) + std::to_string(minor) + "; the device kernels are built for sm_90a (H100) only");
    auto params = std::make_shared<DeviceParams>();
    params->api = &api; params->dev = dev_id;
    std::unique_ptr<DevicePredictor> d(new DevicePredictor(std::move(plan), params));
    d->Validate();
    DeviceGuard g(api, dev_id);
    api.Check(api.stream_create(&d->stream_), "cudaStreamCreate");
    d->Upload();
    d->Bind();
    return d;
  }
  // another handle over the same parameters: own inputs, arena, stream and graph (MultiThread, Reshape)
  std::unique_ptr<DevicePredictor> Clone(const std::map<std::string, Shape>* new_shapes) const {
    std::unique_ptr<DevicePredictor> d(new DevicePredictor(plan_->Clone(new_shapes), params_));
    d->Validate();
    DeviceGuard g(api_, dev_);
    api_.Check(api_.stream_create(&d->stream_), "cudaStreamCreate");
    d->Bind();
    return d;
  }
  ~DevicePredictor() {
    try {
      DeviceGuard g(api_, dev_);
      if (stream_) api_.stream_sync(stream_);
      if (graph_) api_.graph_destroy(graph_);
      if (stream_) api_.stream_destroy(stream_);
      if (mem_) api_.free(mem_);
    } catch (...) {}
  }

  void SetInput(const std::string& key, const float* data, size_t size) {
    auto it = plan_->inputs_.find(key);
    if (it == plan_->inputs_.end()) throw std::runtime_error("SetInput: unknown input " + key);
    if (size != it->second.size()) throw std::runtime_error("SetInput: " + key + " expects " + std::to_string(it->second.size()) + " values, got " + std::to_string(size));
    DeviceGuard g(api_, dev_);
    api_.Check(api_.h2d(input_.at(key), data, size * sizeof(float), stream_), "SetInput: host-to-device copy");
  }
  void Forward() {
    DeviceGuard g(api_, dev_);
    if (graph_ == nullptr) {
      api_.Check(api_.capture_begin(stream_), "cudaStreamBeginCapture");
      try {
        for (int id : plan_->order_) Enqueue(id);
      } catch (...) {
        void* partial = nullptr;
        api_.capture_end(stream_, &partial);
        if (partial) api_.graph_destroy(partial);
        throw;
      }
      api_.Check(api_.capture_end(stream_, &graph_), "Forward: CUDA graph capture");
    }
    api_.Check(api_.graph_launch(graph_, stream_), "Forward: cudaGraphLaunch");
  }
  void PartialForward(int step, int* step_left) {
    const int n = static_cast<int>(plan_->order_.size());
    if (step < 0 || step >= n) { *step_left = 0; return; }
    DeviceGuard g(api_, dev_);
    Enqueue(plan_->order_[step]);
    *step_left = n - step - 1;
  }
  size_t NumOutputs() const { return plan_->NumOutputs(); }
  const Shape& OutputShape(size_t i) const { return plan_->OutputShape(i); }
  void GetOutput(size_t i, float* out, size_t size) {
    const Node& n = plan_->nodes_[plan_->Head(i)];
    if (size != static_cast<size_t>(Numel(n.shape))) throw std::runtime_error("GetOutput: output " + std::to_string(i) + " has " + std::to_string(Numel(n.shape)) + " values, buffer holds " + std::to_string(size));
    DeviceGuard g(api_, dev_);
    api_.Check(api_.d2h(out, ptr_[plan_->StorageOf(plan_->heads_[i])], size * sizeof(float), stream_), "GetOutput: device-to-host copy");
    api_.Check(api_.stream_sync(stream_), "GetOutput: stream synchronisation");
  }
  size_t ArenaBytes() const { return plan_->ArenaBytes(); }
  size_t NumOps() const { return plan_->NumOps(); }

 private:
  DevicePredictor(std::unique_ptr<Predictor> plan, std::shared_ptr<DeviceParams> params)
      : api_(*params->api), plan_(std::move(plan)), params_(std::move(params)), dev_(params_->dev) {}

  const DeviceApi& api_;
  std::unique_ptr<Predictor> plan_;
  std::shared_ptr<DeviceParams> params_;
  int dev_;
  void* stream_ = nullptr;
  void* graph_ = nullptr;
  void* mem_ = nullptr;                          // arena | input slots | convolution workspace
  std::vector<float*> ptr_;                      // device address of every storage of the plan
  std::map<std::string, float*> input_;
  float* ws_ = nullptr;
  long long ws_floats_ = 0;

  const Node& In(const Node& nd, size_t i) const { return plan_->In(nd, i); }
  float* Ptr(const Node& nd) const { return ptr_[nd.storage]; }
  const float* InPtr(const Node& nd, size_t i) const { In(nd, i); return ptr_[plan_->StorageOf(nd.inputs[i])]; }
  bool IsParam(const Node& nd, size_t i) const {
    const Node& s = In(nd, i);
    return s.op == "null" && !plan_->input_shapes_.count(s.name) && plan_->params_->count(s.name);
  }
  static int Int(int64_t v, const Node& nd) {
    if (v < 0 || v > std::numeric_limits<int>::max()) throw std::runtime_error(nd.name + ": a dimension of " + std::to_string(v) + " exceeds the device kernels' 32-bit range");
    return static_cast<int>(v);
  }

  // everything a launch could trip over, rejected before the first one
  void Validate() const {
    const Predictor& p = *plan_;
    for (int id : p.order_) {
      const Node& nd = p.nodes_[id];
      const std::string& op = nd.op;
      if (Predictor::IsView(nd)) continue;
      if (nd.extended) { ValidateExtended(nd); continue; }
      const Attrs& a = nd.attrs;
      if (op == "Activation") {
        const std::string t = a.Str("act_type", "relu");
        if (Predictor::UnaryKind(t) < 0) throw std::runtime_error(nd.name + ": act_type " + t + " is not supported");
      } else if (op == "LeakyReLU") {
        const std::string t = a.Str("act_type", "leaky");
        if (t != "leaky" && t != "elu") throw std::runtime_error(nd.name + ": LeakyReLU act_type " + t + " is not supported");
      } else if (op == "BatchNorm") {
        for (size_t i = 1; i <= 4; ++i)
          if (!IsParam(nd, i)) throw std::runtime_error(nd.name + ": BatchNorm's gamma, beta and statistics must come from the parameter file on the device");
      } else if (op == "transpose" || Predictor::BinaryKind(op) >= 0) {
        if (nd.shape.size() > 8) throw std::runtime_error(nd.name + ": the device kernels take at most 8 axes, got " + ShapeStr(nd.shape));
      } else if (op == "Convolution") {
        // the kernels index in 32 bits: every attribute, every extent, and the furthest input row / column a window reaches
        const Predictor::Conv c = p.ConvAttrs(nd);
        const Shape& xs = In(nd, 0).shape;
        for (int64_t v : {xs[0], xs[1], xs[2], xs[3], nd.shape[1], nd.shape[2], nd.shape[3], c.kh, c.kw, c.sh, c.sw, c.ph, c.pw, c.dh, c.dw, c.groups}) Int(v, nd);
        Int((nd.shape[2] - 1) * c.sh + (c.kh - 1) * c.dh, nd);
        Int((nd.shape[3] - 1) * c.sw + (c.kw - 1) * c.dw, nd);
        const int64_t P = Int(nd.shape[2] * nd.shape[3], nd), K = Int(xs[1] / c.groups * c.kh * c.kw, nd);
        Int(xs[0] * P, nd);
        Int(K * P, nd);
      } else if (op == "FullyConnected") {
        const Shape& w = In(nd, 1).shape;
        Int(Numel(nd.shape) / w[0], nd); Int(w[0], nd); Int(w[1], nd);
      } else if (op == "Pooling") {
        const Shape& xs = In(nd, 0).shape;
        const Predictor::Pool q = p.PoolAttrs(nd, xs);
        for (int64_t v : {xs[0], xs[1], xs[2], xs[3], nd.shape[2], nd.shape[3], q.kh, q.kw, q.sh, q.sw, q.ph, q.pw}) Int(v, nd);
      }
    }
  }

  // parameters, BatchNorm scale / shift and padded convolution weights: one staging buffer, one allocation, one copy
  void Upload() {
    const Predictor& p = *plan_;
    std::vector<float> stage;
    std::vector<std::pair<std::string, size_t>> named;
    std::map<int, std::pair<size_t, size_t>> bn;
    std::map<int, std::pair<size_t, int64_t>> conv;
    auto put = [&](const float* src, size_t n) { const size_t at = stage.size(); stage.insert(stage.end(), src, src + n); stage.resize((stage.size() + 15) / 16 * 16, 0.f); return at; };
    for (const Node& nd : p.nodes_) {
      if (nd.op != "null") continue;
      auto it = p.params_->find(nd.name);
      if (it == p.params_->end() || p.input_shapes_.count(nd.name)) continue;
      bool dup = false;
      for (auto& e : named) dup = dup || e.first == nd.name;
      if (!dup) named.emplace_back(nd.name, put(it->second.second.data(), it->second.second.size()));
    }
    for (int id : p.order_) {
      const Node& nd = p.nodes_[id];
      if (nd.op == "BatchNorm") {       // the host's formula (predict.h Run)
        const Attrs& a = nd.attrs;
        const Shape& xs = In(nd, 0).shape;
        const int64_t C = xs[Predictor::Axis(a.Int("axis", 1), xs.size())];
        const float eps = static_cast<float>(a.Float("eps", 1e-3));
        const bool fix_gamma = a.Bool("fix_gamma", nd.nnvm);
        const float *g = p.InPtr(nd, 1), *b = p.InPtr(nd, 2), *mean = p.InPtr(nd, 3), *var = p.InPtr(nd, 4);
        std::vector<float> scale(C), shift(C);
        for (int64_t c = 0; c < C; ++c) { scale[c] = (fix_gamma ? 1.f : g[c]) / std::sqrt(var[c] + eps); shift[c] = b[c] - mean[c] * scale[c]; }
        const size_t s0 = put(scale.data(), scale.size());
        bn[id] = {s0, put(shift.data(), shift.size())};
      } else if (nd.op == "Convolution" && IsParam(nd, 1)) {
        const Shape& w = In(nd, 1).shape;
        const int64_t K = w[1] * w[2] * w[3];
        if (K % 4 == 0) continue;
        const int64_t ld = (K + 3) / 4 * 4;
        std::vector<float> padded(static_cast<size_t>(w[0] * ld), 0.f);
        const float* src = p.InPtr(nd, 1);
        for (int64_t f = 0; f < w[0]; ++f) std::copy(src + f * K, src + (f + 1) * K, padded.begin() + f * ld);
        conv[id] = {put(padded.data(), padded.size()), ld};
      }
    }
    if (stage.empty()) return;
    api_.Check(api_.malloc(&params_->buf, stage.size() * sizeof(float)), "cudaMalloc of " + std::to_string(stage.size() * sizeof(float)) + " parameter bytes");
    float* base = static_cast<float*>(params_->buf);
    api_.Check(api_.h2d(base, stage.data(), stage.size() * sizeof(float), stream_), "parameter upload");
    api_.Check(api_.stream_sync(stream_), "parameter upload");
    for (auto& e : named) params_->by_name[e.first] = base + e.second;
    for (auto& e : bn) params_->bn[e.first] = {base + e.second.first, base + e.second.second};
    for (auto& e : conv) params_->conv_w[e.first] = {base + e.second.first, e.second.second};
  }

  // one allocation for the arena, the input slots and the convolution workspace; every storage gets its device address
  void Bind() {
    const Predictor& p = *plan_;
    ws_floats_ = 0;
    for (int id : p.order_) {
      const Node& nd = p.nodes_[id];
      if (nd.extended && nd.op == "Deconvolution") {
        const graph::detail::Win w = graph::detail::Window(extended::GraphNode(nd), false, In(nd, 0).shape);
        const Shape& xs = In(nd, 0).shape;
        const int64_t G = graph::AttrView(nd.sattrs).Int("num_group", 1);
        ws_floats_ = std::max(ws_floats_, api_.deconv_workspace((int)xs[0], (int)xs[1], (int)xs[2], (int)xs[3], (int)(nd.shape[1] / G), (int)w.kh, (int)w.kw, (int)G));
        continue;
      }
      if (nd.op != "Convolution" || nd.extended) continue;
      const Predictor::Conv c = p.ConvAttrs(nd);
      const Shape& xs = In(nd, 0).shape;
      const bool pointwise = c.kh == 1 && c.kw == 1 && c.sh == 1 && c.sw == 1 && c.ph == 0 && c.pw == 0;
      ws_floats_ = std::max(ws_floats_, api_.conv_workspace(Int(xs[0], nd), Int(xs[1], nd), Int(nd.shape[2], nd), Int(nd.shape[3], nd), Int(c.kh, nd), Int(c.kw, nd),
                                                            Int(c.groups, nd), pointwise));
    }
    int64_t total = p.arena_floats_;
    std::map<std::string, int64_t> in_off;
    for (auto& kv : p.inputs_) { in_off[kv.first] = total; total += (static_cast<int64_t>(kv.second.size()) + 15) / 16 * 16; }
    const int64_t ws_off = total;
    total += ws_floats_;
    const size_t bytes = static_cast<size_t>(std::max<int64_t>(total, 16)) * sizeof(float);
    api_.Check(api_.malloc(&mem_, bytes), "cudaMalloc of the " + std::to_string(bytes) + "-byte arena");
    api_.Check(api_.memset(mem_, bytes, stream_), "arena initialisation");
    float* base = static_cast<float*>(mem_);
    for (auto& kv : in_off) input_[kv.first] = base + kv.second;
    ws_ = base + ws_off;
    ptr_.assign(p.storages_.size(), nullptr);
    for (size_t s = 0; s < p.storages_.size(); ++s) if (!p.storages_[s].external) ptr_[s] = base + p.storages_[s].offset;
    for (const Node& nd : p.nodes_) {
      if (nd.op != "null" || nd.storage < 0) continue;
      auto in = input_.find(nd.name);
      if (in != input_.end()) { ptr_[nd.storage] = in->second; continue; }
      auto par = params_->by_name.find(nd.name);
      if (par != params_->by_name.end()) ptr_[nd.storage] = par->second;
    }
  }

  void Check(int rc, const Node& nd) const { if (rc != 0) throw std::runtime_error(nd.name + " (" + nd.op + "): device launch failed: " + api_.error_string(rc)); }

  // predict.h Run, on the handle's stream
  void Enqueue(int id) {
    const Predictor& p = *plan_;
    const Node& nd = p.nodes_[id];
    const std::string& op = nd.op;
    if (Predictor::IsView(nd)) return;
    if (nd.extended) { EnqueueExtended(nd); return; }
    const Attrs& a = nd.attrs;
    void* s = stream_;
    float* y = Ptr(nd);
    const long long n = Numel(nd.shape);
    const float* x = InPtr(nd, 0);
    const Shape& xs = In(nd, 0).shape;
    int k;
    if (op == "FullyConnected") {
      const Shape& w = In(nd, 1).shape;
      Check(api_.fc(x, InPtr(nd, 1), a.Bool("no_bias", false) ? nullptr : InPtr(nd, 2), y, static_cast<int>(n / w[0]), static_cast<int>(w[0]), static_cast<int>(w[1]), s), nd);
    } else if (op == "Convolution") {
      const Predictor::Conv c = p.ConvAttrs(nd);
      const Shape& w = In(nd, 1).shape;
      const float* wp = InPtr(nd, 1);
      long long ldw = w[1] * w[2] * w[3];
      auto pad = params_->conv_w.find(id);
      if (pad != params_->conv_w.end()) { wp = pad->second.first; ldw = pad->second.second; }
      Check(api_.conv(x, wp, ldw, a.Bool("no_bias", false) ? nullptr : InPtr(nd, 2), y, ws_, ws_floats_, (int)xs[0], (int)xs[1], (int)xs[2], (int)xs[3],
                      (int)nd.shape[1], (int)nd.shape[2], (int)nd.shape[3], (int)c.kh, (int)c.kw, (int)c.sh, (int)c.sw, (int)c.ph, (int)c.pw, (int)c.dh, (int)c.dw,
                      (int)c.groups, s), nd);
    } else if (op == "Pooling") {
      const Predictor::Pool q = p.PoolAttrs(nd, xs);
      Check(api_.pool(x, y, xs[0] * xs[1], (int)xs[2], (int)xs[3], (int)nd.shape[2], (int)nd.shape[3], (int)q.kh, (int)q.kw, (int)q.sh, (int)q.sw, (int)q.ph,
                      (int)q.pw, q.type, q.count_pad, s), nd);
    } else if (op == "Activation") {
      Check(api_.map(Predictor::UnaryKind(a.Str("act_type", "relu")), x, y, n, s), nd);
    } else if (op == "LeakyReLU") {
      Check(api_.pointwise(a.Str("act_type", "leaky") == "leaky" ? 0 : 1, x, y, n, static_cast<float>(a.Float("slope", 0.25)), 0.f, s), nd);
    } else if ((k = Predictor::UnaryKind(op)) >= 0) {
      Check(api_.map(k, x, y, n, s), nd);
    } else if (op == "clip") {
      const float lo = static_cast<float>(a.Float("a_min", -std::numeric_limits<float>::infinity())), hi = static_cast<float>(a.Float("a_max", std::numeric_limits<float>::infinity()));
      Check(api_.pointwise(2, x, y, n, lo, hi, s), nd);
    } else if (op == "LogisticRegressionOutput") {
      Check(api_.map(1, x, y, n, s), nd);
    } else if (op == "BatchNorm") {
      const int64_t ax = Predictor::Axis(a.Int("axis", 1), xs.size()), C = xs[ax];
      int64_t inner = 1; for (size_t i = ax + 1; i < xs.size(); ++i) inner *= xs[i];
      const auto& ss = params_->bn.at(id);
      Check(api_.affine(x, y, n, C, inner, ss.first, ss.second, s), nd);
    } else if (op == "Concat" || op == "concat") {
      const int64_t ax = Predictor::Axis(a.Int("dim", 1), nd.shape.size());
      int64_t inner = 1; for (size_t i = ax + 1; i < nd.shape.size(); ++i) inner *= nd.shape[i];
      const int64_t outer = n / (nd.shape[ax] * inner);
      int64_t at = 0;
      for (size_t j = 0; j < nd.inputs.size(); ++j) {
        const int64_t c = In(nd, j).shape[ax];
        Check(api_.concat_part(InPtr(nd, j), y, outer, c * inner, nd.shape[ax] * inner, at * inner, s), nd);
        at += c;
      }
    } else if (op == "softmax" || op == "log_softmax") {
      Softmax(nd, nd.shape, x, y, a.Int("axis", -1), op == "log_softmax");
    } else if (op == "SoftmaxOutput" || op == "Softmax") {
      Softmax(nd, nd.shape, x, y, nd.shape.size() < 2 ? 0 : (a.Bool("preserve_shape", false) ? -1 : 1), false);
    } else if (op == "SoftmaxActivation") {
      if (a.Str("mode", "instance") == "channel" || nd.shape.size() <= 2) Softmax(nd, nd.shape, x, y, nd.shape.size() < 2 ? 0 : 1, false);
      else Softmax(nd, Shape{nd.shape[0], n / nd.shape[0]}, x, y, 1, false);     // instance: over everything but the batch axis
    } else if (op == "transpose") {
      auto axes = a.Tuple("axes", {});
      const size_t r = xs.size();
      if (axes.empty()) for (size_t i = 0; i < r; ++i) axes.push_back(static_cast<int64_t>(r - 1 - i));
      std::vector<long long> xstride(r, 1), step(r), shape(nd.shape.begin(), nd.shape.end());
      for (int i = static_cast<int>(r) - 2; i >= 0; --i) xstride[i] = xstride[i + 1] * xs[i + 1];
      for (size_t i = 0; i < r; ++i) step[i] = xstride[Predictor::Axis(axes[i], r)];
      Check(api_.transpose(x, y, n, static_cast<int>(r), shape.data(), step.data(), s), nd);
    } else if (op == "Embedding") {
      const Shape& w = In(nd, 1).shape;
      Check(api_.embedding(x, InPtr(nd, 1), y, Numel(xs), w[0], w[1], s), nd);
    } else if ((k = Predictor::BinaryKind(op)) >= 0) {
      Binary(nd, k);
    } else if ((k = Predictor::ScalarKind(op)) >= 0) {
      Check(api_.pointwise(3 + k, x, y, n, static_cast<float>(a.Float("scalar", 0.0)), 0.f, s), nd);
    } else if (op == "add_n" || op == "ElementWiseSum") {
      std::vector<const float*> in;
      for (size_t j = 0; j < nd.inputs.size(); ++j) in.push_back(InPtr(nd, j));
      Check(api_.add_n(in.data(), static_cast<int>(in.size()), y, n, s), nd);
    } else {
      throw std::runtime_error("operator " + op + " has no device kernel");
    }
  }

  // predict.h RunBinary: operands broadcast over the output's axes
  void Binary(const Node& nd, int k) {
    const float* x = InPtr(nd, 0); float* y = Ptr(nd);
    const long long n = Numel(nd.shape);
    const Shape& ps = In(nd, 0).shape; const Shape& qs = In(nd, 1).shape;
    if (ps == qs) { Check(api_.binary(k, x, InPtr(nd, 1), y, n, 0, nullptr, nullptr, nullptr, stream_), nd); return; }
    const size_t r = nd.shape.size();
    std::vector<long long> sp(r, 0), sq(r, 0), shape(nd.shape.begin(), nd.shape.end());
    auto strides = [&](const Shape& sh, std::vector<long long>& out) {
      long long st = 1;
      for (int i = static_cast<int>(sh.size()) - 1; i >= 0; --i) { out[i + r - sh.size()] = sh[i] == 1 ? 0 : st; st *= sh[i]; }
    };
    strides(ps, sp); strides(qs, sq);
    Check(api_.binary(k, x, InPtr(nd, 1), y, n, static_cast<int>(r), shape.data(), sp.data(), sq.data(), stream_), nd);
  }

  // ---- the device-only set: train_exec.h Run's forward branches

  // the kernels take at most 8 axes and extents in 32 bits; Deconvolution indexes its furthest output row / column and its products in 32 bits
  void ValidateExtended(const Node& nd) const {
    const std::string& op = nd.op;
    std::vector<const Shape*> shapes{&nd.shape};
    for (size_t i = 0; i < nd.inputs.size(); ++i) shapes.push_back(&In(nd, i).shape);
    for (const Shape* sh : shapes) {
      if (sh->size() > 8) throw std::runtime_error(nd.name + ": the device kernels take at most 8 axes, got " + ShapeStr(*sh));
      for (int64_t d : *sh) Int(d, nd);
    }
    if (op == "Deconvolution") {
      const graph::detail::Win w = graph::detail::Window(extended::GraphNode(nd), false, In(nd, 0).shape);
      const Shape& xs = In(nd, 0).shape;
      const int64_t G = graph::AttrView(nd.sattrs).Int("num_group", 1);
      for (int64_t v : {w.kh, w.kw, w.sh, w.sw, w.ph, w.pw, w.dh, w.dw, G}) Int(v, nd);
      Int(nd.shape[2] + w.ph, nd); Int(nd.shape[3] + w.pw, nd);
      Int((w.kh - 1) * w.dh, nd); Int((w.kw - 1) * w.dw, nd);
      Int(xs[2] * xs[3], nd); Int(nd.shape[1] / G * w.kh * w.kw, nd);
    } else if (!(extended::IsGather(op) || extended::IsReduce(op) || extended::UnaryKind(op) >= 0 || extended::BinaryKind(op) >= 0 ||
                 extended::ScalarMode(op) >= 0 || op == "take" || op == "pick" || op == "one_hot" || op == "where" || op == "argmax" || op == "argmin" ||
                 op == "LayerNorm" || op == "InstanceNorm" || op == "L2Normalization" || op == "LRN" || op == "dot" || op == "smooth_l1" ||
                 op == "softmax_cross_entropy")) {
      throw std::runtime_error("operator " + op + " (node " + nd.name + ") has no device kernel");
    }
  }

  void EnqueueExtended(const Node& nd) {
    namespace D = graph::detail;
    const graph::AttrView a(nd.sattrs);
    const std::string& op = nd.op;
    void* s = stream_;
    float* y = Ptr(nd);
    const long long n = Numel(nd.shape);
    const float* x = InPtr(nd, 0);
    const Shape& xs = In(nd, 0).shape;
    int k;
    int64_t outer, C, inner;
    if (op == "SliceChannel") {
      for (int j = 0; j < nd.num_out; ++j) Gather(nd, j, j == 0 ? y : ptr_[nd.more_storage[j - 1]]);
    } else if (extended::IsGather(op)) {
      Gather(nd, 0, y);
    } else if (op == "take" || op == "pick") {
      extended::SplitAxis(xs, D::AxisOf(a.Int("axis", op == "take" ? 0 : -1), xs.size(), nd.name), &outer, &C, &inner);
      Check(api_.take(x, InPtr(nd, 1), y, outer, C, inner, op == "take" ? Numel(In(nd, 1).shape) : 0, s), nd);
    } else if (op == "one_hot") {
      Check(api_.one_hot(x, y, n, nd.shape.back(), static_cast<float>(a.Float("on_value", 1)), static_cast<float>(a.Float("off_value", 0)), s), nd);
    } else if (op == "where") {
      Check(api_.where(x, InPtr(nd, 1), InPtr(nd, 2), y, n, s), nd);
    } else if (op == "argmax" || op == "argmin") {
      extended::SplitAxis(xs, D::AxisOf(a.Int("axis", 0), xs.size(), nd.name), &outer, &C, &inner);
      Check(api_.arg(x, y, outer, C, inner, op == "argmax", s), nd);
    } else if (extended::IsReduce(op)) {
      const auto axes = a.Tuple("axis", {});
      std::vector<char> red(xs.size(), axes.empty());
      for (auto ax : axes) red[D::AxisOf(ax, xs.size(), nd.name)] = 1;
      std::vector<long long> kd, ks, rd, rs;
      long long st = 1;
      for (int i = static_cast<int>(xs.size()) - 1; i >= 0; --i) {
        (red[i] ? rd : kd).insert((red[i] ? rd : kd).begin(), xs[i]);
        (red[i] ? rs : ks).insert((red[i] ? rs : ks).begin(), st);
        st *= xs[i];
      }
      kd.insert(kd.end(), ks.begin(), ks.end()); rd.insert(rd.end(), rs.begin(), rs.end());
      const int kind = op == "max" ? 1 : op == "min" ? 2 : op == "prod" ? 3 : op == "norm" ? 4 : 0;
      const float div = op == "mean" ? static_cast<float>(Numel(xs) / n) : 1.f;
      Check(api_.reduce(kind, x, y, n, static_cast<int>(ks.size()), kd.data(), static_cast<int>(rs.size()), rd.data(), div, s), nd);
    } else if (op == "LayerNorm" || op == "InstanceNorm" || op == "L2Normalization") {
      int mode = 2;
      float eps = static_cast<float>(a.Float("eps", 1e-10));
      if (op == "LayerNorm") { mode = 0; eps = static_cast<float>(a.Float("eps", 1e-5)); extended::SplitAxis(xs, D::AxisOf(a.Int("axis", -1), xs.size(), nd.name), &outer, &C, &inner); }
      else if (op == "InstanceNorm") { mode = 1; eps = static_cast<float>(a.Float("eps", 1e-3)); outer = xs[0]; C = xs[1]; inner = Numel(xs) / (xs[0] * xs[1]); }
      else {                            // train_exec.h NormGroups
        const std::string m = a.Str("mode", "instance");
        const int64_t total = Numel(xs);
        if (m == "instance") { outer = xs[0]; C = total / xs[0]; inner = 1; }
        else if (m == "channel" && xs.size() >= 2) { outer = xs[0]; C = xs[1]; inner = total / (xs[0] * xs[1]); }
        else if (m == "spatial" && xs.size() >= 3) { outer = xs[0] * xs[1]; C = total / (xs[0] * xs[1]); inner = 1; }
        else throw std::runtime_error(nd.name + ": L2Normalization mode " + m + " is not supported for a tensor of shape " + ShapeStr(xs));
      }
      Check(api_.norm(mode, x, mode == 2 ? nullptr : InPtr(nd, 1), mode == 2 ? nullptr : InPtr(nd, 2), y, outer, C, inner, eps, s), nd);
    } else if (op == "LRN") {
      const int64_t ns = a.Int("nsize", 1);
      Check(api_.lrn(x, y, xs[0], xs[1], xs[2] * xs[3], ns / 2, static_cast<float>(a.Float("alpha", 1e-4)) / static_cast<float>(ns),
                     static_cast<float>(a.Float("beta", 0.75)), static_cast<float>(a.Float("knorm", 2)), s), nd);
    } else if (op == "Deconvolution") {
      const D::Win w = D::Window(extended::GraphNode(nd), false, xs);
      Check(api_.deconv(x, InPtr(nd, 1), nd.inputs.size() > 2 ? InPtr(nd, 2) : nullptr, y, ws_, ws_floats_, (int)xs[0], (int)xs[1], (int)xs[2], (int)xs[3],
                        (int)nd.shape[1], (int)nd.shape[2], (int)nd.shape[3], (int)w.kh, (int)w.kw, (int)w.sh, (int)w.sw, (int)w.ph, (int)w.pw, (int)w.dh,
                        (int)w.dw, (int)a.Int("num_group", 1), s), nd);
    } else if (op == "dot") {
      const bool ta = a.Bool("transpose_a", false), tb = a.Bool("transpose_b", false);
      Check(api_.dot(x, InPtr(nd, 1), y, (int)nd.shape[0], (int)nd.shape[1], (int)(ta ? xs[0] : xs[1]), ta, tb, s), nd);
    } else if (op == "smooth_l1") {
      const float sg = static_cast<float>(a.Float("scalar", 1));
      Check(api_.pointwise(13, x, y, n, sg * sg, 0.f, s), nd);
    } else if (op == "softmax_cross_entropy") {
      Check(api_.softmax_ce(x, InPtr(nd, 1), y, xs[0], xs[1], s), nd);
    } else if ((k = extended::UnaryKind(op)) >= 0) {
      Check(api_.map(k, x, y, n, s), nd);
    } else if ((k = extended::BinaryKind(op)) >= 0) {
      Binary(nd, k);
    } else if ((k = extended::ScalarMode(op)) >= 0) {
      Check(api_.pointwise(k, x, y, n, static_cast<float>(a.Float("scalar", 0)), 0.f, s), nd);
    } else {
      throw std::runtime_error("operator " + op + " has no device kernel");
    }
  }

  // train_exec.h BuildMap's per-axis rules as one gather launch; `part` is SliceChannel's output (its slice along the axis)
  void Gather(const Node& nd, int part, float* y) {
    namespace D = graph::detail;
    const graph::AttrView a(nd.sattrs);
    const std::string& op = nd.op;
    const Shape& xs = In(nd, 0).shape;
    Shape os = nd.shape;
    int64_t split_ax = -1;
    if (op == "SliceChannel") { split_ax = D::AxisOf(a.Int("axis", 1), xs.size(), nd.name); os = xs; os[split_ax] = xs[split_ax] / nd.num_out; }   // before squeeze_axis
    const size_t r = os.size();
    Shape in = xs; while (in.size() < r) in.insert(in.begin(), 1);
    std::vector<long long> stride(r, 1), off(r, 0), div(r, 1), before(r, 0), flags(r, 0), perm(r);
    for (int i = static_cast<int>(r) - 2; i >= 0; --i) stride[i] = stride[i + 1] * in[i + 1];
    for (size_t i = 0; i < r; ++i) perm[i] = static_cast<long long>(i);
    int pad_mode = -1;
    float fill = 0.f;
    if (op == "SliceChannel") {
      off[split_ax] = part * os[split_ax];
    } else if (op == "slice_axis") {
      const int64_t ax = D::AxisOf(a.Int("axis", 0), r, nd.name);
      int64_t lo, hi; D::SliceRange(a.Has("begin"), a.Int("begin", 0), a.Has("end"), a.Int("end", 0), in[ax], nd.name, &lo, &hi);
      off[ax] = lo;
    } else if (op == "slice") {
      const auto b = D::TupleOpt(a, "begin"), e = D::TupleOpt(a, "end");
      for (size_t i = 0; i < b.size(); ++i) { int64_t lo, hi; D::SliceRange(b[i].first, b[i].second, e[i].first, e[i].second, in[i], nd.name, &lo, &hi); off[i] = lo; }
    } else if (op == "SwapAxis") {
      std::swap(perm[D::AxisOf(a.Int("dim1", 0), r, nd.name)], perm[D::AxisOf(a.Int("dim2", 0), r, nd.name)]);
    } else if (op == "tile") {
      for (size_t i = 0; i < r; ++i) flags[i] = 1;
    } else if (op == "repeat") {
      div[D::AxisOf(a.Int("axis", 0), r, nd.name)] = a.Int("repeats", 1);
    } else if (op == "UpSampling") {
      div[2] = div[3] = a.Int("scale", 1);
    } else if (op == "reverse") {
      for (auto ax : a.Tuple("axis", {})) flags[D::AxisOf(ax, r, nd.name)] = 2;
    } else if (op == "broadcast_to" || op == "broadcast_axis") {
      for (size_t i = 0; i < r; ++i) flags[i] = in[i] == 1 && os[i] != 1 ? 4 : 0;
    } else if (op == "Pad") {
      const auto pw = a.Tuple("pad_width", {});
      for (size_t i = 0; i < r; ++i) before[i] = pw[2 * i];
      const std::string mode = a.Str("mode", "constant");
      pad_mode = mode == "constant" ? 0 : mode == "edge" ? 1 : 2;
      fill = static_cast<float>(a.Float("constant_value", 0));
    }
    std::vector<long long> rule;
    for (auto* row : {&os, &in}) rule.insert(rule.end(), row->begin(), row->end());
    for (size_t i = 0; i < r; ++i) rule.push_back(stride[perm[i]]);
    for (auto* row : {&before, &div, &off, &flags}) rule.insert(rule.end(), row->begin(), row->end());
    Check(api_.gather(InPtr(nd, 0), y, Numel(os), static_cast<int>(r), rule.data(), pad_mode, fill, stream_), nd);
  }

  // predict.h Softmax: (outer, C, inner) around `axis` of `shape`
  void Softmax(const Node& nd, const Shape& shape, const float* x, float* y, int64_t axis, bool log) {
    const int64_t ax = Predictor::Axis(axis, shape.size()), C = shape[ax];
    int64_t inner = 1; for (size_t i = ax + 1; i < shape.size(); ++i) inner *= shape[i];
    const int64_t outer = Numel(shape) / (C * inner);
    Check(api_.softmax(x, y, outer, C, inner, log ? 1 : 0, stream_), nd);
  }
};

}  // namespace predict
}  // namespace gxrt
