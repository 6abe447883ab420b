// The planned predictor on an H100 (GXPredCreate* with dev_type 2): predict.h's graph, shape inference and liveness-planned arena, run as
// sm_90a kernels (kernels/predict_dev.cu).
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
    sym(a->conv, "gx_pred_conv");
    if (!missing.empty()) return path + " has no entry point " + missing + " (an older build?)";
    return "";
  }
};

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
    api_.Check(api_.d2h(out, ptr_[n.storage], size * sizeof(float), stream_), "GetOutput: device-to-host copy");
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
  const float* InPtr(const Node& nd, size_t i) const { return ptr_[In(nd, i).storage]; }
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
      if (Predictor::IsView(op)) continue;
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
      if (nd.op != "Convolution") continue;
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
    if (Predictor::IsView(op)) return;
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
      const Shape& ps = In(nd, 0).shape; const Shape& qs = In(nd, 1).shape;
      if (ps == qs) { Check(api_.binary(k, x, InPtr(nd, 1), y, n, 0, nullptr, nullptr, nullptr, s), nd); return; }
      const size_t r = nd.shape.size();
      std::vector<long long> sp(r, 0), sq(r, 0), shape(nd.shape.begin(), nd.shape.end());
      auto strides = [&](const Shape& sh, std::vector<long long>& out) {
        long long st = 1;
        for (int i = static_cast<int>(sh.size()) - 1; i >= 0; --i) { out[i + r - sh.size()] = sh[i] == 1 ? 0 : st; st *= sh[i]; }
      };
      strides(ps, sp); strides(qs, sq);
      Check(api_.binary(k, x, InPtr(nd, 1), y, n, static_cast<int>(r), shape.data(), sp.data(), sq.data(), s), nd);
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
