// Fused optimizer / elementwise kernels for sm_90a.
//
// Reference: SGD / SGD-momentum / Adam / DCASGD and the other element-wise rules are 1-3 mshadow MapPlanKernel passes *per parameter*
// (src/operator/optimizer_op-inl.h:86-103,305-326,840-873; DCASGD python/mxnet/optimizer/optimizer.py:872-925), driven by a
// Python loop.  Here:
//   * arena_* : ONE launch updates a whole flat parameter arena (all keys), 128-bit accesses, with the step counter and
//     Adam bias correction kept ON THE DEVICE so the launch is CUDA-graph replayable (no host scalar changes per step).
//     Per-key lr/wd multipliers come from a per-tile table (tile = 1024 floats; keys are tile-aligned in the arena).
//   * multi_tensor_* : one launch over a pointer table (Trainer path for tensors that do not live in an arena).
//   * n-ary sum (CommDevice reduce), scale+cast (the script-level `grad / num_samples` and `.astype('float16')`).
// The update rules themselves (OptHyper, opt_elem / opt_apply4, sched_lr / step_lr) are in optim.cuh, shared with the HiPS fabric kernels.
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include "optim.cuh"

namespace gx {

constexpr int ARENA_TILE = 1024;

// step_state[0] = number of completed updates t, step_state[1] = CTA completion counter (self-resetting)
template <int KIND, bool SCHED>
__global__ void __launch_bounds__(256) arena_opt_kernel(float* __restrict__ w, const float* __restrict__ g, float* __restrict__ s0, float* __restrict__ s1,
                                                         long long n, const float2* __restrict__ tile_mult, OptHyper h, int* __restrict__ step_state,
                                                         float* __restrict__ g_zero) {
  gx::pdl_wait();
  gx::pdl_launch();
  h.kind = KIND;  // a compile-time kind: step_lr and opt_apply4 reduce to this kernel's rule
  const int t = step_state ? (*reinterpret_cast<volatile int*>(step_state)) + 1 : 1;
  const float lr_t = step_lr<SCHED>(h, t);
  const long long n4 = n >> 2;  // arenas are tile-padded, n % 1024 == 0
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    float lr = lr_t, wd = h.wd;
    if (tile_mult) { const float2 m = __ldg(tile_mult + (i * 4) / ARENA_TILE); lr *= m.x; wd *= m.y; }
    float4 W = reinterpret_cast<float4*>(w)[i];
    const float4 G = reinterpret_cast<const float4*>(g)[i];
    float4 A = s0 ? reinterpret_cast<float4*>(s0)[i] : make_float4(0, 0, 0, 0);
    float4 Bv = s1 ? reinterpret_cast<float4*>(s1)[i] : make_float4(0, 0, 0, 0);
    opt_apply4<(KIND > OPT_DCASGD)>(W, G, A, Bv, h, lr, wd);
    reinterpret_cast<float4*>(w)[i] = W;
    if (s0) reinterpret_cast<float4*>(s0)[i] = A;
    if (s1) reinterpret_cast<float4*>(s1)[i] = Bv;
    if (g_zero) reinterpret_cast<float4*>(g_zero)[i] = make_float4(0, 0, 0, 0);  // fused zero_grad for the next step
  }
  if (step_state) {
    __syncthreads();
    if (threadIdx.x == 0) {
      __threadfence();
      const int done = atomicAdd(step_state + 1, 1);
      if (done == (int)gridDim.x - 1) {  // every other CTA has already read t
        step_state[1] = 0;
        step_state[0] = t;
        __threadfence();
      }
    }
  }
}

struct TensorEntry { float* w; const float* g; float* s0; float* s1; long long n; float lr_mult, wd_mult; };

template <int KIND>
__global__ void __launch_bounds__(256) multi_tensor_opt_kernel(const TensorEntry* __restrict__ table, OptHyper h, float lr_t) {
  gx::pdl_wait();
  gx::pdl_launch();
  const TensorEntry e = table[blockIdx.y];
  const float lr = lr_t * e.lr_mult, wd = h.wd * e.wd_mult;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < e.n; i += (long long)gridDim.x * blockDim.x) {
    float W = e.w[i], A = e.s0 ? e.s0[i] : 0.f, Bv = e.s1 ? e.s1[i] : 0.f;
    opt_elem<KIND>(W, e.g[i], A, Bv, h, lr, wd);
    e.w[i] = W;
    if (e.s0) e.s0[i] = A;
    if (e.s1) e.s1[i] = Bv;
  }
}

template <int KIND>
__global__ void __launch_bounds__(256) single_opt_kernel(float* __restrict__ w, const float* __restrict__ g, float* __restrict__ s0, float* __restrict__ s1,
                                                          long long n, OptHyper h, float lr_t) {
  gx::pdl_wait();
  gx::pdl_launch();
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    float W = w[i], A = s0 ? s0[i] : 0.f, Bv = s1 ? s1[i] : 0.f;
    opt_elem<KIND>(W, g[i], A, Bv, h, lr_t, h.wd);
    w[i] = W;
    if (s0) s0[i] = A;
    if (s1) s1[i] = Bv;
  }
}

struct PtrList8 { const float* p[8]; };
__global__ void __launch_bounds__(256) nary_sum_kernel(float* __restrict__ out, PtrList8 in, int cnt, long long n) {
  gx::pdl_wait();
  gx::pdl_launch();
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    float acc = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j)
      if (j < cnt) acc += in.p[j][i];
    out[i] = acc;
  }
}

template <typename T> __device__ __forceinline__ T cvt(float v);
template <> __device__ __forceinline__ float cvt<float>(float v) { return v; }
template <> __device__ __forceinline__ __half cvt<__half>(float v) { return __float2half_rn(v); }
template <> __device__ __forceinline__ __nv_bfloat16 cvt<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }
template <typename T> __device__ __forceinline__ float up(T v);
template <> __device__ __forceinline__ float up<float>(float v) { return v; }
template <> __device__ __forceinline__ float up<__half>(__half v) { return __half2float(v); }
template <> __device__ __forceinline__ float up<__nv_bfloat16>(__nv_bfloat16 v) { return __bfloat162float(v); }

template <typename TI, typename TO>
__global__ void __launch_bounds__(256) scale_cast_kernel(const TI* __restrict__ x, TO* __restrict__ y, float scale, long long n) {
  gx::pdl_wait();
  gx::pdl_launch();
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) y[i] = cvt<TO>(up<TI>(x[i]) * scale);
}

static inline int grid_for(long long n, int per_thread = 1) {
  long long b = (n / per_thread + 255) / 256;
  if (b < 1) b = 1;
  if (b > 148 * 8) b = 148 * 8;
  return (int)b;
}

}  // namespace gx

using namespace gx;

static OptHyper mk(int kind, float lr, float wd, float rescale, float clip, float momentum, float b1, float b2, float eps, float lamda) {
  OptHyper h{};   // the fields of the later kinds 0; sched SCHED_NONE: the constant lr
  h.lr = lr; h.wd = wd; h.rescale = rescale; h.clip = clip; h.momentum = momentum; h.beta1 = b1; h.beta2 = b2; h.eps = eps; h.lamda = lamda;
  h.kind = kind;
  return h;
}

// one case per OptKind: the kernels are instantiated per kind, so that each instance compiles to its own rule only
#define GX_OPT_DISPATCH(kind, LAUNCH)                     \
  switch (kind) {                                         \
    case OPT_SGD: LAUNCH(OPT_SGD); break;                 \
    case OPT_ADAM: LAUNCH(OPT_ADAM); break;               \
    case OPT_DCASGD: LAUNCH(OPT_DCASGD); break;           \
    case OPT_NAG: LAUNCH(OPT_NAG); break;                 \
    case OPT_SIGNUM: LAUNCH(OPT_SIGNUM); break;           \
    case OPT_RMSPROP: LAUNCH(OPT_RMSPROP); break;         \
    case OPT_ADAGRAD: LAUNCH(OPT_ADAGRAD); break;         \
    case OPT_ADADELTA: LAUNCH(OPT_ADADELTA); break;       \
    case OPT_FTRL: LAUNCH(OPT_FTRL); break;               \
    default: return -1;                                   \
  }

// The entry points that take a packed OptHyper (ops/_native_api.py pack_hyper): every kind and all of its hyper-parameters.  The
// schedule travels inside it (h.sched).  n must be a multiple of 4 (arenas are 1024-padded).  step_state: int[2] device or null.
GX_API int gx_arena_opt_h(const void* hyper, float* w, const float* g, float* s0, float* s1, long long n, const void* tile_mult,
                          int* step_state, float* g_zero, cudaStream_t s) {
  const OptHyper h = *reinterpret_cast<const OptHyper*>(hyper);
  const int grid = grid_for(n, 4);
  const float2* tm = reinterpret_cast<const float2*>(tile_mult);
  const bool sched = h.sched.kind != SCHED_NONE;   // the constant-lr or the scheduled instance (step_lr<SCHED>)
#define GX_ARENA(K) launch_pdl(sched ? arena_opt_kernel<K, true> : arena_opt_kernel<K, false>, dim3(grid), dim3(256), 0, s, w, g, s0, s1, n, tm, h, \
                               step_state, g_zero)
  GX_OPT_DISPATCH(h.kind, GX_ARENA)
#undef GX_ARENA
  return GX_CHECK_LAUNCH();
}

// lr_t: the step's lr (Adam: bias-corrected), the same for every tensor; tensors scale it by their lr_mult
GX_API int gx_multi_tensor_opt_h(const void* hyper, const void* table, int num_tensors, long long max_n, float lr_t, cudaStream_t s) {
  const OptHyper h = *reinterpret_cast<const OptHyper*>(hyper);
  int gx_ = grid_for(max_n); if (gx_ > 64) gx_ = 64;
  dim3 grid(gx_, num_tensors);
  const TensorEntry* t = reinterpret_cast<const TensorEntry*>(table);
#define GX_MT(K) launch_pdl(multi_tensor_opt_kernel<K>, dim3(grid), dim3(256), 0, s, t, h, lr_t)
  GX_OPT_DISPATCH(h.kind, GX_MT)
#undef GX_MT
  return GX_CHECK_LAUNCH();
}

GX_API int gx_single_opt_h(const void* hyper, float* w, const float* g, float* s0, float* s1, long long n, float lr_t, cudaStream_t s) {
  const OptHyper h = *reinterpret_cast<const OptHyper*>(hyper);
  const int grid = grid_for(n);
#define GX_SINGLE(K) launch_pdl(single_opt_kernel<K>, dim3(grid), dim3(256), 0, s, w, g, s0, s1, n, h, lr_t)
  GX_OPT_DISPATCH(h.kind, GX_SINGLE)
#undef GX_SINGLE
  return GX_CHECK_LAUNCH();
}

// The positional entry points of SGD / Adam / DCASGD (kind 0 / 1 / 2).  schedule: a host LrSchedule (lr is its base lr), or null for a
// constant lr.
GX_API int gx_arena_opt(int kind, float* w, const float* g, float* s0, float* s1, long long n, const void* tile_mult, float lr, float wd,
                        float rescale, float clip, float momentum, float b1, float b2, float eps, float lamda, int* step_state, float* g_zero,
                        const void* schedule, cudaStream_t s) {
  OptHyper h = mk(kind, lr, wd, rescale, clip, momentum, b1, b2, eps, lamda);
  if (schedule) h.sched = *reinterpret_cast<const LrSchedule*>(schedule);
  return gx_arena_opt_h(&h, w, g, s0, s1, n, tile_mult, step_state, g_zero, s);
}

GX_API int gx_multi_tensor_opt(int kind, const void* table, int num_tensors, long long max_n, float lr_t, float wd, float rescale, float clip,
                               float momentum, float b1, float b2, float eps, float lamda, cudaStream_t s) {
  const OptHyper h = mk(kind, lr_t, wd, rescale, clip, momentum, b1, b2, eps, lamda);
  return gx_multi_tensor_opt_h(&h, table, num_tensors, max_n, lr_t, s);
}

GX_API int gx_single_opt(int kind, float* w, const float* g, float* s0, float* s1, long long n, float lr_t, float wd, float rescale, float clip,
                         float momentum, float b1, float b2, float eps, float lamda, cudaStream_t s) {
  const OptHyper h = mk(kind, lr_t, wd, rescale, clip, momentum, b1, b2, eps, lamda);
  return gx_single_opt_h(&h, w, g, s0, s1, n, lr_t, s);
}

GX_API int gx_nary_sum(float* out, const float* const* inputs, int cnt, long long n, cudaStream_t s) {
  if (cnt < 1 || cnt > 8) return -1;
  PtrList8 l;
  for (int i = 0; i < 8; ++i) l.p[i] = i < cnt ? inputs[i] : nullptr;
  launch_pdl(nary_sum_kernel, dim3(grid_for(n)), dim3(256), 0, s, out, l, cnt, n);
  return GX_CHECK_LAUNCH();
}

// dtype codes: 0 fp32, 1 fp16, 2 bf16
GX_API int gx_scale_cast(const void* x, int in_dt, void* y, int out_dt, float scale, long long n, cudaStream_t s) {
  const int grid = grid_for(n);
#define GX_SC(TI, TO) launch_pdl(scale_cast_kernel<TI, TO>, dim3(grid), dim3(256), 0, s, reinterpret_cast<const TI*>(x), reinterpret_cast<TO*>(y), scale, n)
  if (in_dt == 0 && out_dt == 0) GX_SC(float, float);
  else if (in_dt == 0 && out_dt == 1) GX_SC(float, __half);
  else if (in_dt == 0 && out_dt == 2) GX_SC(float, __nv_bfloat16);
  else if (in_dt == 1 && out_dt == 0) GX_SC(__half, float);
  else if (in_dt == 2 && out_dt == 0) GX_SC(__nv_bfloat16, float);
  else if (in_dt == 1 && out_dt == 1) GX_SC(__half, __half);
  else if (in_dt == 2 && out_dt == 2) GX_SC(__nv_bfloat16, __nv_bfloat16);
  else return -1;
#undef GX_SC
  return GX_CHECK_LAUNCH();
}
