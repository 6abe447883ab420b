// Device side of the C predict API's planned predictor (runtime: csrc/runtime/predict_device.h, host interpreter: predict.h).
//
// One forward kernel per operator family that predict.h's Run and, for the device-only set, train_exec.h's Executor::Run dispatch on, each written to give what the host loop gives, edge cases
// included (Pooling windows clipped to the padded plane, empty max windows = 0, Embedding indices converted and clamped as the host does),
// plus the `gx_pred_*` entry points the runtime reaches through dlopen: device / memory / stream / graph helpers, so that
// libgeomx_capi.so itself never links the CUDA runtime.
//
// Convolution and FullyConnected products go through the wgmma GEMM (gemm_wgmma.cu) at 3xTF32, whatever gx_gemm_set_precision says, with
// its bias and NCHW-scatter epilogues; operands that miss TMA alignment go to its fp32 CUDA-core twin.  Convolution: im2col with groups
// and dilation for a chunk of images into the caller's workspace, then one product per chunk (groups == 1) or per image and group; a 1x1,
// stride-1, unpadded convolution multiplies the input planes directly (MN-major A operand), with no column matrix.
//
// Every kernel follows the library's launch convention (common.cuh): pdl_wait() / pdl_launch() first, launched through launch_pdl, so in the
// handle's CUDA graph each kernel's prologue overlaps the tail of the one before and the shared-memory carve-out stays the GEMM's.
//
// Every entry point returns 0 or a cudaError_t value; shapes arrive validated by the runtime, so no kernel checks them.
#include <cuda.h>

#include <cmath>
#include <cstdint>

#include "common.cuh"

GX_API int gx_gemm_tf32_prec(const float* A, long long lda, int a_mn, const float* B, long long ldb, int b_mn, int M, int N, int K, float* D,
                             long long ldd, const float* bias, const float* mask, long long ldmask, float* colsum, int relu, int accumulate,
                             int store_mode, int hw, float alpha, int split_k, int precision, cudaStream_t stream);
GX_API int gx_gemm_simt(const float* A, long long lda, int a_mn, const float* B, long long ldb, int b_mn, int M, int N, int K, float* D,
                        long long ldd, const float* bias, const float* mask, long long ldmask, float* colsum, int relu, int accumulate,
                        int store_mode, int hw, float alpha, cudaStream_t stream);

namespace gx {
namespace pred {

constexpr int kThreads = 256;
constexpr int kMaxRank = 8;
constexpr int kMaxSum = 8;
// the column matrix of one convolution chunk holds at most this many floats (or one image's, if that is larger)
constexpr long long kConvChunkFloats = 16ll << 20;

inline unsigned blocks_for(long long n) {
  const long long b = (n + kThreads - 1) / kThreads;
  return (unsigned)(b < 1 ? 1 : (b > 65535ll * 16 ? 65535ll * 16 : b));
}

struct Strides {
  int rank;
  long long shape[kMaxRank];
  long long a[kMaxRank];
  long long b[kMaxRank];
};
struct Ptrs { const float* p[kMaxSum]; };

// the host's Act(): relu, sigmoid, tanh, exp, log, sqrt, abs, negative, square, softsign, softrelu; then (11..30) the general executor's
// remaining unary kinds, train_exec.h Un(): sin ... sign
__device__ __forceinline__ float act(int kind, float v) {
  switch (kind) {
    case 0: return v > 0 ? v : 0.f;
    case 1: return 1.f / (1.f + expf(-v));
    case 2: return tanhf(v);
    case 3: return expf(v);
    case 4: return logf(v);
    case 5: return sqrtf(v);
    case 6: return fabsf(v);
    case 7: return -v;
    case 8: return v * v;
    case 9: return v / (1.f + fabsf(v));
    case 10: return v > 20.f ? v : log1pf(expf(v));
    case 11: return sinf(v);
    case 12: return cosf(v);
    case 13: return tanf(v);
    case 14: return asinf(v);
    case 15: return acosf(v);
    case 16: return atanf(v);
    case 17: return sinhf(v);
    case 18: return coshf(v);
    case 19: return log1pf(v);
    case 20: return expm1f(v);
    case 21: return log2f(v);
    case 22: return log10f(v);
    case 23: return 1.f / sqrtf(v);
    case 24: return 1.f / v;
    case 25: return cbrtf(v);
    case 26: return erff(v);
    case 27: return floorf(v);
    case 28: return ceilf(v);
    case 29: return roundf(v);
    default: return v > 0 ? 1.f : v < 0 ? -1.f : 0.f;
  }
}
// std::max / std::min: the first argument wins ties and unordered pairs
__device__ __forceinline__ float smax(float a, float b) { return a < b ? b : a; }
__device__ __forceinline__ float smin(float a, float b) { return b < a ? b : a; }

// 6..12: the general executor's power and comparisons (1.0 / 0.0)
__device__ __forceinline__ float bin(int k, float p, float q) {
  switch (k) {
    case 0: return p + q; case 1: return p - q; case 2: return p * q; case 3: return p / q; case 4: return smax(p, q); case 5: return smin(p, q);
    case 6: return powf(p, q); case 7: return p == q; case 8: return p != q; case 9: return p > q; case 10: return p >= q; case 11: return p < q;
    default: return p <= q;
  }
}

__global__ void __launch_bounds__(kThreads) map_kernel(int kind, const float* x, float* y, long long n) {
  pdl_wait();
  pdl_launch();
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) y[i] = act(kind, x[i]);
}

// mode 0 leaky, 1 elu, 2 clip (a = lo, b = hi), 3..8 scalar ops (+, -, *, /, s - x, s / x with a = s), 9 x ** s, 10 s ** x, 11 max(x, s),
// 12 min(x, s), 13 smooth_l1 with a = sigma^2
__global__ void __launch_bounds__(kThreads) pointwise_kernel(int mode, const float* x, float* y, long long n, float a, float b) {
  pdl_wait();
  pdl_launch();
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const float v = x[i];
    float r;
    switch (mode) {
      case 0: r = v > 0 ? v : a * v; break;
      case 1: r = v > 0 ? v : a * (expf(v) - 1.f); break;
      case 2: r = smin(smax(v, a), b); break;
      case 3: r = v + a; break;
      case 4: r = v - a; break;
      case 5: r = v * a; break;
      case 6: r = v / a; break;
      case 7: r = a - v; break;
      case 8: r = a / v; break;
      case 9: r = powf(v, a); break;
      case 10: r = powf(a, v); break;
      case 11: r = smax(v, a); break;
      case 12: r = smin(v, a); break;
      default: { const float m = fabsf(v); r = m < 1.f / a ? 0.5f * a * m * m : m - 0.5f / a; break; }
    }
    y[i] = r;
  }
}

// BatchNorm at inference: per-channel scale and shift, computed once by the runtime with the host's formula
__global__ void __launch_bounds__(kThreads) affine_kernel(const float* x, float* y, long long n, long long C, long long inner, const float* scale,
                                                          const float* shift) {
  pdl_wait();
  pdl_launch();
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const long long c = (i / inner) % C;
    y[i] = x[i] * scale[c] + shift[c];
  }
}

__global__ void __launch_bounds__(kThreads) binary_same_kernel(int k, const float* p, const float* q, float* y, long long n) {
  pdl_wait();
  pdl_launch();
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) y[i] = bin(k, p[i], q[i]);
}

// broadcast: st.a / st.b are the operands' strides over the output's axes (0 where an operand has extent 1)
__global__ void __launch_bounds__(kThreads) binary_bcast_kernel(int k, const float* p, const float* q, float* y, long long n, Strides st) {
  pdl_wait();
  pdl_launch();
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    long long r = i, ip = 0, iq = 0;
    for (int d = st.rank - 1; d >= 0; --d) {
      const long long c = r % st.shape[d];
      r /= st.shape[d];
      ip += c * st.a[d]; iq += c * st.b[d];
    }
    y[i] = bin(k, p[ip], q[iq]);
  }
}

// transpose: st.a = the input stride that each output axis walks
__global__ void __launch_bounds__(kThreads) transpose_kernel(const float* x, float* y, long long n, Strides st) {
  pdl_wait();
  pdl_launch();
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    long long r = i, src = 0;
    for (int d = st.rank - 1; d >= 0; --d) { const long long c = r % st.shape[d]; r /= st.shape[d]; src += c * st.a[d]; }
    y[i] = x[src];
  }
}

// add_n in the host's order: y = x0 + x1 + ... left to right; `cont` continues a sum that y already holds
__global__ void __launch_bounds__(kThreads) sum_kernel(Ptrs in, int count, int cont, float* y, long long n) {
  pdl_wait();
  pdl_launch();
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    float acc = cont ? y[i] : in.p[0][i];
#pragma unroll
    for (int j = 0; j < kMaxSum; ++j)
      if (j >= 1 - cont && j < count) acc += in.p[j][i];
    y[i] = acc;
  }
}

// one Concat input: `rows` blocks of `len` values land at `at` inside blocks of `ld`
__global__ void __launch_bounds__(kThreads) concat_kernel(const float* p, float* y, long long rows, long long len, long long ld, long long at) {
  pdl_wait();
  pdl_launch();
  const long long n = rows * len;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const long long o = i / len, r = i - o * len;
    y[o * ld + at + r] = p[i];
  }
}

// softmax / log_softmax over axis C of an (outer, C, inner) view: one warp per (outer, inner) row.  Host formula: max in fp32, the sum of
// exp(x - max) in fp64, lse rounded to fp32, y = exp(x - max - lse) (or the exponent itself for log_softmax).  Each term is expf rounded
// to fp32 before the fp64 sum (the fp64 exp's slow path would spill): a relative difference of ~1e-7 in the sum.
__global__ void __launch_bounds__(kThreads) softmax_kernel(const float* x, float* y, long long rows, long long C, long long inner, int log_out) {
  pdl_wait();
  pdl_launch();
  const int lane = threadIdx.x & 31;
  const long long warps = (long long)gridDim.x * (kThreads / 32);
  for (long long r = blockIdx.x * (long long)(kThreads / 32) + (threadIdx.x >> 5); r < rows; r += warps) {
    const long long o = r / inner, in = r - o * inner;
    const float* px = x + o * C * inner + in;
    float* py = y + o * C * inner + in;
    float m = -INFINITY;
    for (long long c = lane; c < C; c += 32) m = smax(m, px[c * inner]);
    for (int s = 16; s; s >>= 1) m = smax(m, __shfl_xor_sync(0xffffffffu, m, s));
    double sum = 0;
    for (long long c = lane; c < C; c += 32) sum += (double)expf(px[c * inner] - m);
    for (int s = 16; s; s >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, s);
    const float lse = (float)log(sum);
    for (long long c = lane; c < C; c += 32) { const float v = px[c * inner] - m - lse; py[c * inner] = log_out ? v : expf(v); }
  }
}

// Embedding: the index is the float converted the way the host's static_cast<int64_t> does on x86-64 (truncation; NaN and values outside
// the int64 range give INT64_MIN), then clamped to [0, rows - 1]
__global__ void __launch_bounds__(kThreads) embedding_kernel(const float* idx, const float* w, float* y, long long n_idx, long long rows, long long dim) {
  pdl_wait();
  pdl_launch();
  const long long n = n_idx * dim;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const long long t = i / dim, d = i - t * dim;
    const float v = idx[t];
    long long r = (v >= -9223372036854775808.f && v < 9223372036854775808.f) ? (long long)v : (long long)(1ull << 63);
    r = r < 0 ? 0 : (r > rows - 1 ? rows - 1 : r);
    y[i] = w[r * dim + d];
  }
}

// Pooling, one thread per output value, exactly the host loop: the window is clipped to the padded plane, then to the input; max over an
// empty window is 0; avg divides by the padded window (count_include_pad) or by the values it covers
__global__ void __launch_bounds__(kThreads) pool_kernel(const float* x, float* y, long long planes, int H, int W, int OH, int OW, int kh, int kw, int sh,
                                                        int sw, int ph, int pw, int type, int count_pad) {
  pdl_wait();
  pdl_launch();
  const long long n = planes * OH * OW;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const long long pl = i / ((long long)OH * OW);
    const int pix = (int)(i - pl * OH * OW), oh = pix / OW, ow = pix - oh * OW;
    const float* src = x + pl * H * W;
    const long long h0 = (long long)oh * sh - ph, w0 = (long long)ow * sw - pw;
    const long long h1 = h0 + kh < (long long)H + ph ? h0 + kh : (long long)H + ph, w1 = w0 + kw < (long long)W + pw ? w0 + kw : (long long)W + pw;
    const long long hs = h0 > 0 ? h0 : 0, ws = w0 > 0 ? w0 : 0, he = h1 < H ? h1 : H, we = w1 < W ? w1 : W;
    float acc = type == 0 ? -INFINITY : 0.f;
    for (long long h = hs; h < he; ++h)
      for (long long w = ws; w < we; ++w) { const float v = src[h * W + w]; acc = type == 0 ? smax(acc, v) : acc + v; }
    if (type == 1) {
      const long long cnt = count_pad ? (h1 - h0) * (w1 - w0) : (he - hs) * (we - ws);
      acc /= (float)(cnt > 1 ? cnt : 1);
    }
    if (type == 0 && (he <= hs || we <= ws)) acc = 0.f;
    y[i] = acc;
  }
}

// ---- the general executor's operators (train_exec.h Run), device-only

// float -> int64 as the host's static_cast<int64_t> does on x86-64 (truncation; NaN and values outside the int64 range give INT64_MIN)
__device__ __forceinline__ long long to_index(float v) {
  return (v >= -9223372036854775808.f && v < 9223372036854775808.f) ? (long long)v : (long long)(1ull << 63);
}
__device__ __forceinline__ long long clamp_index(float v, long long n) {
  const long long r = to_index(v);
  return r < 0 ? 0 : (r > n - 1 ? n - 1 : r);
}

// the per-axis index rules of train_exec.h BuildMap for the layout operators (slice, SwapAxis, tile, repeat, Pad, reverse, broadcast,
// UpSampling, SliceChannel's parts), over the output's axes
struct GatherRule {
  int rank;
  int pad_mode;                   // -1 none, 0 constant (fill), 1 edge, 2 reflect
  float fill;
  long long shape[kMaxRank];      // output extent
  long long in[kMaxRank];         // input extent (the input padded with leading 1s to the output's rank)
  long long stride[kMaxRank];     // input stride that this output axis walks (SwapAxis: of the swapped axis)
  long long before[kMaxRank];     // Pad: leading pad
  long long div[kMaxRank];        // repeat / UpSampling factor
  long long off[kMaxRank];        // slice begin
  int flags[kMaxRank];            // 1 wrap (tile), 2 flip (reverse), 4 broadcast
};

__global__ void __launch_bounds__(kThreads) gather_kernel(const float* x, float* y, long long n, GatherRule g) {
  pdl_wait();
  pdl_launch();
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    long long r = i, src = 0;
    bool constant = false;
    for (int d = g.rank - 1; d >= 0; --d) {
      long long v = r % g.shape[d];
      r /= g.shape[d];
      const long long in = g.in[d];
      if (g.pad_mode >= 0) {
        v -= g.before[d];
        if (v < 0 || v >= in) {
          if (g.pad_mode == 0) constant = true;
          v = g.pad_mode == 1 ? (v < 0 ? 0 : in - 1) : (v < 0 ? -v : 2 * (in - 1) - v);
        }
      }
      v = v / g.div[d] + g.off[d];
      const int f = g.flags[d];
      if (f & 1) v %= in;
      if (f & 2) v = in - 1 - v;
      if (f & 4) v = 0;
      src += v * g.stride[d];
    }
    y[i] = constant ? g.fill : x[src];
  }
}

// take: (outer, ni, inner) <- (outer, C, inner) at row idx[j]; pick (ni = 0): (outer, inner) <- row idx[o * inner + i]
__global__ void __launch_bounds__(kThreads) take_kernel(const float* x, const float* idx, float* y, long long outer, long long C, long long inner,
                                                        long long ni) {
  pdl_wait();
  pdl_launch();
  const long long rows = ni > 0 ? ni : 1, n = outer * rows * inner;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const long long in = i % inner, t = i / inner, j = t % rows, o = t / rows;
    const long long r = clamp_index(idx[ni > 0 ? j : o * inner + in], C);
    y[i] = x[(o * C + r) * inner + in];
  }
}

__global__ void __launch_bounds__(kThreads) one_hot_kernel(const float* idx, float* y, long long n, long long depth, float on, float off) {
  pdl_wait();
  pdl_launch();
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    y[i] = to_index(idx[i / depth]) == i % depth ? on : off;
}

__global__ void __launch_bounds__(kThreads) where_kernel(const float* c, const float* t, const float* f, float* y, long long n) {
  pdl_wait();
  pdl_launch();
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) y[i] = c[i] != 0.f ? t[i] : f[i];
}

// argmax / argmin over the middle axis of (outer, C, inner): the first index of a strict extreme, as the host's loop
__global__ void __launch_bounds__(kThreads) arg_kernel(const float* x, float* y, long long outer, long long C, long long inner, int is_max) {
  pdl_wait();
  pdl_launch();
  const long long n = outer * inner;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const long long o = i / inner, in = i - o * inner;
    const float* p = x + o * C * inner + in;
    long long best = 0;
    float bv = p[0];
    for (long long k = 1; k < C; ++k) {
      const float v = p[k * inner];
      if (is_max ? v > bv : v < bv) { best = k; bv = v; }
    }
    y[i] = (float)best;
  }
}

// reductions, one block per output value: thread t folds the reduced elements t, t + 256, ... in order, then a fixed tree over the block's
// partials, so a replay gives the same bits.  Accumulation is in fp64, as the host's (train_exec.h): a sum that cancels keeps its
// relative accuracy.  kind 0 sum (divided by `div`: mean), 1 max, 2 min, 3 prod, 4 L2 norm.  st.a: the input strides of the kept axes
// (st.shape their extents), red: the reduced axes'.
__device__ __forceinline__ double fold(int kind, double acc, double v) {
  switch (kind) { case 1: return acc < v ? v : acc; case 2: return v < acc ? v : acc; case 3: return acc * v; case 4: return acc + v * v; default: return acc + v; }
}
__device__ __forceinline__ double combine(int kind, double a, double b) { return kind == 4 ? a + b : fold(kind, a, b); }
__global__ void __launch_bounds__(kThreads) reduce_kernel(int kind, const float* x, float* y, long long ny, Strides st, Strides red, long long nred, float div) {
  pdl_wait();
  pdl_launch();
  __shared__ double part[kThreads];
  const double init = kind == 1 ? -INFINITY : kind == 2 ? INFINITY : kind == 3 ? 1.0 : 0.0;
  for (long long o = blockIdx.x; o < ny; o += gridDim.x) {
    long long r = o, base = 0;
    for (int d = st.rank - 1; d >= 0; --d) { base += (r % st.shape[d]) * st.a[d]; r /= st.shape[d]; }
    double acc = init;
    for (long long k = threadIdx.x; k < nred; k += kThreads) {
      long long q = k, off = base;
      for (int d = red.rank - 1; d >= 0; --d) { off += (q % red.shape[d]) * red.a[d]; q /= red.shape[d]; }
      acc = fold(kind, acc, (double)x[off]);
    }
    part[threadIdx.x] = acc;
    __syncthreads();
    for (int s = kThreads / 2; s; s >>= 1) {
      if ((int)threadIdx.x < s) part[threadIdx.x] = combine(kind, part[threadIdx.x], part[threadIdx.x + s]);
      __syncthreads();
    }
    if (threadIdx.x == 0) { const double v = part[0]; y[o] = (float)(kind == 4 ? sqrt(v) : kind == 0 ? v / (double)div : v); }
    __syncthreads();
  }
}

// LayerNorm (mode 0: statistics over C per (outer, inner), gamma / beta by c), InstanceNorm (1: over inner per (outer, c), gamma / beta by
// c) and L2Normalization (2: y = x / sqrt(sum x^2 + eps) over C per (outer, inner)), one warp per group, two passes over the group
__global__ void __launch_bounds__(kThreads) norm_kernel(int mode, const float* x, const float* gamma, const float* beta, float* y, long long outer,
                                                        long long C, long long inner, float eps) {
  pdl_wait();
  pdl_launch();
  const int lane = threadIdx.x & 31;
  const long long warps = (long long)gridDim.x * (kThreads / 32);
  const long long groups = mode == 1 ? outer * C : outer * inner, len = mode == 1 ? inner : C;
  for (long long g = blockIdx.x * (long long)(kThreads / 32) + (threadIdx.x >> 5); g < groups; g += warps) {
    const long long base = mode == 1 ? g * inner : (g / inner) * C * inner + g % inner, step = mode == 1 ? 1 : inner;
    const float* px = x + base;
    float* py = y + base;
    float sum = 0.f;
    for (long long k = lane; k < len; k += 32) sum += mode == 2 ? px[k * step] * px[k * step] : px[k * step];
    for (int s = 16; s; s >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, s);
    if (mode == 2) {
      const float nrm = sqrtf(sum + eps);
      for (long long k = lane; k < len; k += 32) py[k * step] = px[k * step] / nrm;
      continue;
    }
    const float mean = sum / (float)len;
    float sq = 0.f;
    for (long long k = lane; k < len; k += 32) { const float d = px[k * step] - mean; sq += d * d; }
    for (int s = 16; s; s >>= 1) sq += __shfl_xor_sync(0xffffffffu, sq, s);
    const float inv = 1.f / sqrtf(sq / (float)len + eps);
    for (long long k = lane; k < len; k += 32) {
      const long long c = mode == 0 ? k : g % C;
      py[k * step] = (px[k * step] - mean) * inv * gamma[c] + beta[c];
    }
  }
}

// LRN across channels of NCHW, the host's loop: the window's squares summed in fp32 in channel order
__global__ void __launch_bounds__(kThreads) lrn_kernel(const float* x, float* y, long long N, long long C, long long P, long long half, float alpha,
                                                       float beta, float knorm) {
  pdl_wait();
  pdl_launch();
  const long long n = N * C * P;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const long long p = i % P, t = i / P, c = t % C, b = t / C;
    const long long k0 = c - half < 0 ? 0 : c - half, k1 = c + half < C - 1 ? c + half : C - 1;
    float sq = 0.f;
    for (long long k = k0; k <= k1; ++k) { const float v = x[(b * C + k) * P + p]; sq += v * v; }
    y[i] = x[i] * powf(knorm + alpha * sq, -beta);
  }
}

// softmax_cross_entropy of (N, C) against labels: one block; each row's -log p[label] in fp64, the rows summed in a fixed tree
__global__ void __launch_bounds__(kThreads) softmax_ce_kernel(const float* x, const float* label, float* y, long long N, long long C) {
  pdl_wait();
  pdl_launch();
  __shared__ double part[kThreads];
  double acc = 0;
  for (long long i = threadIdx.x; i < N; i += kThreads) {
    const float* p = x + i * C;
    float m = p[0];
    for (long long k = 1; k < C; ++k) m = smax(m, p[k]);
    float z = 0.f;
    for (long long k = 0; k < C; ++k) z += expf(p[k] - m);
    const float q = expf(p[clamp_index(label[i], C)] - m) / z;
    acc -= log((double)smax(q, 1e-30f));
  }
  part[threadIdx.x] = acc;
  __syncthreads();
  for (int s = kThreads / 2; s; s >>= 1) {
    if ((int)threadIdx.x < s) part[threadIdx.x] += part[threadIdx.x + s];
    __syncthreads();
  }
  if (threadIdx.x == 0) y[0] = (float)part[0];
}

// Deconvolution's input rows for one chunk of images: xt[(image, pixel)][c] = x[b0 + image][c][pixel], row stride ldx
__global__ void __launch_bounds__(kThreads) rows_kernel(const float* x, float* xt, long long ldx, int nb, int b0, int C, long long P) {
  pdl_wait();
  pdl_launch();
  const long long n = (long long)nb * C * P;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const long long p = i % P, t = i / P, c = t % C, bl = t / C;
    xt[(bl * P + p) * ldx + c] = x[(long long)b0 * C * P + i];
  }
}

// Deconvolution's col2im in gather form, no atomics: y[b][g*Fg + f][oy][ox] = bias + the sum over the window taps (r, s) that land on it of
// col_g[(b, iy * W + ix)][(f * kh + r) * kw + s], col_g being the chunk's x_g^T . W_g with row stride ldc, one matrix per group
__global__ void __launch_bounds__(kThreads) col2im_kernel(const float* col, long long ldc, const float* bias, float* y, int nb, int b0, int groups, int Fg,
                                                          int H, int W, int OH, int OW, int kh, int kw, int sh, int sw, int ph, int pw, int dh, int dw) {
  pdl_wait();
  pdl_launch();
  const long long F = (long long)groups * Fg, P = (long long)H * W, n = (long long)nb * F * OH * OW;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const int ox = (int)(i % OW), oy = (int)((i / OW) % OH);
    const long long t = i / ((long long)OH * OW), fo = t % F, bl = t / F;
    const int g = (int)(fo / Fg), f = (int)(fo - (long long)g * Fg);
    const float* c = col + ((long long)g * nb + bl) * P * ldc;
    float acc = 0.f;
    for (int r = 0; r < kh; ++r) {
      const int ty = oy + ph - r * dh;
      if (ty < 0 || ty % sh) continue;
      const int iy = ty / sh;
      if (iy >= H) continue;
      for (int s = 0; s < kw; ++s) {
        const int tx = ox + pw - s * dw;
        if (tx < 0 || tx % sw) continue;
        const int ix = tx / sw;
        if (ix >= W) continue;
        acc += c[((long long)iy * W + ix) * ldc + ((long long)f * kh + r) * kw + s];
      }
    }
    y[(long long)b0 * F * OH * OW + i] = acc + (bias ? bias[fo] : 0.f);
  }
}

// im2col of images [b0, b0 + nb) for channel group g: col[(image, oh, ow)][(ci, i, j)] with row stride ldc (>= K, a multiple of 4 for TMA)
__global__ void __launch_bounds__(kThreads) im2col_kernel(const float* x, float* col, long long ldc, int nb, int b0, int C, int H, int W, int OH, int OW,
                                                          int cg, int g, int kh, int kw, int sh, int sw, int ph, int pw, int dh, int dw) {
  pdl_wait();
  pdl_launch();
  const long long K = (long long)cg * kh * kw, P = (long long)OH * OW, n = (long long)nb * P * K;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const long long m = i / K, k = i - m * K;
    const long long bl = m / P;
    const int p = (int)(m - bl * P), oh = p / OW, ow = p - oh * OW;
    const int ci = (int)(k / (kh * kw)), r = (int)(k - (long long)ci * kh * kw), ki = r / kw, kj = r - ki * kw;
    const int ih = oh * sh - ph + ki * dh, iw = ow * sw - pw + kj * dw;
    float v = 0.f;
    if (ih >= 0 && ih < H && iw >= 0 && iw < W) v = x[((((long long)(b0 + bl)) * C + (long long)g * cg + ci) * H + ih) * W + iw];
    col[m * ldc + k] = v;
  }
}

}  // namespace pred
}  // namespace gx

using namespace gx::pred;
using gx::launch_pdl;

// D = A . B^T (+ bias), fp32-accurate: the wgmma kernel at 3xTF32, or the CUDA-core kernel when the wgmma path declines the operands.
// gx_gemm_tf32_prec returns a negative code for every refusal before its launch (-1 TMA alignment, -2 no tensor-map encoder, -(1000 + r)
// a CUresult r from cuTensorMapEncodeTiled) and a cudaError_t from the launch itself; only the latter is an error here.
static int gemm_fp32(const float* A, long long lda, int a_mn, const float* B, long long ldb, int M, int N, int K, float* D, long long ldd,
                     const float* bias, int store_mode, int hw, cudaStream_t s, int b_mn = 0) {
  const int rc = gx_gemm_tf32_prec(A, lda, a_mn, B, ldb, b_mn, M, N, K, D, ldd, bias, nullptr, 0, nullptr, 0, 0, store_mode, hw, 1.f, 1, 3, s);
  if (rc >= 0) return rc;
  return gx_gemm_simt(A, lda, a_mn, B, ldb, b_mn, M, N, K, D, ldd, bias, nullptr, 0, nullptr, 0, 0, store_mode, hw, 1.f, s);
}

// a launch's own error, else whatever an earlier call left behind
static int launched(int rc) { return rc != 0 ? rc : (int)cudaGetLastError(); }

// ------------------------------------------------------------------------------------------------ device, memory, streams, graphs
GX_API int gx_pred_device_count(int* n) { *n = 0; return (int)cudaGetDeviceCount(n); }
GX_API int gx_pred_device_cc(int dev, int* major, int* minor) {
  int rc = (int)cudaDeviceGetAttribute(major, cudaDevAttrComputeCapabilityMajor, dev);
  if (rc == 0) rc = (int)cudaDeviceGetAttribute(minor, cudaDevAttrComputeCapabilityMinor, dev);
  return rc;
}
// *has_context: whether the calling thread has a current CUDA context (cudaGetDevice reports 0 for a thread that never chose a device)
GX_API int gx_pred_get_device(int* dev, int* has_context) {
  typedef CUresult (*GetCurrent)(CUcontext*);
  static GetCurrent get_current = [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    return (cudaGetDriverEntryPoint("cuCtxGetCurrent", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
               ? reinterpret_cast<GetCurrent>(p) : nullptr;
  }();
  CUcontext ctx = nullptr;
  *has_context = (get_current != nullptr && get_current(&ctx) == CUDA_SUCCESS && ctx != nullptr) ? 1 : 0;
  return (int)cudaGetDevice(dev);
}
GX_API int gx_pred_set_device(int dev) { return (int)cudaSetDevice(dev); }
GX_API const char* gx_pred_error_string(int rc) { return cudaGetErrorString((cudaError_t)rc); }
GX_API int gx_pred_malloc(void** p, size_t bytes) { *p = nullptr; return (int)cudaMalloc(p, bytes); }
GX_API int gx_pred_free(void* p) { return (int)cudaFree(p); }
GX_API int gx_pred_h2d(void* dst, const void* src, size_t bytes, void* s) { return (int)cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, (cudaStream_t)s); }
GX_API int gx_pred_d2h(void* dst, const void* src, size_t bytes, void* s) { return (int)cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, (cudaStream_t)s); }
GX_API int gx_pred_memset(void* dst, size_t bytes, void* s) { return (int)cudaMemsetAsync(dst, 0, bytes, (cudaStream_t)s); }
GX_API int gx_pred_stream_create(void** s) { return (int)cudaStreamCreateWithFlags(reinterpret_cast<cudaStream_t*>(s), cudaStreamNonBlocking); }
GX_API int gx_pred_stream_destroy(void* s) { return (int)cudaStreamDestroy((cudaStream_t)s); }
GX_API int gx_pred_stream_sync(void* s) { return (int)cudaStreamSynchronize((cudaStream_t)s); }
// relaxed capture: the GEMM's host side may query attributes while the stream records
GX_API int gx_pred_capture_begin(void* s) { return (int)cudaStreamBeginCapture((cudaStream_t)s, cudaStreamCaptureModeRelaxed); }
// ends the capture that gx_pred_capture_begin started and instantiates it; *exec stays null when either step fails
GX_API int gx_pred_capture_end(void* s, void** exec) {
  *exec = nullptr;
  cudaGraph_t g = nullptr;
  int rc = (int)cudaStreamEndCapture((cudaStream_t)s, &g);
  if (rc == 0) rc = (int)cudaGraphInstantiate(reinterpret_cast<cudaGraphExec_t*>(exec), g, 0);
  if (g) cudaGraphDestroy(g);
  if (rc != 0) { cudaGetLastError(); *exec = nullptr; }
  return rc;
}
GX_API int gx_pred_graph_launch(void* exec, void* s) { return (int)cudaGraphLaunch((cudaGraphExec_t)exec, (cudaStream_t)s); }
GX_API int gx_pred_graph_destroy(void* exec) { return (int)cudaGraphExecDestroy((cudaGraphExec_t)exec); }

// ------------------------------------------------------------------------------------------------ operators
GX_API int gx_pred_map(int kind, const float* x, float* y, long long n, void* s) {
  return launched(launch_pdl(map_kernel, dim3(blocks_for(n)), dim3(kThreads), 0, (cudaStream_t)s, kind, x, y, n));
}
GX_API int gx_pred_pointwise(int mode, const float* x, float* y, long long n, float a, float b, void* s) {
  return launched(launch_pdl(pointwise_kernel, dim3(blocks_for(n)), dim3(kThreads), 0, (cudaStream_t)s, mode, x, y, n, a, b));
}
GX_API int gx_pred_affine(const float* x, float* y, long long n, long long C, long long inner, const float* scale, const float* shift, void* s) {
  return launched(launch_pdl(affine_kernel, dim3(blocks_for(n)), dim3(kThreads), 0, (cudaStream_t)s, x, y, n, C, inner, scale, shift));
}
// sp / sq: the operands' strides over the output axes, null when both operands have the output's shape
GX_API int gx_pred_binary(int kind, const float* p, const float* q, float* y, long long n, int rank, const long long* shape, const long long* sp,
                          const long long* sq, void* s) {
  if (sp == nullptr) {
    return launched(launch_pdl(binary_same_kernel, dim3(blocks_for(n)), dim3(kThreads), 0, (cudaStream_t)s, kind, p, q, y, n));
  }
  if (rank > kMaxRank) return (int)cudaErrorInvalidValue;
  Strides st{};
  st.rank = rank;
  for (int d = 0; d < rank; ++d) { st.shape[d] = shape[d]; st.a[d] = sp[d]; st.b[d] = sq[d]; }
  return launched(launch_pdl(binary_bcast_kernel, dim3(blocks_for(n)), dim3(kThreads), 0, (cudaStream_t)s, kind, p, q, y, n, st));
}
GX_API int gx_pred_transpose(const float* x, float* y, long long n, int rank, const long long* out_shape, const long long* step, void* s) {
  if (rank > kMaxRank) return (int)cudaErrorInvalidValue;
  Strides st{};
  st.rank = rank;
  for (int d = 0; d < rank; ++d) { st.shape[d] = out_shape[d]; st.a[d] = step[d]; }
  return launched(launch_pdl(transpose_kernel, dim3(blocks_for(n)), dim3(kThreads), 0, (cudaStream_t)s, x, y, n, st));
}
GX_API int gx_pred_add_n(const float* const* in, int count, float* y, long long n, void* s) {
  for (int j0 = 0; j0 < count; j0 += kMaxSum) {
    Ptrs p{};
    const int c = count - j0 < kMaxSum ? count - j0 : kMaxSum;
    for (int j = 0; j < c; ++j) p.p[j] = in[j0 + j];
    const int rc = launched(launch_pdl(sum_kernel, dim3(blocks_for(n)), dim3(kThreads), 0, (cudaStream_t)s, p, c, j0 > 0, y, n));
    if (rc) return rc;
  }
  return 0;
}
GX_API int gx_pred_concat_part(const float* p, float* y, long long rows, long long len, long long ld, long long at, void* s) {
  return launched(launch_pdl(concat_kernel, dim3(blocks_for(rows * len)), dim3(kThreads), 0, (cudaStream_t)s, p, y, rows, len, ld, at));
}
GX_API int gx_pred_softmax(const float* x, float* y, long long outer, long long C, long long inner, int log_out, void* s) {
  const long long rows = outer * inner;
  return launched(launch_pdl(softmax_kernel, dim3(blocks_for(rows * 32)), dim3(kThreads), 0, (cudaStream_t)s, x, y, rows, C, inner, log_out));
}
GX_API int gx_pred_embedding(const float* idx, const float* w, float* y, long long n_idx, long long rows, long long dim, void* s) {
  return launched(launch_pdl(embedding_kernel, dim3(blocks_for(n_idx * dim)), dim3(kThreads), 0, (cudaStream_t)s, idx, w, y, n_idx, rows, dim));
}
GX_API int gx_pred_pool(const float* x, float* y, long long planes, int H, int W, int OH, int OW, int kh, int kw, int sh, int sw, int ph, int pw, int type,
                        int count_pad, void* s) {
  return launched(launch_pdl(pool_kernel, dim3(blocks_for(planes * OH * OW)), dim3(kThreads), 0, (cudaStream_t)s, x, y, planes, H, W, OH, OW, kh, kw,
                             sh, sw, ph, pw, type, count_pad));
}
// y[M, N] = x[M, K] . w[N, K]^T (+ bias)
GX_API int gx_pred_fc(const float* x, const float* w, const float* bias, float* y, int M, int N, int K, void* s) {
  return gemm_fp32(x, K, 0, w, K, M, N, K, y, N, bias, 0, 1, (cudaStream_t)s);
}
// floats of workspace gx_pred_conv needs: one chunk of column matrix (none for a 1x1 / stride-1 / unpadded convolution)
GX_API long long gx_pred_conv_workspace(int B, int C, int OH, int OW, int kh, int kw, int groups, int pointwise) {
  if (pointwise) return 0;
  const long long per_image = (long long)OH * OW * ((C / groups * kh * kw + 3) / 4 * 4);
  long long nb = kConvChunkFloats / per_image;
  nb = nb < 1 ? 1 : (nb > B ? B : nb);
  return nb * per_image;
}
// NCHW convolution; w is [F][C / groups * kh * kw] with row stride ldw
GX_API int gx_pred_conv(const float* x, const float* w, long long ldw, const float* bias, float* y, float* ws, long long ws_floats, int B, int C, int H,
                        int W, int F, int OH, int OW, int kh, int kw, int sh, int sw, int ph, int pw, int dh, int dw, int groups, void* sv) {
  cudaStream_t s = (cudaStream_t)sv;
  const int cg = C / groups, fg = F / groups, K = cg * kh * kw, P = OH * OW;
  const bool pointwise = kh == 1 && kw == 1 && sh == 1 && sw == 1 && ph == 0 && pw == 0;
  int rc = 0;
  if (pointwise) {   // A = the image's input planes of the group, [K = cg][M = P] (MN-major)
    for (int b = 0; b < B && !rc; ++b)
      for (int g = 0; g < groups && !rc; ++g)
        rc = gemm_fp32(x + ((long long)b * C + (long long)g * cg) * P, P, 1, w + (long long)g * fg * ldw, ldw, P, fg, K,
                       y + ((long long)b * F + (long long)g * fg) * P, 0, bias ? bias + g * fg : nullptr, 1, P, s);
    return rc;
  }
  const long long ldc = (K + 3) / 4 * 4, per_image = (long long)P * ldc;
  long long nb = ws_floats / per_image;
  if (nb < 1) return (int)cudaErrorInvalidValue;
  if (nb > B) nb = B;
  for (int b0 = 0; b0 < B && !rc; b0 += (int)nb) {
    const int n = (int)(B - b0 < nb ? B - b0 : nb);
    for (int g = 0; g < groups && !rc; ++g) {
      rc = launched(launch_pdl(im2col_kernel, dim3(blocks_for((long long)n * P * K)), dim3(kThreads), 0, s, x, ws, ldc, n, b0, C, H, W, OH, OW, cg, g,
                               kh, kw, sh, sw, ph, pw, dh, dw));
      if (rc) break;
      if (groups == 1) {   // rows (image, pixel) of the whole chunk, scattered to NCHW by the epilogue
        rc = gemm_fp32(ws, ldc, 0, w, ldw, n * P, F, K, y + (long long)b0 * F * P, 0, bias, 1, P, s);
      } else {             // one product per image: the scatter epilogue's image stride is N * hw, here F * P
        for (int bl = 0; bl < n && !rc; ++bl)
          rc = gemm_fp32(ws + (long long)bl * P * ldc, ldc, 0, w + (long long)g * fg * ldw, ldw, P, fg, K,
                         y + ((long long)(b0 + bl) * F + (long long)g * fg) * P, 0, bias ? bias + g * fg : nullptr, 1, P, s);
      }
    }
  }
  return rc;
}

// ------------------------------------------------------------------------------------------------ the general executor's operators
// rule: 7 rows of `rank` values each: output extent, input extent, input stride, Pad's leading pad, divisor, offset, flags (1 wrap, 2 flip,
// 4 broadcast); pad_mode -1 none, 0 constant (fill), 1 edge, 2 reflect
GX_API int gx_pred_gather(const float* x, float* y, long long n, int rank, const long long* rule, int pad_mode, float fill, void* s) {
  if (rank < 1 || rank > kMaxRank) return (int)cudaErrorInvalidValue;
  GatherRule g{};
  g.rank = rank; g.pad_mode = pad_mode; g.fill = fill;
  for (int d = 0; d < rank; ++d) {
    g.shape[d] = rule[d]; g.in[d] = rule[rank + d]; g.stride[d] = rule[2 * rank + d]; g.before[d] = rule[3 * rank + d];
    g.div[d] = rule[4 * rank + d]; g.off[d] = rule[5 * rank + d]; g.flags[d] = (int)rule[6 * rank + d];
  }
  return launched(launch_pdl(gather_kernel, dim3(blocks_for(n)), dim3(kThreads), 0, (cudaStream_t)s, x, y, n, g));
}
// take (ni = the number of indices) and pick (ni = 0)
GX_API int gx_pred_take(const float* x, const float* idx, float* y, long long outer, long long C, long long inner, long long ni, void* s) {
  const long long n = outer * (ni > 0 ? ni : 1) * inner;
  return launched(launch_pdl(take_kernel, dim3(blocks_for(n)), dim3(kThreads), 0, (cudaStream_t)s, x, idx, y, outer, C, inner, ni));
}
GX_API int gx_pred_one_hot(const float* idx, float* y, long long n, long long depth, float on, float off, void* s) {
  return launched(launch_pdl(one_hot_kernel, dim3(blocks_for(n)), dim3(kThreads), 0, (cudaStream_t)s, idx, y, n, depth, on, off));
}
GX_API int gx_pred_where(const float* c, const float* t, const float* f, float* y, long long n, void* s) {
  return launched(launch_pdl(where_kernel, dim3(blocks_for(n)), dim3(kThreads), 0, (cudaStream_t)s, c, t, f, y, n));
}
GX_API int gx_pred_arg(const float* x, float* y, long long outer, long long C, long long inner, int is_max, void* s) {
  return launched(launch_pdl(arg_kernel, dim3(blocks_for(outer * inner)), dim3(kThreads), 0, (cudaStream_t)s, x, y, outer, C, inner, is_max));
}
// keep / red: extents then input strides of the kept and the reduced axes (rank_keep may be 0: one output value)
GX_API int gx_pred_reduce(int kind, const float* x, float* y, long long ny, int rank_keep, const long long* keep, int rank_red, const long long* red,
                          float div, void* s) {
  if (rank_keep < 0 || rank_keep > kMaxRank || rank_red < 1 || rank_red > kMaxRank) return (int)cudaErrorInvalidValue;
  Strides k{}, r{};
  k.rank = rank_keep; r.rank = rank_red;
  long long nred = 1;
  for (int d = 0; d < rank_keep; ++d) { k.shape[d] = keep[d]; k.a[d] = keep[rank_keep + d]; }
  for (int d = 0; d < rank_red; ++d) { r.shape[d] = red[d]; r.a[d] = red[rank_red + d]; nred *= red[d]; }
  const unsigned grid = (unsigned)(ny < 65535ll * 16 ? ny : 65535ll * 16);
  return launched(launch_pdl(reduce_kernel, dim3(grid), dim3(kThreads), 0, (cudaStream_t)s, kind, x, y, ny, k, r, nred, div));
}
GX_API int gx_pred_norm(int mode, const float* x, const float* gamma, const float* beta, float* y, long long outer, long long C, long long inner, float eps,
                        void* s) {
  const long long groups = mode == 1 ? outer * C : outer * inner;
  return launched(launch_pdl(norm_kernel, dim3(blocks_for(groups * 32)), dim3(kThreads), 0, (cudaStream_t)s, mode, x, gamma, beta, y, outer, C, inner, eps));
}
GX_API int gx_pred_lrn(const float* x, float* y, long long N, long long C, long long P, long long half, float alpha, float beta, float knorm, void* s) {
  return launched(launch_pdl(lrn_kernel, dim3(blocks_for(N * C * P)), dim3(kThreads), 0, (cudaStream_t)s, x, y, N, C, P, half, alpha, beta, knorm));
}
GX_API int gx_pred_softmax_ce(const float* x, const float* label, float* y, long long N, long long C, void* s) {
  return launched(launch_pdl(softmax_ce_kernel, dim3(1), dim3(kThreads), 0, (cudaStream_t)s, x, label, y, N, C));
}
// y[M, N] = op(a) . op(b) for 2-D row-major operands: a is [M, K] or, transposed, [K, M]; b is [K, N] or, transposed, [N, K]
GX_API int gx_pred_dot(const float* a, const float* b, float* y, int M, int N, int K, int ta, int tb, void* s) {
  return gemm_fp32(a, ta ? M : K, ta, b, tb ? K : N, M, N, K, y, N, nullptr, 0, 1, (cudaStream_t)s, tb ? 0 : 1);
}
// floats of workspace gx_pred_deconv needs per image: the input rows and the column matrices of every group
static long long deconv_per_image(int C, int H, int W, int Fg, int kh, int kw, int groups) {
  return (long long)H * W * (((long long)C + 3) / 4 * 4 + (long long)groups * (((long long)Fg * kh * kw + 3) / 4 * 4));
}
// floats of workspace gx_pred_deconv needs: one chunk of images
GX_API long long gx_pred_deconv_workspace(int B, int C, int H, int W, int Fg, int kh, int kw, int groups) {
  const long long per_image = deconv_per_image(C, H, W, Fg, kh, kw, groups);
  long long nb = kConvChunkFloats / per_image;
  nb = nb < 1 ? 1 : (nb > B ? B : nb);
  return nb * per_image;
}
// NCHW transposed convolution; w is [C][F / groups][kh][kw].  Per chunk of images: the input as rows (image, pixel) of C values, then per
// group one product col_g[(image, pixel)][Fg*kh*kw] = x_g^T . W_g over the whole chunk (the weight rows as an MN-major B), then the
// gather-form col2im with the bias.
GX_API int gx_pred_deconv(const float* x, const float* w, const float* bias, float* y, float* ws, long long ws_floats, int B, int C, int H, int W, int F,
                          int OH, int OW, int kh, int kw, int sh, int sw, int ph, int pw, int dh, int dw, int groups, void* sv) {
  cudaStream_t s = (cudaStream_t)sv;
  const int cg = C / groups, fg = F / groups, K = fg * kh * kw, P = H * W;
  const long long ldc = (K + 3) / 4 * 4, ldx = (C + 3) / 4 * 4, per_image = deconv_per_image(C, H, W, fg, kh, kw, groups);
  long long nb = ws_floats / per_image;
  if (nb < 1) return (int)cudaErrorInvalidValue;
  if (nb > B) nb = B;
  float* xt = ws + nb * groups * P * ldc;
  int rc = 0;
  for (int b0 = 0; b0 < B && !rc; b0 += (int)nb) {
    const int n = (int)(B - b0 < nb ? B - b0 : nb);
    rc = launched(launch_pdl(rows_kernel, dim3(blocks_for((long long)n * C * P)), dim3(kThreads), 0, s, x, xt, ldx, n, b0, C, (long long)P));
    for (int g = 0; g < groups && !rc; ++g)
      rc = gemm_fp32(xt + (long long)g * cg, ldx, 0, w + (long long)g * cg * K, K, n * P, K, cg, ws + (long long)g * n * P * ldc, ldc, nullptr, 0, 1, s, 1);
    if (!rc)
      rc = launched(launch_pdl(col2im_kernel, dim3(blocks_for((long long)n * F * OH * OW)), dim3(kThreads), 0, s, ws, ldc, bias, y, n, b0, groups, fg, H, W,
                               OH, OW, kh, kw, sh, sw, ph, pw, dh, dw));
  }
  return rc;
}
