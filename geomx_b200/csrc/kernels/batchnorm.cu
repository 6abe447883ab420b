// BatchNorm forward / backward for sm_90a (NCHW or [N,C]).
// Reference: src/operator/nn/batch_norm.cu:247-470 (grid = #channels, warp-shuffle reductions :150), running-stat convention
// running = momentum*running + (1-momentum)*batch  (:262-266, population variance :355-362).
//
// Two forms.  Feature maps (N*HW >= 4096, HW >= 16) are bandwidth problems and use the SPLIT form: a statistics kernel on a (channel, slice)
// grid that fills the machine (one pass over x: sum and sum of squares of x minus a per-channel pivot per thread in fp32, combined across
// CTAs with fp64 atomics; the CTA that draws the last ticket of a channel finalises mean / inv-std / running statistics and re-arms the
// accumulators), then an apply kernel that
// streams every (image, channel) plane with 128-bit accesses.  x is read twice and y written once — 3 passes at HBM rate instead of the 4
// strided passes of a one-CTA-per-channel kernel.
// Small problems (Dense + BN, tiny maps) keep the one-CTA-per-channel kernels: they are latency-bound and one launch beats two.
#include <mutex>

#include "common.cuh"

namespace gx {

__device__ __forceinline__ float block_sum(float v, float* red) {
  v = warp_sum(v);
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  __syncthreads();
  if (lane == 0) red[wid] = v;
  __syncthreads();
  float s = 0.f;
  const int nw = blockDim.x >> 5;
  for (int j = 0; j < nw; ++j) s += red[j];
  return s;
}

__global__ void __launch_bounds__(512) bn_fwd_kernel(const float* __restrict__ x, const float* __restrict__ gamma, const float* __restrict__ beta,
                                                      float* __restrict__ running_mean, float* __restrict__ running_var, float* __restrict__ y,
                                                      float* __restrict__ save_mean, float* __restrict__ save_invstd, int N, int C, int HW,
                                                      int training, float momentum, float eps) {
  gx::pdl_wait();
  gx::pdl_launch();
  __shared__ float red[16];
  const int c = blockIdx.x;
  const long long cnt = (long long)N * HW;
  float mean, invstd;
  if (training) {
    float s = 0.f;
    for (long long i = threadIdx.x; i < cnt; i += blockDim.x) s += x[((i / HW) * C + c) * HW + i % HW];
    mean = block_sum(s, red) / (float)cnt;
    float q = 0.f;
    for (long long i = threadIdx.x; i < cnt; i += blockDim.x) {
      const float d = x[((i / HW) * C + c) * HW + i % HW] - mean;
      q = fmaf(d, d, q);
    }
    const float var = block_sum(q, red) / (float)cnt;
    invstd = rsqrtf(var + eps);
    if (threadIdx.x == 0) {
      running_mean[c] = momentum * running_mean[c] + (1.f - momentum) * mean;
      running_var[c] = momentum * running_var[c] + (1.f - momentum) * var;
      save_mean[c] = mean;
      save_invstd[c] = invstd;
    }
  } else {
    mean = running_mean[c];
    invstd = rsqrtf(running_var[c] + eps);
  }
  const float g = gamma ? gamma[c] : 1.f, b = beta ? beta[c] : 0.f;
  const float a = g * invstd, off = b - mean * a;
  for (long long i = threadIdx.x; i < cnt; i += blockDim.x) {
    const long long o = ((i / HW) * C + c) * HW + i % HW;
    y[o] = fmaf(x[o], a, off);
  }
}

__global__ void __launch_bounds__(512) bn_bwd_kernel(const float* __restrict__ x, const float* __restrict__ dy, const float* __restrict__ gamma,
                                                      const float* __restrict__ save_mean, const float* __restrict__ save_invstd,
                                                      float* __restrict__ dx, float* __restrict__ dgamma, float* __restrict__ dbeta, int N, int C, int HW,
                                                      int fixed_stats) {
  gx::pdl_wait();
  gx::pdl_launch();
  __shared__ float red[16];
  const int c = blockIdx.x;
  const long long cnt = (long long)N * HW;
  const float mean = save_mean[c], invstd = save_invstd[c];
  float sdy = 0.f, sdyx = 0.f;
  for (long long i = threadIdx.x; i < cnt; i += blockDim.x) {
    const long long o = ((i / HW) * C + c) * HW + i % HW;
    const float g = dy[o];
    sdy += g;
    sdyx = fmaf(g, (x[o] - mean) * invstd, sdyx);
  }
  sdy = block_sum(sdy, red);
  sdyx = block_sum(sdyx, red);
  if (threadIdx.x == 0) {
    if (dgamma) dgamma[c] = sdyx;
    if (dbeta) dbeta[c] = sdy;
  }
  const float g = gamma ? gamma[c] : 1.f;
  const float k = g * invstd, inv_cnt = 1.f / (float)cnt;
  for (long long i = threadIdx.x; i < cnt; i += blockDim.x) {
    const long long o = ((i / HW) * C + c) * HW + i % HW;
    if (fixed_stats) { dx[o] = k * dy[o]; continue; }
    const float xh = (x[o] - mean) * invstd;
    dx[o] = k * (dy[o] - (sdy + xh * sdyx) * inv_cnt);
  }
}

// ------------------------------------------------------------------------------------------------------------------ split form
struct BnAcc { double a, b; };   // per channel: (sum x, sum x^2) forward, (sum dy, sum dy*xhat) backward

__device__ __forceinline__ void bn_block_sum2(float& u, float& v, float* red) {
  u = warp_sum(u); v = warp_sum(v);
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
  if (lane == 0) { red[wid] = u; red[16 + wid] = v; }
  __syncthreads();
  if (threadIdx.x < 32) {
    float a = threadIdx.x < nw ? red[threadIdx.x] : 0.f, b = threadIdx.x < nw ? red[16 + threadIdx.x] : 0.f;
    u = warp_sum(a); v = warp_sum(b);
  }
}

// grid (C, S), 256 threads: CTA (c, s) covers images s, s+S, ...
// Every CTA of a channel accumulates x - p for the same pivot p = x[0, c, 0], so the fp32 partial sums stay of the size of the spread of x,
// not of its mean: E[x^2] - mean^2 of raw values loses the variance to cancellation once |mean| / std is in the hundreds.
__global__ void __launch_bounds__(256) bn_stats_kernel(const float* __restrict__ x, float* __restrict__ running_mean, float* __restrict__ running_var,
                                                        float* __restrict__ save_mean, float* __restrict__ save_invstd, BnAcc* __restrict__ acc,
                                                        int* __restrict__ tickets, int N, int C, int HW, float momentum, float eps) {
  gx::pdl_wait();
  gx::pdl_launch();
  __shared__ float red[32];
  const int c = blockIdx.x, S = gridDim.y;
  const float p = __ldg(x + (long long)c * HW);
  float s = 0.f, q = 0.f;
  if ((HW & 3) == 0) {
    // flattened (image, 128-bit chunk) index: all 256 threads stay busy whatever HW is, four independent loads in flight per thread
    const int hw4 = HW >> 2, imgs = (N - (int)blockIdx.y + S - 1) / S, total = imgs * hw4;
    const long long img_stride = (long long)S * C * HW;
    const float* base = x + ((long long)blockIdx.y * C + c) * HW;
    auto at = [&](int j) {
      const int k = j / hw4;
      const float4 v = __ldg(reinterpret_cast<const float4*>(base + k * img_stride) + (j - k * hw4));
      return make_float4(v.x - p, v.y - p, v.z - p, v.w - p);
    };
    int j = threadIdx.x;
    for (; j + 768 < total; j += 1024) {
      const float4 v0 = at(j), v1 = at(j + 256), v2 = at(j + 512), v3 = at(j + 768);
      s += ((v0.x + v0.y) + (v0.z + v0.w)) + ((v1.x + v1.y) + (v1.z + v1.w)) + ((v2.x + v2.y) + (v2.z + v2.w)) + ((v3.x + v3.y) + (v3.z + v3.w));
      q = fmaf(v0.x, v0.x, fmaf(v0.y, v0.y, fmaf(v0.z, v0.z, fmaf(v0.w, v0.w, q))));
      q = fmaf(v1.x, v1.x, fmaf(v1.y, v1.y, fmaf(v1.z, v1.z, fmaf(v1.w, v1.w, q))));
      q = fmaf(v2.x, v2.x, fmaf(v2.y, v2.y, fmaf(v2.z, v2.z, fmaf(v2.w, v2.w, q))));
      q = fmaf(v3.x, v3.x, fmaf(v3.y, v3.y, fmaf(v3.z, v3.z, fmaf(v3.w, v3.w, q))));
    }
    for (; j < total; j += 256) {
      const float4 v = at(j);
      s += (v.x + v.y) + (v.z + v.w);
      q = fmaf(v.x, v.x, fmaf(v.y, v.y, fmaf(v.z, v.z, fmaf(v.w, v.w, q))));
    }
  } else {
    for (int n = blockIdx.y; n < N; n += S) {
      const float* px = x + ((long long)n * C + c) * HW;
      for (int i = threadIdx.x; i < HW; i += 256) { const float v = __ldg(px + i) - p; s += v; q = fmaf(v, v, q); }
    }
  }
  bn_block_sum2(s, q, red);
  if (threadIdx.x == 0) {
    atomicAdd(&acc[c].a, (double)s);
    atomicAdd(&acc[c].b, (double)q);
    __threadfence();
    if (atomicAdd(tickets + c, 1) == S - 1) {          // every slice of this channel has been added
      __threadfence();
      const double cnt = (double)N * HW;
      const double sum = *reinterpret_cast<volatile double*>(&acc[c].a), sq = *reinterpret_cast<volatile double*>(&acc[c].b);
      const double dm = sum / cnt, mean = (double)p + dm;   // sums are of x - p
      double var = sq / cnt - dm * dm;
      if (var < 0.0) var = 0.0;
      save_mean[c] = (float)mean;
      save_invstd[c] = rsqrtf((float)var + eps);
      running_mean[c] = momentum * running_mean[c] + (1.f - momentum) * (float)mean;
      running_var[c] = momentum * running_var[c] + (1.f - momentum) * (float)var;
      acc[c].a = 0.0; acc[c].b = 0.0; tickets[c] = 0;   // re-armed for the next launch (stream order makes this visible)
    }
  }
}

// grid: one CTA per `planes_per_cta` (image, channel) planes; y = x * a[c] + off[c]
__global__ void __launch_bounds__(256) bn_apply_kernel(const float* __restrict__ x, const float* __restrict__ gamma, const float* __restrict__ beta,
                                                        const float* __restrict__ mean_src, const float* __restrict__ var_or_invstd, int is_var,
                                                        float eps, float* __restrict__ y, long long planes, int C, int HW) {
  gx::pdl_wait();
  gx::pdl_launch();
  if ((HW & 3) == 0) {
    // the tensor is one flat array of planes: grid-stride over its 128-bit chunks, two in flight per thread; a chunk never straddles a plane
    const long long total = planes * (HW >> 2), stride = (long long)gridDim.x * 256;
    const int hw4 = HW >> 2;
    auto coef = [&](long long i, float& a, float& off) {
      const int c = (int)((i / hw4) % C);
      const float invstd = is_var ? rsqrtf(__ldg(var_or_invstd + c) + eps) : __ldg(var_or_invstd + c);
      a = (gamma ? __ldg(gamma + c) : 1.f) * invstd;
      off = (beta ? __ldg(beta + c) : 0.f) - __ldg(mean_src + c) * a;
    };
    long long i = (long long)blockIdx.x * 256 + threadIdx.x;
    for (; i + stride < total; i += 2 * stride) {
      const float4 v0 = __ldg(reinterpret_cast<const float4*>(x) + i), v1 = __ldg(reinterpret_cast<const float4*>(x) + i + stride);
      float a0, o0, a1, o1;
      coef(i, a0, o0); coef(i + stride, a1, o1);
      reinterpret_cast<float4*>(y)[i] = make_float4(fmaf(v0.x, a0, o0), fmaf(v0.y, a0, o0), fmaf(v0.z, a0, o0), fmaf(v0.w, a0, o0));
      reinterpret_cast<float4*>(y)[i + stride] = make_float4(fmaf(v1.x, a1, o1), fmaf(v1.y, a1, o1), fmaf(v1.z, a1, o1), fmaf(v1.w, a1, o1));
    }
    for (; i < total; i += stride) {
      const float4 v = __ldg(reinterpret_cast<const float4*>(x) + i);
      float a, o;
      coef(i, a, o);
      reinterpret_cast<float4*>(y)[i] = make_float4(fmaf(v.x, a, o), fmaf(v.y, a, o), fmaf(v.z, a, o), fmaf(v.w, a, o));
    }
    return;
  }
  for (long long pl = blockIdx.x; pl < planes; pl += gridDim.x) {
    const int c = (int)(pl % C);
    const float invstd = is_var ? rsqrtf(var_or_invstd[c] + eps) : var_or_invstd[c];
    const float a = (gamma ? gamma[c] : 1.f) * invstd, off = (beta ? beta[c] : 0.f) - mean_src[c] * a;
    const float* px = x + pl * HW; float* py = y + pl * HW;
    for (int i = threadIdx.x; i < HW; i += 256) py[i] = fmaf(__ldg(px + i), a, off);
  }
}

__global__ void __launch_bounds__(256) bn_bwd_stats_kernel(const float* __restrict__ x, const float* __restrict__ dy, const float* __restrict__ save_mean,
                                                            const float* __restrict__ save_invstd, float* __restrict__ dgamma, float* __restrict__ dbeta,
                                                            float* __restrict__ sums, BnAcc* __restrict__ acc, int* __restrict__ tickets, int N, int C, int HW) {
  gx::pdl_wait();
  gx::pdl_launch();
  __shared__ float red[32];
  const int c = blockIdx.x, S = gridDim.y;
  const float mean = save_mean[c], invstd = save_invstd[c];
  float sdy = 0.f, sdyx = 0.f;
  if ((HW & 3) == 0) {
    const int hw4 = HW >> 2, imgs = (N - (int)blockIdx.y + S - 1) / S, total = imgs * hw4;
    const long long img_stride = (long long)S * C * HW, o0 = ((long long)blockIdx.y * C + c) * HW;
    auto off = [&](int j) { const int k = j / hw4; return o0 + k * img_stride + 4LL * (j - k * hw4); };
    int j = threadIdx.x;
    for (; j + 256 < total; j += 512) {
      const long long oa = off(j), ob = off(j + 256);
      const float4 va = __ldg(reinterpret_cast<const float4*>(x + oa)), ga = __ldg(reinterpret_cast<const float4*>(dy + oa));
      const float4 vb = __ldg(reinterpret_cast<const float4*>(x + ob)), gb = __ldg(reinterpret_cast<const float4*>(dy + ob));
      sdy += ((ga.x + ga.y) + (ga.z + ga.w)) + ((gb.x + gb.y) + (gb.z + gb.w));
      sdyx = fmaf(ga.x, va.x - mean, fmaf(ga.y, va.y - mean, fmaf(ga.z, va.z - mean, fmaf(ga.w, va.w - mean, sdyx))));
      sdyx = fmaf(gb.x, vb.x - mean, fmaf(gb.y, vb.y - mean, fmaf(gb.z, vb.z - mean, fmaf(gb.w, vb.w - mean, sdyx))));
    }
    for (; j < total; j += 256) {
      const long long oa = off(j);
      const float4 v = __ldg(reinterpret_cast<const float4*>(x + oa)), g = __ldg(reinterpret_cast<const float4*>(dy + oa));
      sdy += (g.x + g.y) + (g.z + g.w);
      sdyx = fmaf(g.x, v.x - mean, fmaf(g.y, v.y - mean, fmaf(g.z, v.z - mean, fmaf(g.w, v.w - mean, sdyx))));
    }
  } else {
    for (int n = blockIdx.y; n < N; n += S) {
      const long long o = ((long long)n * C + c) * HW;
      for (int i = threadIdx.x; i < HW; i += 256) { const float g = __ldg(dy + o + i); sdy += g; sdyx = fmaf(g, __ldg(x + o + i) - mean, sdyx); }
    }
  }
  sdyx *= invstd;
  bn_block_sum2(sdy, sdyx, red);
  if (threadIdx.x == 0) {
    atomicAdd(&acc[c].a, (double)sdy);
    atomicAdd(&acc[c].b, (double)sdyx);
    __threadfence();
    if (atomicAdd(tickets + c, 1) == S - 1) {
      __threadfence();
      const float a = (float)*reinterpret_cast<volatile double*>(&acc[c].a), b = (float)*reinterpret_cast<volatile double*>(&acc[c].b);
      if (dbeta) dbeta[c] = a;
      if (dgamma) dgamma[c] = b;
      sums[2 * c] = a; sums[2 * c + 1] = b;
      acc[c].a = 0.0; acc[c].b = 0.0; tickets[c] = 0;
    }
  }
}

__global__ void __launch_bounds__(256) bn_bwd_apply_kernel(const float* __restrict__ x, const float* __restrict__ dy, const float* __restrict__ gamma,
                                                            const float* __restrict__ save_mean, const float* __restrict__ save_invstd,
                                                            const float* __restrict__ sums, float* __restrict__ dx, long long planes, int C, int HW, float inv_cnt,
                                                            int fixed_stats) {
  gx::pdl_wait();
  gx::pdl_launch();
  if ((HW & 3) == 0) {
    const long long total = planes * (HW >> 2), stride = (long long)gridDim.x * 256;
    const int hw4 = HW >> 2;
    for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < total; i += stride) {
      const int c = (int)((i / hw4) % C);
      const float mean = __ldg(save_mean + c), invstd = __ldg(save_invstd + c);
      const float k = (gamma ? __ldg(gamma + c) : 1.f) * invstd;
      const float m_dy = __ldg(sums + 2 * c) * inv_cnt, m_dyx = __ldg(sums + 2 * c + 1) * inv_cnt * invstd;
      const float4 g = __ldg(reinterpret_cast<const float4*>(dy) + i);
      if (fixed_stats) { reinterpret_cast<float4*>(dx)[i] = make_float4(k * g.x, k * g.y, k * g.z, k * g.w); continue; }
      const float4 v = __ldg(reinterpret_cast<const float4*>(x) + i);
      float4 o;
      o.x = k * (g.x - m_dy - (v.x - mean) * m_dyx); o.y = k * (g.y - m_dy - (v.y - mean) * m_dyx);
      o.z = k * (g.z - m_dy - (v.z - mean) * m_dyx); o.w = k * (g.w - m_dy - (v.w - mean) * m_dyx);
      reinterpret_cast<float4*>(dx)[i] = o;
    }
    return;
  }
  for (long long pl = blockIdx.x; pl < planes; pl += gridDim.x) {
    const int c = (int)(pl % C);
    const float mean = save_mean[c], invstd = save_invstd[c];
    const float k = (gamma ? gamma[c] : 1.f) * invstd;
    const float m_dy = sums[2 * c] * inv_cnt, m_dyx = sums[2 * c + 1] * inv_cnt * invstd;   // dx = k * (dy - mean(dy) - xhat * mean(dy*xhat))
    const float* px = x + pl * HW; const float* pg = dy + pl * HW; float* pd = dx + pl * HW;
    if (fixed_stats) { for (int i = threadIdx.x; i < HW; i += 256) pd[i] = k * __ldg(pg + i); continue; }
    for (int i = threadIdx.x; i < HW; i += 256) pd[i] = k * (__ldg(pg + i) - m_dy - (__ldg(px + i) - mean) * m_dyx);
  }
}

}  // namespace gx

using namespace gx;

// persistent accumulators of the split form, one set per (device, stream) so that BatchNorm layers running concurrently on different streams
// never share them (self-cleaning: the finalising CTA zeroes what it consumed)
constexpr int BN_MAX_C = 16384;
struct BnWorkspace { int dev = -1; cudaStream_t stream = nullptr; BnAcc* acc = nullptr; int* tickets = nullptr; float* sums = nullptr; };
static BnWorkspace g_bn_ws[64];
static int g_bn_ws_used = 0;
static std::mutex g_bn_ws_mu;
static BnWorkspace* bn_workspace_find(int dev, cudaStream_t s) {
  for (int i = 0; i < g_bn_ws_used; ++i) if (g_bn_ws[i].dev == dev && g_bn_ws[i].stream == s) return &g_bn_ws[i];
  return nullptr;
}
static BnWorkspace* bn_workspace_lookup(cudaStream_t s) {
  int dev = 0;
  cudaGetDevice(&dev);
  std::lock_guard<std::mutex> lk(g_bn_ws_mu);
  return bn_workspace_find(dev, s);
}
static BnWorkspace* bn_workspace(cudaStream_t s) {
  BnWorkspace* ws = g_bn_ws;
  int& used = g_bn_ws_used;
  int dev = 0;
  cudaGetDevice(&dev);
  std::lock_guard<std::mutex> lk(g_bn_ws_mu);
  if (BnWorkspace* w = bn_workspace_find(dev, s)) return w;
  // first use on this stream: allocation is not allowed while the stream is being captured into a graph (the caller then uses the
  // single-kernel form for this launch; warm-up steps normally run before a capture and allocate here)
  cudaStreamCaptureStatus st = cudaStreamCaptureStatusNone;
  if (cudaStreamIsCapturing(s, &st) != cudaSuccess || st != cudaStreamCaptureStatusNone || used == 64) { cudaGetLastError(); return nullptr; }
  BnWorkspace w;
  w.dev = dev; w.stream = s;
  if (cudaMalloc(&w.acc, BN_MAX_C * sizeof(BnAcc)) != cudaSuccess || cudaMalloc(&w.tickets, BN_MAX_C * sizeof(int)) != cudaSuccess ||
      cudaMalloc(&w.sums, BN_MAX_C * 2 * sizeof(float)) != cudaSuccess) { cudaGetLastError(); return nullptr; }
  cudaMemset(w.acc, 0, BN_MAX_C * sizeof(BnAcc));
  cudaMemset(w.tickets, 0, BN_MAX_C * sizeof(int));
  cudaDeviceSynchronize();
  ws[used] = w;
  return &ws[used++];
}
// 1 when the split form's accumulators already exist for the calling device and stream `s` (introspection for tests: the first BatchNorm
// on a stream that is being captured into a graph cannot allocate them and runs the one-CTA form)
GX_API int gx_bn_workspace_ready(cudaStream_t s) {
  return bn_workspace_lookup(s) != nullptr ? 1 : 0;
}
static bool bn_split_form(int N, int C, int HW) { return (long long)N * HW >= 4096 && HW >= 16 && C <= BN_MAX_C; }
static int bn_slices(int N, int C) {
  int sms = 148, dev = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  int s = (8 * sms + C - 1) / C;          // ~8 CTAs of 256 threads per SM
  if (s > N) s = N;
  return s < 1 ? 1 : s;
}

GX_API int gx_bn_fwd(const float* x, const float* gamma, const float* beta, float* rm, float* rv, float* y, float* save_mean, float* save_invstd,
                     int N, int C, int HW, int training, float momentum, float eps, cudaStream_t s) {
  BnWorkspace* w = bn_split_form(N, C, HW) ? bn_workspace(s) : nullptr;
  if (w != nullptr) {
    int sms = 148, dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    const long long planes = (long long)N * C;
    const unsigned grid = (unsigned)(planes < 16LL * sms ? planes : 16LL * sms);
    if (training) {
      launch_pdl(bn_stats_kernel, dim3(C, bn_slices(N, C)), dim3(256), 0, s, x, rm, rv, save_mean, save_invstd, w->acc, w->tickets, N, C, HW, momentum, eps);
      if (int rc = GX_CHECK_LAUNCH()) return rc;
      launch_pdl(bn_apply_kernel, dim3(grid), dim3(256), 0, s, x, gamma, beta, (const float*)save_mean, (const float*)save_invstd, 0, eps, y, planes, C, HW);
    } else {
      launch_pdl(bn_apply_kernel, dim3(grid), dim3(256), 0, s, x, gamma, beta, (const float*)rm, (const float*)rv, 1, eps, y, planes, C, HW);
    }
    return GX_CHECK_LAUNCH();
  }
  launch_pdl(bn_fwd_kernel, dim3(C), dim3(512), 0, s, x, gamma, beta, rm, rv, y, save_mean, save_invstd, N, C, HW, training, momentum, eps);
  return GX_CHECK_LAUNCH();
}
// fixed_stats: save_mean / save_invstd are the running statistics the forward pass normalised with (inference mode, use_global_stats), which
// do not depend on x, so dx = dy * gamma * invstd (reference batch_norm.cu, is_train_and_not_global_stats); dgamma / dbeta are the same sums.
GX_API int gx_bn_bwd(const float* x, const float* dy, const float* gamma, const float* save_mean, const float* save_invstd, float* dx, float* dgamma,
                     float* dbeta, int N, int C, int HW, int fixed_stats, cudaStream_t s) {
  BnWorkspace* w = bn_split_form(N, C, HW) ? bn_workspace(s) : nullptr;
  if (w != nullptr) {
    int sms = 148, dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    const long long planes = (long long)N * C;
    const unsigned grid = (unsigned)(planes < 16LL * sms ? planes : 16LL * sms);
    launch_pdl(bn_bwd_stats_kernel, dim3(C, bn_slices(N, C)), dim3(256), 0, s, x, dy, save_mean, save_invstd, dgamma, dbeta, w->sums, w->acc, w->tickets, N, C, HW);
    if (int rc = GX_CHECK_LAUNCH()) return rc;
    launch_pdl(bn_bwd_apply_kernel, dim3(grid), dim3(256), 0, s, x, dy, gamma, save_mean, save_invstd, (const float*)w->sums, dx, planes, C, HW,
               1.f / ((float)N * (float)HW), fixed_stats);
    return GX_CHECK_LAUNCH();
  }
  launch_pdl(bn_bwd_kernel, dim3(C), dim3(512), 0, s, x, dy, gamma, save_mean, save_invstd, dx, dgamma, dbeta, N, C, HW, fixed_stats);
  return GX_CHECK_LAUNCH();
}
