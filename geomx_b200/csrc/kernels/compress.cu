// Gradient-compression kernels for sm_90a: 2-bit (residual), Bi-Sparse (BSC), block-scaled fp8, DGT contribution.
//
// Reference behaviour (see geomx_b200/kvstore/compression.py for the full contract):
//   2bit  : src/kvstore/gradient_compression-inl.h:40-139 — one thread per 16-value word, byte-wise bit twiddling.
//           Here: one thread packs 16 values from four 128-bit loads, identical bit layout.
//   BSC   : src/kvstore/gradient_compression.cc:191-336 — single-threaded CPU lambdas (shuffle + heap + linear scans).
//           Here: one CTA per tensor does momentum correction, sampled-threshold selection (radix select of the k-th
//           largest sample) and *index-ordered* stream compaction with a block-wide scan, all in one launch;
//           several tensors are batched as blockIdx.x.
//   fp8   : new on H100 — e4m3 payload + fp32 scale per 128 values, error feedback in `residual`.
//   DGT   : 3rdparty/ps-lite/include/ps/kv_app.h:853-876 EvalMsgContribution — EMA of mean |g| per 4096-byte block.
#include <cuda_fp8.h>

#include "common.cuh"

namespace gx {

// ------------------------------------------------------------------------------------------------ 2-bit
__global__ void __launch_bounds__(256) quantize_2bit_kernel(const float* __restrict__ grad, float* __restrict__ residual, uint32_t* __restrict__ out,
                                                             long long n, float thr) {
  gx::pdl_wait();
  gx::pdl_launch();
  const long long words = (n + 15) / 16;
  for (long long wi = blockIdx.x * (long long)blockDim.x + threadIdx.x; wi < words; wi += (long long)gridDim.x * blockDim.x) {
    uint32_t word = 0;
    const long long base = wi * 16;
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const long long i = base + j;
      if (i < n) {
        float r = residual[i] + grad[i];
        uint32_t code = 0;
        if (r >= thr) { code = 3; r -= thr; }
        else if (r <= -thr) { code = 2; r += thr; }
        residual[i] = r;
        // value j lives in byte j>>2 (little-endian within the word), bit pair 6-2*(j&3)
        word |= code << (((j >> 2) << 3) + (6 - 2 * (j & 3)));
      }
    }
    out[wi] = word;
  }
}
__global__ void __launch_bounds__(256) dequantize_2bit_kernel(const uint32_t* __restrict__ in, float* __restrict__ out, long long n, float thr,
                                                               int accumulate) {
  gx::pdl_wait();
  gx::pdl_launch();
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const uint32_t word = in[i >> 4];
    const int j = (int)(i & 15);
    const uint32_t code = (word >> (((j >> 2) << 3) + (6 - 2 * (j & 3)))) & 3u;
    const float v = code == 3 ? thr : (code == 2 ? -thr : 0.f);
    out[i] = accumulate ? out[i] + v : v;
  }
}

// ------------------------------------------------------------------------------------------------ BSC
struct BscSeg {
  const float* grad;   // may be null for pull-compress
  float* u; float* v;  // error-feedback state (null for pull-compress: v := dense input)
  float* out;          // [2k]: vals | idx
  long long n;
  int k, sample, k_sample;
};

constexpr int BSC_THREADS = 1024;
constexpr int BSC_ITEMS = 4;

__device__ __forceinline__ int block_exclusive_scan(int val, int* total, int* smem_warp) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  int inc = val;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int t = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += t;
  }
  if (lane == 31) smem_warp[wid] = inc;
  __syncthreads();
  if (wid == 0) {
    int w = lane < (BSC_THREADS / 32) ? smem_warp[lane] : 0;
    int winc = w;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int t = __shfl_up_sync(0xffffffffu, winc, o);
      if (lane >= o) winc += t;
    }
    smem_warp[lane] = winc - w;            // exclusive prefix of warp totals
    if (lane == 31) smem_warp[32] = winc;  // block total
  }
  __syncthreads();
  const int res = smem_warp[wid] + inc - val;
  *total = smem_warp[32];
  __syncthreads();
  return res;
}

// mode 0: BSCompress (momentum correction + sampled threshold + ordered compaction + state reset)
// mode 1: BSCPullCompress (keep non-zeros in index order)
template <int MODE>
__global__ void __launch_bounds__(BSC_THREADS, 1) bsc_kernel(const BscSeg* __restrict__ segs, float momentum) {
  gx::pdl_wait();
  gx::pdl_launch();
  const BscSeg sg = segs[blockIdx.x];
  __shared__ int s_warp[33];
  __shared__ int s_hist[256];
  __shared__ int s_sel[2];
  const long long n = sg.n;
  const float* src = MODE == 0 ? sg.v : sg.grad;
  float boundary = 0.f;
  if (MODE == 0) {
    // 1) momentum correction  u = m*u + g ; v += u
    for (long long i = threadIdx.x; i < n; i += BSC_THREADS) {
      const float u = momentum * sg.u[i] + sg.grad[i];
      sg.u[i] = u;
      sg.v[i] += u;
    }
    __syncthreads();
    // 2) boundary = k_sample-th largest |v| over a strided sample: 8-bit radix select on the bit patterns of |v| (which order like the
    //    values), four passes over the sample in global memory, so any sample size fits
    const int S = sg.sample;
    const long long stride = n / S > 0 ? n / S : 1;
    uint32_t prefix = 0, mask = 0;
    int remaining = sg.k_sample < S ? sg.k_sample : S;  // k_sample > sample: the smallest sampled |v|, as the reference's heap gives
    for (int shift = 24; shift >= 0; shift -= 8) {
      if (threadIdx.x < 256) s_hist[threadIdx.x] = 0;
      __syncthreads();
      for (int j = threadIdx.x; j < S; j += BSC_THREADS) {
        const uint32_t key = __float_as_uint(sg.v[(long long)j * stride]) & 0x7fffffffu;
        if ((key & mask) == prefix) atomicAdd(&s_hist[(key >> shift) & 255u], 1);
      }
      __syncthreads();
      const int h = threadIdx.x < 256 ? s_hist[255 - threadIdx.x] : 0;  // thread i owns bin 255-i: the scan counts the keys in higher bins
      int total;
      const int above = block_exclusive_scan(h, &total, s_warp);
      if (threadIdx.x < 256 && above < remaining && above + h >= remaining) { s_sel[0] = 255 - (int)threadIdx.x; s_sel[1] = remaining - above; }
      __syncthreads();
      prefix |= (uint32_t)s_sel[0] << shift;
      mask |= 255u << shift;
      remaining = s_sel[1];
    }
    boundary = __uint_as_float(prefix);
  }
  // 3) index-ordered compaction, at most k entries
  const int k = sg.k;
  int base = 0;
  for (long long chunk = 0; chunk < n && base < k; chunk += (long long)BSC_THREADS * BSC_ITEMS) {
    const long long i0 = chunk + (long long)threadIdx.x * BSC_ITEMS;
    float vals[BSC_ITEMS];
    int flags = 0, cnt = 0;
#pragma unroll
    for (int j = 0; j < BSC_ITEMS; ++j) {
      const long long i = i0 + j;
      vals[j] = i < n ? src[i] : 0.f;
      const bool keep = i < n && (MODE == 0 ? fabsf(vals[j]) >= boundary : vals[j] != 0.f);
      if (keep) { flags |= 1 << j; ++cnt; }
    }
    int total;
    int pos = base + block_exclusive_scan(cnt, &total, s_warp);
#pragma unroll
    for (int j = 0; j < BSC_ITEMS; ++j) {
      if (flags & (1 << j)) {
        if (pos < k) {
          sg.out[pos] = vals[j];
          sg.out[k + pos] = (float)(i0 + j);
          if (MODE == 0) { sg.v[i0 + j] = 0.f; sg.u[i0 + j] = 0.f; }
        }
        ++pos;
      }
    }
    base += total;
  }
  // 4) sentinel padding
  const int filled = base < k ? base : k;
  for (int j = filled + threadIdx.x; j < k; j += BSC_THREADS) {
    sg.out[j] = -65530.f;
    sg.out[k + j] = -1.f;
  }
}

__global__ void __launch_bounds__(256) bsc_decompress_kernel(const float* __restrict__ zipped, float* __restrict__ out, int k) {
  gx::pdl_wait();
  gx::pdl_launch();
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < k; j += gridDim.x * blockDim.x) {
    const float fi = zipped[k + j];
    if (fi >= 0.f) atomicAdd(out + (long long)fi, zipped[j]);
  }
}

// ------------------------------------------------------------------------------------------------ block-scaled fp8 (e4m3, 128 values / scale)
__global__ void __launch_bounds__(128) fp8_block_quantize_kernel(const float* __restrict__ x, float* __restrict__ residual, uint8_t* __restrict__ q,
                                                                  float* __restrict__ scale, long long n) {
  gx::pdl_wait();
  gx::pdl_launch();
  const long long blk = blockIdx.x;
  const long long i = blk * 128 + threadIdx.x;
  float v = 0.f;
  if (i < n) v = x[i] + (residual ? residual[i] : 0.f);
  float a = warp_max(fabsf(v));
  __shared__ float red[4];
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = a;
  __syncthreads();
  a = fmaxf(fmaxf(red[0], red[1]), fmaxf(red[2], red[3]));
  const float sc = a > 0.f ? a / 448.f : 1.f;
  const __nv_fp8_storage_t b = __nv_cvt_float_to_fp8(v / sc, __NV_SATFINITE, __NV_E4M3);
  q[i] = (uint8_t)b;
  if (threadIdx.x == 0) scale[blk] = sc;
  if (residual && i < n) {
    const float deq = __half2float(__half(__nv_cvt_fp8_to_halfraw(b, __NV_E4M3))) * sc;
    residual[i] = v - deq;
  }
}
__global__ void __launch_bounds__(256) fp8_block_dequantize_kernel(const uint8_t* __restrict__ q, const float* __restrict__ scale, float* __restrict__ out,
                                                                    long long n, int accumulate) {
  gx::pdl_wait();
  gx::pdl_launch();
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const float v = __half2float(__half(__nv_cvt_fp8_to_halfraw((__nv_fp8_storage_t)q[i], __NV_E4M3))) * scale[i >> 7];
    out[i] = accumulate ? out[i] + v : v;
  }
}

// ------------------------------------------------------------------------------------------------ DGT block contribution
// contrib[b] = alpha * contrib[b] + (1-alpha) * mean(|g| over block b)     (kv_app.h:853-876)
__global__ void __launch_bounds__(256) dgt_contrib_kernel(const float* __restrict__ g, float* __restrict__ contrib, long long n, int block_elems,
                                                           float alpha, int first) {
  gx::pdl_wait();
  gx::pdl_launch();
  const long long b = blockIdx.x;
  const long long lo = b * block_elems, hi = lo + block_elems < n ? lo + block_elems : n;
  float acc = 0.f;
  for (long long i = lo + threadIdx.x; i < hi; i += blockDim.x) acc += fabsf(g[i]);
  acc = warp_sum(acc);
  __shared__ float red[8];
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float s = 0.f;
    for (int j = 0; j < 8; ++j) s += red[j];
    const float mean = s / (float)(hi - lo);
    contrib[b] = first ? mean : alpha * contrib[b] + (1.f - alpha) * mean;
  }
}

static inline int cgrid(long long n) {
  long long b = (n + 255) / 256;
  return (int)(b < 1 ? 1 : (b > 148 * 8 ? 148 * 8 : b));
}

}  // namespace gx

using namespace gx;

GX_API int gx_quantize_2bit(const float* grad, float* residual, void* out, long long n, float thr, cudaStream_t s) {
  launch_pdl(quantize_2bit_kernel, dim3(cgrid((n + 15) / 16)), dim3(256), 0, s, grad, residual, reinterpret_cast<uint32_t*>(out), n, thr);
  return GX_CHECK_LAUNCH();
}
GX_API int gx_dequantize_2bit(const void* in, float* out, long long n, float thr, int accumulate, cudaStream_t s) {
  launch_pdl(dequantize_2bit_kernel, dim3(cgrid(n)), dim3(256), 0, s, reinterpret_cast<const uint32_t*>(in), out, n, thr, accumulate);
  return GX_CHECK_LAUNCH();
}
// segs: device array of BscSeg (see struct above), one CTA each.
GX_API int gx_bsc_compress_batch(const void* segs, int num_segs, float momentum, cudaStream_t s) {
  if (num_segs == 0) return 0;
  launch_pdl(bsc_kernel<0>, dim3(num_segs), dim3(BSC_THREADS), 0, s, reinterpret_cast<const BscSeg*>(segs), momentum);
  return GX_CHECK_LAUNCH();
}
GX_API int gx_bsc_pull_compress_batch(const void* segs, int num_segs, cudaStream_t s) {
  if (num_segs == 0) return 0;
  launch_pdl(bsc_kernel<1>, dim3(num_segs), dim3(BSC_THREADS), 0, s, reinterpret_cast<const BscSeg*>(segs), 0.f);
  return GX_CHECK_LAUNCH();
}
GX_API int gx_bsc_decompress(const float* zipped, float* out, long long n, int k, int accumulate, cudaStream_t s) {
  if (!accumulate) cudaMemsetAsync(out, 0, (size_t)n * sizeof(float), s);
  if (k > 0) launch_pdl(bsc_decompress_kernel, dim3(cgrid(k)), dim3(256), 0, s, zipped, out, k);
  return GX_CHECK_LAUNCH();
}
GX_API int gx_fp8_block_quantize(const float* x, float* residual, void* q, float* scale, long long n, cudaStream_t s) {
  const long long nb = (n + 127) / 128;
  if (nb == 0) return 0;
  launch_pdl(fp8_block_quantize_kernel, dim3((unsigned)nb), dim3(128), 0, s, x, residual, reinterpret_cast<uint8_t*>(q), scale, n);
  return GX_CHECK_LAUNCH();
}
GX_API int gx_fp8_block_dequantize(const void* q, const float* scale, float* out, long long n, int accumulate, cudaStream_t s) {
  launch_pdl(fp8_block_dequantize_kernel, dim3(cgrid(n)), dim3(256), 0, s, reinterpret_cast<const uint8_t*>(q), scale, out, n, accumulate);
  return GX_CHECK_LAUNCH();
}
GX_API int gx_dgt_contrib(const float* g, float* contrib, long long n, int block_elems, float alpha, int first, cudaStream_t s) {
  const long long nb = (n + block_elems - 1) / block_elems;
  if (nb == 0) return 0;
  launch_pdl(dgt_contrib_kernel, dim3((unsigned)nb), dim3(256), 0, s, g, contrib, n, block_elems, alpha, first);
  return GX_CHECK_LAUNCH();
}
GX_API int gx_bsc_seg_size() { return (int)sizeof(BscSeg); }
