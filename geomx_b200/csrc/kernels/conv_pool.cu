// Convolution-side kernels for sm_90a (CUDA-core parts; the GEMMs run on wgmma in gemm_wgmma.cu):
//   * im2col / col2im for the whole batch in ONE launch (the reference launches im2col + cublasSgemm once per image:
//     src/operator/nn/im2col.cuh:79-187, src/operator/nn/convolution-inl.h:165-284)
//   * fused direct conv + bias + ReLU + 2x2 max-pool forward for skinny-K first layers (K = Cin*kh*kw < 32, where a
//     128xNx8 tensor-core tile would be >75 % padding), and the matching fused pool/ReLU-backward + weight-gradient
//   * 2x2/2 max-pool forward/backward with argmax (reference src/operator/nn/pool.cuh:128-165,379-432)
//   * fused pool-backward + ReLU-backward + NCHW->pixel-major transpose + bias-gradient (feeds the dgrad/wgrad GEMMs)
//   * ReLU fwd/bwd, NCHW<->rows transposes, column sums (bias gradients)
#include "common.cuh"

namespace gx {

// ------------------------------------------------------------------------------------------------ im2col / col2im
// col[(n,oh,ow)][k], k = (c*KH + kh)*KW + kw, row stride ldc (>= K, multiple of 4; pad columns are zeroed)
__global__ void __launch_bounds__(256) im2col_kernel(const float* __restrict__ x, float* __restrict__ col, int N, int C, int H, int W,
                                                      int KH, int KW, int OH, int OW, int sh, int sw, int ph, int pw, int K, int ldc) {
  gx::pdl_wait();
  gx::pdl_launch();
  const long long total = (long long)N * OH * OW * ldc;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int k = (int)(i % ldc);
    const long long row = i / ldc;
    float v = 0.f;
    if (k < K) {
      const int kw = k % KW, kh = (k / KW) % KH, c = k / (KW * KH);
      const int ow = (int)(row % OW), oh = (int)((row / OW) % OH), n = (int)(row / ((long long)OW * OH));
      const int h = oh * sh - ph + kh, w = ow * sw - pw + kw;
      if (h >= 0 && h < H && w >= 0 && w < W) v = __ldg(x + (((long long)n * C + c) * H + h) * W + w);
    }
    col[i] = v;
  }
}

// gather-form col2im (no atomics): dx[n,c,h,w] = sum over (kh,kw) of dcol[(n,oh,ow)][(c,kh,kw)] with oh*sh-ph+kh == h
__global__ void __launch_bounds__(256) col2im_kernel(const float* __restrict__ dcol, float* __restrict__ dx, int N, int C, int H, int W,
                                                      int KH, int KW, int OH, int OW, int sh, int sw, int ph, int pw, int ldc) {
  gx::pdl_wait();
  gx::pdl_launch();
  const long long total = (long long)N * C * H * W;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int w = (int)(i % W), h = (int)((i / W) % H), c = (int)((i / ((long long)W * H)) % C), n = (int)(i / ((long long)W * H * C));
    float acc = 0.f;
    for (int kh = 0; kh < KH; ++kh) {
      const int hh = h + ph - kh;
      if (hh < 0 || hh % sh) continue;
      const int oh = hh / sh;
      if (oh >= OH) continue;
      for (int kw = 0; kw < KW; ++kw) {
        const int ww = w + pw - kw;
        if (ww < 0 || ww % sw) continue;
        const int ow = ww / sw;
        if (ow >= OW) continue;
        acc += __ldg(dcol + (((long long)n * OH + oh) * OW + ow) * ldc + (c * KH + kh) * KW + kw);
      }
    }
    dx[i] = acc;
  }
}

// Shared-memory tiled variants for stride-1 / pad-0 convolutions (the demo network): one CTA per (image, group of CG channels).
// im2col: the CG input planes are staged in smem once, the CTA then writes its [OH*OW][CG*KH*KW] slab of `col` with fully coalesced stores.
template <int CG>
__global__ void __launch_bounds__(256) im2col_tiled_kernel(const float* __restrict__ x, float* __restrict__ col, int C, int H, int W, int KH, int KW,
                                                            int OH, int OW, int ldc) {
  gx::pdl_wait();
  gx::pdl_launch();
  extern __shared__ float sm[];
  const int n = blockIdx.x, c0 = blockIdx.y * CG;
  const int cg = min(CG, C - c0);
  for (int i = threadIdx.x; i < cg * H * W; i += blockDim.x) sm[i] = x[((long long)n * C + c0) * H * W + i];
  __syncthreads();
  const int KK = KH * KW, span = cg * KK;
  for (int i = threadIdx.x; i < OH * OW * span; i += blockDim.x) {
    const int kk = i % span, row = i / span;
    const int cl = kk / KK, t = kk - cl * KK, kh = t / KW, kw = t - kh * KW;
    const int oh = row / OW, ow = row - oh * OW;
    col[((long long)n * OH * OW + row) * ldc + c0 * KK + kk] = sm[cl * H * W + (oh + kh) * W + ow + kw];
  }
}
// col2im: the [OH*OW][CG*KH*KW] slab of dcol is staged in smem (coalesced), every input-gradient pixel then gathers its <= KH*KW taps from smem.
template <int CG>
__global__ void __launch_bounds__(256) col2im_tiled_kernel(const float* __restrict__ dcol, float* __restrict__ dx, int C, int H, int W, int KH, int KW,
                                                            int OH, int OW, int ldc) {
  gx::pdl_wait();
  gx::pdl_launch();
  extern __shared__ float sm[];
  const int n = blockIdx.x, c0 = blockIdx.y * CG;
  const int cg = min(CG, C - c0);
  const int KK = KH * KW, span = cg * KK;
  for (int i = threadIdx.x; i < OH * OW * span; i += blockDim.x) {
    const int kk = i % span, row = i / span;
    sm[row * span + kk] = dcol[((long long)n * OH * OW + row) * ldc + c0 * KK + kk];
  }
  __syncthreads();
  for (int i = threadIdx.x; i < cg * H * W; i += blockDim.x) {
    const int w = i % W, h = (i / W) % H, cl = i / (W * H);
    float acc = 0.f;
    for (int kh = 0; kh < KH; ++kh) {
      const int oh = h - kh;
      if (oh < 0 || oh >= OH) continue;
      for (int kw = 0; kw < KW; ++kw) {
        const int ow = w - kw;
        if (ow < 0 || ow >= OW) continue;
        acc += sm[(oh * OW + ow) * span + cl * KK + kh * KW + kw];
      }
    }
    dx[((long long)n * C + c0) * H * W + i] = acc;
  }
}

// ------------------------------------------------------------------------------------------------ transposes / reductions
// y[(n,hw)][c] = x[n,c,hw]
__global__ void __launch_bounds__(256) nchw_to_rows_kernel(const float* __restrict__ x, float* __restrict__ y, int N, int C, int HW) {
  gx::pdl_wait();
  gx::pdl_launch();
  __shared__ float tile[32][33];
  const int n = blockIdx.z;
  const int c0 = blockIdx.y * 32, p0 = blockIdx.x * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;  // 32 x 8
  for (int j = ty; j < 32; j += 8) {
    const int c = c0 + j, p = p0 + tx;
    tile[j][tx] = (c < C && p < HW) ? x[((long long)n * C + c) * HW + p] : 0.f;
  }
  __syncthreads();
  for (int j = ty; j < 32; j += 8) {
    const int p = p0 + j, c = c0 + tx;
    if (p < HW && c < C) y[((long long)n * HW + p) * C + c] = tile[tx][j];
  }
}

// out[c] (+)= sum_r x[r][c]   (bias gradients)
__global__ void __launch_bounds__(256) colsum_kernel(const float* __restrict__ x, float* __restrict__ out, long long R, int C, long long ld, int accumulate) {
  gx::pdl_wait();
  gx::pdl_launch();
  const int c = blockIdx.x * 32 + (threadIdx.x & 31);
  const int ty = threadIdx.x >> 5;
  __shared__ float part[8][33];
  float acc = 0.f;
  if (c < C)
    for (long long r = ty; r < R; r += 8) acc += x[r * ld + c];
  part[ty][threadIdx.x & 31] = acc;
  __syncthreads();
  if (ty == 0 && c < C) {
    float s = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) s += part[j][threadIdx.x & 31];
    if (accumulate) out[c] += s;
    else out[c] = s;
  }
}

// NCHW per-channel sum: out[c] = sum_{n,hw} x[n,c,hw]   (conv bias gradient on NCHW dy)
__global__ void __launch_bounds__(256) chansum_nchw_kernel(const float* __restrict__ x, float* __restrict__ out, int N, int C, int HW) {
  gx::pdl_wait();
  gx::pdl_launch();
  const int c = blockIdx.x;
  float acc = 0.f;
  for (long long i = threadIdx.x; i < (long long)N * HW; i += blockDim.x) {
    const int n = (int)(i / HW), p = (int)(i % HW);
    acc += x[((long long)n * C + c) * HW + p];
  }
  __shared__ float red[8];
  acc = warp_sum(acc);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float s = 0.f;
    for (int j = 0; j < (int)(blockDim.x >> 5); ++j) s += red[j];
    out[c] = s;
  }
}

// ------------------------------------------------------------------------------------------------ ReLU
// Each thread owns 4 consecutive elements: one 128-bit access per tensor when every pointer is 16-byte aligned (uniform over the grid),
// scalar accesses otherwise (a contiguous view such as x[1:] or a slice handed over by cat / split backward starts anywhere).
// fmaxf maps NaN to 0, like the reference's mshadow_op::relu (torch.relu would propagate it).
__global__ void __launch_bounds__(256) relu_fwd_kernel(const float* __restrict__ x, float* __restrict__ y, long long n) {
  gx::pdl_wait();
  gx::pdl_launch();
  const long long i4 = (blockIdx.x * (long long)blockDim.x + threadIdx.x) * 4;
  const bool vec = ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(y)) & 15) == 0;
  if (vec && i4 + 3 < n) {
    float4 v = *reinterpret_cast<const float4*>(x + i4);
    v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); v.z = fmaxf(v.z, 0.f); v.w = fmaxf(v.w, 0.f);
    *reinterpret_cast<float4*>(y + i4) = v;
  } else {
    for (long long i = i4; i < n && i < i4 + 4; ++i) y[i] = fmaxf(x[i], 0.f);
  }
}
__global__ void __launch_bounds__(256) relu_bwd_kernel(const float* __restrict__ y, const float* __restrict__ dy, float* __restrict__ dx, long long n) {
  gx::pdl_wait();
  gx::pdl_launch();
  const long long i4 = (blockIdx.x * (long long)blockDim.x + threadIdx.x) * 4;
  const bool vec = ((reinterpret_cast<uintptr_t>(y) | reinterpret_cast<uintptr_t>(dy) | reinterpret_cast<uintptr_t>(dx)) & 15) == 0;
  if (vec && i4 + 3 < n) {
    const float4 a = *reinterpret_cast<const float4*>(y + i4);
    float4 g = *reinterpret_cast<const float4*>(dy + i4);
    g.x = a.x > 0.f ? g.x : 0.f; g.y = a.y > 0.f ? g.y : 0.f; g.z = a.z > 0.f ? g.z : 0.f; g.w = a.w > 0.f ? g.w : 0.f;
    *reinterpret_cast<float4*>(dx + i4) = g;
  } else {
    for (long long i = i4; i < n && i < i4 + 4; ++i) dx[i] = y[i] > 0.f ? dy[i] : 0.f;
  }
}

// ------------------------------------------------------------------------------------------------ 2x2/2 max-pool
__global__ void __launch_bounds__(256) maxpool2x2_fwd_kernel(const float* __restrict__ x, float* __restrict__ y, uint8_t* __restrict__ idx,
                                                              long long NC, int H, int W) {
  gx::pdl_wait();
  gx::pdl_launch();
  const int PH = H >> 1, PW = W >> 1;
  const long long total = NC * PH * PW;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int pw = (int)(i % PW), ph = (int)((i / PW) % PH);
    const long long nc = i / ((long long)PW * PH);
    const float* src = x + (nc * H + 2 * ph) * W + 2 * pw;
    const float2 r0 = *reinterpret_cast<const float2*>(src);
    const float2 r1 = *reinterpret_cast<const float2*>(src + W);
    float best = r0.x; int b = 0;
    if (r0.y > best) { best = r0.y; b = 1; }
    if (r1.x > best) { best = r1.x; b = 2; }
    if (r1.y > best) { best = r1.y; b = 3; }
    y[i] = best;
    if (idx) idx[i] = (uint8_t)b;
  }
}
__global__ void __launch_bounds__(256) maxpool2x2_bwd_kernel(const float* __restrict__ dy, const uint8_t* __restrict__ idx, float* __restrict__ dx,
                                                              long long NC, int H, int W) {
  gx::pdl_wait();
  gx::pdl_launch();
  const int PH = H >> 1, PW = W >> 1;
  const long long total = NC * PH * PW;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int pw = (int)(i % PW), ph = (int)((i / PW) % PH);
    const long long nc = i / ((long long)PW * PH);
    const float g = dy[i];
    const int b = idx[i];
    float* dst = dx + (nc * H + 2 * ph) * W + 2 * pw;
    *reinterpret_cast<float2*>(dst) = make_float2(b == 0 ? g : 0.f, b == 1 ? g : 0.f);
    *reinterpret_cast<float2*>(dst + W) = make_float2(b == 2 ? g : 0.f, b == 3 ? g : 0.f);
  }
}

// Fused: pool-backward + ReLU-backward (pooled>0) + NCHW -> pixel-major rows [(n,h,w)][C] + bias gradient.
//   dz[(n,2ph+dy,2pw+dx)][c] = (argmax==(dy,dx) && pooled>0) ? dpooled[n,c,ph,pw] : 0 ;  dbias[c] += sum dz[:, c]
// one CTA per (n, ph) pooled row; dbias must be zeroed by the caller.
__global__ void __launch_bounds__(256) pool_relu_bwd_rows_kernel(const float* __restrict__ dpooled, const float* __restrict__ pooled,
                                                                  const uint8_t* __restrict__ idx, float* __restrict__ dz_rows,
                                                                  float* __restrict__ dbias, int N, int C, int PH, int PW) {
  gx::pdl_wait();
  gx::pdl_launch();
  const int n = blockIdx.x / PH, ph = blockIdx.x % PH;
  const int W = 2 * PW, H = 2 * PH;
  for (int e = threadIdx.x; e < PW * C; e += blockDim.x) {
    const int c = e % C, pw = e / C;  // c fastest -> coalesced row writes
    const long long pi = (((long long)n * C + c) * PH + ph) * PW + pw;
    const float g = pooled[pi] > 0.f ? dpooled[pi] : 0.f;
    const int b = idx[pi];
    const long long r0 = ((long long)n * H + 2 * ph) * W + 2 * pw;
    dz_rows[(r0)*C + c] = b == 0 ? g : 0.f;
    dz_rows[(r0 + 1) * C + c] = b == 1 ? g : 0.f;
    dz_rows[(r0 + W) * C + c] = b == 2 ? g : 0.f;
    dz_rows[(r0 + W + 1) * C + c] = b == 3 ? g : 0.f;
    if (dbias != nullptr && g != 0.f) atomicAdd(dbias + c, g);
  }
}

// ------------------------------------------------------------------------------------------------ skinny-K first layer (direct conv)
// y_pooled[n,co,ph,pw] = max_{dy,dx} relu(conv(x)[n,co,2ph+dy,2pw+dx] + b[co]);  valid conv, stride 1, Cin*KH*KW <= 64.
// grid (N, ceil(Cout/CO_PER_BLOCK)); the whole input image and CO_PER_BLOCK filters live in smem.
template <int CO_PER_BLOCK>
__global__ void __launch_bounds__(256) conv_relu_pool_fwd_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ b,
                                                                  float* __restrict__ y, uint8_t* __restrict__ idx, int Cin, int H, int W, int Cout,
                                                                  int KH, int KW) {
  gx::pdl_wait();
  gx::pdl_launch();
  extern __shared__ float sm[];
  const int K = Cin * KH * KW;
  float* sx = sm;                 // Cin*H*W
  float* sw = sm + Cin * H * W;   // CO_PER_BLOCK * K
  const int n = blockIdx.x, co0 = blockIdx.y * CO_PER_BLOCK;
  for (int i = threadIdx.x; i < Cin * H * W; i += blockDim.x) sx[i] = x[(long long)n * Cin * H * W + i];
  for (int i = threadIdx.x; i < CO_PER_BLOCK * K; i += blockDim.x) {
    const int co = co0 + i / K;
    sw[i] = co < Cout ? w[(long long)co * K + i % K] : 0.f;
  }
  __syncthreads();
  const int OH = H - KH + 1, OW = W - KW + 1, PH = OH >> 1, PW = OW >> 1;
  for (int e = threadIdx.x; e < CO_PER_BLOCK * PH * PW; e += blockDim.x) {
    const int pw = e % PW, ph = (e / PW) % PH, cl = e / (PW * PH);
    const int co = co0 + cl;
    if (co >= Cout) continue;
    float a00 = 0.f, a01 = 0.f, a10 = 0.f, a11 = 0.f;
    const float* wf = sw + cl * K;
    for (int c = 0; c < Cin; ++c) {
      const float* xin = sx + c * H * W + (2 * ph) * W + 2 * pw;
      for (int kh = 0; kh < KH; ++kh) {
#pragma unroll 5
        for (int kw = 0; kw < KW; ++kw) {
          const float wv = wf[(c * KH + kh) * KW + kw];
          const float* px = xin + kh * W + kw;
          a00 = fmaf(wv, px[0], a00);
          a01 = fmaf(wv, px[1], a01);
          a10 = fmaf(wv, px[W], a10);
          a11 = fmaf(wv, px[W + 1], a11);
        }
      }
    }
    float best = a00; int bi = 0;
    if (a01 > best) { best = a01; bi = 1; }
    if (a10 > best) { best = a10; bi = 2; }
    if (a11 > best) { best = a11; bi = 3; }
    best = fmaxf(best + b[co], 0.f);
    const long long o = (((long long)n * Cout + co) * PH + ph) * PW + pw;
    y[o] = best;
    idx[o] = (uint8_t)bi;
  }
}

// Same as conv_relu_pool_fwd_kernel, plus the im2col slab of the NEXT convolution (stride 1, no padding, kernel KH2 x KW2) for the
// CO_PER_BLOCK pooled planes this CTA just produced:  col[(n,oh2,ow2)][(co*KH2+kh)*KW2+kw] = y[n,co,oh2+kh,ow2+kw].   One launch less, and
// the pooled activations never travel through L2 between the two steps.
template <int CO_PER_BLOCK>
__global__ void __launch_bounds__(256) conv_relu_pool_im2col_fwd_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ b,
                                                                         float* __restrict__ y, uint8_t* __restrict__ idx, float* __restrict__ col, int Cin,
                                                                         int H, int W, int Cout, int KH, int KW, int KH2, int KW2, int ldc) {
  gx::pdl_wait();
  gx::pdl_launch();
  extern __shared__ float sm[];
  const int K = Cin * KH * KW;
  const int OH = H - KH + 1, OW = W - KW + 1, PH = OH >> 1, PW = OW >> 1;
  float* sx = sm;                              // Cin*H*W
  float* sw = sx + Cin * H * W;                // CO_PER_BLOCK * K
  float* sp = sw + CO_PER_BLOCK * K;           // CO_PER_BLOCK * PH * PW pooled planes
  const int n = blockIdx.x, co0 = blockIdx.y * CO_PER_BLOCK;
  for (int i = threadIdx.x; i < Cin * H * W; i += blockDim.x) sx[i] = x[(long long)n * Cin * H * W + i];
  for (int i = threadIdx.x; i < CO_PER_BLOCK * K; i += blockDim.x) {
    const int co = co0 + i / K;
    sw[i] = co < Cout ? w[(long long)co * K + i % K] : 0.f;
  }
  __syncthreads();
  for (int e = threadIdx.x; e < CO_PER_BLOCK * PH * PW; e += blockDim.x) {
    const int pw = e % PW, ph = (e / PW) % PH, cl = e / (PW * PH);
    const int co = co0 + cl;
    float best = 0.f; int bi = 0;
    if (co < Cout) {
      float a00 = 0.f, a01 = 0.f, a10 = 0.f, a11 = 0.f;
      const float* wf = sw + cl * K;
      for (int c = 0; c < Cin; ++c) {
        const float* xin = sx + c * H * W + (2 * ph) * W + 2 * pw;
        for (int kh = 0; kh < KH; ++kh) {
#pragma unroll 5
          for (int kw = 0; kw < KW; ++kw) {
            const float wv = wf[(c * KH + kh) * KW + kw];
            const float* px = xin + kh * W + kw;
            a00 = fmaf(wv, px[0], a00); a01 = fmaf(wv, px[1], a01); a10 = fmaf(wv, px[W], a10); a11 = fmaf(wv, px[W + 1], a11);
          }
        }
      }
      best = a00;
      if (a01 > best) { best = a01; bi = 1; }
      if (a10 > best) { best = a10; bi = 2; }
      if (a11 > best) { best = a11; bi = 3; }
      best = fmaxf(best + b[co], 0.f);
      const long long o = (((long long)n * Cout + co) * PH + ph) * PW + pw;
      y[o] = best;
      idx[o] = (uint8_t)bi;
    }
    sp[e] = best;
  }
  __syncthreads();
  const int OH2 = PH - KH2 + 1, OW2 = PW - KW2 + 1, KK2 = KH2 * KW2;
  const int cg = min(CO_PER_BLOCK, Cout - co0), span = cg * KK2;
  for (int i = threadIdx.x; i < OH2 * OW2 * span; i += blockDim.x) {
    const int kk = i % span, row = i / span;
    const int cl = kk / KK2, t = kk - cl * KK2, kh = t / KW2, kw = t - kh * KW2;
    const int oh = row / OW2, ow = row - oh * OW2;
    col[((long long)n * OH2 * OW2 + row) * ldc + co0 * KK2 + kk] = sp[cl * PH * PW + (oh + kh) * PW + ow + kw];
  }
}

// Fused backward of the same layer (no dx needed for a first layer):
//   g = (pooled>0) ? dpooled : 0 at the arg-max position;  dW[co][c,kh,kw] += g * x[n,c,2ph+dy+kh,2pw+dx+kw];  db[co] += g
// grid (Cout, NSPLIT): block (co, s) reduces images n = s, s+NSPLIT, ... ; one (c,kh,kw) tap per thread-group, smem reduce, atomics.
__global__ void __launch_bounds__(256) conv_relu_pool_wgrad_kernel(const float* __restrict__ x, const float* __restrict__ dpooled,
                                                                    const float* __restrict__ pooled, const uint8_t* __restrict__ idx,
                                                                    float* __restrict__ dw, float* __restrict__ db, int N, int Cin, int H, int W,
                                                                    int Cout, int KH, int KW) {
  gx::pdl_wait();
  gx::pdl_launch();
  const int co = blockIdx.x;
  const int OH = H - KH + 1, OW = W - KW + 1, PH = OH >> 1, PW = OW >> 1;
  const int K = Cin * KH * KW;
  extern __shared__ float sm[];
  float* sg = sm;                      // PH*PW gradients of this (n, co) plane
  int* spos = reinterpret_cast<int*>(sm + PH * PW);  // top-left input offset of the arg-max window
  float* sx = sm + 2 * PH * PW;        // Cin*H*W input image
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
  float acc[8];  // up to 8 taps per warp round (K <= 64, 8 warps)
#pragma unroll
  for (int t = 0; t < 8; ++t) acc[t] = 0.f;
  float bacc = 0.f;
  for (int n = blockIdx.y; n < N; n += gridDim.y) {
    __syncthreads();
    for (int i = threadIdx.x; i < Cin * H * W; i += blockDim.x) sx[i] = x[(long long)n * Cin * H * W + i];
    for (int i = threadIdx.x; i < PH * PW; i += blockDim.x) {
      const long long pi = ((long long)n * Cout + co) * PH * PW + i;
      const float g = pooled[pi] > 0.f ? dpooled[pi] : 0.f;
      const int b = idx[pi];
      const int ph = i / PW, pw = i % PW;
      sg[i] = g;
      spos[i] = (2 * ph + (b >> 1)) * W + 2 * pw + (b & 1);
      if (g != 0.f) bacc += g;
    }
    __syncthreads();
    // warp `wid` owns taps k = wid, wid+nw, ... ; lanes stride over pooled positions
    int t = 0;
    for (int k = wid; k < K; k += nw, ++t) {
      const int kw = k % KW, kh = (k / KW) % KH, c = k / (KW * KH);
      const float* xin = sx + c * H * W + kh * W + kw;
      float a = 0.f;
      for (int i = lane; i < PH * PW; i += 32) a = fmaf(sg[i], xin[spos[i]], a);
      acc[t] += a;
    }
  }
  int t = 0;
  for (int k = wid; k < K; k += nw, ++t) {
    const float s = warp_sum(acc[t]);
    if (lane == 0) atomicAdd(dw + (long long)co * K + k, s);
  }
  bacc = warp_sum(bacc);
  if (lane == 0 && bacc != 0.f && db != nullptr) atomicAdd(db + co, bacc);
}

// conv_relu_pool_wgrad_kernel with the col2im of the NEXT convolution's input gradient fused in: the gradient w.r.t. this layer's pooled
// output plane (n, co) is gathered from dcol[(n,oh2,ow2)][(co*KH2+kh)*KW2+kw] (stride-1 / valid KH2 x KW2 conv) inside the CTA.
__global__ void __launch_bounds__(256) conv_relu_pool_wgrad_col2im_kernel(const float* __restrict__ x, const float* __restrict__ dcol,
                                                                           const float* __restrict__ pooled, const uint8_t* __restrict__ idx,
                                                                           float* __restrict__ dw, float* __restrict__ db, int N, int Cin, int H, int W,
                                                                           int Cout, int KH, int KW, int KH2, int KW2, int ldc) {
  gx::pdl_wait();
  gx::pdl_launch();
  const int co = blockIdx.x, n = blockIdx.y;
  const int OH = H - KH + 1, OW = W - KW + 1, PH = OH >> 1, PW = OW >> 1;
  const int OH2 = PH - KH2 + 1, OW2 = PW - KW2 + 1, KK2 = KH2 * KW2;
  const int K = Cin * KH * KW;
  extern __shared__ float sm[];
  float* sg = sm;                                     // PH*PW
  int* spos = reinterpret_cast<int*>(sm + PH * PW);   // PH*PW
  float* sx = sm + 2 * PH * PW;                       // Cin*H*W
  float* sd = sx + Cin * H * W;                       // OH2*OW2*KK2 slab of dcol
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
  for (int i = threadIdx.x; i < Cin * H * W; i += blockDim.x) sx[i] = x[(long long)n * Cin * H * W + i];
  for (int i = threadIdx.x; i < OH2 * OW2 * KK2; i += blockDim.x) {
    const int kk = i % KK2, row = i / KK2;
    sd[i] = dcol[((long long)n * OH2 * OW2 + row) * ldc + co * KK2 + kk];
  }
  __syncthreads();
  float bacc = 0.f;
  for (int i = threadIdx.x; i < PH * PW; i += blockDim.x) {
    const int ph = i / PW, pw = i - ph * PW;
    float da = 0.f;
    for (int kh = 0; kh < KH2; ++kh) {
      const int oh = ph - kh;
      if (oh < 0 || oh >= OH2) continue;
      for (int kw = 0; kw < KW2; ++kw) {
        const int ow = pw - kw;
        if (ow < 0 || ow >= OW2) continue;
        da += sd[(oh * OW2 + ow) * KK2 + kh * KW2 + kw];
      }
    }
    const long long pi = ((long long)n * Cout + co) * PH * PW + i;
    const float g = pooled[pi] > 0.f ? da : 0.f;
    const int bsel = idx[pi];
    sg[i] = g;
    spos[i] = (2 * ph + (bsel >> 1)) * W + 2 * pw + (bsel & 1);
    bacc += g;
  }
  __syncthreads();
  for (int k = wid; k < K; k += nw) {
    const int kw = k % KW, kh = (k / KW) % KH, c = k / (KW * KH);
    const float* xin = sx + c * H * W + kh * W + kw;
    float a = 0.f;
    for (int i = lane; i < PH * PW; i += 32) a = fmaf(sg[i], xin[spos[i]], a);
    a = warp_sum(a);
    if (lane == 0) atomicAdd(dw + (long long)co * K + k, a);
  }
  bacc = warp_sum(bacc);
  if (lane == 0 && bacc != 0.f && db != nullptr) atomicAdd(db + co, bacc);
}

static inline int nblocks(long long total, int per = 256, int cap = 148 * 16) {
  long long b = (total + per - 1) / per;
  return (int)(b < 1 ? 1 : (b > cap ? cap : b));
}

}  // namespace gx

using namespace gx;

GX_API int gx_im2col(const float* x, float* col, int N, int C, int H, int W, int KH, int KW, int sh, int sw, int ph, int pw, int ldc,
                     cudaStream_t s) {
  const int OH = (H + 2 * ph - KH) / sh + 1, OW = (W + 2 * pw - KW) / sw + 1;
  const long long total = (long long)N * OH * OW * ldc;
  constexpr int CG = 4;
  if (sh == 1 && sw == 1 && ph == 0 && pw == 0 && ldc == C * KH * KW && (size_t)CG * H * W * sizeof(float) <= 96 * 1024) {
    static bool set = false;
    if (!set) { cudaFuncSetAttribute(im2col_tiled_kernel<CG>, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024); set = true; }
    launch_pdl(im2col_tiled_kernel<CG>, dim3(N, (C + CG - 1) / CG), dim3(256), (size_t)CG * H * W * sizeof(float), s, x, col, C, H, W, KH, KW, OH, OW, ldc);
    return GX_CHECK_LAUNCH();
  }
  launch_pdl(im2col_kernel, dim3(nblocks(total)), dim3(256), 0, s, x, col, N, C, H, W, KH, KW, OH, OW, sh, sw, ph, pw, C * KH * KW, ldc);
  return GX_CHECK_LAUNCH();
}
GX_API int gx_col2im(const float* dcol, float* dx, int N, int C, int H, int W, int KH, int KW, int sh, int sw, int ph, int pw, int ldc,
                     cudaStream_t s) {
  const int OH = (H + 2 * ph - KH) / sh + 1, OW = (W + 2 * pw - KW) / sw + 1;
  constexpr int CG = 4;
  if (sh == 1 && sw == 1 && ph == 0 && pw == 0 && (size_t)OH * OW * CG * KH * KW * sizeof(float) <= 160 * 1024) {
    static bool set = false;
    if (!set) { cudaFuncSetAttribute(col2im_tiled_kernel<CG>, cudaFuncAttributeMaxDynamicSharedMemorySize, 160 * 1024); set = true; }
    launch_pdl(col2im_tiled_kernel<CG>, dim3(N, (C + CG - 1) / CG), dim3(256), (size_t)OH * OW * CG * KH * KW * sizeof(float), s, dcol, dx, C, H, W, KH, KW,
               OH, OW, ldc);
    return GX_CHECK_LAUNCH();
  }
  launch_pdl(col2im_kernel, dim3(nblocks((long long)N * C * H * W)), dim3(256), 0, s, dcol, dx, N, C, H, W, KH, KW, OH, OW, sh, sw, ph, pw, ldc);
  return GX_CHECK_LAUNCH();
}
GX_API int gx_nchw_to_rows(const float* x, float* y, int N, int C, int HW, cudaStream_t s) {
  dim3 grid((HW + 31) / 32, (C + 31) / 32, N);
  launch_pdl(nchw_to_rows_kernel, dim3(grid), dim3(256), 0, s, x, y, N, C, HW);
  return GX_CHECK_LAUNCH();
}
GX_API int gx_colsum(const float* x, float* out, long long R, int C, long long ld, int accumulate, cudaStream_t s) {
  launch_pdl(colsum_kernel, dim3((C + 31) / 32), dim3(256), 0, s, x, out, R, C, ld, accumulate);
  return GX_CHECK_LAUNCH();
}
GX_API int gx_chansum_nchw(const float* x, float* out, int N, int C, int HW, cudaStream_t s) {
  launch_pdl(chansum_nchw_kernel, dim3(C), dim3(256), 0, s, x, out, N, C, HW);
  return GX_CHECK_LAUNCH();
}
GX_API int gx_relu_fwd(const float* x, float* y, long long n, cudaStream_t s) {
  if (n <= 0) return 0;
  launch_pdl(relu_fwd_kernel, dim3((unsigned)((n + 1023) / 1024)), dim3(256), 0, s, x, y, n);
  return GX_CHECK_LAUNCH();
}
GX_API int gx_relu_bwd(const float* y, const float* dy, float* dx, long long n, cudaStream_t s) {
  if (n <= 0) return 0;
  launch_pdl(relu_bwd_kernel, dim3((unsigned)((n + 1023) / 1024)), dim3(256), 0, s, y, dy, dx, n);
  return GX_CHECK_LAUNCH();
}
GX_API int gx_maxpool2x2_fwd(const float* x, float* y, uint8_t* idx, long long NC, int H, int W, cudaStream_t s) {
  launch_pdl(maxpool2x2_fwd_kernel, dim3(nblocks(NC * (H / 2) * (W / 2))), dim3(256), 0, s, x, y, idx, NC, H, W);
  return GX_CHECK_LAUNCH();
}
GX_API int gx_maxpool2x2_bwd(const float* dy, const uint8_t* idx, float* dx, long long NC, int H, int W, cudaStream_t s) {
  launch_pdl(maxpool2x2_bwd_kernel, dim3(nblocks(NC * (H / 2) * (W / 2))), dim3(256), 0, s, dy, idx, dx, NC, H, W);
  return GX_CHECK_LAUNCH();
}
GX_API int gx_pool_relu_bwd_rows(const float* dpooled, const float* pooled, const uint8_t* idx, float* dz_rows, float* dbias, int N, int C,
                                 int PH, int PW, cudaStream_t s) {
  launch_pdl(pool_relu_bwd_rows_kernel, dim3(N * PH), dim3(256), 0, s, dpooled, pooled, idx, dz_rows, dbias, N, C, PH, PW);
  return GX_CHECK_LAUNCH();
}
GX_API int gx_conv_relu_pool_fwd(const float* x, const float* w, const float* b, float* y, uint8_t* idx, int N, int Cin, int H, int W, int Cout,
                                 int KH, int KW, cudaStream_t s) {
  constexpr int CPB = 4;
  const size_t smem = ((size_t)Cin * H * W + (size_t)CPB * Cin * KH * KW) * sizeof(float);
  if (smem > 200 * 1024) return -1;
  static bool set = false;
  if (!set) { cudaFuncSetAttribute(conv_relu_pool_fwd_kernel<CPB>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024); set = true; }
  dim3 grid(N, (Cout + CPB - 1) / CPB);
  launch_pdl(conv_relu_pool_fwd_kernel<CPB>, dim3(grid), dim3(192), smem, s, x, w, b, y, idx, Cin, H, W, Cout, KH, KW);
  return GX_CHECK_LAUNCH();
}
GX_API int gx_conv_relu_pool_wgrad(const float* x, const float* dpooled, const float* pooled, const uint8_t* idx, float* dw, float* db, int N,
                                   int Cin, int H, int W, int Cout, int KH, int KW, cudaStream_t s) {
  const int OH = H - KH + 1, OW = W - KW + 1, PH = OH / 2, PW = OW / 2;
  if (Cin * KH * KW > 64) return -1;
  const size_t smem = ((size_t)2 * PH * PW + (size_t)Cin * H * W) * sizeof(float);
  if (smem > 200 * 1024) return -1;
  static bool set = false;
  if (!set) { cudaFuncSetAttribute(conv_relu_pool_wgrad_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024); set = true; }
  dim3 grid(Cout, N);   // one (co, image) plane per CTA: a single round of (cold) loads, 25 atomics per CTA
  launch_pdl(conv_relu_pool_wgrad_kernel, dim3(grid), dim3(256), smem, s, x, dpooled, pooled, idx, dw, db, N, Cin, H, W, Cout, KH, KW);
  return GX_CHECK_LAUNCH();
}

GX_API int gx_conv_relu_pool_im2col_fwd(const float* x, const float* w, const float* b, float* y, uint8_t* idx, float* col, int N, int Cin, int H, int W,
                                        int Cout, int KH, int KW, int KH2, int KW2, int ldc, cudaStream_t s) {
  constexpr int CPB = 4;
  const int PH = (H - KH + 1) / 2, PW = (W - KW + 1) / 2;
  const size_t smem = ((size_t)Cin * H * W + (size_t)CPB * Cin * KH * KW + (size_t)CPB * PH * PW) * sizeof(float);
  if (smem > 200 * 1024 || ldc != Cout * KH2 * KW2) return -1;
  static bool set = false;
  if (!set) { cudaFuncSetAttribute(conv_relu_pool_im2col_fwd_kernel<CPB>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024); set = true; }
  launch_pdl(conv_relu_pool_im2col_fwd_kernel<CPB>, dim3(N, (Cout + CPB - 1) / CPB), dim3(256), smem, s, x, w, b, y, idx, col, Cin, H, W, Cout, KH, KW, KH2,
             KW2, ldc);
  return GX_CHECK_LAUNCH();
}
GX_API int gx_conv_relu_pool_wgrad_col2im(const float* x, const float* dcol, const float* pooled, const uint8_t* idx, float* dw, float* db, int N, int Cin,
                                          int H, int W, int Cout, int KH, int KW, int KH2, int KW2, int ldc, cudaStream_t s) {
  const int PH = (H - KH + 1) / 2, PW = (W - KW + 1) / 2, OH2 = PH - KH2 + 1, OW2 = PW - KW2 + 1;
  if (Cin * KH * KW > 2048) return -1;
  const size_t smem = ((size_t)2 * PH * PW + (size_t)Cin * H * W + (size_t)OH2 * OW2 * KH2 * KW2) * sizeof(float);
  if (smem > 200 * 1024) return -1;
  static bool set = false;
  if (!set) { cudaFuncSetAttribute(conv_relu_pool_wgrad_col2im_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024); set = true; }
  launch_pdl(conv_relu_pool_wgrad_col2im_kernel, dim3(Cout, N), dim3(256), smem, s, x, dcol, pooled, idx, dw, db, N, Cin, H, W, Cout, KH, KW, KH2, KW2, ldc);
  return GX_CHECK_LAUNCH();
}
