// Softmax cross-entropy kernels for sm_90a.
//   * warp-per-row log-softmax + pick + loss forward / backward (reference: three launches — softmax_compute_kernel
//     <<<N,128>>> src/operator/nn/softmax-inl.h:166-204, pick src/operator/tensor/broadcast_reduce_op_index.cu:39-45 and
//     their gradients :223-250)
//   * classifier head fused forward+backward: logits = a·Wᵀ + b, softmax-CE loss, d_logits, dW, db, and the input
//     gradient already masked by the previous ReLU plus its bias gradient — ONE launch for what the reference runs
//     as FullyConnected fwd + log_softmax + pick + 3 backward ops (fully_connected-inl.h:71-173).
#include "common.cuh"

namespace gx {

// loss[r] = -log_softmax(x[r])[label[r]]
__global__ void __launch_bounds__(256) softmax_ce_fwd_kernel(const float* __restrict__ x, const float* __restrict__ label, float* __restrict__ loss,
                                                              int R, int C) {
  gx::pdl_wait();
  gx::pdl_launch();
  const int r = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (r >= R) return;
  const int lane = threadIdx.x & 31;
  const float* row = x + (long long)r * C;
  float mx = -INFINITY;
  for (int c = lane; c < C; c += 32) mx = fmaxf(mx, row[c]);
  mx = warp_max(mx);
  float s = 0.f;
  for (int c = lane; c < C; c += 32) s += __expf(row[c] - mx);
  s = warp_sum(s);
  if (lane == 0) {
    const int l = (int)label[r];
    loss[r] = -(row[l] - mx - __logf(s));
  }
}
// dx[r][c] = (softmax(x[r])[c] - [c==label[r]]) * dloss[r]
__global__ void __launch_bounds__(256) softmax_ce_bwd_kernel(const float* __restrict__ x, const float* __restrict__ label, const float* __restrict__ dloss,
                                                              float* __restrict__ dx, int R, int C) {
  gx::pdl_wait();
  gx::pdl_launch();
  const int r = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (r >= R) return;
  const int lane = threadIdx.x & 31;
  const float* row = x + (long long)r * C;
  float mx = -INFINITY;
  for (int c = lane; c < C; c += 32) mx = fmaxf(mx, row[c]);
  mx = warp_max(mx);
  float s = 0.f;
  for (int c = lane; c < C; c += 32) s += __expf(row[c] - mx);
  s = warp_sum(s);
  const float inv = 1.f / s, g = dloss ? dloss[r] : 1.f;
  const int l = (int)label[r];
  for (int c = lane; c < C; c += 32) dx[(long long)r * C + c] = (__expf(row[c] - mx) * inv - (c == l ? 1.f : 0.f)) * g;
}

// Fused classifier head, single CTA (B*C <= 8192, C <= 32, B*K + C*K floats of smem):
//   phase 0 : stage a[B][K] and W[C][K] in shared memory with coalesced 128-bit loads (everything is cold in L2/HBM after the step's
//             L2 flush, so all global reads are issued up front)
//   phase 1 : warp per sample: logits, loss, dlogits -> smem
//   phase 2 : dW[c][k] = sum_b dl[b][c]*a[b][k] ; db[c] = sum_b dl[b][c]
//             da[b][k] = (a[b][k] > 0 ? sum_c dl[b][c]*W[c][k] : 0)  over all B*K outputs in parallel;  dbias_prev[k] = sum_b da[b][k]
// WEIGHTED: the dlogits of sample b are scaled by coef[b] in phase 1 (the per-row gradient coefficient of a short or sample-weighted batch),
// so every gradient carries it; the loss stays unweighted.  Instantiated twice: head_fwd_bwd_kernel (WEIGHTED = false) compiles to the code
// it had before the weighted head existed; head_fwd_bwd_weighted_kernel.
template <bool WEIGHTED>
__device__ __forceinline__ void head_fwd_bwd_body(const float* __restrict__ a, const float* __restrict__ W, const float* __restrict__ bias,
                                                  const float* __restrict__ label, float* __restrict__ loss, float* __restrict__ logits_out,
                                                  float* __restrict__ dW, float* __restrict__ db, float* __restrict__ da,
                                                  float* __restrict__ dbias_prev, int B, int K, int C, int relu_mask,
                                                  const float* __restrict__ coef) {
  gx::pdl_wait();
  gx::pdl_launch();
  extern __shared__ float sm[];
  float* sa = sm;               // [B][K]
  float* sw = sa + B * K;       // [C][K]
  float* dl = sw + C * K;       // [B][C]
  float* sda = dl + B * C;      // [B][K] masked input gradient (for the column sums)
  float* sbias = sda + B * K;   // [C]
  float* slab = sbias + 32;     // [B]
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
  for (int i = threadIdx.x; i < (B * K) / 4; i += blockDim.x) reinterpret_cast<float4*>(sa)[i] = reinterpret_cast<const float4*>(a)[i];
  for (int i = threadIdx.x; i < (C * K) / 4; i += blockDim.x) reinterpret_cast<float4*>(sw)[i] = reinterpret_cast<const float4*>(W)[i];
  if (threadIdx.x < C) sbias[threadIdx.x] = bias[threadIdx.x];
  for (int i = threadIdx.x; i < B; i += blockDim.x) slab[i] = label[i];
  __syncthreads();
  for (int b = wid; b < B; b += nw) {
    const float* ab = sa + b * K;
    float mylogit = 0.f;  // lane c (< C) keeps logit c
    for (int c = 0; c < C; ++c) {
      float p = 0.f;
      const float* wc = sw + c * K;
      for (int k = lane; k < K; k += 32) p = fmaf(ab[k], wc[k], p);
      p = warp_sum(p) + sbias[c];
      if (lane == c) mylogit = p;
    }
    float mx = lane < C ? mylogit : -INFINITY;
    mx = warp_max(mx);
    const float e = lane < C ? __expf(mylogit - mx) : 0.f;
    const float s = warp_sum(e);
    const int l = (int)slab[b];
    if (lane < C) {
      const float d = e / s - (lane == l ? 1.f : 0.f);
      dl[b * C + lane] = WEIGHTED ? __fmul_rn(d, coef[b]) : d;
      if (logits_out) logits_out[(long long)b * C + lane] = mylogit;
    }
    const float picked = __shfl_sync(0xffffffffu, mylogit, l & 31);
    if (lane == 0) loss[b] = -(picked - mx - __logf(s));
  }
  __syncthreads();
  for (int i = threadIdx.x; i < C * K; i += blockDim.x) {   // dW
    const int c = i / K, k = i - c * K;
    float acc = 0.f;
    for (int b = 0; b < B; ++b) acc = fmaf(dl[b * C + c], sa[b * K + k], acc);
    dW[i] = acc;
  }
  for (int c = threadIdx.x; c < C; c += blockDim.x) {       // db
    float acc = 0.f;
    for (int b = 0; b < B; ++b) acc += dl[b * C + c];
    db[c] = acc;
  }
  for (int i = threadIdx.x; i < B * K; i += blockDim.x) {   // da (+ ReLU mask)
    const int b = i / K, k = i - b * K;
    float acc = 0.f;
    for (int c = 0; c < C; ++c) acc = fmaf(dl[b * C + c], sw[c * K + k], acc);
    if (relu_mask && !(sa[i] > 0.f)) acc = 0.f;
    da[i] = acc;
    sda[i] = acc;
  }
  if (dbias_prev) {
    __syncthreads();
    for (int k = threadIdx.x; k < K; k += blockDim.x) {
      float acc = 0.f;
      for (int b = 0; b < B; ++b) acc += sda[b * K + k];
      dbias_prev[k] = acc;
    }
  }
}
__global__ void __launch_bounds__(1024) head_fwd_bwd_kernel(const float* __restrict__ a, const float* __restrict__ W, const float* __restrict__ bias,
                                                             const float* __restrict__ label, float* __restrict__ loss, float* __restrict__ logits_out,
                                                             float* __restrict__ dW, float* __restrict__ db, float* __restrict__ da,
                                                             float* __restrict__ dbias_prev, int B, int K, int C, int relu_mask) {
  head_fwd_bwd_body<false>(a, W, bias, label, loss, logits_out, dW, db, da, dbias_prev, B, K, C, relu_mask, nullptr);
}
__global__ void __launch_bounds__(1024) head_fwd_bwd_weighted_kernel(const float* __restrict__ a, const float* __restrict__ W,
                                                                      const float* __restrict__ bias, const float* __restrict__ label,
                                                                      float* __restrict__ loss, float* __restrict__ logits_out, float* __restrict__ dW,
                                                                      float* __restrict__ db, float* __restrict__ da, float* __restrict__ dbias_prev,
                                                                      int B, int K, int C, int relu_mask, const float* __restrict__ coef) {
  head_fwd_bwd_body<true>(a, W, bias, label, loss, logits_out, dW, db, da, dbias_prev, B, K, C, relu_mask, coef);
}

}  // namespace gx

using namespace gx;

GX_API int gx_softmax_ce_fwd(const float* x, const float* label, float* loss, int R, int C, cudaStream_t s) {
  launch_pdl(softmax_ce_fwd_kernel, dim3((R + 7) / 8), dim3(256), 0, s, x, label, loss, R, C);
  return GX_CHECK_LAUNCH();
}
GX_API int gx_softmax_ce_bwd(const float* x, const float* label, const float* dloss, float* dx, int R, int C, cudaStream_t s) {
  launch_pdl(softmax_ce_bwd_kernel, dim3((R + 7) / 8), dim3(256), 0, s, x, label, dloss, dx, R, C);
  return GX_CHECK_LAUNCH();
}
// coef [B] (may be null): the dlogits of sample b are scaled by coef[b] (head_fwd_bwd_weighted_kernel); the loss is not
GX_API int gx_head_fwd_bwd(const float* a, const float* W, const float* bias, const float* label, float* loss, float* logits, float* dW,
                           float* db, float* da, float* dbias_prev, const float* coef, int B, int K, int C, int relu_mask, cudaStream_t s) {
  const size_t smem = ((size_t)2 * B * K + (size_t)C * K + (size_t)B * C + 32 + (size_t)B) * sizeof(float);
  if (C > 32 || (long long)B * C > 8192 || smem > 200 * 1024 || (K & 3)) return -1;
  if (coef != nullptr) {
    static bool set_w = false;
    if (!set_w) { cudaFuncSetAttribute(head_fwd_bwd_weighted_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024); set_w = true; }
    launch_pdl(head_fwd_bwd_weighted_kernel, dim3(1), dim3(1024), smem, s, a, W, bias, label, loss, logits, dW, db, da, dbias_prev, B, K, C,
               relu_mask, coef);
    return GX_CHECK_LAUNCH();
  }
  static bool set = false;
  if (!set) { cudaFuncSetAttribute(head_fwd_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024); set = true; }
  launch_pdl(head_fwd_bwd_kernel, dim3(1), dim3(1024), smem, s, a, W, bias, label, loss, logits, dW, db, da, dbias_prev, B, K, C, relu_mask);
  return GX_CHECK_LAUNCH();
}
