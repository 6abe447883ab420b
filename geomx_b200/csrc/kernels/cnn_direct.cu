// Direct (fp32 FMA) convolution kernels for the small-batch regime of the reference's demo CNN
//   Conv2D(16,k5,relu) -> MaxPool2 -> Conv2D(32,k5,relu) -> MaxPool2      (examples/cnn.py:56-60, input 1x28x28)
// forward and backward, TWO launches in total:
//   cnn_fwd_kernel      x -> a1 (+argmax) -> a2 (+argmax)          both convolutions, bias, ReLU and both max-pools; one 4-CTA cluster per
//                       image: each CTA computes a quarter of conv0 and shares it through distributed shared memory, so conv0 runs once
//                       (cnn_fwd_dense0_kernel, even batches <= 32: the same, in clusters of two images, followed by the first dense
//                       layer a2 -> a3, so that the dense-chain cluster kernel starts from a3; in the classic training step also by the
//                       rest of the row-separable chain, dense1, classifier, softmax-CE, dz4 and dz3, so that it only computes da2)
//   cnn_bwd_all_kernel  one heterogeneous grid in clusters of two: CTAs [256, 256+4B)  da2 -> da1 (shared memory only) -> dW0, db0   (conv1
//                       data gradient gathered from the non-zeros of dz2 + pool/ReLU backward of both layers + conv0 weight gradient), CTAs
//                       [0, 256)  da2, a1 -> dW1, db1 (conv1 weight gradient, each cluster's two CTAs splitting the batch and combining their
//                       sums in shared memory); both exploit the sparsity of dz2 (one non-zero per pooling window).  Both bodies resolve
//                       the programmatic grid dependency only AFTER the staging that does not depend on the preceding kernel, so the CTAs
//                       become resident and stage while that kernel still runs — at B <= 32 the whole grid, in one wave.
//                       (cnn_bwd_kernel / cnn_wgrad1_kernel: the same bodies as separate launches; cnn_bwd_exchange_kernel: the same bodies
//                       in one grid without clusters (data-gradient CTAs first, one weight-gradient CTA per output slice) whose last CTAs also
//                       perform the conv keys' exchange — measured, no gain, opt-in.)
// and, for inference, ONE launch for any number of images:
//   cnn_eval_kernel     x -> logits, softmax-CE loss, arg-max and correct flag per image: the convolutions and dense0 of cnn_fwd_dense0_kernel
//                       (clusters of two images, without the stores only the backward pass needs), then dense1 and the classifier in the
//                       same cluster (HipsCNNTrainStep.evaluate / predict)
//
// Why not the tensor-core GEMM here: with a per-worker batch of 32 the conv1 products are M = 2048 x N = 32 x K = 400 — 16 tensor-core
// tiles.  Forward + dgrad + wgrad + im2col/col2im traffic through the GEMM path is several launches of latency-bound work on 16 SMs, while
// the same 78 MFLOP spread over 128 CTAs of plain FMAs finish in a few microseconds, in exact fp32 (the reference's cublasSgemmEx precision).  The max-pool makes
// the backward pass 4x sparse (one non-zero per 2x2 window), which both conv1 gradients exploit.  Larger batches / other geometries use
// the wgmma GEMM path (ops/functional.py conv2d).
//
// Reference kernels replaced: im2col_gpu_kernel / col2im_gpu_kernel (src/operator/nn/im2col.cuh:79-187), per-image cublasSgemmEx
// (convolution-inl.h:165-284), bias broadcast, ReLU (activation-inl.h:89-121), pool_max_2d / unpool (pool.cuh:128-165, 379-432).
#include "common.cuh"
#include "hips_ll.cuh"

#include <cooperative_groups.h>

namespace cg = cooperative_groups;

namespace gx {

// geometry (compile time)
constexpr int CD_H = 28, CD_K = 5;
constexpr int CD_C1 = 16, CD_P1 = 12;            // conv0: 16 channels, 24x24 -> pooled 12x12
constexpr int CD_C2 = 32, CD_P2 = 4;             // conv1: 32 channels,  8x8  -> pooled 4x4
constexpr int CD_W1PAD = 28;                     // 25 taps padded to 28 floats (16-byte rows)

// asynchronous global -> shared copies: all of a CTA's operand loads are in flight at once instead of one dependent round trip per element
__device__ __forceinline__ void cpa4(float* sdst, const float* gsrc) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(smem_u32(sdst)), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void cpa16(float* sdst, const float* gsrc) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(sdst)), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void cpa_wait_all() { asm volatile("cp.async.commit_group;\ncp.async.wait_group 0;" ::: "memory"); }

// 2x2 output window of a 5x5 valid convolution from a 6x6 input patch: acc[dy*2+dx] += sum_{r,s} patch[dy+r][dx+s] * w[r*5+s]
__device__ __forceinline__ void window_fma(const float (&pt)[6][6], const float (&w)[28], float (&acc)[4]) {
#pragma unroll
  for (int r = 0; r < 5; ++r)
#pragma unroll
    for (int s = 0; s < 5; ++s) {
      const float wv = w[r * 5 + s];
      acc[0] = fmaf(wv, pt[r][s], acc[0]);
      acc[1] = fmaf(wv, pt[r][s + 1], acc[1]);
      acc[2] = fmaf(wv, pt[r + 1][s], acc[2]);
      acc[3] = fmaf(wv, pt[r + 1][s + 1], acc[3]);
    }
}
// 6x6 patch whose top-left corner is `p` (8-byte aligned, row stride `ld` floats, ld even)
__device__ __forceinline__ void load_patch(const float* p, int ld, float (&pt)[6][6]) {
#pragma unroll
  for (int r = 0; r < 6; ++r)
#pragma unroll
    for (int q = 0; q < 3; ++q) {
      const float2 v = *reinterpret_cast<const float2*>(p + r * ld + 2 * q);
      pt[r][2 * q] = v.x; pt[r][2 * q + 1] = v.y;
    }
}
__device__ __forceinline__ void load_w28(const float* p, float (&w)[28]) {
#pragma unroll
  for (int q = 0; q < 7; ++q) {
    const float4 v = *reinterpret_cast<const float4*>(p + 4 * q);
    w[4 * q] = v.x; w[4 * q + 1] = v.y; w[4 * q + 2] = v.z; w[4 * q + 3] = v.w;
  }
}
// max-pool of a window's four pre-bias values (first maximum wins, like maxpool2x2_fwd_kernel), then bias + ReLU
__device__ __forceinline__ float pool4(const float (&a)[4], float bias, int& bi) {
  float best = a[0]; bi = 0;
  if (a[1] > best) { best = a[1]; bi = 1; }
  if (a[2] > best) { best = a[2]; bi = 2; }
  if (a[3] > best) { best = a[3]; bi = 3; }
  return fmaxf(best + bias, 0.f);
}

// ------------------------------------------------------------------------------------------------------------------ forward
struct CnnFwdSmem {
  __align__(16) float sx[CD_H * CD_H];
  __align__(16) float sw0[4 * CD_W1PAD];
  float sb0[4];
  __align__(16) float sa1[CD_C1 * CD_P1 * CD_P1];
  __align__(16) float sw1[8 * CD_C1 * CD_W1PAD];
  float sb1[8];
  __align__(16) float spart[4 * 64 * 8];
};

// Both convolutions of image b in CTA g of its four, IMGS images per cluster (the four CTAs of image b are cluster ranks bl + IMGS r,
// bl = b % IMGS).  CTA (b, g) computes conv0 channels [4g, 4g+4) and stores them into the conv0 map of all four CTAs of its image
// (distributed shared memory), then conv1 for output channels [8g, 8g+8) over all 16.  Returns, in threads tid < 128, the pooled conv1
// value that thread stored to a2 and its offset within the image's 512 (channel * 16 + window).  The kernel arms whatever its cluster
// needs before this body's start-up cluster barrier.
// TRAIN = false (inference): none of the stores the backward pass needs (a1, idx1, a2, idx2, carry, x_keep), and the image is read from
// x[min(b, n_img - 1)], so that the missing second image of an odd batch's last cluster reads nothing past the batch.
template <int IMGS, bool TRAIN = true>
__device__ __forceinline__ float cnn_fwd_convs(CnnFwdSmem& s, const float* __restrict__ x, const float* __restrict__ w0,
                                               const float* __restrict__ b0, const float* __restrict__ w1, const float* __restrict__ b1,
                                               float* __restrict__ a1, unsigned char* __restrict__ idx1, float* __restrict__ a2,
                                               unsigned char* __restrict__ idx2, const float* __restrict__ carry_src, float* __restrict__ carry_dst,
                                               int carry_n, float* __restrict__ x_keep, unsigned long long* dbg, int& a2_off, int n_img = 0) {
  float* sx = s.sx; float* sw0 = s.sw0; float* sb0 = s.sb0; float* sa1 = s.sa1; float* sw1 = s.sw1; float* sb1 = s.sb1; float* spart = s.spart;
  cg::cluster_group cluster = cg::this_cluster();
  const bool dbg_on = dbg != nullptr && blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0;
  auto stamp = [&](int slot) { if (dbg_on) { unsigned long long t; asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t)); dbg[slot] = t; } };
  // the conv0 stores below go into the other CTAs' shared memory, which must exist by then: arrive now, wait after the staging
  cluster.barrier_arrive();
  pdl_wait();
  pdl_launch();
  const int b = blockIdx.x, g = blockIdx.y, tid = threadIdx.x, bl = b % IMGS;     // g == the image's rank among its four CTAs
  // look-ahead steps: this launch is the tail of the previous batch's step; it hands the labels that arrived with its image batch over to
  // the buffer the classifier head of the NEXT launch reads (a 128-byte side job instead of a copy node in the step graph)
  if (TRAIN && carry_n > 0 && b == 0 && g == 0) for (int i = tid; i < carry_n; i += 256) carry_dst[i] = carry_src[i];
  const int bx = TRAIN ? b : min(b, n_img - 1);
  for (int i = tid; i < CD_H * CD_H / 4; i += 256) cpa16(sx + 4 * i, x + (long long)bx * CD_H * CD_H + 4 * i);
  if (tid < 4 * 25) { const int cl = tid / 25, t = tid - cl * 25; cpa4(sw0 + cl * CD_W1PAD + t, w0 + 4 * g * 25 + tid); }
  if (tid < 4 * 3) sw0[(tid / 3) * CD_W1PAD + 25 + tid % 3] = 0.f;                                   // pad taps 25..27
  if (tid < 4) sb0[tid] = b0[4 * g + tid];
  {
    const float* wsrc = w1 + (long long)(8 * g) * CD_C1 * 25;      // the 8 output channels of this CTA: 3200 contiguous floats
    for (int i = tid; i < 8 * CD_C1 * 25; i += 256) { const int r = i / 25, t = i - r * 25; cpa4(sw1 + r * CD_W1PAD + t, wsrc + i); }
    for (int i = tid; i < 8 * CD_C1 * 3; i += 256) sw1[(i / 3) * CD_W1PAD + 25 + i % 3] = 0.f;
  }
  if (tid < 8) sb1[tid] = b1[8 * g + tid];
  cpa_wait_all();
  __syncthreads();
  cluster.barrier_wait();
  stamp(1);
  // look-ahead steps: the backward pass of this batch runs in the NEXT launch, after the following batch has overwritten x — keep a copy
  if (TRAIN && x_keep != nullptr && g == 0) for (int i = tid; i < CD_H * CD_H / 4; i += 256)
    reinterpret_cast<float4*>(x_keep + (long long)b * CD_H * CD_H)[i] = reinterpret_cast<const float4*>(sx)[i];
  // ---- conv0 + bias + ReLU + pool of this CTA's 4 channels: thread -> channel 4g + tid/64, windows (tid%64) + 64 j
  {
    const int cl = tid >> 6, sub = tid & 63, ch = 4 * g + cl;
    float w[28];
    load_w28(sw0 + cl * CD_W1PAD, w);
    const float bias = sb0[cl];
#pragma unroll 1
    for (int win = sub; win < CD_P1 * CD_P1; win += 64) {
      const int ph = win / CD_P1, pw = win - ph * CD_P1;
      float pt[6][6];
      load_patch(sx + (2 * ph) * CD_H + 2 * pw, CD_H, pt);
      float acc[4] = {0.f, 0.f, 0.f, 0.f};
      window_fma(pt, w, acc);
      int bi;
      const float v = pool4(acc, bias, bi);
#pragma unroll
      for (int r = 0; r < 4; ++r) cluster.map_shared_rank(sa1, r * IMGS + bl)[ch * CD_P1 * CD_P1 + win] = v;
      if (TRAIN) {
        const long long o = ((long long)b * CD_C1 + ch) * (CD_P1 * CD_P1) + win;
        a1[o] = v; idx1[o] = (unsigned char)bi;
      }
    }
  }
  cluster.sync();      // all 16 conv0 channels of image b are in every CTA's sa1
  stamp(2);
  // ---- conv1: thread -> input-channel quarter cq, output-channel pair op, pooling window win; 2 oc x 4 pixels accumulators
  {
    const int cq = tid >> 6, t64 = tid & 63, op = t64 >> 4, win = t64 & 15, ph = win >> 2, pw = win & 3;
    float acc0[4] = {0.f, 0.f, 0.f, 0.f}, acc1[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll 1
    for (int cc = 0; cc < 4; ++cc) {
      const int c = 4 * cq + cc;
      float pt[6][6], w[28];
      load_patch(sa1 + c * (CD_P1 * CD_P1) + (2 * ph) * CD_P1 + 2 * pw, CD_P1, pt);
      load_w28(sw1 + ((2 * op) * CD_C1 + c) * CD_W1PAD, w);
      window_fma(pt, w, acc0);
      load_w28(sw1 + ((2 * op + 1) * CD_C1 + c) * CD_W1PAD, w);
      window_fma(pt, w, acc1);
    }
    float4* dst = reinterpret_cast<float4*>(spart + (cq * 64 + t64) * 8);
    dst[0] = make_float4(acc0[0], acc0[1], acc0[2], acc0[3]);
    dst[1] = make_float4(acc1[0], acc1[1], acc1[2], acc1[3]);
  }
  __syncthreads();
  stamp(3);
  float v = 0.f;
  a2_off = 0;
  if (tid < 128) {
    const int i64 = tid >> 1, which = tid & 1, op = i64 >> 4, win = i64 & 15, ol = 2 * op + which;
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int cq = 0; cq < 4; ++cq) {
      const float4 t = *reinterpret_cast<const float4*>(spart + (cq * 64 + i64) * 8 + which * 4);
      acc[0] += t.x; acc[1] += t.y; acc[2] += t.z; acc[3] += t.w;
    }
    int bi;
    v = pool4(acc, sb1[ol], bi);
    a2_off = (8 * g + ol) * (CD_P2 * CD_P2) + win;
    if (TRAIN) {
      const long long o = (long long)b * CD_C2 * (CD_P2 * CD_P2) + a2_off;
      a2[o] = v; idx2[o] = (unsigned char)bi;
    }
  }
  return v;
}

// grid (B, 4), 256 threads, clusters of (1, 4, 1): the four CTAs of image b
__global__ void __cluster_dims__(1, 4, 1) __launch_bounds__(256)
    cnn_fwd_kernel(const float* __restrict__ x, const float* __restrict__ w0, const float* __restrict__ b0, const float* __restrict__ w1,
                   const float* __restrict__ b1, float* __restrict__ a1, unsigned char* __restrict__ idx1, float* __restrict__ a2,
                   unsigned char* __restrict__ idx2, const float* __restrict__ carry_src, float* __restrict__ carry_dst, int carry_n,
                   float* __restrict__ x_keep, unsigned long long* dbg) {
  __shared__ CnnFwdSmem s;
  const bool dbg_on = dbg != nullptr && blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0;
  auto stamp = [&](int slot) { if (dbg_on) { unsigned long long t; asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t)); dbg[slot] = t; } };
  stamp(0);
  int a2_off;
  cnn_fwd_convs<1>(s, x, w0, b0, w1, b1, a1, idx1, a2, idx2, carry_src, carry_dst, carry_n, x_keep, dbg, a2_off);
  stamp(4);
}

// ---- the same convolutions, followed by the first dense layer of the head: a3 = relu(a2 Wd^T + bd), Wd [256][512].  dense0 is
// row-separable (a3[b] needs only a2[b]), so it runs on the forward grid instead of the 16 SMs of the dense-chain cluster.
// grid (B, 4), B even, 256 threads, clusters of (2, 4, 1): the four CTAs of images b0 and b0 + 1 (b0 even; conv0 is shared within each
// image's four).  After the conv1 epilogue every CTA pushes its 128 a2 values (st.async, transaction mbarrier) into the a2 buffer of all 8
// CTAs; cluster rank r then computes a3[b0 .. b0+1][32 r .. 32 r + 32]: 8 threads per output column, each over every 8th float4 of the
// column's W0 row (its K-segment; 8 neighbouring lanes read 128 contiguous bytes of the row, and distinct 16-byte chunks of a2 in shared
// memory), every W0 load used for both images; the 8 partials are summed in a fixed shuffle order.
struct CnnFwdDense0Smem {
  CnnFwdSmem conv;
  __align__(16) float a2[2 * CD_C2 * CD_P2 * CD_P2];   // both images' a2, as pushed by the 8 CTAs
  uint64_t bar_a2;
};
constexpr int CD_D1 = 256, CD_D0 = CD_C2 * CD_P2 * CD_P2;    // dense0: 512 -> 256
constexpr int CD_D2 = 128, CD_NC = 10;                       // dense1: 256 -> 128, classifier: 128 -> 10

// thread 0, before cnn_fwd_convs: arms the a2 buffer and has the first cluster prefetch W0 into L2
__device__ __forceinline__ void fwd_dense0_arm(CnnFwdDense0Smem& s, const float* __restrict__ wd) {
  // the a2 buffer expects all 1024 floats; the peers push only after the body's start-up cluster barrier, so it is armed in time
  mbar_init(&s.bar_a2, 1);
  mbar_arrive_expect_tx(&s.bar_a2, 2 * CD_D0 * 4);
  fence_barrier_init();
  // W0 into L2 now: it is read at the very end of the kernel, and the step may start with L2 cold.  The first cluster prefetches it (each
  // CTA its 64 KB, rows 32 r .. 32 r + 31) and every cluster reads it from L2.  (Every cluster prefetching its own copy was measured
  // 0.4 us slower per step: 8 MiB of prefetch traffic at B = 32 slowed the staging of the images.)
  if (blockIdx.x < 2) {
    const float* slice = wd + (long long)32 * cg::this_cluster().block_rank() * CD_D0;
    for (int k = 0; k < 4; ++k)
      asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(slice + k * 8 * CD_D0), "r"(8 * CD_D0 * 4) : "memory");
  }
}

// after cnn_fwd_convs<2> (v, a2_off: what it returned): the a2 hand-off to all 8 CTAs and dense0 of the cluster's two images.  The threads
// with j = tid % 8 < 2 call store(j, a3[bpair + j][32 cr + tid / 8]) (cr = cluster rank).
template <class Store>
__device__ __forceinline__ void fwd_dense0(CnnFwdDense0Smem& s, float v, int a2_off, int cr, const float* __restrict__ wd,
                                          const float* __restrict__ bd, unsigned long long* dbg, Store store) {
  const bool dbg_on = dbg != nullptr && blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0;
  auto stamp = [&](int slot) { if (dbg_on) { unsigned long long t; asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t)); dbg[slot] = t; } };
  const int tid = threadIdx.x, bl = blockIdx.x & 1;
  const float* wrow = wd + (long long)(32 * cr + (tid >> 3)) * CD_D0;   // the W0 row of this thread's output column
  // ---- a2 hand-off: lane 2 win + which holds window win of channel 8g + 2 op + which (op = warp); lanes 8k + which + {0, 2, 4, 6} hold
  // windows 4k .. 4k + 3 of one channel, gathered into one float4 push
  if (tid < 128) {
    const float v1 = __shfl_down_sync(0xffffffffu, v, 2), v2 = __shfl_down_sync(0xffffffffu, v, 4), v3 = __shfl_down_sync(0xffffffffu, v, 6);
    if ((tid & 6) == 0) push_all<8>(s.a2, bl * CD_D0 + a2_off, &s.bar_a2, cr, make_float4(v, v1, v2, v3));
  }
  // ---- dense0: thread -> column n = 32 r + tid / 8, K-segment j = tid % 8: float4 chunks j, j + 8, ... of the row (k = 32 q + 4 j)
  const int j = tid & 7;
  const float bias = __ldg(bd + 32 * cr + (tid >> 3));
  constexpr int NB = 8;   // float4 of W0 in flight per thread: two batches cover the row segment (16 float4), in 32 of the 64 registers
  float4 w[NB];
#pragma unroll
  for (int i = 0; i < NB; ++i) w[i] = __ldg(reinterpret_cast<const float4*>(wrow) + 8 * i + j);   // first batch: in flight while a2 lands
  wait_landed(&s.bar_a2);
  stamp(5);
  float acc0 = 0.f, acc1 = 0.f;
#pragma unroll 1
  for (int q0 = 0; q0 < CD_D0 / 32; q0 += NB) {
    if (q0 > 0) {
#pragma unroll
      for (int i = 0; i < NB; ++i) w[i] = __ldg(reinterpret_cast<const float4*>(wrow) + 8 * (q0 + i) + j);
    }
#pragma unroll
    for (int i = 0; i < NB; ++i) {
      const float4 x0 = reinterpret_cast<const float4*>(s.a2)[8 * (q0 + i) + j];
      const float4 x1 = reinterpret_cast<const float4*>(s.a2 + CD_D0)[8 * (q0 + i) + j];
      acc0 = fmaf(w[i].x, x0.x, acc0); acc0 = fmaf(w[i].y, x0.y, acc0); acc0 = fmaf(w[i].z, x0.z, acc0); acc0 = fmaf(w[i].w, x0.w, acc0);
      acc1 = fmaf(w[i].x, x1.x, acc1); acc1 = fmaf(w[i].y, x1.y, acc1); acc1 = fmaf(w[i].z, x1.z, acc1); acc1 = fmaf(w[i].w, x1.w, acc1);
    }
  }
#pragma unroll
  for (int o = 4; o > 0; o >>= 1) {
    acc0 += __shfl_xor_sync(0xffffffffu, acc0, o);
    acc1 += __shfl_xor_sync(0xffffffffu, acc1, o);
  }
  if (j < 2) store(j, fmaxf((j == 0 ? acc0 : acc1) + bias, 0.f));
}

// ---- dense1 and the classifier in the same clusters: the part cnn_eval_kernel and the training head of cnn_fwd_dense0_kernel share.
//   dense1       every CTA pushes its 32 a3 columns of both images into all 8 CTAs (st.async, second transaction mbarrier); cluster rank r
//                computes a4[.][16 r .. 16 r + 16): 16 threads per column, each over every 16th float4 of the column's W1 row, summed in a
//                fixed shuffle order (W1, 128 KB, is read from L2 by every cluster)
//   a4 hand-off  every CTA pushes its 16 a4 columns of both images into all 8 CTAs (third mbarrier)
//   logits       16 threads per logit (thread t < 160: class t / 16, float4 chunks j and j + 16 of its W2 row), fixed shuffle order
struct CnnHeadSmem {
  CnnFwdDense0Smem d0;
  __align__(16) float a3[2 * CD_D1];        // both images' a3, as pushed by the 8 CTAs
  __align__(16) float a4[2 * CD_D2];        // both images' a4, as pushed by the 8 CTAs
  __align__(16) float a3own[2 * 32];        // this CTA's a3 columns of both images, gathered into float4 pushes
  __align__(16) float a4own[2 * 16];        // ... and its a4 columns
  float logit[2 * 16];                      // [image][class]
  uint64_t bar_a3, bar_a4;
};

// thread 0, before fwd_dense0_arm (whose barrier-init fence covers these barriers too): arms the a3 and a4 buffers, and has the first cluster
// prefetch W1 (each CTA its 16 KB, rows 16 r .. 16 r + 15) and W2 into L2, as fwd_dense0_arm does for W0
__device__ __forceinline__ void fwd_head_arm(CnnHeadSmem& s, const float* __restrict__ wd1, const float* __restrict__ wd2) {
  mbar_init(&s.bar_a3, 1);
  mbar_arrive_expect_tx(&s.bar_a3, 2 * CD_D1 * 4);
  mbar_init(&s.bar_a4, 1);
  mbar_arrive_expect_tx(&s.bar_a4, 2 * CD_D2 * 4);
  if (blockIdx.x < 2) {
    const int r = (int)cg::this_cluster().block_rank();
    asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(wd1 + (long long)16 * r * CD_D1), "r"(16 * CD_D1 * 4) : "memory");
    if (r == 0) asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(wd2), "r"(CD_NC * CD_D2 * 4) : "memory");
  }
}

// after fwd_dense0 has left this CTA's a3 columns of both images in s.a3own: the a3 hand-off and dense1.  Leaves this CTA's a4 columns in
// s.a4own; the caller then runs fwd_a4_handoff (loads it issues in between are in flight while a4 is gathered).
__device__ __forceinline__ void fwd_dense1(CnnHeadSmem& s, int cr, const float* __restrict__ wd1, const float* __restrict__ bd1,
                                           unsigned long long* dbg) {
  const bool dbg_on = dbg != nullptr && blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0;
  auto stamp = [&](int slot) { if (dbg_on) { unsigned long long t; asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t)); dbg[slot] = t; } };
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  // ---- a3 hand-off: warp w wrote columns 32 r + 4 w .. 4 w + 3 of both images; its lanes 0 and 1 push those of image 0 and 1
  __syncwarp();
  if (lane < 2) push_all<8>(s.a3, lane * CD_D1 + 32 * cr + 4 * warp, &s.bar_a3, cr, reinterpret_cast<const float4*>(s.a3own)[lane * 8 + warp]);
  // ---- dense1: thread -> column n = 16 r + tid / 16, K-segment j = tid % 16: float4 chunks j, j + 16, j + 32, j + 48 of the row
  const int j = tid & 15, n = 16 * cr + (tid >> 4);
  const float* wrow = wd1 + (long long)n * CD_D1;
  float4 w[4];
#pragma unroll
  for (int q = 0; q < 4; ++q) w[q] = __ldg(reinterpret_cast<const float4*>(wrow) + 16 * q + j);   // in flight while a3 lands
  const float bias1 = __ldg(bd1 + n);
  wait_landed(&s.bar_a3);
  stamp(7);
  float acc0 = 0.f, acc1 = 0.f;
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const float4 x0 = reinterpret_cast<const float4*>(s.a3)[16 * q + j];
    const float4 x1 = reinterpret_cast<const float4*>(s.a3 + CD_D1)[16 * q + j];
    acc0 = fmaf(w[q].x, x0.x, acc0); acc0 = fmaf(w[q].y, x0.y, acc0); acc0 = fmaf(w[q].z, x0.z, acc0); acc0 = fmaf(w[q].w, x0.w, acc0);
    acc1 = fmaf(w[q].x, x1.x, acc1); acc1 = fmaf(w[q].y, x1.y, acc1); acc1 = fmaf(w[q].z, x1.z, acc1); acc1 = fmaf(w[q].w, x1.w, acc1);
  }
#pragma unroll
  for (int o = 8; o > 0; o >>= 1) {
    acc0 += __shfl_xor_sync(0xffffffffu, acc0, o);
    acc1 += __shfl_xor_sync(0xffffffffu, acc1, o);
  }
  if (j < 2) s.a4own[j * 16 + (tid >> 4)] = fmaxf((j == 0 ? acc0 : acc1) + bias1, 0.f);
}
// every CTA: returns once a4 of both images has landed in s.a4 (so that nothing is still pushed into its shared memory when it exits)
__device__ __forceinline__ void fwd_a4_handoff(CnnHeadSmem& s, int cr) {
  const int tid = threadIdx.x;
  __syncthreads();
  // 8 float4 (image tid / 4, columns 16 r + 4 (tid % 4) ..) into all 8 CTAs
  if (tid < 8) push_all<8>(s.a4, (tid >> 2) * CD_D2 + 16 * cr + 4 * (tid & 3), &s.bar_a4, cr, reinterpret_cast<const float4*>(s.a4own)[tid]);
  wait_landed(&s.bar_a4);
}
// the W2 row chunks of logit c: float4 j and j + 16 (j = tid % 16)
__device__ __forceinline__ void fwd_w2_row(const float* __restrict__ wd2, int c, int j, float4 (&w2)[2]) {
  w2[0] = __ldg(reinterpret_cast<const float4*>(wd2 + c * CD_D2) + j);
  w2[1] = __ldg(reinterpret_cast<const float4*>(wd2 + c * CD_D2) + 16 + j);
}
// logit c of the a4 row `a4r`, without its bias: the 16 threads of the logit (j = tid % 16) sum in a fixed shuffle order and all return it
__device__ __forceinline__ float fwd_logit(const float* a4r, const float4 (&w2)[2], int j) {
  const float4 x0 = reinterpret_cast<const float4*>(a4r)[j];
  const float4 x1 = reinterpret_cast<const float4*>(a4r)[16 + j];
  float acc = 0.f;
  acc = fmaf(w2[0].x, x0.x, acc); acc = fmaf(w2[0].y, x0.y, acc); acc = fmaf(w2[0].z, x0.z, acc); acc = fmaf(w2[0].w, x0.w, acc);
  acc = fmaf(w2[1].x, x1.x, acc); acc = fmaf(w2[1].y, x1.y, acc); acc = fmaf(w2[1].z, x1.z, acc); acc = fmaf(w2[1].w, x1.w, acc);
#pragma unroll
  for (int o = 8; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  return acc;
}

// ---- the training head of cnn_fwd_dense0_kernel.  Everything from a3 to dz3 is row-separable (only the weight gradients mix images), so the
// forward clusters compute it for their two images and the dense-chain cluster kernel is left with da2 = dz3 W0 only.
struct FwdHeadArgs {
  const float* wd1; const float* bd1; const float* wd2; const float* bd2;   // [128][256], [128], [10][128], [10]
  const float* label;                                                       // [B] class index as float
  float* loss; float* logits;                                               // [B], [B][10] (logits may be null)
  float* a4; float* dz4; float* dz3; float* dl;                              // [B][128], [B][128], [B][256], [B][16] (classes >= 10 zero)
};
struct CnnFwdHeadSmem {
  CnnHeadSmem h;
  __align__(16) float dz4[2 * CD_D2];       // both images' dz4, computed whole by every CTA
  __align__(16) float part[8 * 2 * 32];     // dz3 partial sums [warp][image][column]
  float dl[2 * 16];                         // both images' dlogits
};
static_assert(sizeof(CnnFwdHeadSmem) == CNN_FWD_DENSE0_SMEM_BYTES, "CNN_FWD_DENSE0_SMEM_BYTES (common.cuh) must match");

// After fwd_dense0 (this CTA's a3 columns in s.h.a3own): dense1 and the a4 hand-off, then on every CTA the logits, softmax-CE (the dense
// chain's, softmax_ce_quad) and the whole dz4 of the cluster's two images, and from dz4 this CTA's dz3 columns 32 r .. 32 r + 32: warp w
// sums over W1 rows 16 w .. 16 w + 15 (lane = column, so a warp reads 128 contiguous bytes of a row from L2), the 8 partials are added in
// warp order.  Stores this CTA's a4, dz4 and dz3 columns; ranks 0 and 1 store the loss, logits and dlogits of image bpair + rank.  Every
// output has one writer and a fixed summation order: two launches give the same bits.
// WEIGHTED: the dlogits of image b are scaled by coef[b] (the per-row gradient coefficient of a short or sample-weighted batch) where they
// are produced, so that dz4, dz3 and every weight gradient carry it; the loss stays unweighted.
template <bool WEIGHTED>
__device__ __forceinline__ void fwd_train_head(CnnFwdHeadSmem& s, const FwdHeadArgs& hd, int cr, int bpair, unsigned long long* dbg,
                                               const float* __restrict__ coef) {
  const bool dbg_on = dbg != nullptr && blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0;
  auto stamp = [&](int slot) { if (dbg_on) { unsigned long long t; asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t)); dbg[slot] = t; } };
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, j = tid & 15, c = tid >> 4;
  fwd_dense1(s.h, cr, hd.wd1, hd.bd1, dbg);
  float4 w2[2] = {make_float4(0.f, 0.f, 0.f, 0.f), make_float4(0.f, 0.f, 0.f, 0.f)};
  float bias2 = 0.f;
  if (c < CD_NC) { fwd_w2_row(hd.wd2, c, j, w2); bias2 = __ldg(hd.bd2 + c); }
  fwd_a4_handoff(s.h, cr);
  stamp(14);
  float w1c[16];                            // the dz3 operands W1[16 warp + k][32 r + lane], in flight during the classifier
#pragma unroll
  for (int k = 0; k < 16; ++k) w1c[k] = __ldg(hd.wd1 + (long long)(16 * warp + k) * CD_D1 + 32 * cr + lane);
  if (c < CD_NC) {
    const float l0 = fwd_logit(s.h.a4, w2, j) + bias2, l1 = fwd_logit(s.h.a4 + CD_D2, w2, j) + bias2;
    if (j == 0) { s.h.logit[c] = l0; s.h.logit[16 + c] = l1; }
  }
  __syncthreads();
  if (warp == 0) {
    // lanes 4 i + q (i < 2) hold classes 4 q .. 4 q + 3 of image i; lanes >= 8 repeat lanes 0 .. 7 (the shuffles take the whole warp)
    const int i = (lane >> 2) & 1, c0 = 4 * (lane & 3), b = bpair + i;
    float lg[4], dl[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) lg[k] = c0 + k < CD_NC ? s.h.logit[16 * i + c0 + k] : 0.f;
    const float loss = softmax_ce_quad(lg, CD_NC, (int)__ldg(hd.label + b), dl);
    if (WEIGHTED) {
      const float cb = __ldg(coef + b);
#pragma unroll
      for (int k = 0; k < 4; ++k) dl[k] = __fmul_rn(dl[k], cb);
    }
    if (lane < 8) {
      *reinterpret_cast<float4*>(s.dl + 16 * i + c0) = make_float4(dl[0], dl[1], dl[2], dl[3]);
      if (cr == i) {
        *reinterpret_cast<float4*>(hd.dl + (long long)b * 16 + c0) = make_float4(dl[0], dl[1], dl[2], dl[3]);
        if (c0 == 0) hd.loss[b] = loss;
        if (hd.logits != nullptr)
#pragma unroll
          for (int k = 0; k < 4; ++k) if (c0 + k < CD_NC) hd.logits[(long long)b * CD_NC + c0 + k] = lg[k];
      }
    }
  }
  __syncthreads();
  {
    // dz4[i][m] = relu'(a4[i][m]) * sum_c dl[i][c] * W2[c][m]: thread -> image tid / 128, column m = tid % 128 (c ascending, as the chain)
    const int i = tid >> 7, m = tid & (CD_D2 - 1);
    float d = 0.f;
#pragma unroll
    for (int cc = 0; cc < CD_NC; ++cc) d = fmaf(s.dl[16 * i + cc], __ldg(hd.wd2 + cc * CD_D2 + m), d);
    if (!(s.h.a4[i * CD_D2 + m] > 0.f)) d = 0.f;
    s.dz4[i * CD_D2 + m] = d;
    if ((m >> 4) == cr) hd.dz4[(long long)(bpair + i) * CD_D2 + m] = d;
    if (tid < 8)
      *reinterpret_cast<float4*>(hd.a4 + (long long)(bpair + (tid >> 2)) * CD_D2 + 16 * cr + 4 * (tid & 3)) = reinterpret_cast<const float4*>(s.h.a4own)[tid];
  }
  __syncthreads();
  {
    float acc0 = 0.f, acc1 = 0.f;
#pragma unroll
    for (int k = 0; k < 16; ++k) {
      acc0 = fmaf(s.dz4[16 * warp + k], w1c[k], acc0);
      acc1 = fmaf(s.dz4[CD_D2 + 16 * warp + k], w1c[k], acc1);
    }
    s.part[(2 * warp) * 32 + lane] = acc0;
    s.part[(2 * warp + 1) * 32 + lane] = acc1;
  }
  __syncthreads();
  if (tid < 64) {
    const int i = tid >> 5;
    float d = s.part[i * 32 + lane];
#pragma unroll
    for (int w = 1; w < 8; ++w) d += s.part[(2 * w + i) * 32 + lane];
    if (!(s.h.a3own[i * 32 + lane] > 0.f)) d = 0.f;
    hd.dz3[(long long)(bpair + i) * CD_D1 + 32 * cr + lane] = d;
  }
  stamp(15);
}

// grid (B, 4), B even, 256 threads, clusters of (2, 4, 1).  Without the head's outputs (hd.a4 == nullptr) it ends with a3 (stamps 5 a2 landed,
// 6 a3 stored); with them it also runs fwd_train_head (stamps 7 a3 landed, 14 a4 landed, 15 dz3 stored).  Slot 4 is the end of the kernel.
// Instantiated twice: cnn_fwd_dense0_kernel (WEIGHTED = false) compiles to the code it had before the weighted head existed;
// cnn_fwd_dense0_weighted_kernel scales the dlogits by coef.
template <bool WEIGHTED>
__device__ __forceinline__ void cnn_fwd_dense0_body(const float* __restrict__ x, const float* __restrict__ w0, const float* __restrict__ b0,
                                                    const float* __restrict__ w1, const float* __restrict__ b1, const float* __restrict__ wd,
                                                    const float* __restrict__ bd, float* __restrict__ a1, unsigned char* __restrict__ idx1,
                                                    float* __restrict__ a2, unsigned char* __restrict__ idx2, float* __restrict__ a3,
                                                    const float* __restrict__ carry_src, float* __restrict__ carry_dst, int carry_n,
                                                    float* __restrict__ x_keep, unsigned long long* dbg, const FwdHeadArgs& hd,
                                                    const float* __restrict__ coef) {
  __shared__ CnnFwdHeadSmem s;
  const bool dbg_on = dbg != nullptr && blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0;
  auto stamp = [&](int slot) { if (dbg_on) { unsigned long long t; asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t)); dbg[slot] = t; } };
  stamp(0);
  const bool head = hd.a4 != nullptr;
  if (threadIdx.x == 0) {
    if (head) fwd_head_arm(s.h, hd.wd1, hd.wd2);
    fwd_dense0_arm(s.h.d0, wd);
  }
  int a2_off;
  const float v = cnn_fwd_convs<2>(s.h.d0.conv, x, w0, b0, w1, b1, a1, idx1, a2, idx2, carry_src, carry_dst, carry_n, x_keep, dbg, a2_off);
  // (computed after the convolutions, which need every register they can get)
  const int tid = threadIdx.x, cr = (int)cg::this_cluster().block_rank(), bl = blockIdx.x & 1, bpair = blockIdx.x - bl;
  fwd_dense0(s.h.d0, v, a2_off, cr, wd, bd, dbg, [&](int j, float y) {
    a3[(long long)(bpair + j) * CD_D1 + 32 * cr + (tid >> 3)] = y;
    s.h.a3own[j * 32 + (tid >> 3)] = y;
  });
  stamp(6);
  if (head) fwd_train_head<WEIGHTED>(s, hd, cr, bpair, dbg, coef);
  stamp(4);      // (slot 4 stays the end of the forward kernel)
}

__global__ void __cluster_dims__(2, 4, 1) __launch_bounds__(256, 4)   // <= 64 registers: fits beside a dense_tail_kernel CTA
    cnn_fwd_dense0_kernel(const float* __restrict__ x, const float* __restrict__ w0, const float* __restrict__ b0, const float* __restrict__ w1,
                          const float* __restrict__ b1, const float* __restrict__ wd, const float* __restrict__ bd, float* __restrict__ a1,
                          unsigned char* __restrict__ idx1, float* __restrict__ a2, unsigned char* __restrict__ idx2, float* __restrict__ a3,
                          const float* __restrict__ carry_src, float* __restrict__ carry_dst, int carry_n, float* __restrict__ x_keep,
                          unsigned long long* dbg, const FwdHeadArgs hd) {
  cnn_fwd_dense0_body<false>(x, w0, b0, w1, b1, wd, bd, a1, idx1, a2, idx2, a3, carry_src, carry_dst, carry_n, x_keep, dbg, hd, nullptr);
}

// coef [B]: the gradient coefficient of each row (see fwd_train_head); always launched with the head
__global__ void __cluster_dims__(2, 4, 1) __launch_bounds__(256, 4)   // <= 64 registers, as its unweighted twin
    cnn_fwd_dense0_weighted_kernel(const float* __restrict__ x, const float* __restrict__ w0, const float* __restrict__ b0,
                                   const float* __restrict__ w1, const float* __restrict__ b1, const float* __restrict__ wd,
                                   const float* __restrict__ bd, float* __restrict__ a1, unsigned char* __restrict__ idx1, float* __restrict__ a2,
                                   unsigned char* __restrict__ idx2, float* __restrict__ a3, const float* __restrict__ carry_src,
                                   float* __restrict__ carry_dst, int carry_n, float* __restrict__ x_keep, unsigned long long* dbg,
                                   const FwdHeadArgs hd, const float* __restrict__ coef) {
  cnn_fwd_dense0_body<true>(x, w0, b0, w1, b1, wd, bd, a1, idx1, a2, idx2, a3, carry_src, carry_dst, carry_n, x_keep, dbg, hd, coef);
}

// ------------------------------------------------------------------------------------------------------------------ inference
// The whole forward pass of N images (any N >= 1) and its per-sample scores, in one launch: grid (N rounded up to even, 4), clusters of
// (2, 4, 1) as in cnn_fwd_dense0_kernel, whose convolutions (without the stores only training needs), dense0 and dense1 it runs.  Then
// rank i < 2 (the g = 0 CTA of image bpair + i) computes that image's 10 logits, softmax-CE with fp32 expf / logf and the arg-max (first
// maximum wins, like torch.argmax).
// The missing second image of an odd N's last cluster is computed from a copy of image N - 1 and takes part in every push; nothing of it is
// written.  No atomics: two launches on the same inputs give the same bits.
__global__ void __cluster_dims__(2, 4, 1) __launch_bounds__(256)
    cnn_eval_kernel(const float* __restrict__ x, const float* __restrict__ w0, const float* __restrict__ b0, const float* __restrict__ w1,
                    const float* __restrict__ b1, const float* __restrict__ wd0, const float* __restrict__ bd0, const float* __restrict__ wd1,
                    const float* __restrict__ bd1, const float* __restrict__ wd2, const float* __restrict__ bd2, const float* __restrict__ label,
                    float* __restrict__ logits, float* __restrict__ loss, int* __restrict__ pred, int* __restrict__ correct, int N) {
  __shared__ CnnHeadSmem s;
  if (threadIdx.x == 0) {
    fwd_head_arm(s, wd1, wd2);
    fwd_dense0_arm(s.d0, wd0);
  }
  int a2_off;
  const float v = cnn_fwd_convs<2, false>(s.d0.conv, x, w0, b0, w1, b1, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, 0, nullptr, nullptr,
                                          a2_off, N);
  const int tid = threadIdx.x, cr = (int)cg::this_cluster().block_rank(), j = tid & 15, c = tid >> 4;
  fwd_dense0(s.d0, v, a2_off, cr, wd0, bd0, nullptr, [&](int jj, float y) { s.a3own[jj * 32 + (tid >> 3)] = y; });
  fwd_dense1(s, cr, wd1, bd1, nullptr);
  // classifier operands in flight while a4 is gathered
  float4 w2[2] = {make_float4(0.f, 0.f, 0.f, 0.f), make_float4(0.f, 0.f, 0.f, 0.f)};
  float bias2 = 0.f;
  if (cr < 2 && c < CD_NC) { fwd_w2_row(wd2, c, j, w2); bias2 = __ldg(bd2 + c); }
  fwd_a4_handoff(s, cr);
  if (cr >= 2) return;
  const int b = (blockIdx.x & ~1) + cr;      // ranks 0 and 1 are the g = 0 CTAs of images bpair and bpair + 1
  if (c < CD_NC) {
    const float acc = fwd_logit(s.a4 + cr * CD_D2, w2, j);
    if (j == 0) {
      s.logit[c] = acc + bias2;
      if (logits != nullptr && b < N) logits[(long long)b * CD_NC + c] = acc + bias2;
    }
  }
  __syncthreads();
  if (tid == 0 && b < N) {
    float mx = s.logit[0];
    int am = 0;
#pragma unroll
    for (int k = 1; k < CD_NC; ++k) if (s.logit[k] > mx) { mx = s.logit[k]; am = k; }
    pred[b] = am;
    if (label != nullptr) {
      float se = 0.f;
#pragma unroll
      for (int k = 0; k < CD_NC; ++k) se += expf(s.logit[k] - mx);
      // a label that is not an integer in [0, 10) (NaN included) scores NaN and is never counted correct; it indexes nothing
      const float yl = label[b];
      const bool ok = yl >= 0.f && yl < (float)CD_NC && yl == truncf(yl);
      const int yi = ok ? (int)yl : 0;
      loss[b] = ok ? -(s.logit[yi] - mx - logf(se)) : __int_as_float(0x7fc00000);
      correct[b] = ok && yi == am ? 1 : 0;
    }
  }
}

// ------------------------------------------------------------------------------------------------------------------ backward (data + conv0)
// grid (B, 4), 288 threads.  CTA (b, cg): conv1-input channels [4cg, 4cg+4) of image b.
//   dz2 (32 x 8 x 8) has at most one non-zero per 2x2 pooling window: at the window's arg-max, where a2 > 0.  Those non-zeros are listed per
//   window position (16 lists of up to 32 output channels) and da1 is gathered from them: an output pixel (y, x) of the 12x12 map can only be
//   reached by the 3x3 pooling windows around window (y/2 - 1, x/2 - 1), so it runs over those lists, i.e. over the non-zeros only.  The filter
//   planes are zero-padded to 7x7, so that the one or two arg-max positions of a window that fall just outside a pixel's 5x5 footprint add 0
//   instead of needing a test.  da1 never leaves shared memory: it is max-pool / ReLU routed straight into conv0's weight and bias gradient (the
//   first layer needs no input gradient).
struct CnnBwdSmem {
  static constexpr int WT = 0;                                   // [2 cl pairs][32 oc][7][7] float2: W1[oc][4cg+2cp+{0,1}][r-1][s-1], 0 on the border
  static constexpr int X = WT + 2 * CD_C2 * 49 * 2;              // [28][28]
  static constexpr int A1 = X + CD_H * CD_H;                     // [4][144] pooled conv0 activations (ReLU mask)
  static constexpr int DA1 = A1 + 4 * 144;                       // [4][144] -> routed gradient g
  static constexpr int POS = DA1 + 4 * 144;                      // [4][144] int: top-left of the arg-max pixel in the 24x24 map (as x offset)
  static constexpr int NZ = POS + 4 * 144;                       // [16 windows][32] float2 {dz2 value, weight offset oc*49 - (iy*7 + ix)}
  static constexpr int NZSRC = NZ + 16 * 32 * 2;                 // [16][32] int: oc*16 + window (index into the image's dz2 / da2)
  static constexpr int NZCNT = NZSRC + 16 * 32;                  // [16] int: list lengths
  static constexpr int TOTAL = NZCNT + 16;
  static constexpr int BYTES = TOTAL * 4;
};
constexpr int CNN_BWD_CTA_STAMPS = 320;   // CTAs of cnn_bwd_all_kernel that record (start, end, SM) in the debug buffer (see there)

__device__ __forceinline__ void cnn_bwd_body(float* sm, const int b, const int cg, const float* __restrict__ x, const float* __restrict__ w1,
                                             const float* __restrict__ a1, const unsigned char* __restrict__ idx1, const float* __restrict__ a2,
                                             const unsigned char* __restrict__ idx2, const float* __restrict__ da2, float* __restrict__ dw0,
                                             float* __restrict__ db0, unsigned long long* dbg) {
  using L = CnnBwdSmem;
  float* swt = sm + L::WT; float* sx = sm + L::X; float* sa1 = sm + L::A1; float* sda1 = sm + L::DA1;
  int* spos = reinterpret_cast<int*>(sm + L::POS); float2* snz = reinterpret_cast<float2*>(sm + L::NZ);
  int* snzsrc = reinterpret_cast<int*>(sm + L::NZSRC); int* snzcnt = reinterpret_cast<int*>(sm + L::NZCNT);
  const bool dbg_on = dbg != nullptr && b == 0 && cg == 0 && threadIdx.x == 0;
  auto stamp = [&](int slot) { if (dbg_on) { unsigned long long t; asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t)); dbg[slot] = t; } };
  stamp(8);
  const int tid = threadIdx.x;
  // swt[((cp*32 + oc)*49 + r*7 + s)*2 + k] = W1[oc][4cg + 2cp + k][r-1][s-1] for r, s in 1..5, 0 on the border of the 7x7 plane.  The taps are
  // copied in source order (100 contiguous floats per oc), so that a warp's loads are coalesced.
  for (int i = tid; i < CD_C2 * 4 * 25; i += 288) {
    const int oc = i / 100, rem = i - oc * 100, cl = rem / 25, tap = rem - cl * 25, r = tap / 5, t = tap - r * 5;
    cpa4(swt + (((cl >> 1) * CD_C2 + oc) * 49 + (r + 1) * 7 + t + 1) * 2 + (cl & 1), w1 + ((long long)oc * CD_C1 + 4 * cg) * 25 + rem);
  }
  for (int i = tid; i < 2 * CD_C2 * 24; i += 288) {          // the 24 border taps of every (cp, oc) plane: rows 0 and 6, then columns 0 and 6
    const int plane = i / 24, j = i - plane * 24;
    const int t7 = j < 7 ? j : j < 14 ? 42 + (j - 7) : j < 19 ? (j - 13) * 7 : (j - 18) * 7 + 6;
    reinterpret_cast<float2*>(swt)[plane * 49 + t7] = make_float2(0.f, 0.f);
  }
  stamp(25);
  for (int i = tid; i < CD_H * CD_H / 4; i += 288) cpa16(sx + 4 * i, x + (long long)b * CD_H * CD_H + 4 * i);
  for (int i = tid; i < 4 * 144 / 4; i += 288) cpa16(sa1 + 4 * i, a1 + ((long long)b * CD_C1 + 4 * cg) * 144 + 4 * i);
  for (int i = tid; i < 4 * 144; i += 288) {
    const long long o = ((long long)b * CD_C1 + 4 * cg) * 144 + i;
    const int win = i % 144, id = idx1[o];
    spos[i] = (2 * (win / CD_P1) + (id >> 1)) * CD_H + 2 * (win % CD_P1) + (id & 1);
  }
  stamp(26);
  // where dz2 can be non-zero (a2 > 0, at the arg-max idx2) is known from the forward pass: one warp per pooling window lists its output
  // channels in ascending order, with the weight offset that places the arg-max pixel; only the values (da2) wait for the grid dependency
  {
    const int oc = tid & 31, wa = tid >> 5, wb = wa + 9;      // 9 warps: windows wa and wa + 9 (< 16); all loads issued before the first ballot
    const long long oa = ((long long)b * CD_C2 + oc) * 16 + wa, ob = ((long long)b * CD_C2 + oc) * 16 + (wb < 16 ? wb : wa);
    const float ava = a2[oa], avb = a2[ob];
    const int ida = idx2[oa], idb = idx2[ob];
    auto list = [&](int w, float av, int id) {
      const unsigned m = __ballot_sync(0xffffffffu, av > 0.f);
      if (av > 0.f) {
        const int k = __popc(m & ((1u << oc) - 1u));
        snz[w * 32 + k].y = __int_as_float(oc * 49 - ((id >> 1) * 7 + (id & 1)));
        snzsrc[w * 32 + k] = oc * 16 + w;
      }
      if (oc == 0) snzcnt[w] = __popc(m);
    };
    list(wa, ava, ida);
    if (wb < 16) list(wb, avb, idb);
  }
  stamp(27);
  cpa_wait_all();
  __syncthreads();
  stamp(9);
  // Everything staged so far was produced by the forward kernel (complete long ago); da2 comes from the kernel right before this one.
  // The grid dependency is resolved HERE, so that with programmatic dependent launch these CTAs become resident on the SMs the 16-CTA
  // dense-chain cluster leaves idle and finish their staging while it is still running.
  pdl_wait();
  pdl_launch();
  // the non-zero values of dz2 (pool + ReLU backward of conv1's output)
  for (int e = tid; e < 16 * 32; e += 288)
    if ((e & 31) < snzcnt[e >> 5]) snz[e].x = da2[(long long)b * CD_C2 * 16 + snzsrc[e]];
  __syncthreads();
  stamp(10);
  // ---- conv1 data gradient, routed through conv0's ReLU: thread -> channel pair cp, pixel (y, x) = (2py + qy, 2px + qx) of the 12x12 map
  //   da1[c][y][x] = sum_{wh, ww} sum_{oc in list (wh, ww)} dz2 * W1[oc][c][y - oh][x - ow]   (windows and list entries in ascending order)
  // a pixel whose a1 <= 0 gets no gradient (the ReLU routes it to 0), so its sum is skipped.  Pixels with the same (qy, qx) share a warp.
  {
    const int cp = tid / 144, p = tid - cp * 144, q = p / 36, r = p - q * 36, qy = q >> 1, qx = q & 1, py = r / 6, px = r - py * 6;
    const int pix = (2 * py + qy) * CD_P1 + 2 * px + qx;
    const float m0 = sa1[(2 * cp) * 144 + pix], m1 = sa1[(2 * cp + 1) * 144 + pix];
    float acc0 = 0.f, acc1 = 0.f;
    if (m0 > 0.f || m1 > 0.f) {
      const float2* wcp = reinterpret_cast<const float2*>(swt) + cp * CD_C2 * 49;
      for (int wh = max(py - 2, 0); wh <= min(py, 3); ++wh)
        for (int ww = max(px - 2, 0); ww <= min(px, 3); ++ww) {
          // 7x7 tap of the window's top-left pixel: (dy + 1, dx + 1) with dy = y - 2wh in 0..5; the entry's offset subtracts the arg-max shift
          const float2* wp = wcp + (2 * (py - wh) + qy + 1) * 7 + 2 * (px - ww) + qx + 1;
          const float2* nz = snz + (wh * 4 + ww) * 32;
          const int n = snzcnt[wh * 4 + ww];
#pragma unroll 4
          for (int k = 0; k < n; ++k) {
            const float2 e = nz[k];
            const float2 wv = wp[__float_as_int(e.y)];
            acc0 = fmaf(e.x, wv.x, acc0);
            acc1 = fmaf(e.x, wv.y, acc1);
          }
        }
    }
    sda1[(2 * cp) * 144 + pix] = m0 > 0.f ? acc0 : 0.f;
    sda1[(2 * cp + 1) * 144 + pix] = m1 > 0.f ? acc1 : 0.f;
  }
  __syncthreads();
  stamp(11);
  stamp(12);     // (the ReLU routing is part of the data-gradient phase)
  // ---- conv0 weight / bias gradient of this image (4 channels): dW0[ch][kh][kw] += sum_windows g * x[oh+kh][ow+kw]
  // 200 threads: (tap, channel) x 2 halves of the 144 windows; four independent accumulators break the FMA dependency chain
  if (tid < 200) {
    const int half = tid / 100, t = tid - half * 100, cl = t / 25, tap = t % 25, koff = (tap / 5) * CD_H + tap % 5;
    const float* gp = sda1 + cl * 144 + half * 72;
    const int* pp = spos + cl * 144 + half * 72;
    float a0 = 0.f, a1_ = 0.f, a2_ = 0.f, a3 = 0.f;
#pragma unroll 2
    for (int p = 0; p < 72; p += 4) {
      a0 = fmaf(gp[p], sx[pp[p] + koff], a0);
      a1_ = fmaf(gp[p + 1], sx[pp[p + 1] + koff], a1_);
      a2_ = fmaf(gp[p + 2], sx[pp[p + 2] + koff], a2_);
      a3 = fmaf(gp[p + 3], sx[pp[p + 3] + koff], a3);
    }
    atomicAdd(dw0 + (4 * cg + cl) * 25 + tap, (a0 + a1_) + (a2_ + a3));
  } else if (tid >= 224 && tid < 228) {
    const int cl = tid - 224;
    float acc = 0.f;
    for (int p = 0; p < 144; ++p) acc += sda1[cl * 144 + p];
    atomicAdd(db0 + 4 * cg + cl, acc);
    if (dbg != nullptr && b == 0 && cg == 0 && cl == 0) { unsigned long long t; asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t)); dbg[28] = t; }
  }
  stamp(13);
}

// ------------------------------------------------------------------------------------------------------------------ conv1 weight gradient
// CTA (oc, cg, h), 256 threads, owns dW1[oc][4cg..4cg+3][5][5] (100 outputs, written once: no atomics) over images [h NI, (h+1) NI):
//   dW1[oc][c][kh][kw] = sum_{b, window} g[b][oc][window] * a1[b][c][oh+kh][ow+kw]     (g != 0 only at the window's arg-max where a2 > 0)
// PAIR: NI = B / 2 and the two CTAs h = 0, 1 of a cluster of two split the batch (half the staging, half the sums per CTA); h = 1 pushes its
// 100 partial sums (and db1's) into h = 0 (st.async, transaction mbarrier), which adds them in the order h0 + h1 and stores.  Otherwise
// NI = B, h = 0.  Where g can be non-zero (a2 > 0) is known from the forward pass: the staging lists those (image, window) entries in
// ascending order, with the arg-max pixel's offset into the staged planes, so that after the grid dependency only their da2 values are
// loaded and only they are summed.
__host__ __device__ constexpr int wgrad1_list(int ni) { return ni * 16 + 8; }       // entry list, padded for the 2 x 4-way split below
// dynamic shared memory of the body for NI images: planes, list values + positions, warp counts, partials, received partials, mbarrier
__host__ __device__ constexpr int wgrad1_smem_bytes(int ni) { return (ni * 576 + 2 * wgrad1_list(ni) + 16 + 256 + 128 + 4) * 4; }

__device__ __forceinline__ void cluster_arrive() { asm volatile("barrier.cluster.arrive;" ::: "memory"); }   // (release)
__device__ __forceinline__ void cluster_wait() { asm volatile("barrier.cluster.wait;" ::: "memory"); }       // (acquire)

template <bool PAIR>
__device__ __forceinline__ void cnn_wgrad1_body(float* sm, const int oc, const int cg, const int h, const float* __restrict__ a1,
                                                const float* __restrict__ a2, const unsigned char* __restrict__ idx2, const float* __restrict__ da2,
                                                float* __restrict__ dw1, float* __restrict__ db1, int B, unsigned long long* dbg) {
  const int ni = PAIR ? B / 2 : B, b0 = h * ni, L = wgrad1_list(ni);
  float* sa = sm;                                      // [ni][4][144] the four input-channel planes of every image
  float* sg = sa + ni * 576;                           // [L] listed entries: da2 offset (int bits) until the grid dependency, then g
  int* sp = reinterpret_cast<int*>(sg + L);            // [L] arg-max pixel as offset into sa (image * 576 + offset in a 12x12 plane)
  int* scnt = sp + L;                                  // [8] per-warp entry counts of one listing round
  float* sacc = reinterpret_cast<float*>(scnt + 16);   // [2][128]
  float* srecv = sacc + 256;                           // PAIR, h = 0: the partner's 100 partial sums, db1's at [100]
  uint64_t* bar = reinterpret_cast<uint64_t*>(srecv + 128);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const bool dbg_on = dbg != nullptr && oc == 0 && cg == 0 && h == 0 && tid == 0;
  auto stamp = [&](int slot) { if (dbg_on) { unsigned long long t; asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t)); dbg[slot] = t; } };
  stamp(16);
  if (PAIR) {
    if (h == 0 && tid == 0) {
      mbar_init(bar, 1);
      mbar_arrive_expect_tx(bar, (cg == 0 ? 26 : 25) * 16);    // 25 float4 of dW1 partials (+ one carrying db1's)
      fence_barrier_init();
    }
    cluster_arrive();        // h = 1 pushes only after its wait for this arrive: the barrier above is armed by then
  }
  for (int i = tid; i < ni * 144; i += 256) {          // 144 float4 per image: 4 contiguous planes
    const int bb = i / 144, r = i - bb * 144;
    cpa16(sa + 4 * i, a1 + ((long long)(b0 + bb) * CD_C1 + 4 * cg) * 144 + 4 * r);
  }
  // the list: rounds of 256 entries, each thread one entry, ranked by warp ballots and the counts of the warps before it
  int n = 0;
  for (int base = 0; base < ni * 16; base += 256) {
    const int e = base + tid, bb = e >> 4, win = e & 15;
    const int src = ((b0 + bb) * CD_C2 + oc) * 16 + win;
    const bool nz = e < ni * 16 && a2[src] > 0.f;
    const unsigned m = __ballot_sync(0xffffffffu, nz);
    if (lane == 0) scnt[warp] = __popc(m);
    __syncthreads();
    int k = n, tot = n;
#pragma unroll
    for (int w = 0; w < 8; ++w) { const int c = scnt[w]; k += w < warp ? c : 0; tot += c; }
    if (nz) {
      const int id = idx2[src];
      k += __popc(m & ((1u << lane) - 1u));
      sg[k] = __int_as_float(src);
      sp[k] = bb * 576 + (2 * (win >> 2) + (id >> 1)) * CD_P1 + 2 * (win & 3) + (id & 1);
    }
    n = tot;
    __syncthreads();         // (scnt is rewritten by the next round)
  }
  if (tid < 8) { sg[n + tid] = 0.f; sp[n + tid] = 0; }   // pad to a multiple of 8 with entries that add 0
  pdl_wait();            // (see cnn_bwd_body: only da2 depends on the preceding kernel)
  pdl_launch();
  for (int k = tid; k < n; k += 256) sg[k] = da2[__float_as_int(sg[k])];
  cpa_wait_all();
  __syncthreads();
  stamp(17);
  // thread -> (input channel cl, tap) = t < 100, half q of the list; four independent accumulators per thread
  const int q = tid >> 7, t = tid & 127, hn = ((n + 7) & ~7) >> 1;
  float acc = 0.f;
  if (t < 100) {
    const int cl = t / 25, tap = t % 25, koff = (tap / 5) * CD_P1 + tap % 5;
    float c0 = 0.f, c1 = 0.f, c2 = 0.f, c3 = 0.f;
    const float* sak = sa + cl * 144 + koff;
#pragma unroll 2
    for (int k = q * hn; k < (q + 1) * hn; k += 4) {    // hn is a multiple of 4: float4 / int4 reads of the list
      const float4 g = *reinterpret_cast<const float4*>(sg + k);
      const int4 p = *reinterpret_cast<const int4*>(sp + k);
      c0 = fmaf(g.x, sak[p.x], c0);
      c1 = fmaf(g.y, sak[p.y], c1);
      c2 = fmaf(g.z, sak[p.z], c2);
      c3 = fmaf(g.w, sak[p.w], c3);
    }
    acc = (c0 + c1) + (c2 + c3);
  }
  sacc[q * 128 + t] = acc;
  __syncthreads();
  float s = 0.f;                                       // warp 7, cg == 0: db1's part = sum of the listed routed gradients
  if (cg == 0 && warp == 7) {
    for (int k = lane; k < n; k += 32) s += sg[k];
    s = warp_sum(s);
  }
  float* dst = dw1 + ((long long)oc * CD_C1 + 4 * cg) * 25;
  if (!PAIR) {
    if (tid < 100) dst[tid] = sacc[tid] + sacc[128 + tid];
    if (cg == 0 && tid == 224) db1[oc] = s;
  } else if (h == 1) {
    cluster_wait();
    if (tid < 25) {
      const float4 v = make_float4(sacc[4 * tid] + sacc[128 + 4 * tid], sacc[4 * tid + 1] + sacc[129 + 4 * tid],
                                   sacc[4 * tid + 2] + sacc[130 + 4 * tid], sacc[4 * tid + 3] + sacc[131 + 4 * tid]);
      push_all<2, 1>(srecv, 4 * tid, bar, 1, v);
    }
    if (cg == 0 && tid == 224) push_all<2, 1>(srecv, 100, bar, 1, make_float4(s, 0.f, 0.f, 0.f));
  } else {
    cluster_wait();
    wait_landed(bar);
    if (tid < 100) dst[tid] = (sacc[tid] + sacc[128 + tid]) + srecv[tid];
    if (cg == 0 && tid == 224) db1[oc] = s + srecv[100];
  }
  stamp(18);
}

__global__ void __launch_bounds__(288) cnn_bwd_kernel(const float* x, const float* w1, const float* a1, const unsigned char* idx1, const float* a2,
                                                       const unsigned char* idx2, const float* da2, float* dw0, float* db0, unsigned long long* dbg) {
  extern __shared__ __align__(16) float sm[];
  cnn_bwd_body(sm, blockIdx.x, blockIdx.y, x, w1, a1, idx1, a2, idx2, da2, dw0, db0, dbg);
}
// grid (32 oc, 4 cg, 2 h), 256 threads, clusters of (1, 1, 2): the two CTAs that split the batch for one (oc, cg)
__global__ void __cluster_dims__(1, 1, 2) __launch_bounds__(256) cnn_wgrad1_kernel(const float* a1, const float* a2, const unsigned char* idx2,
                                                                                    const float* da2, float* dw1, float* db1, int B,
                                                                                    unsigned long long* dbg) {
  extern __shared__ __align__(16) float sm[];
  cnn_wgrad1_body<true>(sm, blockIdx.x, blockIdx.y, blockIdx.z, a1, a2, idx2, da2, dw1, db1, B, dbg);
}
// The whole convolution backward pass as ONE launch, in clusters of two CTAs: CTAs [0, 256) run the conv1 weight-gradient body (CTA
// 8 oc + 2 cg + h: pairs of CTAs that split the batch), CTAs [256, 256 + 4B) the data-gradient / conv0 body (CTA 256 + 4 b + cg; a cluster
// never mixes the two bodies, and the data-gradient CTAs do not use theirs).  Two independent jobs that read the same inputs; a single
// heterogeneous grid saves a stream fork / join in the step graph.  The grid's dynamic shared memory is the larger body's: at B <= 32 the
// data-gradient body's 41,344 bytes, so that the whole grid is resident at once (5 CTAs per SM, one beside each CTA of the dense-chain
// cluster) while the dense chain still runs, and every CTA has finished its staging when da2 arrives.
__global__ void __launch_bounds__(288) __cluster_dims__(2, 1, 1)
    cnn_bwd_all_kernel(const float* x, const float* w1, const float* a1, const unsigned char* idx1, const float* a2, const unsigned char* idx2,
                       const float* da2, float* dw0, float* db0, float* dw1, float* db1, int B, unsigned long long* dbg) {
  extern __shared__ __align__(16) float sm[];
  const int i = blockIdx.x;      // (the grid dependency is resolved inside the bodies, after their independent staging)
  // debug: the last CNN_BWD_CTA_STAMPS CTAs record (start, end, SM id) at dbg[64 + 3 k ..], k = i - (grid - CNN_BWD_CTA_STAMPS) (all CTAs of
  // a smaller grid: k = i), so that tools/step_timeline.py can show how the grid packs onto the SMs; slots stay below 64 + 3 * 320 = 1024
  unsigned long long t0 = 0;
  if (dbg != nullptr && threadIdx.x == 0) asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t0));
  if (i >= 8 * CD_C2) {
    const int j = i - 8 * CD_C2;
    cnn_bwd_body(sm, j >> 2, j & 3, x, w1, a1, idx1, a2, idx2, da2, dw0, db0, dbg);
  } else if (threadIdx.x < 256) {            // (no thread of this CTA takes the other branch, so its __syncthreads pair up among these 256)
    cnn_wgrad1_body<true>(sm, i >> 3, (i >> 1) & 3, i & 1, a1, a2, idx2, da2, dw1, db1, B, dbg);
  } else {                                   // threads 256..287 take part in the pair's cluster barrier, which would otherwise wait for them
    cluster_arrive();
    cluster_wait();
  }
  const int k = i - max((int)gridDim.x - CNN_BWD_CTA_STAMPS, 0);
  if (dbg != nullptr && threadIdx.x == 0 && k >= 0) {
    unsigned long long t1; unsigned smid;
    asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t1));
    asm volatile("mov.u32 %0, %smid;" : "=r"(smid));
    dbg[64 + 3 * k] = t0; dbg[65 + 3 * k] = t1; dbg[66 + 3 * k] = smid;
  }
}

// The convolution backward pass AND the exchange of the four conv keys (push -> both server tiers -> optimizer -> pull, the replicated one-hop
// mode of hips_fabric.cu's direct protocol) as ONE launch.  The bodies of cnn_bwd_all_kernel, without clusters: CTAs [0, 4B) data gradient,
// [4B, 4B+128) conv1 weight gradient, one CTA per (oc, cg) over the whole batch.  Every CTA takes a ticket when its
// gradients are written; the CTAs that draw the last `n_active` tickets wait until the ticket counter shows that the whole grid has finished
// and then each serve one 1024-float tile of the conv keys: gradient -> LL packets into every rank's slot, poll the packets of all ranks, sum
// in the hierarchy's order (party sums, push_scale, sum over parties), optimizer on this rank's replica of the server state, fresh weights
// into the parameter arena.  Compared with a separate exchange launch this removes the grid drain + launch between the last gradient store and
// the first packet: the tail CTAs are already running when the last gradient lands.
//   state words of the channel (FabricParams::state): [0] round, [1] tail completion counter, [2] optimizer step, [5] protocol error, [6] tickets.
// All 256 CTAs are co-resident (2 per SM on 132 SMs), so spinning on the ticket counter cannot starve the CTAs it waits for.
template <bool SCHED, bool EXT>
__global__ void __launch_bounds__(288) cnn_bwd_exchange_kernel(const float* x, const float* w1, const float* a1, const unsigned char* idx1, const float* a2,
                                                                const unsigned char* idx2, const float* da2, float* dw0, float* db0, float* dw1, float* db1,
                                                                int B, unsigned long long* dbg, const __grid_constant__ FabricParams p,
                                                                const int* __restrict__ tile_list, int n_active) {
  extern __shared__ __align__(16) float sm[];
  __shared__ int s_ticket;
  const int i = blockIdx.x;
  if (i < 4 * B) {
    cnn_bwd_body(sm, i >> 2, i & 3, x, w1, a1, idx1, a2, idx2, da2, dw0, db0, dbg);
  } else if (threadIdx.x < 256) {
    const int j = i - 4 * B;
    cnn_wgrad1_body<false>(sm, j >> 2, j & 3, 0, a1, a2, idx2, da2, dw1, db1, B, dbg);
  }
  if (threadIdx.x >= FAB_THREADS) return;                       // the exchange tail is written for 256 threads (one float4 of a tile each)
  // the channel's round / optimizer step (they can only advance after every CTA of this launch has drawn its ticket below)
  const uint32_t round = (uint32_t)(*reinterpret_cast<volatile int*>(p.state)) + 1u;
  const int opt_t = (*reinterpret_cast<volatile int*>(p.state + 2)) + 1;
  auto bar = [] { asm volatile("bar.sync 1, 256;" ::: "memory"); };
  bar();                                                         // every gradient store / atomic of this CTA has been issued
  if (threadIdx.x == 0) { __threadfence(); s_ticket = atomicAdd(p.state + 6, 1); }
  bar();
  const int first = (int)gridDim.x - n_active;
  if (s_ticket < first) return;
  const bool dbg_on = dbg != nullptr && s_ticket == first && threadIdx.x == 0;
  auto stamp = [&](int slot) { if (dbg_on) { unsigned long long t; asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t)); dbg[slot] = t; } };
  stamp(20);
  if (threadIdx.x == 0) {
    while (*reinterpret_cast<volatile int*>(p.state + 6) < (int)gridDim.x) {}
    __threadfence();
  }
  bar();
  stamp(21);
  const int t = tile_list[s_ticket - first];
  const uint32_t epoch = (round << 3) | (uint32_t)(p.channel_id & 7);
  int* err = p.state + 5;
  const int f = grad_fmt(fmt_of(p, t));
  const long long off = (long long)t * TILE + threadIdx.x * 4;
  float* g = p.grad[p.rank] + off;
  const float4 v = __ldcg(reinterpret_cast<const float4*>(g));  // written by other CTAs of this launch: read at L2
  if (p.zero_grad) *reinterpret_cast<float4*>(g) = make_float4(0.f, 0.f, 0.f, 0.f);
  const bool wire = p.ll_d[p.rank] != nullptr;                   // false: single rank without loop-back — nothing to exchange
  if (wire) direct_send_all(p, off, v, f, epoch);
  stamp(22);
  TileState s = tile_state_load(p, t, off, step_lr<SCHED>(p.h, opt_t));  // state loads overlap the flight of the packets
  const float4 agg = wire ? direct_recv_sum(p, off, f, epoch, err) : f4_scale(v, p.push_scale);
  stamp(23);
  const float4 W = tile_state_apply<EXT>(p, off, s, agg);
  *reinterpret_cast<float4*>(p.param[p.rank] + off) = W;        // the pull is a local store: every rank holds the fresh replica
  if (threadIdx.x == 0) {
    const int done = atomicAdd(p.state + 1, 1);
    if (done == n_active - 1) {                                  // every tail CTA is past the ticket spin: the counters can be re-armed
      p.state[1] = 0;
      p.state[6] = 0;
      p.state[2] = opt_t;
      p.state[0] = (int)round;
    }
  }
  stamp(24);
}

}  // namespace gx

using namespace gx;

static unsigned long long* g_cnn_dbg = nullptr;      // optional %globaltimer stamps of CTA (0,0): fwd 0-6, bwd 8-13 and 25-28, wgrad1 16-18
GX_API int gx_cnn_set_debug(unsigned long long* p) { g_cnn_dbg = p; return 0; }

// x [B,1,28,28]; w0 [16,1,5,5]; w1 [32,16,5,5]; writes a1 [B,16,12,12] + idx1, a2 [B,32,4,4] + idx2
GX_API int gx_cnn_fwd(const float* x, const float* w0, const float* b0, const float* w1, const float* b1, float* a1, unsigned char* idx1, float* a2,
                      unsigned char* idx2, const float* carry_src, float* carry_dst, int carry_n, float* x_keep, int B, cudaStream_t s) {
  if (B < 1) return 0;
  launch_pdl(cnn_fwd_kernel, dim3(B, 4), dim3(256), 0, s, x, w0, b0, w1, b1, a1, idx1, a2, idx2, carry_src, carry_dst, carry_n, x_keep, g_cnn_dbg);
  return GX_CHECK_LAUNCH();
}
// the same, plus the first dense layer: a3 [B,256] = relu(a2 [B,512] · wd [256,512]^T + bd).  With a4 non-null also the training head
// (fwd_train_head): wd1 [128,256], bd1, wd2 [10,128], bd2, label [B] in; loss [B], logits [B,10] (unless null), a4 [B,128], dz4 [B,128],
// dz3 [B,256] and dl [B,16] out.  coef [B] (with the head only; may be null): the dlogits of row b are scaled by coef[b] before anything is
// derived from them (cnn_fwd_dense0_weighted_kernel); the loss is not.  Only for even B <= 32 (clusters of two images); returns -1 without
// launching otherwise, or for coef without the head.
GX_API int gx_cnn_fwd_dense0(const float* x, const float* w0, const float* b0, const float* w1, const float* b1, const float* wd, const float* bd,
                             float* a1, unsigned char* idx1, float* a2, unsigned char* idx2, float* a3, const float* carry_src, float* carry_dst,
                             int carry_n, float* x_keep, const float* wd1, const float* bd1, const float* wd2, const float* bd2, const float* label,
                             float* loss, float* logits, float* a4, float* dz4, float* dz3, float* dl, const float* coef, int B, cudaStream_t s) {
  if (B < 2 || (B & 1) || B > 32 || (coef != nullptr && a4 == nullptr)) return -1;
  const FwdHeadArgs hd = {wd1, bd1, wd2, bd2, label, loss, logits, a4, dz4, dz3, dl};
  if (coef != nullptr)
    launch_pdl(cnn_fwd_dense0_weighted_kernel, dim3(B, 4), dim3(256), 0, s, x, w0, b0, w1, b1, wd, bd, a1, idx1, a2, idx2, a3, carry_src, carry_dst,
               carry_n, x_keep, g_cnn_dbg, hd, coef);
  else
    launch_pdl(cnn_fwd_dense0_kernel, dim3(B, 4), dim3(256), 0, s, x, w0, b0, w1, b1, wd, bd, a1, idx1, a2, idx2, a3, carry_src, carry_dst, carry_n,
               x_keep, g_cnn_dbg, hd);
  return GX_CHECK_LAUNCH();
}
// inference of the whole demo CNN (cnn_eval_kernel): x [N,1,28,28], the ten parameters in CNN_PARAM_SHAPES order; writes logits [N,10] (unless
// null), pred [N] (int32 arg-max) and, when `label` [N] (float class ids) is given, loss [N] (softmax-CE) and correct [N] (int32 0 / 1).
// Returns -1 without launching for N < 1.
GX_API int gx_cnn_eval(const float* x, const float* w0, const float* b0, const float* w1, const float* b1, const float* wd0, const float* bd0,
                       const float* wd1, const float* bd1, const float* wd2, const float* bd2, const float* label, float* logits, float* loss,
                       int* pred, int* correct, int N, cudaStream_t s) {
  if (N < 1) return -1;
  launch_pdl(cnn_eval_kernel, dim3(N + (N & 1), 4), dim3(256), 0, s, x, w0, b0, w1, b1, wd0, bd0, wd1, bd1, wd2, bd2, label, logits, loss, pred,
             correct, N);
  return GX_CHECK_LAUNCH();
}
// accumulates into dw0 [16,25] / db0 [16] (atomics: zero them first)
GX_API int gx_cnn_bwd(const float* x, const float* w1, const float* a1, const unsigned char* idx1, const float* a2, const unsigned char* idx2,
                      const float* da2, float* dw0, float* db0, int B, cudaStream_t s) {
  if (B < 1) return 0;
  static bool attr = false;
  if (!attr) {
    cudaError_t e = cudaFuncSetAttribute(cnn_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, CnnBwdSmem::BYTES);
    if (e != cudaSuccess) return (int)e;
    attr = true;
  }
  launch_pdl(cnn_bwd_kernel, dim3(B, 4), dim3(288), (size_t)CnnBwdSmem::BYTES, s, x, w1, a1, idx1, a2, idx2, da2, dw0, db0, g_cnn_dbg);
  return GX_CHECK_LAUNCH();
}
// overwrites dw1 [32,16,5,5] and db1 [32].  B even, B <= 64 (shared-memory planes of half the images per CTA).
GX_API int gx_cnn_wgrad1(const float* a1, const float* a2, const unsigned char* idx2, const float* da2, float* dw1, float* db1, int B, cudaStream_t s) {
  if (B < 2 || (B & 1) || B > 64) return -1;
  const size_t smem = (size_t)wgrad1_smem_bytes(B / 2);
  static size_t attr = 0;
  if (smem > attr) {
    cudaError_t e = cudaFuncSetAttribute(cnn_wgrad1_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return (int)e;
    attr = smem;
  }
  launch_pdl(cnn_wgrad1_kernel, dim3(CD_C2, 4, 2), dim3(256), smem, s, a1, a2, idx2, da2, dw1, db1, B, g_cnn_dbg);
  return GX_CHECK_LAUNCH();
}

// grid and dynamic shared memory of cnn_bwd_all_kernel at batch B (0 for batches it does not cover)
static int bwd_all_grid(int B) { return 8 * CD_C2 + 4 * B; }
static size_t bwd_all_smem(int B) {
  const size_t w = (size_t)wgrad1_smem_bytes(B / 2);
  return w > (size_t)CnnBwdSmem::BYTES ? w : (size_t)CnnBwdSmem::BYTES;
}
static int bwd_all_prepare(size_t smem) {
  static size_t attr = 0;
  if (smem > attr) {
    cudaError_t e = cudaFuncSetAttribute(cnn_bwd_all_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return (int)e;
    attr = smem;
  }
  return 0;
}

// conv backward in one launch (see cnn_bwd_all_kernel): accumulates dw0 / db0 (zero them first), overwrites dw1 / db1.  B even, <= 64.
GX_API int gx_cnn_bwd_all(const float* x, const float* w1, const float* a1, const unsigned char* idx1, const float* a2, const unsigned char* idx2,
                          const float* da2, float* dw0, float* db0, float* dw1, float* db1, int B, cudaStream_t s) {
  if (B < 2 || (B & 1) || B > 64) return -1;
  const size_t smem = bwd_all_smem(B);
  if (int e = bwd_all_prepare(smem)) return e;
  launch_pdl(cnn_bwd_all_kernel, dim3(bwd_all_grid(B)), dim3(288), smem, s, x, w1, a1, idx1, a2, idx2, da2, dw0, db0, dw1, db1, B, g_cnn_dbg);
  return GX_CHECK_LAUNCH();
}

// how cnn_bwd_all_kernel runs at batch B, for tests and tools: out[0] CTAs of the grid, [1] its dynamic shared memory (bytes), [2] the
// data-gradient body's, [3] the weight-gradient body's, [4] CTAs resident per SM on an idle device, [5] clusters of two resident at once
// on the whole idle device (cudaOccupancyMaxActiveClusters), [6] registers per thread, [7] CTAs whose (start, end, SM) the debug buffer
// records (the last ones of the grid).  Returns -1 for batches it does not cover.
GX_API int gx_cnn_bwd_all_geometry(int B, int* out) {
  if (B < 2 || (B & 1) || B > 64) return -1;
  const size_t smem = bwd_all_smem(B);
  if (int e = bwd_all_prepare(smem)) return e;
  int per_sm = 0, clusters = 0;
  cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, cnn_bwd_all_kernel, 288, smem);
  if (e != cudaSuccess) return (int)e;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(bwd_all_grid(B)); cfg.blockDim = dim3(288); cfg.dynamicSmemBytes = smem;
  e = cudaOccupancyMaxActiveClusters(&clusters, cnn_bwd_all_kernel, &cfg);
  if (e != cudaSuccess) return (int)e;
  cudaFuncAttributes fa;
  e = cudaFuncGetAttributes(&fa, cnn_bwd_all_kernel);
  if (e != cudaSuccess) return (int)e;
  out[0] = bwd_all_grid(B); out[1] = (int)smem; out[2] = CnnBwdSmem::BYTES; out[3] = wgrad1_smem_bytes(B / 2);
  out[4] = per_sm; out[5] = clusters; out[6] = fa.numRegs; out[7] = min(bwd_all_grid(B), CNN_BWD_CTA_STAMPS);
  return 0;
}

// conv backward + exchange of the conv keys in one launch (see cnn_bwd_exchange_kernel).  `params`: FabricParams block of the channel
// (replicated mode), `tile_list` / `n_active`: the channel's tiles.  Returns -1 for shapes the kernel does not cover.
GX_API int gx_cnn_bwd_exchange(const float* x, const float* w1, const float* a1, const unsigned char* idx1, const float* a2, const unsigned char* idx2,
                               const float* da2, float* dw0, float* db0, float* dw1, float* db1, int B, const void* params, const int* tile_list,
                               int n_active, cudaStream_t s) {
  if (B < 2 || (B & 1) || B > 64) return -1;
  const int grid = 4 * B + 4 * CD_C2;
  if (n_active < 1 || n_active > grid) return -1;
  int dev = 0, sms = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  if (grid > 2 * sms) return -1;                                  // the ticket wait needs the whole grid resident (2 CTAs per SM)
  const size_t smem_w = (size_t)wgrad1_smem_bytes(B);
  const size_t smem = smem_w > (size_t)CnnBwdSmem::BYTES ? smem_w : (size_t)CnnBwdSmem::BYTES;
  static size_t attr = 0;
  if (smem > attr) {
    for (const void* k : {(const void*)cnn_bwd_exchange_kernel<false, false>, (const void*)cnn_bwd_exchange_kernel<true, false>,
                          (const void*)cnn_bwd_exchange_kernel<false, true>, (const void*)cnn_bwd_exchange_kernel<true, true>}) {
      cudaError_t e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
      if (e != cudaSuccess) return (int)e;
    }
    attr = smem;
  }
  const FabricParams p = *reinterpret_cast<const FabricParams*>(params);
  // the constant-lr or the scheduled instance (step_lr<SCHED>), with the later optimizer kinds or without (opt_apply4<EXT>)
  launch_pdl(GX_FAB_INSTANCE(cnn_bwd_exchange_kernel, p), dim3(grid), dim3(288), smem, s, x, w1, a1, idx1, a2, idx2, da2, dw0, db0, dw1, db1, B, g_cnn_dbg, p, tile_list,
             n_active);
  return GX_CHECK_LAUNCH();
}
