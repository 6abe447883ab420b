// Fused small-batch MLP head: dense0 -> dense1 -> classifier -> softmax-CE, forward AND backward, in ONE thread-block-cluster launch.
//
// Reference path (examples/cnn.py:60-64 Dense(256,relu)/Dense(128,relu)/Dense(10) + SoftmaxCrossEntropyLoss, run as FullyConnected
// forward/backward ops src/operator/nn/fully_connected-inl.h:71-173 -> cublasSgemmEx linalg_impl.h:196-214, log_softmax softmax-inl.h:166-250,
// pick broadcast_reduce_op_index.cu:39-45): 3 forward GEMMs + 6 backward GEMMs + bias / activation / softmax kernels, each a separate engine op.
//
// With a per-worker batch of 32 every one of those GEMMs has M = 32: a 128-row tensor-core tile would be 3/4 padding and each launch is pure latency
// (the tensor pipe stays almost idle).  Here the whole chain is one kernel on a cluster of CS CTAs
// (16 — a non-portable cluster size, opted into at launch — or 8 when the device cannot co-schedule 16; GEOMX_MLP_CLUSTER):
//   * every CTA owns a 1/CS column slice of each layer; weights are staged in shared memory ONCE (cp.async, issued before griddepcontrol.wait
//     so the 150 KB of weight traffic overlaps the tail of the convolution kernels) and reused by forward and backward;
//   * products run on the fp32 FMA pipes (exact fp32, like the reference's SGEMM): 4x4 register tiles, K split over warps, operands read with
//     conflict-free 128-bit shared loads from XOR-swizzled tiles, partial sums reduced through shared memory;
//   * layer outputs (a3, a4, dz3) are pushed to every CTA of the cluster with st.async into distributed shared memory; each store
//     completes its bytes on a transaction mbarrier in the receiving CTA, and a consumer waits on its own barrier only.  Each receive buffer
//     is written once per launch, so after start-up there is no cluster-wide barrier (and no GPU-scope fence, no L1 invalidation) between
//     layers: a CTA starts a layer as soon as its own inputs have landed.  dz4 is not handed off: once a4 has landed every CTA holds all
//     of its inputs (a4, W2, dlogits) and computes the whole of it;
//   * epilogues fused: bias, ReLU, ReLU masks of the backward pass, softmax / loss / dlogits.
//   * 512 threads: all of them on dense0, dz4 and dx; dense1, the logits and dz3 are too small for a deeper K split to pay.
// The cluster kernel computes only what the convolution backward pass waits for (loss, logits, da2).  Nothing in the step reads the dense
// weight gradients before the dense keys' exchange, so they are a second, ordinary grid (dense_wgrad_kernel) on a parallel branch: the
// cluster kernel stores what they need (a3, a4, dz4, dz3, dlogits; about 50 KB) and the weight-gradient kernel turns them into dW0 / dW1 /
// dW2 and the bias gradients.  Two launches replace what used to be seven (dense0, dense1, head, dW1, dz3, dW0, da2); tools/kernel_times.py
// times the chain with per-phase %globaltimer stamps.
// dense0 is row-separable (a3[b] needs only the pooled conv output of image b), so where the direct forward kernel runs (even batches <= 32)
// it computes a3 on its 128 SMs (cnn_fwd_dense0_kernel, cnn_direct.cu) and the cluster kernel is dense_tail_kernel: the same chain from a3
// on, through the same body (dense_chain_body), with no x tile, no dense0 phase and no a3 hand-off.  In the classic training step the
// forward kernel also computes everything down to dz3 (all of it row-separable), and dense_tail_kernel runs from dz3: P5 (dx) only, over
// one cluster per four batch rows (dense_dx_rows).
//
// Shapes are compile-time (D0 -> D1 -> D2 -> C<=16, batch <= 32): the demo CNN's 512 -> 256 -> 128 -> 10.  Other shapes use the wgmma GEMMs.
#include <cooperative_groups.h>

#include "common.cuh"

namespace cg = cooperative_groups;

namespace gx {

constexpr int MC_THREADS = 512;   // 16 warps
constexpr int MC_HALF = 256;      // warp-group 0: dense1, the logits and dz3
constexpr int MC_B = 32;      // batch rows held (rows >= B are zero)
constexpr int MC_CMAX = 16;   // classes (padded)
constexpr int DX_THREADS = 128;   // dense_tail_kernel from dz3: threads per CTA

struct MlpChainParams {
  const float* x;       // [B][D0]   input activations (flattened pooled conv output)
  const float* w0; const float* b0;   // [D1][D0], [D1]
  const float* w1; const float* b1;   // [D2][D1], [D2]
  const float* w2; const float* b2;   // [C][D2],  [C]
  const float* label;   // [B] class index as float
  float* loss;          // [B]
  float* logits;        // [B][C] or nullptr
  float* dx;            // [B][D0]   gradient w.r.t. x
  // what the weight gradients need (rows b < B): a3 [B][D1], a4 [B][D2], dz4 [B][D2], dz3 [B][D1], dlogits [B][16] (classes >= C zero)
  // (dense_tail_kernel: a3 is its input, x and b0 are unused)
  float* a3; float* a4; float* dz4; float* dz3; float* dl;
  int B, C;
  int from_dz3;              // dense_tail_kernel: dz3 is the input (cnn_fwd_dense0_kernel's training head computed it) and dx the only output
  unsigned long long* dbg;   // optional %globaltimer stamps of cluster CTA 0 (tools/kernel_times.py)
  const float* coef;         // [B] per-row gradient coefficient: read by the weighted instances only (dense_chain_body's W)
};

// 16-byte chunk swizzle of a K-major [rows][K] tile: chunk (k>>2) is XORed with (row>>2)&7, so the 8 row-groups a warp touches in one
// 128-bit load land in 8 different bank groups
__device__ __forceinline__ int sw_off(int row, int k, int K) { return row * K + ((((k >> 2) ^ ((row >> 2) & 7))) << 2) + (k & 3); }

__device__ __forceinline__ void cp_async16(float* smem_dst, const float* gsrc) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(smem_dst)), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// (the point-to-point hand-offs between the CTAs of the cluster, push_all / wait_landed, are in common.cuh)

// stage `rows` x K floats (global row stride ld) into a swizzled K-major tile
__device__ __forceinline__ void stage_swizzled_async(float* dst, const float* src, int rows, int K, long long ld) {
  const int chunks = rows * (K >> 2);
  for (int c = threadIdx.x; c < chunks; c += MC_THREADS) {
    const int r = c / (K >> 2), q = c - r * (K >> 2);
    cp_async16(dst + sw_off(r, q << 2, K), src + (long long)r * ld + (q << 2));
  }
}
// stage `rows` x `cols` floats into a plain row-major tile [rows][cols]
__device__ __forceinline__ void stage_plain_async(float* dst, const float* src, int rows, int cols, long long ld) {
  const int chunks = rows * (cols >> 2);
  for (int c = threadIdx.x; c < chunks; c += MC_THREADS) {
    const int r = c / (cols >> 2), q = c - r * (cols >> 2);
    cp_async16(dst + r * cols + (q << 2), src + (long long)r * ld + (q << 2));
  }
}

// ---- register-tile products.  Thread (tb, tn, ks): rows 4tb..4tb+3 of X, 4 output columns, K chunks ks, ks+KS, ...
// NT: W is a swizzled K-major tile [NC][K]
template <int K, int KS>
__device__ __forceinline__ void prod_nt(const float* __restrict__ sX, const float* __restrict__ sW, int tb, int tn, int ks, float (&acc)[4][4]) {
#pragma unroll 2
  for (int kq = ks; kq < K / 4; kq += KS) {
    float4 x[4], w[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) x[i] = *reinterpret_cast<const float4*>(sX + (4 * tb + i) * K + ((kq ^ (tb & 7)) << 2));
#pragma unroll
    for (int j = 0; j < 4; ++j) w[j] = *reinterpret_cast<const float4*>(sW + (4 * tn + j) * K + ((kq ^ (tn & 7)) << 2));
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        acc[i][j] = fmaf(x[i].x, w[j].x, acc[i][j]);
        acc[i][j] = fmaf(x[i].y, w[j].y, acc[i][j]);
        acc[i][j] = fmaf(x[i].z, w[j].z, acc[i][j]);
        acc[i][j] = fmaf(x[i].w, w[j].w, acc[i][j]);
      }
  }
}
// NN: W is a plain tile [K][NC] (output columns contiguous): out[b][n] = sum_k X[b][k] * W[k][n]
template <int K, int NC, int KS>
__device__ __forceinline__ void prod_nn(const float* __restrict__ sX, const float* __restrict__ sW, int tb, int tn, int ks, float (&acc)[4][4]) {
#pragma unroll 2
  for (int kq = ks; kq < K / 4; kq += KS) {
    float4 x[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) x[i] = *reinterpret_cast<const float4*>(sX + (4 * tb + i) * K + ((kq ^ (tb & 7)) << 2));
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      const float4 w = *reinterpret_cast<const float4*>(sW + (4 * kq + kk) * NC + 4 * tn);
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float xv = kk == 0 ? x[i].x : kk == 1 ? x[i].y : kk == 2 ? x[i].z : x[i].w;
        acc[i][0] = fmaf(xv, w.x, acc[i][0]);
        acc[i][1] = fmaf(xv, w.y, acc[i][1]);
        acc[i][2] = fmaf(xv, w.z, acc[i][2]);
        acc[i][3] = fmaf(xv, w.w, acc[i][3]);
      }
    }
  }
}
// write this thread's 4x4 partial tile into scratch [KS][32][NC]
template <int NC>
__device__ __forceinline__ void put_partial(float* scratch, int tb, int tn, int ks, const float (&acc)[4][4]) {
#pragma unroll
  for (int i = 0; i < 4; ++i)
    *reinterpret_cast<float4*>(scratch + (ks * MC_B + 4 * tb + i) * NC + 4 * tn) = make_float4(acc[i][0], acc[i][1], acc[i][2], acc[i][3]);
}
template <int NC, int KS>
__device__ __forceinline__ float4 sum_partials(const float* scratch, int b, int n4) {
  float4 s = *reinterpret_cast<const float4*>(scratch + b * NC + 4 * n4);
#pragma unroll
  for (int k = 1; k < KS; ++k) {
    const float4 t = *reinterpret_cast<const float4*>(scratch + (k * MC_B + b) * NC + 4 * n4);
    s.x += t.x; s.y += t.y; s.z += t.z; s.w += t.w;
  }
  return s;
}
// wgrad: dW[n][k] = sum_{b < B} DZ[b][n] * X[b][k] for rows n0 .. n0+3 (those < nrows are stored) and columns k0 .. k0+3, read from global
// memory (DZ: [B][LDZ], X and dW: [.][LDX]).  One fmaf chain per output over b ascending.
template <int LDZ, int LDX>
__device__ __forceinline__ void wgrad_4x4(const float* __restrict__ dz, const float* __restrict__ x, int B, int n0, int k0, int nrows,
                                          float* __restrict__ out) {
  float acc[4][4] = {};
#pragma unroll 4
  for (int b = 0; b < B; ++b) {
    const float4 d = *reinterpret_cast<const float4*>(dz + b * LDZ + n0);
    const float4 v = *reinterpret_cast<const float4*>(x + b * LDX + k0);
    const float dd[4] = {d.x, d.y, d.z, d.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      acc[i][0] = fmaf(dd[i], v.x, acc[i][0]);
      acc[i][1] = fmaf(dd[i], v.y, acc[i][1]);
      acc[i][2] = fmaf(dd[i], v.z, acc[i][2]);
      acc[i][3] = fmaf(dd[i], v.w, acc[i][3]);
    }
  }
#pragma unroll
  for (int i = 0; i < 4; ++i)
    if (n0 + i < nrows) *reinterpret_cast<float4*>(out + (n0 + i) * LDX + k0) = make_float4(acc[i][0], acc[i][1], acc[i][2], acc[i][3]);
}
// bias gradient: db[n] = sum_{b < B} DZ[b][n], b ascending
template <int LDZ>
__device__ __forceinline__ float colsum(const float* __restrict__ dz, int B, int n) {
  float s = 0.f;
  for (int b = 0; b < B; ++b) s += dz[b * LDZ + n];
  return s;
}

// W2 as a swizzled K-major tile [16][D2] (rows >= C zero), b1 slice, b2 (classes >= C zero)
template <int D2, int NS2>
__device__ __forceinline__ void stage_head_async(float* sW2, float* sB1, float* sB2, const float* w2, const float* b1, const float* b2, int cr,
                                                 int C) {
  const int tid = threadIdx.x;
  for (int c = tid; c < MC_CMAX * (D2 >> 2); c += MC_THREADS) {
    const int r = c / (D2 >> 2), q = c - r * (D2 >> 2);
    float* dst = sW2 + sw_off(r, q << 2, D2);
    if (r < C) cp_async16(dst, w2 + (long long)r * D2 + (q << 2));
    else *reinterpret_cast<float4*>(dst) = make_float4(0.f, 0.f, 0.f, 0.f);
  }
  if (tid < NS2) sB1[tid] = b1[cr * NS2 + tid];
  if (tid < 16) sB2[tid] = tid < C ? b2[tid] : 0.f;
}

// Shared-memory layout of mlp_chain_kernel (starts from x and computes dense0 itself).  Both kernels name the same buffers (W0, W1, A3, A4,
// DZ4, W2, DL, MISC, A3OWN, SCRATCH, BAR) so that dense_chain_body serves both.
template <int D0, int D1, int D2, int CS>
struct MlpSmem {
  static constexpr int NS1 = D1 / CS, NS2 = D2 / CS, KS0 = D0 / CS;
  // float offsets
  static constexpr int X = 0;                                  // [32][D0] swizzled  (dead after P1: P4 / P5 scratch)
  static constexpr int SCRATCH = X, SCRATCH_SZ = MC_B * D0;
  static constexpr int W0 = X + MC_B * D0;                     // fwd: [NS1][D0] swizzled;  bwd: [D1][KS0] plain
  static constexpr int W0_SZ = (NS1 * D0 > D1 * KS0) ? NS1 * D0 : D1 * KS0;
  static constexpr int W1 = W0 + W0_SZ;                        // fwd: [NS2][D1] swizzled;  bwd: [D2][NS1] plain
  static constexpr int W1_SZ = (NS2 * D1 > D2 * NS1) ? NS2 * D1 : D2 * NS1;
  // receive buffers: each is written by the peers exactly once per launch.  No peer can produce dz3 before it holds this CTA's a4, and
  // this CTA pushes a4 only after its P2 products have finished reading a3, so dz3 lands in the a3 buffer without a write-after-read barrier
  static constexpr int A3 = W1 + W1_SZ;                        // [32][D1] swizzled  (later: dz3)
  static constexpr int A4 = A3 + MC_B * D1;                    // [32][D2] swizzled  (earlier: P1 scratch)
  static constexpr int DZ4 = A4 + MC_B * D2;                   // [32][D2] swizzled, computed locally  (earlier: P1 / P2 / logit scratch)
  static constexpr int W2 = DZ4 + MC_B * D2;                   // [16][D2] swizzled, rows >= C zero
  static constexpr int DL = W2 + MC_CMAX * D2;                 // [32][16] dlogits
  static constexpr int MISC = DL + MC_B * MC_CMAX;             // b0 slice [NS1] | b1 slice [NS2] | b2 [16] | label [32]
  static constexpr int A3OWN = MISC + NS1 + NS2 + 16 + 32;     // [32][NS1] plain: this CTA's a3 columns (ReLU mask of dz3)
  static constexpr int BAR = A3OWN + MC_B * NS1;               // 3 mbarriers: a3, a4, dz3 landed
  static constexpr int TOTAL = BAR + 3 * 2;
  static constexpr int BYTES = TOTAL * 4;
};
// Shared-memory layout of dense_tail_kernel (starts from a3, which the forward kernel computed): no x tile, W0 only as the column slice of
// the backward pass, and a scratch of its own for the P4 / P5 partials.  The A3 buffer is staged from global memory and later receives dz3,
// the only hand-off into it (write-once as in MlpSmem: no peer can push dz3 before it holds this CTA's a4).
template <int D0, int D1, int D2, int CS>
struct TailSmem {
  static constexpr int NS1 = D1 / CS, NS2 = D2 / CS, KS0 = D0 / CS;
  static constexpr int W0 = 0;                                 // [D1][KS0] plain
  static constexpr int W1 = W0 + D1 * KS0;                     // fwd: [NS2][D1] swizzled;  bwd: [D2][NS1] plain
  static constexpr int W1_SZ = (NS2 * D1 > D2 * NS1) ? NS2 * D1 : D2 * NS1;
  static constexpr int A3 = W1 + W1_SZ;                        // [32][D1] swizzled, rows >= B zero  (later: dz3)
  static constexpr int A4 = A3 + MC_B * D1;                    // [32][D2] swizzled
  static constexpr int DZ4 = A4 + MC_B * D2;                   // [32][D2] swizzled, computed locally  (earlier: P2 / logit scratch)
  static constexpr int W2 = DZ4 + MC_B * D2;                   // [16][D2] swizzled, rows >= C zero
  static constexpr int DL = W2 + MC_CMAX * D2;                 // [32][16] dlogits
  static constexpr int MISC = DL + MC_B * MC_CMAX;             // (unused) [NS1] | b1 slice [NS2] | b2 [16] | label [32]
  static constexpr int A3OWN = MISC + NS1 + NS2 + 16 + 32;     // [32][NS1] plain: this CTA's a3 columns (ReLU mask of dz3)
  static constexpr int SCRATCH = A3OWN + MC_B * NS1;           // P4 / P5 partials
  static constexpr int SCRATCH_SZ = (MC_THREADS / (2 * KS0)) * MC_B * KS0;
  static constexpr int BAR = SCRATCH + SCRATCH_SZ;             // 2 mbarriers: a4, dz3 landed
  static constexpr int TOTAL = BAR + 2 * 2;
  static constexpr int BYTES = TOTAL * 4;
  // from dz3 (dense_dx_rows): the W0 column slice [D1][KS0], DX_ROWS rows of dz3 and the partial sums of the K splits
  static constexpr int DX_ROWS = 4, DX_KS = DX_THREADS / KS0;
  static constexpr int DX_BYTES = (D1 * KS0 + DX_ROWS * D1 + DX_KS * DX_ROWS * KS0) * 4;
};
// the tail's CTAs stage their weights on the SMs beside the forward kernel's CTAs (one each: 256 x 64 + 512 x 96 = 65,536 registers), so
// both kernels' shared memory, with the 1 KB the runtime reserves per CTA, has to fit into the SM's 228 KB
static_assert(TailSmem<512, 256, 128, 16>::BYTES + CNN_FWD_DENSE0_SMEM_BYTES + 2048 <= 233472, "dense_tail_kernel fits beside cnn_fwd_dense0_kernel");

// P5 of the chain: dx[:, slice of D0] = dz3 * W0[:, slice], with dz3 (rows >= B zero) whole in the A3 buffer and the W0 column slice staged.
// NC = KS0, K = D1, split over all 16 warps.
template <class L, int D0, int D1, class Stamp>
__device__ __forceinline__ void dense_dx(float* sm, const MlpChainParams& p, const int cr, Stamp&& stamp) {
  constexpr int KS0 = L::KS0, PER = 2 * KS0, KS = MC_THREADS / PER;
  const float* sDZ3 = sm + L::A3; const float* sW0 = sm + L::W0;
  float* scratch = sm + L::SCRATCH;
  const int tid = threadIdx.x, ks = tid / PER, tile = tid % PER, tb = tile & 7, tn = tile >> 3;
  float acc[4][4] = {};
  prod_nn<D1, KS0, KS>(sDZ3, sW0, tb, tn, ks, acc);
  stamp(14);
  put_partial<KS0>(scratch, tb, tn, ks, acc);
  __syncthreads();
  for (int e = tid; e < MC_B * KS0 / 4; e += MC_THREADS) {
    const int b = e / (KS0 / 4), n4 = e % (KS0 / 4);
    if (b < p.B) *reinterpret_cast<float4*>(p.dx + (long long)b * D0 + cr * KS0 + 4 * n4) = sum_partials<KS0, KS>(scratch, b, n4);
  }
  stamp(9);
}

// dense_tail_kernel from dz3: dx = dz3 W0, one DX_ROWS x KS0 tile per CTA.  The kernel runs over ceil(B / DX_ROWS) clusters: cluster g takes
// rows [g DX_ROWS, (g + 1) DX_ROWS), rank cr the columns of its W0 slice, so that da2 is computed on up to 128 SMs instead of one cluster's.
// DX_THREADS threads (the tail's 512 would hold 49 K registers on every SM the grid lands on, where the convolution backward grid that
// follows becomes resident).  The W0 slice is staged before the grid dependency, only the tile's dz3 rows after it.  Thread -> column
// n = tid % KS0 and K split ks = tid / KS0, one fmaf chain per row over its K range; the splits are added in ascending order, so that
// two launches give the same bits.
template <class L, int D0, int D1, int CS, class Stamp>
__device__ __forceinline__ void dense_dx_rows(float* sm, const MlpChainParams& p, const int cr, Stamp&& stamp) {
  constexpr int R = L::DX_ROWS, KS0 = L::KS0, KS = L::DX_KS, KL = D1 / KS;
  static_assert(DX_THREADS % KS0 == 0 && KL % 4 == 0, "dx tile splits");
  float* sW = sm; float* sZ = sW + D1 * KS0; float* sP = sZ + R * D1;
  const int tid = threadIdx.x, row0 = (blockIdx.x / CS) * R;
  for (int c = tid; c < D1 * (KS0 / 4); c += DX_THREADS) {
    const int r = c / (KS0 / 4), q = c - r * (KS0 / 4);
    cp_async16(sW + r * KS0 + 4 * q, p.w0 + (long long)r * D0 + cr * KS0 + 4 * q);
  }
  cp_async_commit();
  stamp(1);
  pdl_wait();
  pdl_launch();
  stamp(2);
  for (int c = tid; c < R * (D1 / 4); c += DX_THREADS) {
    const int r = c / (D1 / 4), q = c - r * (D1 / 4);
    if (row0 + r < p.B) cp_async16(sZ + r * D1 + 4 * q, p.dz3 + (long long)(row0 + r) * D1 + 4 * q);
    else *reinterpret_cast<float4*>(sZ + r * D1 + 4 * q) = make_float4(0.f, 0.f, 0.f, 0.f);
  }
  cp_async_commit();
  cp_async_wait<0>();
  __syncthreads();
  stamp(3);
  const int n = tid % KS0, ks = tid / KS0;
  float acc[R] = {};
#pragma unroll 2
  for (int k = ks * KL; k < (ks + 1) * KL; k += 4) {
    const float w[4] = {sW[k * KS0 + n], sW[(k + 1) * KS0 + n], sW[(k + 2) * KS0 + n], sW[(k + 3) * KS0 + n]};
#pragma unroll
    for (int r = 0; r < R; ++r) {
      const float4 z = *reinterpret_cast<const float4*>(sZ + r * D1 + k);
      acc[r] = fmaf(z.x, w[0], acc[r]); acc[r] = fmaf(z.y, w[1], acc[r]); acc[r] = fmaf(z.z, w[2], acc[r]); acc[r] = fmaf(z.w, w[3], acc[r]);
    }
  }
  stamp(14);
#pragma unroll
  for (int r = 0; r < R; ++r) sP[(ks * R + r) * KS0 + n] = acc[r];
  __syncthreads();
  for (int e = tid; e < R * KS0; e += DX_THREADS) {
    const int r = e / KS0, c = e - r * KS0;
    float s = sP[e];
#pragma unroll
    for (int k = 1; k < KS; ++k) s += sP[k * R * KS0 + e];
    if (row0 + r < p.B) p.dx[(long long)(row0 + r) * D0 + cr * KS0 + c] = s;
  }
  stamp(9);
}

// P2 .. P5 of the chain, the part both cluster kernels share: a4 = relu(a3 W1^T + b1) with the a4 hand-off, the classifier, softmax-CE and
// the whole dz4, dz3 with its hand-off, and dx.  On entry the weights are staged (W0 as the column slice for dx still in flight, W1 as the
// row slice), a3 is in the A3 buffer (FROM_X: as it lands from the peers) and in A3OWN (this CTA's columns), the labels and biases are
// staged and the cluster has met once.  FROM_X (mlp_chain_kernel) also waits for a3 and stores this CTA's a3 columns.  W (the weighted
// instances): the dlogits of row b are scaled by p.coef[b] where they are produced, so that dz4, dz3, dx and every weight gradient carry it;
// the loss stays unweighted.
template <class L, int D0, int D1, int D2, int CS, bool FROM_X, bool W, class Stamp>
__device__ __forceinline__ void dense_chain_body(float* sm, const MlpChainParams& p, const int cr, uint64_t* bar_a3, uint64_t* bar_a4,
                                                 uint64_t* bar_dz3, Stamp&& stamp) {
  constexpr int NS1 = L::NS1, NS2 = L::NS2, KS0 = L::KS0;
  static_assert(MC_HALF % (2 * NS1) == 0 && MC_HALF % (2 * NS2) == 0 && MC_THREADS % (2 * KS0) == 0, "K splits");
  static_assert(MC_HALF / (2 * NS1) * MC_B * NS1 <= L::SCRATCH_SZ && MC_THREADS / (2 * KS0) * MC_B * KS0 <= L::SCRATCH_SZ, "P4 / P5 scratch");
  static_assert(MC_B * NS1 / 4 <= MC_HALF && MC_B * NS2 / 4 <= MC_HALF, "one thread per float4 of a3 / a4");
  float* sW0 = sm + L::W0; float* sW1 = sm + L::W1; float* sA3 = sm + L::A3; float* sA4 = sm + L::A4;
  float* sDZ4 = sm + L::DZ4; float* sW2 = sm + L::W2; float* sDL = sm + L::DL; float* sA3own = sm + L::A3OWN;
  float* sB1 = sm + L::MISC + NS1; float* sB2 = sB1 + NS2; float* sLab = sB2 + 16;
  const int tid = threadIdx.x;
  const int B = p.B, C = p.C;
  // ---------------- P2: a4[:, slice] = relu(a3 * W1[slice]^T + b1)         NC = 16, K = D1, KS = 8
  {
    constexpr int PER = 2 * NS2, KS = MC_HALF / PER;     // this layer is small: warp-group 0 only
    if (tid < MC_HALF) {
      if (FROM_X) {
        wait_landed(bar_a3);
        stamp(4);
      }
      const int ks = tid / PER, tile = tid % PER, tb = tile & 7, tn = tile >> 3;
      float acc[4][4] = {};
      prod_nt<D1, KS>(sA3, sW1, tb, tn, ks, acc);
      put_partial<NS2>(sDZ4, tb, tn, ks, acc);
    }
    __syncthreads();     // from here on the full a3 buffer is dead: it receives dz3
    stage_plain_async(sW1, p.w1 + cr * NS1, D2, NS1, D1);   // W1[:, slice of D1] for dz3
    cp_async_commit();
    if (tid < MC_B * NS2 / 4) {
      const int b = tid / (NS2 / 4), n4 = tid % (NS2 / 4);
      float4 v = sum_partials<NS2, KS>(sDZ4, b, n4);
      v.x = fmaxf(v.x + sB1[4 * n4], 0.f); v.y = fmaxf(v.y + sB1[4 * n4 + 1], 0.f);
      v.z = fmaxf(v.z + sB1[4 * n4 + 2], 0.f); v.w = fmaxf(v.w + sB1[4 * n4 + 3], 0.f);
      if (b >= B) v = make_float4(0.f, 0.f, 0.f, 0.f);
      push_all<CS>(sA4, sw_off(b, cr * NS2 + 4 * n4, D2), bar_a4, cr, v);
      if (b < B) *reinterpret_cast<float4*>(p.a4 + b * D2 + cr * NS2 + 4 * n4) = v;
    } else if (FROM_X && tid >= MC_HALF && tid - MC_HALF < MC_B * NS1 / 4) {
      // warp-group 1 is idle in P2: it stores this CTA's a3 columns for the weight-gradient kernel
      const int b = (tid - MC_HALF) / (NS1 / 4), n4 = (tid - MC_HALF) % (NS1 / 4);
      if (b < B) *reinterpret_cast<float4*>(p.a3 + b * D1 + cr * NS1 + 4 * n4) = *reinterpret_cast<const float4*>(sA3own + b * NS1 + 4 * n4);
    }
  }
  // ---------------- P3: classifier + softmax-CE (every CTA redundantly: 32 x C logits), the whole dz4, dW2 slice, db2
  {
    wait_landed(bar_a4);
    stamp(5);
    constexpr int PER = 8 * (MC_CMAX / 4), KS = MC_HALF / PER;   // 32 logit tiles x 8 K splits on warp-group 0: NC = 16, K = D2
    static_assert(KS * MC_B * MC_CMAX <= MC_B * D2, "logit partials fit the dz4 buffer");
    if (tid < MC_HALF) {
      // The dz4 buffer still holds P2's partials, but every one of them was read before this CTA's own a4 slice was pushed (the pushed
      // values depend on those reads), and bar_a4 has counted that slice.  Rows >= C of W2 are zero, so their logits are just b2.
      const int ks = tid / PER, tile = tid % PER, tb = tile & 7, tn = tile >> 3;
      float acc[4][4] = {};
      prod_nt<D2, KS>(sA4, sW2, tb, tn, ks, acc);
      put_partial<MC_CMAX>(sDZ4, tb, tn, ks, acc);
    }
    __syncthreads();
    if (tid < MC_B * MC_CMAX / 4) {
      // softmax-CE: four consecutive lanes hold one row, lane n4 of the four its classes 4 n4 .. 4 n4 + 3
      const int b = tid >> 2, n4 = tid & 3, c0 = 4 * n4;
      const float4 s4 = sum_partials<MC_CMAX, KS>(sDZ4, b, n4);
      const float lg[4] = {s4.x + sB2[c0], s4.y + sB2[c0 + 1], s4.z + sB2[c0 + 2], s4.w + sB2[c0 + 3]};
      float dl[4];
      const float loss = softmax_ce_quad(lg, C, (int)sLab[b], dl);
      if (b >= B) dl[0] = dl[1] = dl[2] = dl[3] = 0.f;
      if (W && b < B) {
        const float cb = __ldg(p.coef + b);
#pragma unroll
        for (int j = 0; j < 4; ++j) dl[j] = __fmul_rn(dl[j], cb);
      }
      *reinterpret_cast<float4*>(sDL + b * MC_CMAX + c0) = make_float4(dl[0], dl[1], dl[2], dl[3]);
      if (cr == 0 && b < B) {
        *reinterpret_cast<float4*>(p.dl + b * MC_CMAX + c0) = make_float4(dl[0], dl[1], dl[2], dl[3]);
        if (n4 == 0) p.loss[b] = loss;
        if (p.logits != nullptr)
#pragma unroll
          for (int j = 0; j < 4; ++j) if (c0 + j < C) p.logits[(long long)b * C + c0 + j] = lg[j];
      }
    }
    __syncthreads();             // dlogits complete, the logit partials read
    {
      // dz4[b][m] = relu'(a4[b][m]) * sum_c dl[b][c] * W2[c][m] over all of D2: four columns m of the rows b0, b0 + 16 per thread, which
      // share each W2 load.  Every CTA runs the same loop over c on the same data, so all of them hold the same bits.
      constexpr int RSTEP = MC_THREADS / (D2 / 4), NR = MC_B / RSTEP;
      static_assert(MC_THREADS % (D2 / 4) == 0 && MC_B % RSTEP == 0, "dz4 rows split evenly over the threads");
      const int b0 = tid / (D2 / 4), m = 4 * (tid % (D2 / 4));
      float4 s[NR];
#pragma unroll
      for (int r = 0; r < NR; ++r) s[r] = make_float4(0.f, 0.f, 0.f, 0.f);
      for (int c = 0; c < C; ++c) {
        const float4 w = *reinterpret_cast<const float4*>(sW2 + sw_off(c, m, D2));
#pragma unroll
        for (int r = 0; r < NR; ++r) {
          const float d = sDL[(b0 + r * RSTEP) * MC_CMAX + c];
          s[r].x = fmaf(d, w.x, s[r].x); s[r].y = fmaf(d, w.y, s[r].y); s[r].z = fmaf(d, w.z, s[r].z); s[r].w = fmaf(d, w.w, s[r].w);
        }
      }
#pragma unroll
      for (int r = 0; r < NR; ++r) {
        const int o = sw_off(b0 + r * RSTEP, m, D2);
        const float4 a = *reinterpret_cast<const float4*>(sA4 + o);
        float4 v = s[r];
        if (!(a.x > 0.f)) v.x = 0.f;
        if (!(a.y > 0.f)) v.y = 0.f;
        if (!(a.z > 0.f)) v.z = 0.f;
        if (!(a.w > 0.f)) v.w = 0.f;
        *reinterpret_cast<float4*>(sDZ4 + o) = v;
        if (b0 + r * RSTEP < B && m / NS2 == cr)     // this CTA's column slice, for the weight-gradient kernel
          *reinterpret_cast<float4*>(p.dz4 + (b0 + r * RSTEP) * D2 + m) = v;
      }
    }
    cp_async_wait<0>();          // W1 column slice (and W0 column slice) landed: first read in P4, so the head does not wait for them
    __syncthreads();             // dz4 complete, the staged slices visible
    stamp(6);
  }
  // ---------------- P4: dz3[:, slice] = relu'(a3) * (dz4 * W1[:, slice])          NC = NS1, K = D2, split over warp-group 0
  // (split over all 16 warps, the deeper reduction made "dz3 pushed" slower: 2.4 us instead of 2.0)
  float* sDZ3 = sA3;
  float* scratch = sm + L::SCRATCH;                      // P4 / P5 partials
  {
    constexpr int PER = 2 * NS1, KS = MC_HALF / PER;
    if (tid < MC_HALF) {
      const int ks = tid / PER, tile = tid % PER, tb = tile & 7, tn = tile >> 3;
      float acc[4][4] = {};
      prod_nn<D2, NS1, KS>(sDZ4, sW1, tb, tn, ks, acc);
      put_partial<NS1>(scratch, tb, tn, ks, acc);
    }
    __syncthreads();
    if (tid < MC_B * NS1 / 4) {
      const int b = tid / (NS1 / 4), n4 = tid % (NS1 / 4);
      float4 dz3v = sum_partials<NS1, KS>(scratch, b, n4);
      const float4 a3 = *reinterpret_cast<const float4*>(sA3own + b * NS1 + 4 * n4);
      dz3v.x = a3.x > 0.f ? dz3v.x : 0.f; dz3v.y = a3.y > 0.f ? dz3v.y : 0.f; dz3v.z = a3.z > 0.f ? dz3v.z : 0.f; dz3v.w = a3.w > 0.f ? dz3v.w : 0.f;
      const int o = sw_off(b, cr * NS1 + 4 * n4, D1);
      push_all<CS, CS - 1>(sDZ3, o, bar_dz3, cr, dz3v);
      *reinterpret_cast<float4*>(sDZ3 + o) = dz3v;   // own columns: stored locally
      if (b < B) *reinterpret_cast<float4*>(p.dz3 + b * D1 + cr * NS1 + 4 * n4) = dz3v;
    }
    stamp(7);
    __syncthreads();                                     // own dz3 columns stored, the P4 partials read
  }
  wait_landed(bar_dz3);                                  // the peers' columns
  stamp(8);
  dense_dx<L, D0, D1>(sm, p, cr, stamp);
}

// CS = CTAs per cluster: 8 (portable) or 16 (non-portable size, one GPC): every layer is cut into CS column slices.  Instantiated twice:
// mlp_chain_kernel (W = false) compiles to the code it had before the weighted chain existed; mlp_chain_weighted_kernel scales the dlogits.
template <int D0, int D1, int D2, int CS, bool W>
__device__ __forceinline__ void mlp_chain_body(const MlpChainParams& p) {
  using L = MlpSmem<D0, D1, D2, CS>;
  constexpr int NS1 = L::NS1, NS2 = L::NS2;
  static_assert((CS & (CS - 1)) == 0, "cluster size must be a power of two");
  static_assert(D0 % 64 == 0 && D1 % 64 == 0 && D2 % 64 == 0, "layer widths must be multiples of 64");
  static_assert(NS1 % 8 == 0 && NS2 % 4 == 0 && L::KS0 % 4 == 0, "slices must hold whole register tiles");
  static_assert(MC_THREADS / (2 * NS1) * MC_B * NS1 <= 2 * MC_B * D2, "P1 scratch fits the a4 and dz4 buffers");
  static_assert(L::BAR % 2 == 0, "mbarriers are 8-byte aligned");
  extern __shared__ __align__(16) float sm[];
  float* sX = sm + L::X; float* sW0 = sm + L::W0; float* sW1 = sm + L::W1; float* sA3 = sm + L::A3; float* sA4 = sm + L::A4;
  float* sW2 = sm + L::W2; float* sA3own = sm + L::A3OWN;
  float* sB0 = sm + L::MISC; float* sB1 = sB0 + NS1; float* sB2 = sB1 + NS2; float* sLab = sB2 + 16;
  uint64_t* bar = reinterpret_cast<uint64_t*>(sm + L::BAR);
  uint64_t* bar_a3 = bar; uint64_t* bar_a4 = bar + 1; uint64_t* bar_dz3 = bar + 2;
  cg::cluster_group cluster = cg::this_cluster();
  const int cr = (int)cluster.block_rank();
  const int tid = threadIdx.x;
  const int B = p.B, C = p.C;
  // stamp by thread 0 of cluster CTA 0
  auto stamp = [&](int slot) {
    if (p.dbg != nullptr && cr == 0 && tid == 0) { unsigned long long t; asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t)); p.dbg[slot] = t; }
  };
  stamp(0);

  // ---------------- start-up: each receive barrier expects its whole buffer (dz3: all but this CTA's own columns, which are stored locally).
  // The peers push into this CTA's shared memory only after the cluster barrier below, so the barriers are armed before any byte arrives.
  if (tid == 0) {
    for (int i = 0; i < 3; ++i) mbar_init(bar + i, 1);
    mbar_arrive_expect_tx(bar_a3, MC_B * D1 * 4);
    mbar_arrive_expect_tx(bar_a4, MC_B * D2 * 4);
    mbar_arrive_expect_tx(bar_dz3, (CS - 1) * MC_B * NS1 * 4);
    fence_barrier_init();      // (the release the peers need: nothing else this CTA wrote so far is read by them)
  }
  asm volatile("barrier.cluster.arrive.relaxed.aligned;" ::: "memory");   // waited for once the inputs are staged: the loads overlap the rendezvous

  // ---------------- prologue: weights do not depend on the preceding kernel (they were written by the previous step's exchange, which a
  // kernel further up the stream has already waited for) -> stage them before griddepcontrol.wait
  stage_swizzled_async(sW0, p.w0 + (long long)cr * NS1 * D0, NS1, D0, D0);
  stage_swizzled_async(sW1, p.w1 + (long long)cr * NS2 * D1, NS2, D1, D1);
  stage_head_async<D2, NS2>(sW2, sB1, sB2, p.w2, p.b1, p.b2, cr, C);
  if (tid < NS1) sB0[tid] = p.b0[cr * NS1 + tid];
  cp_async_commit();
  stamp(1);
  pdl_wait();
  pdl_launch();
  stamp(2);
  // input activations (full copy per CTA) + labels
  for (int c = tid; c < MC_B * (D0 >> 2); c += MC_THREADS) {
    const int r = c / (D0 >> 2), q = c - r * (D0 >> 2);
    if (r < B) cp_async16(sX + sw_off(r, q << 2, D0), p.x + (long long)r * D0 + (q << 2));
    else *reinterpret_cast<float4*>(sX + sw_off(r, q << 2, D0)) = make_float4(0.f, 0.f, 0.f, 0.f);
  }
  if (tid < MC_B) sLab[tid] = tid < B ? p.label[tid] : 0.f;
  cp_async_commit();
  cp_async_wait<0>();
  __syncthreads();
  cluster.barrier_wait();   // every CTA of the cluster is running with its barriers armed (the pushes below target its shared memory)
  stamp(3);

  // tile coordinates shared by the 32-row products: 8 row groups x (NC/4) column groups per K split
  // ---------------- P1: a3[:, slice] = relu(x * W0[slice]^T + b0)          NC = 32, K = D0, KS = 4
  {
    constexpr int PER = 2 * NS1, KS = MC_THREADS / PER;  // 8 row groups x NS1/4 column groups per split; K split over all 16 warps
    const int ks = tid / PER, tile = tid % PER, tb = tile & 7, tn = tile >> 3;
    float acc[4][4] = {};
    prod_nt<D0, KS>(sX, sW0, tb, tn, ks, acc);
    stamp(10);
    float* scratch = sA4;                                // [sA4 | sDZ4] = 32 KB contiguous, both unused until the end of P2 / P3
    put_partial<NS1>(scratch, tb, tn, ks, acc);
    __syncthreads();
    // W0's row slice is no longer needed: start fetching the COLUMN slice W0[:, cr*KS0 ...] for the backward pass (da2) underneath P2..P4
    stamp(11);
    stage_plain_async(sW0, p.w0 + cr * L::KS0, D1, L::KS0, D0);
    cp_async_commit();
    stamp(12);
    if (tid < MC_B * NS1 / 4) {
      const int b = tid / (NS1 / 4), n4 = tid % (NS1 / 4);   // 32 x NS1/4 float4 outputs
      float4 v = sum_partials<NS1, KS>(scratch, b, n4);
      v.x = fmaxf(v.x + sB0[4 * n4], 0.f); v.y = fmaxf(v.y + sB0[4 * n4 + 1], 0.f);
      v.z = fmaxf(v.z + sB0[4 * n4 + 2], 0.f); v.w = fmaxf(v.w + sB0[4 * n4 + 3], 0.f);
      if (b >= B) v = make_float4(0.f, 0.f, 0.f, 0.f);
      *reinterpret_cast<float4*>(sA3own + b * NS1 + 4 * n4) = v;
      // the pushed value depends on this thread's scratch reads, so no peer can write a4 into the scratch before they are done
      push_all<CS>(sA3, sw_off(b, cr * NS1 + 4 * n4, D1), bar_a3, cr, v);
    }
    stamp(13);
  }
  dense_chain_body<L, D0, D1, D2, CS, true, W>(sm, p, cr, bar_a3, bar_a4, bar_dz3, stamp);
}
template <int D0, int D1, int D2, int CS>
__global__ void __cluster_dims__(CS, 1, 1) __launch_bounds__(MC_THREADS, 1) mlp_chain_kernel(const MlpChainParams p) {
  mlp_chain_body<D0, D1, D2, CS, false>(p);
}
template <int D0, int D1, int D2, int CS>
__global__ void __cluster_dims__(CS, 1, 1) __launch_bounds__(MC_THREADS, 1) mlp_chain_weighted_kernel(const MlpChainParams p) {
  mlp_chain_body<D0, D1, D2, CS, true>(p);
}

// The chain from a3 on, for a step whose forward kernel (cnn_fwd_dense0_kernel) has already computed a3 = relu(x W0^T + b0): P2 .. P5 of
// mlp_chain_kernel, unchanged, on the same cluster.  Everything but a3 and the labels (the W1 row slice, W2, the biases and the W0 column
// slice of dx) is staged before griddepcontrol.wait, i.e. while the forward kernel still runs; then a3 (32 KB) is the only input left.
// Instantiated twice, as mlp_chain_kernel: dense_tail_kernel (W = false) and dense_tail_weighted_kernel.
template <int D0, int D1, int D2, int CS, bool W>
__device__ __forceinline__ void dense_tail_body(const MlpChainParams& p) {
  using L = TailSmem<D0, D1, D2, CS>;
  constexpr int NS1 = L::NS1, NS2 = L::NS2;
  static_assert((CS & (CS - 1)) == 0, "cluster size must be a power of two");
  static_assert(NS1 % 8 == 0 && NS2 % 4 == 0 && L::KS0 % 4 == 0, "slices must hold whole register tiles");
  static_assert(L::BAR % 2 == 0 && L::SCRATCH % 4 == 0, "mbarriers are 8-byte aligned, the scratch 16-byte aligned");
  extern __shared__ __align__(16) float sm[];
  float* sW0 = sm + L::W0; float* sW1 = sm + L::W1; float* sA3 = sm + L::A3; float* sW2 = sm + L::W2; float* sA3own = sm + L::A3OWN;
  float* sB1 = sm + L::MISC + NS1; float* sB2 = sB1 + NS2; float* sLab = sB2 + 16;
  uint64_t* bar = reinterpret_cast<uint64_t*>(sm + L::BAR);
  uint64_t* bar_a4 = bar; uint64_t* bar_dz3 = bar + 1;
  cg::cluster_group cluster = cg::this_cluster();
  const int cr = (int)cluster.block_rank();
  const int tid = threadIdx.x;
  const int B = p.B, C = p.C;
  auto stamp = [&](int slot) {
    if (p.dbg != nullptr && blockIdx.x == 0 && tid == 0) { unsigned long long t; asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t)); p.dbg[slot] = t; }
  };
  stamp(0);
  if (p.from_dz3) {     // dx = dz3 W0 only, nothing exchanged between the CTAs
    dense_dx_rows<L, D0, D1, CS>(sm, p, cr, stamp);
    return;
  }
  if (tid == 0) {
    for (int i = 0; i < 2; ++i) mbar_init(bar + i, 1);
    mbar_arrive_expect_tx(bar_a4, MC_B * D2 * 4);
    mbar_arrive_expect_tx(bar_dz3, (CS - 1) * MC_B * NS1 * 4);
    fence_barrier_init();
  }
  asm volatile("barrier.cluster.arrive.relaxed.aligned;" ::: "memory");
  // ---------------- prologue (independent of the forward kernel)
  stage_swizzled_async(sW1, p.w1 + (long long)cr * NS2 * D1, NS2, D1, D1);
  stage_head_async<D2, NS2>(sW2, sB1, sB2, p.w2, p.b1, p.b2, cr, C);
  stage_plain_async(sW0, p.w0 + cr * L::KS0, D1, L::KS0, D0);
  cp_async_commit();
  stamp(1);
  pdl_wait();
  pdl_launch();
  stamp(2);
  // a3 (rows >= B zero), this CTA's own a3 columns, the labels
  for (int c = tid; c < MC_B * (D1 >> 2); c += MC_THREADS) {
    const int r = c / (D1 >> 2), q = c - r * (D1 >> 2);
    if (r < B) cp_async16(sA3 + sw_off(r, q << 2, D1), p.a3 + (long long)r * D1 + (q << 2));
    else *reinterpret_cast<float4*>(sA3 + sw_off(r, q << 2, D1)) = make_float4(0.f, 0.f, 0.f, 0.f);
  }
  for (int c = tid; c < MC_B * (NS1 >> 2); c += MC_THREADS) {
    const int r = c / (NS1 >> 2), q = c - r * (NS1 >> 2);
    if (r < B) cp_async16(sA3own + r * NS1 + (q << 2), p.a3 + (long long)r * D1 + cr * NS1 + (q << 2));
    else *reinterpret_cast<float4*>(sA3own + r * NS1 + (q << 2)) = make_float4(0.f, 0.f, 0.f, 0.f);
  }
  if (tid < MC_B) sLab[tid] = tid < B ? p.label[tid] : 0.f;
  cp_async_commit();
  cp_async_wait<0>();
  __syncthreads();
  cluster.barrier_wait();
  stamp(3);
  dense_chain_body<L, D0, D1, D2, CS, false, W>(sm, p, cr, nullptr, bar_a4, bar_dz3, stamp);
}
template <int D0, int D1, int D2, int CS>
__global__ void __cluster_dims__(CS, 1, 1) __launch_bounds__(MC_THREADS, 1) dense_tail_kernel(const MlpChainParams p) {
  dense_tail_body<D0, D1, D2, CS, false>(p);
}
template <int D0, int D1, int D2, int CS>
__global__ void __cluster_dims__(CS, 1, 1) __launch_bounds__(MC_THREADS, 1) dense_tail_weighted_kernel(const MlpChainParams p) {
  dense_tail_body<D0, D1, D2, CS, true>(p);
}

// ---- the dense weight gradients, from what mlp_chain_kernel stored: dW0 = dz3^T x, dW1 = dz4^T a3, dW2 = dl^T a4, and the bias gradients
// as column sums.  K = B <= 32, so every output is one register-held fmaf chain over b; one thread per 4 x 4 tile (or per bias element).
struct DenseWgradParams {
  const float* x; const float* a3; const float* a4; const float* dz4; const float* dz3; const float* dl;   // rows b < B
  float* dw0; float* db0; float* dw1; float* db1; float* dw2; float* db2;
  int B, C;
  unsigned long long* dbg;   // optional: 16 start of CTA 0 | 17 its grid dependency resolved | 18 end of the last CTA
};
constexpr int WG_THREADS = 256;
template <int D0, int D1, int D2>
struct DenseWgradGrid {
  static constexpr int T0 = (D1 / 4) * (D0 / 4), T1 = (D2 / 4) * (D1 / 4), T2 = (MC_CMAX / 4) * (D2 / 4);   // 4 x 4 tiles of dW0, dW1, dW2
  static constexpr int THREADS = T0 + T1 + T2 + D1 + D2 + MC_CMAX;                                            // + db0, db1, db2
  static constexpr int CTAS = (THREADS + WG_THREADS - 1) / WG_THREADS;
};

template <int D0, int D1, int D2>
__global__ void __launch_bounds__(WG_THREADS) dense_wgrad_kernel(const DenseWgradParams p) {
  using G = DenseWgradGrid<D0, D1, D2>;
  const bool stamps = p.dbg != nullptr && threadIdx.x == 0;
  auto now = [] { unsigned long long t; asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t)); return t; };
  if (stamps && blockIdx.x == 0) p.dbg[16] = now();
  pdl_launch();   // the dense keys' exchange behind this kernel may become resident and stage; its own griddepcontrol.wait covers this grid
  pdl_wait();
  if (stamps && blockIdx.x == 0) p.dbg[17] = now();
  const int B = p.B;
  int t = blockIdx.x * WG_THREADS + threadIdx.x;
  if (t < G::T0) {
    wgrad_4x4<D1, D0>(p.dz3, p.x, B, 4 * (t / (D0 / 4)), 4 * (t % (D0 / 4)), D1, p.dw0);
  } else if ((t -= G::T0) < G::T1) {
    wgrad_4x4<D2, D1>(p.dz4, p.a3, B, 4 * (t / (D1 / 4)), 4 * (t % (D1 / 4)), D2, p.dw1);
  } else if ((t -= G::T1) < G::T2) {
    wgrad_4x4<MC_CMAX, D2>(p.dl, p.a4, B, 4 * (t / (D2 / 4)), 4 * (t % (D2 / 4)), p.C, p.dw2);
  } else if ((t -= G::T2) < D1) {
    p.db0[t] = colsum<D1>(p.dz3, B, t);
  } else if ((t -= D1) < D2) {
    p.db1[t] = colsum<D2>(p.dz4, B, t);
  } else if ((t -= D2) < p.C) {
    p.db2[t] = colsum<MC_CMAX>(p.dl, B, t);
  }
  if (p.dbg != nullptr) {
    __syncthreads();
    if (threadIdx.x == 0) atomicMax(p.dbg + 18, now());
  }
}

}  // namespace gx

using namespace gx;

// 512 -> 256 -> 128 -> C (C <= 16), B <= 32.  TAIL: dense_tail_kernel, else mlp_chain_kernel; W: their weighted instances.  Returns -2 when
// this cluster size cannot be scheduled on this device.
template <bool TAIL, bool W, int CS>
static int mlp_launch(const MlpChainParams& p, cudaStream_t stream) {
  constexpr int BYTES = TAIL ? TailSmem<512, 256, 128, CS>::BYTES : MlpSmem<512, 256, 128, CS>::BYTES;
  auto kern = TAIL ? (W ? dense_tail_weighted_kernel<512, 256, 128, CS> : dense_tail_kernel<512, 256, 128, CS>)
                   : (W ? mlp_chain_weighted_kernel<512, 256, 128, CS> : mlp_chain_kernel<512, 256, 128, CS>);
  static int ready = 0;      // 0 = not configured, 1 = ok, -1 = this cluster size cannot be scheduled on this device
  if (ready == 0) {
    ready = -1;
    if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, BYTES) == cudaSuccess &&
        (CS <= 8 || cudaFuncSetAttribute(kern, cudaFuncAttributeNonPortableClusterSizeAllowed, 1) == cudaSuccess)) {
      cudaLaunchConfig_t cfg = {};
      cfg.gridDim = dim3(CS); cfg.blockDim = dim3(MC_THREADS); cfg.dynamicSmemBytes = BYTES;
      cudaLaunchAttribute at[1];
      at[0].id = cudaLaunchAttributeClusterDimension; at[0].val.clusterDim.x = CS; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
      cfg.attrs = at; cfg.numAttrs = 1;
      int nclusters = 0;
      if (cudaOccupancyMaxActiveClusters(&nclusters, kern, &cfg) == cudaSuccess && nclusters >= 1) ready = 1;
    }
    cudaGetLastError();
  }
  if (ready < 0) return -2;
  static int use_pdl = -1;
  if (use_pdl < 0) { const char* e = getenv("GEOMX_MLP_PDL"); use_pdl = (e && e[0] == '0') ? 0 : 1; }
  // dense_tail_kernel from dz3 (dense_dx_rows): one cluster per DX_ROWS rows, DX_THREADS threads, only the smem that mode uses
  using T = TailSmem<512, 256, 128, CS>;
  const bool dx_only = TAIL && p.from_dz3;
  const dim3 grid(dx_only ? CS * ((p.B + T::DX_ROWS - 1) / T::DX_ROWS) : CS), block(dx_only ? DX_THREADS : MC_THREADS);
  const size_t smem = dx_only ? (size_t)T::DX_BYTES : (size_t)BYTES;
  if (use_pdl) launch_pdl(kern, grid, block, smem, stream, p);
  else kern<<<grid, block, smem, stream>>>(p);
  return GX_CHECK_LAUNCH();
}
// cluster of 16 CTAs (one GPC) halves every slice; fall back to the portable size 8 when the device cannot co-schedule 16
template <bool TAIL, bool W>
static int mlp_launch_any(const MlpChainParams& p, cudaStream_t stream) {
  static int want = -1;
  if (want < 0) { const char* e = getenv("GEOMX_MLP_CLUSTER"); want = e ? atoi(e) : 16; }
  if (want >= 16) {
    const int rc = mlp_launch<TAIL, W, 16>(p, stream);
    if (rc != -2) return rc;
    want = 8;
  }
  return mlp_launch<TAIL, W, 8>(p, stream);
}

static unsigned long long* g_mlp_dbg = nullptr;
GX_API int gx_mlp_chain_set_debug(unsigned long long* p) { g_mlp_dbg = p; return 0; }

// the data path: loss, logits, dx; stores a3, a4, dz4, dz3 and the dlogits (rows b < B) for gx_dense_wgrad.  coef [B] (may be null): the
// dlogits of row b are scaled by coef[b] before anything is derived from them (mlp_chain_weighted_kernel); the loss is not.  Returns -1 for
// unsupported shapes (caller uses the per-layer kernels).
GX_API int gx_mlp_chain(const float* x, const float* w0, const float* b0, const float* w1, const float* b1, const float* w2, const float* b2,
                        const float* label, float* loss, float* logits, float* dx, float* a3, float* a4, float* dz4, float* dz3, float* dl,
                        const float* coef, int B, int D0, int D1, int D2, int C, cudaStream_t stream) {
  if (D0 != 512 || D1 != 256 || D2 != 128 || C < 1 || C > MC_CMAX || B < 1 || B > MC_B) return -1;
  MlpChainParams p;
  p.x = x; p.w0 = w0; p.b0 = b0; p.w1 = w1; p.b1 = b1; p.w2 = w2; p.b2 = b2; p.label = label; p.loss = loss; p.logits = logits; p.dx = dx;
  p.a3 = a3; p.a4 = a4; p.dz4 = dz4; p.dz3 = dz3; p.dl = dl; p.B = B; p.C = C; p.dbg = g_mlp_dbg; p.coef = coef;
  return coef != nullptr ? mlp_launch_any<false, true>(p, stream) : mlp_launch_any<false, false>(p, stream);
}

// the same data path from a3 [B][D1] (computed by gx_cnn_fwd_dense0): loss, logits, dx; stores a4, dz4, dz3 and the dlogits for
// gx_dense_wgrad.  w0 is read only as the column slices of dx.  from_dz3 != 0: dx = dz3 [B][D1] · w0 only (dz3 computed by gx_cnn_fwd_dense0's
// training head); nothing else is read or written.  coef [B] (may be null, and must be without from_dz3, whose dz3 already carries it): the
// dlogits of row b are scaled by coef[b] (dense_tail_weighted_kernel), as in gx_mlp_chain.  Returns -1 for unsupported shapes.
GX_API int gx_dense_tail(const float* a3, const float* w0, const float* w1, const float* b1, const float* w2, const float* b2, const float* label,
                         float* loss, float* logits, float* dx, float* a4, float* dz4, float* dz3, float* dl, const float* coef, int B, int D0, int D1,
                         int D2, int C, int from_dz3, cudaStream_t stream) {
  if (D0 != 512 || D1 != 256 || D2 != 128 || C < 1 || C > MC_CMAX || B < 1 || B > MC_B || (coef != nullptr && from_dz3)) return -1;
  MlpChainParams p = {};
  p.w0 = w0; p.w1 = w1; p.b1 = b1; p.w2 = w2; p.b2 = b2; p.label = label; p.loss = loss; p.logits = logits; p.dx = dx;
  p.a3 = const_cast<float*>(a3); p.a4 = a4; p.dz4 = dz4; p.dz3 = dz3; p.dl = dl; p.B = B; p.C = C; p.dbg = g_mlp_dbg;
  p.from_dz3 = from_dz3 != 0;
  p.coef = coef;
  return coef != nullptr ? mlp_launch_any<true, true>(p, stream) : mlp_launch_any<true, false>(p, stream);
}

// dW0 / db0, dW1 / db1, dW2 / db2 (overwritten) from what gx_mlp_chain stored; x has exactly B rows, dl rows hold 16 floats
GX_API int gx_dense_wgrad(const float* x, const float* a3, const float* a4, const float* dz4, const float* dz3, const float* dl, float* dw0,
                          float* db0, float* dw1, float* db1, float* dw2, float* db2, int B, int D0, int D1, int D2, int C, cudaStream_t stream) {
  if (D0 != 512 || D1 != 256 || D2 != 128 || C < 1 || C > MC_CMAX || B < 1 || B > MC_B) return -1;
  DenseWgradParams p;
  p.x = x; p.a3 = a3; p.a4 = a4; p.dz4 = dz4; p.dz3 = dz3; p.dl = dl;
  p.dw0 = dw0; p.db0 = db0; p.dw1 = dw1; p.db1 = db1; p.dw2 = dw2; p.db2 = db2; p.B = B; p.C = C; p.dbg = g_mlp_dbg;
  launch_pdl(dense_wgrad_kernel<512, 256, 128>, dim3(DenseWgradGrid<512, 256, 128>::CTAS), dim3(WG_THREADS), 0, stream, p);
  return GX_CHECK_LAUNCH();
}
GX_API int gx_mlp_chain_smem_bytes() { return MlpSmem<512, 256, 128, 8>::BYTES; }
GX_API int gx_dense_tail_smem_bytes() { return TailSmem<512, 256, 128, 16>::BYTES; }
