// wgmma / TMA GEMM for sm_90a:   D[M,N] = epilogue( alpha * A[M,K] * B[N,K]^T )
//
//  * operands are fp32 in global memory, multiplied on the Hopper tensor cores as TF32 (wgmma .f32.tf32.tf32) with fp32
//    accumulation in registers — the closest tensor-core analogue of the reference's cublasSgemmEx path
//    (reference src/operator/linalg_impl.h:196-214, FullyConnected src/operator/nn/fully_connected-inl.h:71-173,
//    Convolution im2col+GEMM src/operator/nn/convolution-inl.h:165-284).
//  * each operand may be K-major (row-major [rows][K]) or MN-major (row-major [K][rows]) so that forward, dgrad
//    (dY*W) and wgrad (dY^T*X) all read the tensors where they already live — no transposes are materialised in global memory.
//    wgmma takes tf32 operands K-major only, so an MN-major tile is transposed in shared memory on its way to the tensor core.
//  * warp-specialised, one 128 x BLOCK_N tile per CTA, 384 threads: warp 0 = TMA producer (cp.async.bulk.tensor, mbarrier ring),
//    warps 1-3 = staging (3xTF32 hi/lo split, MN-major -> K-major SWIZZLE_128B transpose), warps 4-11 = two consumer warpgroups of
//    64 rows each (wgmma issue, then the epilogue through shared memory: fused bias / ReLU / ReLU-mask / column-sum (bias gradient) /
//    NCHW scatter / 2x2 max-pool / split-K atomic accumulate).
//
// Precision: the default is **3xTF32** (fp32-accurate): every operand tile that TMA lands in shared memory is split by the staging warps
// into hi = rn_tf32(x) and lo = rn_tf32(x - hi); the consumer warpgroups then issue lo*hi + hi*lo + hi*hi into the same fp32 accumulator.
// The dropped lo*lo term and the rounding of lo are ~2^-22 relative per product, i.e. the result matches an fp32 SGEMM (the reference's
// cublasSgemmEx with CUDA_R_32F, linalg_impl.h:196-214) to fp32 rounding.  `gx_gemm_set_precision(1)` / GEOMX_GEMM_PRECISION=tf32 selects
// plain TF32 (one MMA per K step; K-major operands then go from TMA straight to the tensor core).
//
// Tile shapes: wgmma M=64 per warpgroup (BLOCK_M = 128), N=BLOCK_N in {16,32,64,128}, K=8 per instruction (32 B of tf32), BLOCK_K = 32
// fp32 = one 128-byte swizzle atom per row.  Out-of-bounds rows/cols/k are zero-filled by TMA, masked in the epilogue.
#include <cuda.h>

#include <atomic>

#include "common.cuh"

namespace gx {

constexpr int BLOCK_M = 128;
constexpr int BLOCK_K = 32;
constexpr int WG_K = 8;                   // K of one wgmma instruction
constexpr int GEMM_THREADS = 384;         // warp 0 TMA, warps 1-3 staging, warps 4-11 two consumer warpgroups
constexpr int STAGE_THREADS = 96;
constexpr int CONSUMER_THREADS = 256;
constexpr int ACC_CHUNK_KB = 4;           // 3xTF32: K blocks accumulated by the tensor core before the partial sum is added in fp32 registers
constexpr int A_TILE_BYTES = BLOCK_M * BLOCK_K * 4;  // 16 KiB
constexpr int MN_BOX_BYTES = 32 * BLOCK_K * 4;       // one 32(MN) x 32(K) box = 4 KiB
constexpr int MAX_STAGES = 8;
constexpr int SMEM_BUDGET = 200 * 1024;

struct GemmParams {
  int M, N, K;
  int kb_per_split;
  float* D;
  long long ldd;
  const float* bias;
  const float* mask;
  long long ldmask;
  float* colsum;
  int relu, accumulate, store_mode, hw;
  int pool_w;              // store_mode 2: width of the (pre-pool) feature map; rows are (image, oh, ow)
  unsigned char* pool_idx; // store_mode 2: arg-max position (0..3) of every pooled element, same layout as D
  float alpha;
  int a_boxes, b_boxes;    // MN-major operands: number of 32-wide TMA boxes that are (partly) in bounds for this problem
  int a_bytes, b_bytes;    // bytes of the A / B tile that TMA actually fills per stage (what the staging warps have to touch)
  int tx_bytes;            // bytes that land per stage (A box(es) + B box(es)); out-of-range rows/boxes are never requested
  int stages;              // TMA ring depth actually used (<= SmemLayout::STAGES)
  unsigned long long* dbg; // optional: %globaltimer stamps of CTA (0,0,0) phases (tools/kernel_times.py)
};

// One ring stage: [A as landed | B as landed | A transposed (A MN-major) | B transposed (B MN-major) | A lo | B lo (3xTF32)].
// A K-major operand lands in the wgmma layout (TMA SWIZZLE_128B) and is split in place; an MN-major one lands as plain 32x32 boxes.
template <int BLOCK_N, bool A_MN, bool B_MN, bool SPLIT>
struct SmemLayout {
  static_assert(BLOCK_N >= 16 && BLOCK_N % 16 == 0, "wgmma N");
  static constexpr int B_TILE_BYTES = BLOCK_N * BLOCK_K * 4;
  static constexpr int A_RAW = 0, B_RAW = A_TILE_BYTES;
  static constexpr int A_T = A_TILE_BYTES + B_TILE_BYTES;
  static constexpr int B_T = A_T + (A_MN ? A_TILE_BYTES : 0);
  static constexpr int A_LO = B_T + (B_MN ? B_TILE_BYTES : 0);
  static constexpr int B_LO = A_LO + A_TILE_BYTES;
  static constexpr int STAGE_BYTES = SPLIT ? B_LO + B_TILE_BYTES : A_LO;
  static constexpr int A_OP = A_MN ? A_T : A_RAW, B_OP = B_MN ? B_T : B_RAW;   // what the tensor core reads (hi parts in 3xTF32)
  static constexpr bool STAGING = SPLIT || A_MN || B_MN;
  static constexpr int STAGES = SMEM_BUDGET / STAGE_BYTES < MAX_STAGES ? SMEM_BUDGET / STAGE_BYTES : MAX_STAGES;
  static constexpr int EPI_LD = BLOCK_N + 1;                                  // output tile staged for the row-wise epilogue
  static constexpr int EPI_BYTES = BLOCK_M * EPI_LD * 4;
  static constexpr int bytes(int stages) { return (stages * STAGE_BYTES > EPI_BYTES ? stages * STAGE_BYTES : EPI_BYTES) + 1024; }
};

// hi = rn_tf32(x) (low 13 mantissa bits zero), lo = rn_tf32(x - hi): x = hi + lo up to ~2^-22 |x|
__device__ __forceinline__ void split_tf32(float x, float& hi, float& lo) {
  uint32_t h, l;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(h) : "f"(x));
  hi = __uint_as_float(h);
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(l) : "f"(x - hi));
  lo = __uint_as_float(l);
}
__device__ __forceinline__ float4 split4(float4 v, float4& lo) {
  float4 h;
  split_tf32(v.x, h.x, lo.x); split_tf32(v.y, h.y, lo.y); split_tf32(v.z, h.z, lo.z); split_tf32(v.w, h.w, lo.w);
  return h;
}
// K-major tile: split `bytes` in place (hi) and into the lo copy `lo_off` bytes further; element-wise => swizzle agnostic
__device__ __forceinline__ void split_region(uint8_t* base, int bytes, int lo_off, int tid) {
  for (int off = tid * 16; off < bytes; off += STAGE_THREADS * 16) {
    float4 l;
    const float4 h = split4(*reinterpret_cast<const float4*>(base + off), l);
    *reinterpret_cast<float4*>(base + off) = h;
    *reinterpret_cast<float4*>(base + off + lo_off) = l;
  }
}
// MN-major tile: `rows` rows of 32-wide boxes [box][k][32] -> K-major SWIZZLE_128B [row][k] (16-B chunk c of row r at
// r*128 + ((c ^ (r & 7)) << 4), the layout TMA would have produced), hi and (3xTF32) lo
template <bool SPLIT>
__device__ __forceinline__ void transpose_region(const uint8_t* raw, uint8_t* hi, uint8_t* lo, int rows, int tid) {
  for (int i = tid; i < rows * 8; i += STAGE_THREADS) {
    const int c = i / rows, r = i - c * rows;
    const float* src = reinterpret_cast<const float*>(raw + (r >> 5) * MN_BOX_BYTES) + (r & 31) + c * 4 * 32;
    const float4 v = make_float4(src[0], src[32], src[64], src[96]);
    const int off = r * 128 + ((c ^ (r & 7)) << 4);
    if constexpr (SPLIT) {
      float4 l;
      *reinterpret_cast<float4*>(hi + off) = split4(v, l);
      *reinterpret_cast<float4*>(lo + off) = l;
    } else {
      *reinterpret_cast<float4*>(hi + off) = v;
    }
  }
}

template <int BLOCK_N>
__device__ __forceinline__ void wgmma_tf32(float (&d)[BLOCK_N / 2], uint64_t da, uint64_t db, uint32_t scale_d) {
  if constexpr (BLOCK_N == 16) wgmma_tf32_n16(d, da, db, scale_d);
  else if constexpr (BLOCK_N == 32) wgmma_tf32_n32(d, da, db, scale_d);
  else if constexpr (BLOCK_N == 64) wgmma_tf32_n64(d, da, db, scale_d);
  else wgmma_tf32_n128(d, da, db, scale_d);
}

template <int BLOCK_N, bool A_MN, bool B_MN, bool SPLIT>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_tf32_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const GemmParams p) {
  using L = SmemLayout<BLOCK_N, A_MN, B_MN, SPLIT>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  __shared__ __align__(8) uint64_t full_bar[MAX_STAGES], empty_bar[MAX_STAGES], ready_bar[MAX_STAGES];
  __shared__ float s_bias[BLOCK_N];
  const int STAGES = p.stages;

  pdl_launch();  // let the next kernel begin its own prologue right away
  const bool dbg_on = p.dbg != nullptr && blockIdx.x == 0 && blockIdx.y == 0 && blockIdx.z == 0;
  auto stamp = [&](int slot) { if (dbg_on) { unsigned long long t; asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t)); p.dbg[slot] = t; } };
  if (threadIdx.x == 0) stamp(0);
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int n0 = blockIdx.x * BLOCK_N;
  const int m0 = blockIdx.y * BLOCK_M;
  const int num_kb = (p.K + BLOCK_K - 1) / BLOCK_K;
  const int kb_begin = blockIdx.z * p.kb_per_split;
  const int kb_end = min(num_kb, kb_begin + p.kb_per_split);

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], CONSUMER_THREADS / 32);
      mbar_init(&ready_bar[s], STAGE_THREADS);
    }
    fence_barrier_init();
  }
  __syncthreads();
  if (threadIdx.x == 0) stamp(1);
  pdl_wait();    // everything above overlapped the previous kernel's tail; from here on we touch its outputs
  if (threadIdx.x == 0) stamp(2);

  if (warp == 0) {
    // ================================ TMA producer ================================
    if (lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int kb = kb_begin; kb < kb_end; ++kb) {
        mbar_wait(&empty_bar[stage], phase ^ 1u);
        uint8_t* sA = smem + stage * L::STAGE_BYTES + L::A_RAW;
        uint8_t* sB = smem + stage * L::STAGE_BYTES + L::B_RAW;
        mbar_arrive_expect_tx(&full_bar[stage], p.tx_bytes);
        const int k0 = kb * BLOCK_K;
        if constexpr (!A_MN) {
          tma_load_2d(sA, &tmA, &full_bar[stage], k0, m0);
        } else {
#pragma unroll
          for (int j = 0; j < BLOCK_M / 32; ++j)
            if (j < p.a_boxes) tma_load_2d(sA + j * MN_BOX_BYTES, &tmA, &full_bar[stage], m0 + 32 * j, k0);
        }
        if constexpr (!B_MN) {
          tma_load_2d(sB, &tmB, &full_bar[stage], k0, n0);
        } else {
#pragma unroll
          for (int j = 0; j < BLOCK_N / 32; ++j)
            if (j < p.b_boxes) tma_load_2d(sB + j * MN_BOX_BYTES, &tmB, &full_bar[stage], n0 + 32 * j, k0);
        }
        if (++stage == STAGES) { stage = 0; phase ^= 1u; }
      }
    }
    return;
  }
  if (warp < 4) {
    // ================================ staging (warps 1-3): landed stage -> wgmma operands ================================
    if constexpr (L::STAGING) {
      const int et = threadIdx.x - 32;
      int stage = 0;
      uint32_t phase = 0;
      for (int kb = kb_begin; kb < kb_end; ++kb) {
        mbar_wait(&full_bar[stage], phase);
        uint8_t* base = smem + stage * L::STAGE_BYTES;
        if constexpr (A_MN) transpose_region<SPLIT>(base + L::A_RAW, base + L::A_T, base + L::A_LO, 32 * p.a_boxes, et);
        else if constexpr (SPLIT) split_region(base + L::A_RAW, p.a_bytes, L::A_LO - L::A_RAW, et);
        if constexpr (B_MN) transpose_region<SPLIT>(base + L::B_RAW, base + L::B_T, base + L::B_LO, 32 * p.b_boxes, et);
        else if constexpr (SPLIT) split_region(base + L::B_RAW, p.b_bytes, L::B_LO - L::B_RAW, et);
        fence_proxy_async_smem();      // generic-proxy writes -> visible to the tensor core's (async proxy) operand reads
        mbar_arrive(&ready_bar[stage]);
        if (++stage == STAGES) { stage = 0; phase ^= 1u; }
      }
    }
    return;
  }

  // ================================ consumers (warps 4-11): wgmma main loop ================================
  constexpr int R = BLOCK_N / 2;          // accumulator registers per thread (64 x BLOCK_N per warpgroup)
  const int wg = (warp - 4) >> 2;
  const int ct = threadIdx.x - 128;
  const bool wg_rows = m0 + 64 * wg < p.M;   // warpgroup-uniform: a warpgroup whose 64 rows are all out of range issues no MMA
  float acc[R];
  float sum[SPLIT ? R : 1];   // 3xTF32: running fp32 sum of the finished accumulator chunks (IEEE adds in registers)
#pragma unroll
  for (int j = 0; j < R; ++j) acc[j] = 0.f;
#pragma unroll
  for (int j = 0; j < (SPLIT ? R : 1); ++j) sum[j] = 0.f;
  {
    int stage = 0;
    uint32_t phase = 0;
    for (int kb = kb_begin; kb < kb_end; ++kb) {
      // The tensor core's fp32 accumulation is not round-to-nearest: its error is biased and grows with the number of MMAs folded into one
      // accumulator.  The 3xTF32 mode therefore lets the tensor core accumulate at most ACC_CHUNK_KB K blocks (48 MMAs) and adds every
      // finished chunk into fp32 registers with IEEE adds.
      const int rel = kb - kb_begin;
      const bool chunk_first = SPLIT ? (rel % ACC_CHUNK_KB) == 0 : rel == 0;
      const bool chunk_last = SPLIT && ((rel % ACC_CHUNK_KB) == ACC_CHUNK_KB - 1 || kb == kb_end - 1);
      mbar_wait(L::STAGING ? &ready_bar[stage] : &full_bar[stage], phase);
      if (kb == kb_begin && ct == 0) stamp(3);
      if (wg_rows) {
        uint8_t* base = smem + stage * L::STAGE_BYTES;
        const uint32_t a_hi = smem_u32(base + L::A_OP) + wg * 64 * 128, b_hi = smem_u32(base + L::B_OP);
        const uint32_t a_lo = smem_u32(base + L::A_LO) + wg * 64 * 128, b_lo = smem_u32(base + L::B_LO);
        wgmma_fence_regs(acc);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BLOCK_K / WG_K; ++k) {
          const uint32_t o = k * WG_K * 4;
          const uint32_t sc = (chunk_first && k == 0) ? 0u : 1u;
          if constexpr (SPLIT) {
            // small terms first: a_lo*b_hi + a_hi*b_lo + a_hi*b_hi, all into the same fp32 accumulator
            wgmma_tf32<BLOCK_N>(acc, gmma_desc_sw128(a_lo + o), gmma_desc_sw128(b_hi + o), sc);
            wgmma_tf32<BLOCK_N>(acc, gmma_desc_sw128(a_hi + o), gmma_desc_sw128(b_lo + o), 1u);
            wgmma_tf32<BLOCK_N>(acc, gmma_desc_sw128(a_hi + o), gmma_desc_sw128(b_hi + o), 1u);
          } else {
            wgmma_tf32<BLOCK_N>(acc, gmma_desc_sw128(a_hi + o), gmma_desc_sw128(b_hi + o), sc);
          }
        }
        wgmma_commit();
        wgmma_wait_all();
        wgmma_fence_regs(acc);
        if constexpr (SPLIT) {
          if (chunk_last) {
#pragma unroll
            for (int j = 0; j < R; ++j) sum[j] += acc[j];
          }
        }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty_bar[stage]);   // this warp's reads of the stage are complete
      if (++stage == STAGES) { stage = 0; phase ^= 1u; }
    }
  }
  if (ct == 0) stamp(4);

  // ================================ epilogue: accumulators -> smem tile -> one row per thread ================================
  named_bar_sync(1, CONSUMER_THREADS);   // every consumer is done with the ring: it becomes the output tile
  float* sD = reinterpret_cast<float*>(smem);
  {
    const int r0 = 64 * wg + 16 * ((warp - 4) & 3) + (lane >> 2), c0 = 2 * (lane & 3);
#pragma unroll
    for (int i = 0; i < BLOCK_N / 8; ++i) {
      const float* f = SPLIT ? sum : acc;
      sD[r0 * L::EPI_LD + 8 * i + c0] = f[4 * i];
      sD[r0 * L::EPI_LD + 8 * i + c0 + 1] = f[4 * i + 1];
      sD[(r0 + 8) * L::EPI_LD + 8 * i + c0] = f[4 * i + 2];
      sD[(r0 + 8) * L::EPI_LD + 8 * i + c0 + 1] = f[4 * i + 3];
    }
    for (int j = ct; j < BLOCK_N; j += CONSUMER_THREADS) s_bias[j] = (p.bias != nullptr && n0 + j < p.N && blockIdx.z == 0) ? __ldg(p.bias + n0 + j) : 0.f;
  }
  named_bar_sync(1, CONSUMER_THREADS);
  if (ct == 0) stamp(5);
  // thread ct owns row ct % 128 and half of the columns; a warp = 32 consecutive rows (the fused pooling's windows never leave it)
  constexpr int HALF = BLOCK_N / 2;
  const int row = ct & (BLOCK_M - 1), cb = (ct / BLOCK_M) * HALF;
  const int m = m0 + row;
  const bool row_ok = m < p.M;
  const bool warp_has_rows = (m0 + (row & ~31)) < p.M;   // warp-uniform
  const bool have_acc = kb_end > kb_begin;
  if (warp_has_rows) {
#pragma unroll
    for (int c0 = cb; c0 < cb + HALF; c0 += 4) {
      if (n0 + c0 >= p.N) break;  // warp-uniform
      const bool full = n0 + c0 + 4 <= p.N;
      float v[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int n = n0 + c0 + j;
        float x = have_acc ? sD[row * L::EPI_LD + c0 + j] * p.alpha : 0.f;
        x += s_bias[c0 + j];
        if (p.relu) x = fmaxf(x, 0.f);
        if (p.mask != nullptr) x = (row_ok && n < p.N && __ldg(p.mask + (long long)m * p.ldmask + n) > 0.f) ? x : 0.f;
        v[j] = (row_ok && n < p.N) ? x : 0.f;
      }
      if (p.colsum != nullptr) {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float s = warp_sum(v[j]);
          if (lane == 0 && n0 + c0 + j < p.N) atomicAdd(p.colsum + n0 + c0 + j, s);
        }
      }
      if (p.store_mode == 2) {
        // fused 2x2/2 max-pool of an NCHW feature map (ReLU already applied): row m = (image, oh, ow); the three partners of a window's
        // top-left element sit 1, W and W+1 lanes further in the same warp (host guarantees 32 % (2W) == 0 and hw % 32 == 0).
        // First maximum wins, like maxpool2x2_fwd_kernel; only pooled values + arg-max leave the SM.
        const int W = p.pool_w, pix = m % p.hw, oh = pix / W, ow = pix - oh * W, img = m / p.hw;
        const bool base = row_ok && ((oh & 1) == 0) && ((ow & 1) == 0);
        const int PW = W >> 1, PHW = p.hw >> 2;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float a01 = __shfl_down_sync(0xffffffffu, v[j], 1), a10 = __shfl_down_sync(0xffffffffu, v[j], W),
                      a11 = __shfl_down_sync(0xffffffffu, v[j], W + 1);
          const int n = n0 + c0 + j;
          if (base && n < p.N) {
            float best = v[j]; int bi = 0;
            if (a01 > best) { best = a01; bi = 1; }
            if (a10 > best) { best = a10; bi = 2; }
            if (a11 > best) { best = a11; bi = 3; }
            const long long o = ((long long)img * p.N + n) * PHW + (oh >> 1) * PW + (ow >> 1);
            p.D[o] = best;
            p.pool_idx[o] = (unsigned char)bi;
          }
        }
      } else if (row_ok) {
        if (p.store_mode == 0) {
          float* dst = p.D + (long long)m * p.ldd + n0 + c0;
          if (((p.ldd & 3) == 0) && ((reinterpret_cast<uintptr_t>(p.D) & 15) == 0) && full && !p.accumulate) {
            *reinterpret_cast<float4*>(dst) = make_float4(v[0], v[1], v[2], v[3]);
          } else {
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              if (n0 + c0 + j < p.N) {
                if (p.accumulate) atomicAdd(dst + j, v[j]);
                else dst[j] = v[j];
              }
            }
          }
        } else {
          // NCHW scatter: row m = (image, pixel), column n = channel
          const int img = m / p.hw, pix = m - img * p.hw;
          float* dst = p.D + ((long long)img * p.N) * p.hw + pix;
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const int n = n0 + c0 + j;
            if (n < p.N) {
              if (p.accumulate) atomicAdd(dst + (long long)n * p.hw, v[j]);
              else dst[(long long)n * p.hw] = v[j];
            }
          }
        }
      }
    }
  }
  if (ct == 0) stamp(6);
}

// ------------------------------------------------------------------------------------------------ host
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                    const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiled get_encode() {
  static PFN_encodeTiled fn = nullptr;
  if (fn == nullptr) {
    void* ptr = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<PFN_encodeTiled>(ptr);
  }
  return fn;
}

// inner = contiguous dimension (elements), outer = strided dimension, ld = elements between outer rows
static int make_tmap(CUtensorMap* tm, const float* base, long long inner, long long outer, long long ld, int box_inner, int box_outer, bool mn_major) {
  PFN_encodeTiled enc = get_encode();
  if (enc == nullptr) return -2;
  cuuint64_t gdim[2] = {(cuuint64_t)inner, (cuuint64_t)outer};
  cuuint64_t gstride[1] = {(cuuint64_t)ld * 4};
  cuuint32_t box[2] = {(cuuint32_t)box_inner, (cuuint32_t)box_outer};
  cuuint32_t estr[2] = {1, 1};
  // driver entry points need a current context on the calling thread (autograd worker threads may never have made a runtime call)
  static thread_local bool ctx_bound = false;
  if (!ctx_bound) { cudaFree(nullptr); ctx_bound = true; }
  CUresult r = enc(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(base), gdim, gstride, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   mn_major ? CU_TENSOR_MAP_SWIZZLE_NONE : CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? 0 : -(1000 + (int)r);
}

template <int BLOCK_N, bool A_MN, bool B_MN, bool SPLIT>
static int launch(const CUtensorMap& ta, const CUtensorMap& tb, GemmParams p, dim3 grid, cudaStream_t stream) {
  using L = SmemLayout<BLOCK_N, A_MN, B_MN, SPLIT>;
  static int env_stages = -1;
  if (env_stages < 0) { const char* e = getenv("GEOMX_GEMM_STAGES"); env_stages = e ? atoi(e) : 0; }
  int stages = L::STAGES;
  if (p.kb_per_split < stages) stages = p.kb_per_split;   // never more ring slots than K blocks
  if (env_stages > 0 && env_stages < stages) stages = env_stages;
  if (stages < 1) stages = 1;
  p.stages = stages;
  // the dynamic shared-memory limit is an attribute of the function in each device's context: set once per device, not once per process
  static std::atomic<unsigned long long> attr_set{0};
  auto kern = gemm_tf32_kernel<BLOCK_N, A_MN, B_MN, SPLIT>;
  int dev = 0;
  cudaGetDevice(&dev);
  const unsigned long long bit = dev < 64 ? 1ull << dev : 0ull;
  if (bit == 0 || !(attr_set.load(std::memory_order_acquire) & bit)) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, L::bytes(L::STAGES));
    if (e != cudaSuccess) return (int)e;
    attr_set.fetch_or(bit, std::memory_order_release);
  }
  launch_pdl(kern, dim3(grid), dim3(GEMM_THREADS), L::bytes(stages), stream, ta, tb, p);
  return (int)cudaGetLastError();
}

template <int BLOCK_N, bool SPLIT>
static int dispatch_major2(bool a_mn, bool b_mn, const CUtensorMap& ta, const CUtensorMap& tb, const GemmParams& p, dim3 grid, cudaStream_t s) {
  if (!a_mn && !b_mn) return launch<BLOCK_N, false, false, SPLIT>(ta, tb, p, grid, s);
  if (!a_mn && b_mn) return launch<BLOCK_N, false, true, SPLIT>(ta, tb, p, grid, s);
  if (a_mn && !b_mn) return launch<BLOCK_N, true, false, SPLIT>(ta, tb, p, grid, s);
  return launch<BLOCK_N, true, true, SPLIT>(ta, tb, p, grid, s);
}
template <int BLOCK_N>
static int dispatch_major(bool split, bool a_mn, bool b_mn, const CUtensorMap& ta, const CUtensorMap& tb, const GemmParams& p, dim3 grid, cudaStream_t s) {
  return split ? dispatch_major2<BLOCK_N, true>(a_mn, b_mn, ta, tb, p, grid, s) : dispatch_major2<BLOCK_N, false>(a_mn, b_mn, ta, tb, p, grid, s);
}

}  // namespace gx

static unsigned long long* g_gemm_dbg = nullptr;
// 3 = 3xTF32 (fp32-accurate, default), 1 = TF32.  Process-wide; GEOMX_GEMM_PRECISION=tf32|3xtf32 sets the initial value.
static int g_gemm_prec = -1;
static int gemm_precision() {
  if (g_gemm_prec < 0) { const char* e = getenv("GEOMX_GEMM_PRECISION"); g_gemm_prec = (e && (e[0] == 't' || e[0] == '1')) ? 1 : 3; }
  return g_gemm_prec;
}
GX_API int gx_gemm_set_precision(int prec) { g_gemm_prec = (prec == 1) ? 1 : 3; return g_gemm_prec; }
GX_API int gx_gemm_get_precision() { return gemm_precision(); }
GX_API int gx_gemm_set_debug(unsigned long long* p) { g_gemm_dbg = p; return 0; }

// A: K-major -> [M][K] with row stride lda; MN-major -> [K][M] with row stride lda.  Same for B with N.
// returns 0 on success, -1 if the operands do not satisfy TMA alignment or K <= 0 (caller falls back to gx_gemm_simt, which writes
// D = epi(0) for an empty K, the same contract), -2 for a ReLU epilogue with
// split_k > 1: every split applies the epilogue to its partial sum before the atomic add, which is right for the bias (split 0 only), the
// mask and the column sum (linear), but would give sum(relu(partial)) instead of relu(sum).
static int gemm_tf32_impl(const float* A, long long lda, int a_mn, const float* B, long long ldb, int b_mn, int M, int N, int K, float* D,
                          long long ldd, const float* bias, const float* mask, long long ldmask, float* colsum, int relu, int accumulate,
                          int store_mode, int hw, float alpha, int split_k,
                          int pool_w, unsigned char* pool_idx, int precision, cudaStream_t stream) {
  using namespace gx;
  if (relu && split_k > 1) return -2;
  if (M <= 0 || N <= 0) return 0;
  if (K <= 0) return -1;
  if (store_mode == 2) {   // fused pooling: whole windows must live inside one warp's 32 rows, no split-K / accumulate
    if (pool_w < 2 || (pool_w & 1) || (32 % (2 * pool_w)) != 0 || hw % 32 != 0 || (hw % pool_w) != 0 || ((hw / pool_w) & 1) || M % 32 != 0 ||
        split_k > 1 || accumulate || pool_idx == nullptr) return -1;
  }
  if ((lda & 3) || (ldb & 3) || (reinterpret_cast<uintptr_t>(A) & 15) || (reinterpret_cast<uintptr_t>(B) & 15)) return -1;
  // tile width: these problems are bound by how fast ONE SM can pull its operand panel out of L2, so small problems are cut into narrow
  // tiles to spread the B panel over many SMs; large ones use 128-wide tiles.
  int block_n = 16;
  const long long mt = ceil_div(M, BLOCK_M);
  for (int bn : {128, 64, 32, 16}) {
    if (mt * ceil_div(N, bn) >= 24 || bn == 16) { block_n = bn; break; }
  }
  static int sms = 0;
  if (sms == 0) { int dev = 0; cudaGetDevice(&dev); cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev); }
  if (mt * ceil_div(N, 128) >= sms) block_n = 128;   // 128-wide tiles once they alone fill every SM
  if (b_mn && block_n < 32) block_n = 32;   // an MN-major B tile is made of 32-wide TMA boxes
  CUtensorMap ta, tb;
  int rc;
  // TMA cost is per requested row, so boxes are trimmed to the rows that exist when the whole problem fits one tile in that dimension; the
  // untouched smem rows feed accumulator rows / columns that the epilogue never stores.
  const int a_rows = (mt == 1) ? (int)((M + 7) / 8 * 8) : BLOCK_M;
  const int nt = (int)ceil_div(N, block_n);
  const int b_rows = (nt == 1) ? (int)((N + 7) / 8 * 8 < block_n ? (N + 7) / 8 * 8 : block_n) : block_n;
  const int a_boxes = (mt == 1) ? (int)ceil_div(M, 32) : BLOCK_M / 32;
  const int b_boxes = (nt == 1) ? (int)ceil_div(N, 32) : block_n / 32;
  if (!a_mn) rc = make_tmap(&ta, A, K, M, lda, BLOCK_K, a_rows, false);
  else rc = make_tmap(&ta, A, M, K, lda, 32, BLOCK_K, true);
  if (rc) return rc;
  if (!b_mn) rc = make_tmap(&tb, B, K, N, ldb, BLOCK_K, b_rows, false);
  else rc = make_tmap(&tb, B, N, K, ldb, 32, BLOCK_K, true);
  if (rc) return rc;
  const int num_kb = (int)ceil_div(K, BLOCK_K);
  if (split_k < 1) split_k = 1;
  if (split_k > num_kb) split_k = num_kb;
  GemmParams p;
  p.M = M; p.N = N; p.K = K;
  p.kb_per_split = (int)ceil_div(num_kb, split_k);
  split_k = (int)ceil_div(num_kb, p.kb_per_split);
  p.D = D; p.ldd = ldd; p.bias = bias; p.mask = mask; p.ldmask = ldmask; p.colsum = colsum;
  p.relu = relu; p.accumulate = (accumulate || split_k > 1) ? 1 : 0; p.store_mode = store_mode; p.hw = hw > 0 ? hw : 1; p.alpha = alpha;
  p.stages = 0; p.dbg = g_gemm_dbg;
  p.pool_w = pool_w; p.pool_idx = pool_idx;
  p.a_boxes = a_boxes < 1 ? 1 : a_boxes; p.b_boxes = b_boxes < 1 ? 1 : b_boxes;
  p.a_bytes = a_mn ? p.a_boxes * MN_BOX_BYTES : a_rows * BLOCK_K * 4;
  p.b_bytes = b_mn ? p.b_boxes * MN_BOX_BYTES : b_rows * BLOCK_K * 4;
  p.tx_bytes = p.a_bytes + p.b_bytes;
  const bool split = precision == 3;
  dim3 grid((unsigned)ceil_div(N, block_n), (unsigned)mt, (unsigned)split_k);
  switch (block_n) {
    case 16: return dispatch_major<16>(split, a_mn, b_mn, ta, tb, p, grid, stream);
    case 32: return dispatch_major<32>(split, a_mn, b_mn, ta, tb, p, grid, stream);
    case 64: return dispatch_major<64>(split, a_mn, b_mn, ta, tb, p, grid, stream);
    default: return dispatch_major<128>(split, a_mn, b_mn, ta, tb, p, grid, stream);
  }
}

GX_API int gx_gemm_tf32(const float* A, long long lda, int a_mn, const float* B, long long ldb, int b_mn, int M, int N, int K, float* D,
                        long long ldd, const float* bias, const float* mask, long long ldmask, float* colsum, int relu, int accumulate,
                        int store_mode, int hw, float alpha, int split_k, cudaStream_t stream) {
  return gemm_tf32_impl(A, lda, a_mn, B, ldb, b_mn, M, N, K, D, ldd, bias, mask, ldmask, colsum, relu, accumulate, store_mode == 2 ? 1 : store_mode, hw,
                        alpha, split_k, 0, nullptr, gemm_precision(), stream);
}
// gx_gemm_tf32 at an explicit precision (3 = 3xTF32, 1 = TF32) that leaves the process-wide setting alone: for callers whose results must
// not depend on it (the device predictor, predict_dev.cu)
GX_API int gx_gemm_tf32_prec(const float* A, long long lda, int a_mn, const float* B, long long ldb, int b_mn, int M, int N, int K, float* D,
                             long long ldd, const float* bias, const float* mask, long long ldmask, float* colsum, int relu, int accumulate,
                             int store_mode, int hw, float alpha, int split_k, int precision, cudaStream_t stream) {
  return gemm_tf32_impl(A, lda, a_mn, B, ldb, b_mn, M, N, K, D, ldd, bias, mask, ldmask, colsum, relu, accumulate, store_mode == 2 ? 1 : store_mode, hw,
                        alpha, split_k, 0, nullptr, precision == 1 ? 1 : 3, stream);
}
// Convolution-as-GEMM with the 2x2/2 max-pool fused into the epilogue: rows of A are (image, oh, ow) with ow fastest and `hw` = OH*OW,
// `pool_w` = OW.  D receives the POOLED NCHW map [images][N][OH/2][OW/2], `pool_idx` the arg-max position of every pooled element.
// returns -1 when the geometry does not fit the in-warp pooling (caller runs GEMM + pool kernels instead).
GX_API int gx_gemm_tf32_pool(const float* A, long long lda, int a_mn, const float* B, long long ldb, int b_mn, int M, int N, int K, float* D,
                             const float* bias, int relu, int hw, int pool_w, unsigned char* pool_idx, float alpha, cudaStream_t stream) {
  return gemm_tf32_impl(A, lda, a_mn, B, ldb, b_mn, M, N, K, D, N, bias, nullptr, 0, nullptr, relu, 0, 2, hw, alpha, 1, pool_w,
                        pool_idx, gemm_precision(), stream);
}

// ------------------------------------------------------------------------------------------------
// CUDA-core fallback for operands that violate TMA alignment (odd leading dimensions, e.g. N=10 classifier heads).
// Same contract as gx_gemm_tf32 (fp32 FMA).  64x64 tile, 16-deep smem panels.
namespace gx {
__global__ void __launch_bounds__(256) gemm_simt_kernel(const float* __restrict__ A, long long lda, int a_mn, const float* __restrict__ B,
                                                         long long ldb, int b_mn, int M, int N, int K, GemmParams p) {
  gx::pdl_wait();
  gx::pdl_launch();
  __shared__ float sA[16][64 + 1];
  __shared__ float sB[16][64 + 1];
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  const int m0 = blockIdx.y * 64, n0 = blockIdx.x * 64;
  float acc[4][4] = {};
  for (int k0 = 0; k0 < K; k0 += 16) {
    for (int i = threadIdx.x; i < 16 * 64; i += 256) {
      const int kk = i / 64, r = i % 64;
      const int k = k0 + kk;
      float a = 0.f, b = 0.f;
      if (k < K && m0 + r < M) a = a_mn ? A[(long long)k * lda + m0 + r] : A[(long long)(m0 + r) * lda + k];
      if (k < K && n0 + r < N) b = b_mn ? B[(long long)k * ldb + n0 + r] : B[(long long)(n0 + r) * ldb + k];
      sA[kk][r] = a;
      sB[kk][r] = b;
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < 16; ++kk) {
      float a[4], b[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) { a[i] = sA[kk][ty * 4 + i]; b[i] = sB[kk][tx * 4 + i]; }
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int m = m0 + ty * 4 + i;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int n = n0 + tx * 4 + j;
      if (m >= M || n >= N) continue;
      float x = acc[i][j] * p.alpha;
      if (p.bias) x += p.bias[n];
      if (p.relu) x = fmaxf(x, 0.f);
      if (p.mask) x = p.mask[(long long)m * p.ldmask + n] > 0.f ? x : 0.f;
      if (p.colsum) atomicAdd(p.colsum + n, x);
      float* dst = p.store_mode == 0 ? p.D + (long long)m * p.ldd + n
                                     : p.D + ((long long)(m / p.hw) * N + n) * p.hw + (m % p.hw);
      if (p.accumulate) atomicAdd(dst, x);
      else *dst = x;
    }
  }
}
}  // namespace gx

GX_API int gx_gemm_simt(const float* A, long long lda, int a_mn, const float* B, long long ldb, int b_mn, int M, int N, int K, float* D,
                        long long ldd, const float* bias, const float* mask, long long ldmask, float* colsum, int relu, int accumulate,
                        int store_mode, int hw, float alpha, cudaStream_t stream) {
  using namespace gx;
  if (M <= 0 || N <= 0) return 0;
  GemmParams p;
  p.M = M; p.N = N; p.K = K; p.kb_per_split = 0; p.D = D; p.ldd = ldd; p.bias = bias; p.mask = mask; p.ldmask = ldmask; p.colsum = colsum;
  p.relu = relu; p.accumulate = accumulate; p.store_mode = store_mode; p.hw = hw > 0 ? hw : 1; p.alpha = alpha; p.stages = 0; p.dbg = nullptr; p.a_boxes = p.b_boxes = 0; p.tx_bytes = 0; p.a_bytes = p.b_bytes = 0;
  dim3 grid((unsigned)ceil_div(N, 64), (unsigned)ceil_div(M, 64));
  launch_pdl(gemm_simt_kernel, dim3(grid), dim3(256), 0, stream, A, lda, a_mn, B, ldb, b_mn, M, N, K, p);
  return (int)cudaGetLastError();
}
