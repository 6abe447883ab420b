// Shared device helpers for the sm_90a kernels: mbarrier / TMA / wgmma PTX wrappers,
// system-scope flag primitives for the in-kernel collectives, and small utilities.
//
// Everything here is written against the PTX ISA for sm_90a (CUDA 12.9): wgmma.mma_async -> HGMMA, cp.async.bulk.tensor -> UTMALDG,
// multimem.* -> peer/multicast loads & stores.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#define GX_API extern "C" __attribute__((visibility("default")))
#define GX_CHECK_LAUNCH() (int)cudaGetLastError()

#include <cstdlib>
#include <utility>

namespace gx {

// ------------------------------------------------------------------------------------------------ programmatic dependent launch (PDL)
// Every kernel of this library begins with pdl_wait() (griddepcontrol.wait: block until the preceding grid in the stream has completed and
// its memory is visible) and pdl_launch() (griddepcontrol.launch_dependents: let the NEXT grid start its prologue — block scheduling,
// smem carve-up, barrier init, tensormap prefetch — while this one is still running).  Launches go through launch_pdl(), which
// sets cudaLaunchAttributeProgrammaticStreamSerialization; in a CUDA graph the edges become programmatic dependencies.  GEOMX_PDL=0 disables.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

inline bool pdl_enabled() {
  static int v = -1;
  if (v < 0) { const char* e = getenv("GEOMX_PDL"); v = (e && e[0] == '0') ? 0 : 1; }
  return v == 1;
}
// All kernels ask for the same (maximum) shared-memory carve-out: a GEMM CTA needs ~200 KB while the element-wise kernels need none, and an
// SM cannot run two kernels with different L1/smem splits side by side — with per-kernel defaults every GEMM <-> non-GEMM boundary of the step
// would drain and reconfigure the SMs and defeat programmatic dependent launch.  GEOMX_CARVEOUT=0 keeps the driver defaults.
inline void unify_carveout(const void* fn) {
  static const void* seen[256];
  static int nseen = 0;
  static int enabled = -1;
  if (enabled < 0) { const char* e = getenv("GEOMX_CARVEOUT"); enabled = (e && e[0] == '0') ? 0 : 1; }
  if (!enabled) return;
  for (int i = 0; i < nseen; ++i) if (seen[i] == fn) return;
  if (nseen < 256) seen[nseen++] = fn;
  cudaFuncSetAttribute(fn, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
}

template <typename... KArgs, typename... Args>
inline int launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, Args&&... args) {
  unify_carveout(reinterpret_cast<const void*>(kernel));
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr; cfg.numAttrs = pdl_enabled() ? 1 : 0;
  return (int)cudaLaunchKernelEx(&cfg, kernel, KArgs(std::forward<Args>(args))...);
}

// ------------------------------------------------------------------------------------------------ misc
__host__ __device__ __forceinline__ int64_t ceil_div(int64_t a, int64_t b) { return (a + b - 1) / b; }

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ uint32_t lane_id() { return threadIdx.x & 31u; }

__device__ __forceinline__ bool elect_one() {
  uint32_t pred = 0;
  asm volatile(
      "{\n\t.reg .pred P;\n\t"
      "elect.sync _|P, 0xffffffff;\n\t"
      "selp.b32 %0, 1, 0, P;\n\t}\n"
      : "=r"(pred));
  return pred != 0;
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// ------------------------------------------------------------------------------------------------ mbarrier
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n\t.reg .pred P1;\n\t"
      "LAB_WAIT:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n\t"
      "@P1 bra DONE;\n\t"
      "bra LAB_WAIT;\n\t"
      "DONE:\n\t}\n" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}
// generic-proxy smem writes -> visible to the async proxy (TMA / wgmma operand reads)
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// ------------------------------------------------------------------------------------------------ point-to-point cluster hand-offs
// A producer pushes its slice into the receive buffer of every CTA of the cluster with st.async; each store completes its bytes on a
// transaction mbarrier in the receiving CTA, which waits on its own barrier only (no cluster-wide barrier, no GPU-scope fence).
__device__ __forceinline__ uint32_t mapa_u32(uint32_t local_smem_addr, int rank) {
  uint32_t a;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(a) : "r"(local_smem_addr), "r"(rank));
  return a;
}
// push v to float offset o of `buf` in the N CTAs of the cluster that follow rank cr (N = CS: every CTA including this one, this one last;
// N = CS - 1: the peers only), so that the CTAs do not all hit rank 0 first; each store completes 16 bytes on the receiver's barrier `bar`
template <int CS, int N = CS>
__device__ __forceinline__ void push_all(const float* buf, int o, uint64_t* bar, int cr, float4 v) {
  const uint32_t a = smem_u32(buf + o), m = smem_u32(bar);
#pragma unroll 4   // a full unroll hoists all 2 N remote addresses and pushes mlp_chain_kernel past 96 registers (co-residency with cnn_fwd)
  for (int i = 0; i < N; ++i) {
    const int r = (cr + 1 + i) & (CS - 1);
    asm volatile("st.async.shared::cluster.mbarrier::complete_tx::bytes.v4.f32 [%0], {%1, %2, %3, %4}, [%5];"
                 ::"r"(mapa_u32(a, r)), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w), "r"(mapa_u32(m, r)) : "memory");
  }
}
// wait until every byte announced on this CTA's (single-use) barrier has landed.  The acquire that makes the peers' stores visible is
// restricted to shared::cluster memory: a plain acquire.cluster wait would also invalidate L1, for no data the kernels read through it.
__device__ __forceinline__ void wait_landed(uint64_t* bar) {
  asm volatile(
      "{\n\t.reg .pred P1;\n\t"
      "WAIT_LANDED:\n\t"
      "mbarrier.try_wait.parity.relaxed.cluster.shared::cta.b64 P1, [%0], 0;\n\t"
      "@!P1 bra WAIT_LANDED;\n\t}\n"
      "fence.acquire.sync_restrict::shared::cluster.cluster;" ::"r"(smem_u32(bar))
      : "memory");
}

// softmax cross-entropy of one row whose logits four consecutive lanes hold (the lane with lane % 4 == q: classes 4 q .. 4 q + 3; classes
// >= C are ignored), label l: dl = softmax - one-hot (0 for classes >= C); returns the row's loss, in all four lanes.  Every lane of the warp
// takes part (shuffles).  The dense chain (mlp_chain.cu) and the training head of cnn_fwd_dense0_kernel (cnn_direct.cu) share it, so that both
// round the same way.
__device__ __forceinline__ float softmax_ce_quad(const float (&lg)[4], int C, int l, float (&dl)[4]) {
  const int lane = threadIdx.x & 31, c0 = 4 * (lane & 3);
  float mx = -INFINITY;
#pragma unroll
  for (int j = 0; j < 4; ++j) if (c0 + j < C) mx = fmaxf(mx, lg[j]);
  mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
  mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
  float e[4], s = 0.f;
#pragma unroll
  for (int j = 0; j < 4; ++j) { e[j] = c0 + j < C ? __expf(lg[j] - mx) : 0.f; s += e[j]; }
  s += __shfl_xor_sync(0xffffffffu, s, 1);
  s += __shfl_xor_sync(0xffffffffu, s, 2);
#pragma unroll
  for (int j = 0; j < 4; ++j) dl[j] = c0 + j < C ? e[j] / s - (c0 + j == l ? 1.f : 0.f) : 0.f;
  const int q = l & 3;
  const float mine = q == 0 ? lg[0] : q == 1 ? lg[1] : q == 2 ? lg[2] : lg[3];
  const float picked = __shfl_sync(0xffffffffu, mine, (lane & ~3) | ((l >> 2) & 3));
  return -(picked - mx - __logf(s));
}

// Static shared memory of cnn_fwd_dense0_kernel (cnn_direct.cu asserts it).  Its successor in the step, dense_tail_kernel (mlp_chain.cu),
// stages its weights while the forward kernel runs, on the SMs beside its CTAs: mlp_chain.cu checks that both fit into one SM.
constexpr int CNN_FWD_DENSE0_SMEM_BYTES = 46288;

// ------------------------------------------------------------------------------------------------ TMA
__device__ __forceinline__ void tma_prefetch_desc(const void* tmap) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(tmap)) : "memory");
}
// 2-D tiled load: box lands at smem_dst, completion signalled on bar (complete_tx::bytes)
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const void* tmap, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(
          smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(tmap)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}

// ------------------------------------------------------------------------------------------------ wgmma (sm_90a warpgroup MMA)
__device__ __forceinline__ void named_bar_sync(uint32_t id, uint32_t nthreads) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory"); }
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// keeps the compiler from moving accumulator reads / writes across the asynchronous MMAs that own those registers
template <int R>
__device__ __forceinline__ void wgmma_fence_regs(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// wgmma shared-memory matrix descriptor (sm_90 GMMA layout):
//  [0,14) start>>4 | [16,30) LBO>>4 | [32,46) SBO>>4 | [49,52) base_offset | [62,64) layout (1 = SWIZZLE_128B)
// K-major SWIZZLE_128B operand: rows of 128 B (32 fp32 = one swizzle atom), 8-row groups SBO = 1024 B apart, LBO unused; the tile base is
// 1024-B aligned and a K step inside the atom advances the start address (32 B per k8 tf32 instruction).
__device__ __forceinline__ uint64_t gmma_desc_sw128(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFFu) >> 4);
  d |= static_cast<uint64_t>(1u) << 16;
  d |= static_cast<uint64_t>(1024u >> 4) << 32;
  d |= 1ull << 62;
  return d;
}

// D[64 x N] (+)= A[64 x 8] * B[N x 8]^T, tf32 operands (K-major, from shared memory), fp32 accumulators in registers.
// Fragment of thread t (warp w = t/32, lane l): d[4i + {0,1,2,3}] = D[16w + l/4 + {0,0,8,8}][8i + 2(l%4) + {0,1,0,1}].
__device__ __forceinline__ void wgmma_tf32_n16(float (&d)[8], uint64_t da, uint64_t db, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n16k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
      : "l"(da), "l"(db), "r"(scale_d));
}
__device__ __forceinline__ void wgmma_tf32_n32(float (&d)[16], uint64_t da, uint64_t db, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(da), "l"(db), "r"(scale_d));
}
__device__ __forceinline__ void wgmma_tf32_n64(float (&d)[32], uint64_t da, uint64_t db, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(da), "l"(db), "r"(scale_d));
}
__device__ __forceinline__ void wgmma_tf32_n128(float (&d)[64], uint64_t da, uint64_t db, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(da), "l"(db), "r"(scale_d));
}

// ------------------------------------------------------------------------------------------------ system-scope flags (in-kernel collectives)
__device__ __forceinline__ void st_release_sys(uint32_t* p, uint32_t v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ uint32_t ld_relaxed_sys(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.relaxed.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void red_add_release_sys(uint32_t* p, uint32_t v) {
  asm volatile("red.release.sys.global.add.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ void fence_sys() { asm volatile("fence.acq_rel.sys;" ::: "memory"); }

// 16-byte peer / streaming accesses
__device__ __forceinline__ float4 ld_f4_sys(const float* p) {  // peer memory: bypass L1 so re-reads see remote stores
  float4 v;
  asm volatile("ld.relaxed.sys.global.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_f4_sys(float* p, float4 v) {
  asm volatile("st.relaxed.sys.global.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}
// NVLS: switch-side reduction / multicast store on a multicast (multimem) address
__device__ __forceinline__ float4 multimem_ld_reduce_f4(const float* mc) {
  float4 v;
  asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w)
               : "l"(mc)
               : "memory");
  return v;
}
__device__ __forceinline__ void multimem_st_f4(float* mc, float4 v) {
  asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(mc), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w)
               : "memory");
}

}  // namespace gx
