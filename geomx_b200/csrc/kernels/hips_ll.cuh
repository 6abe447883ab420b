// Shared device-side pieces of the HiPS fabric kernels: the launch parameter block, the per-tile server update, the LL ("low latency") packet
// protocol and the replicated direct-protocol exchange of one tile.  Included by hips_fabric.cu (the exchange kernels) and by cnn_direct.cu
// (the convolution backward kernel whose tail performs the conv keys' exchange itself).  The optimizer rules are in optim.cuh.
#pragma once
#include <cuda_fp16.h>
#include <cuda_fp8.h>
#include "optim.cuh"

namespace gx {

constexpr int MAX_RANKS = 16;
constexpr int TILE = 1024;           // floats per tile (= 4 KiB = one 256-thread float4 sweep)
constexpr int FAB_THREADS = 256;


struct FabricParams {
  int world, rank, party_size, num_parties, party, local;
  int num_gs;
  int gs_rank[MAX_RANKS];
  float* grad[MAX_RANKS];      // peer pointers, indexed by global rank (only own party required)
  float* param[MAX_RANKS];     // peer pointers, all ranks
  float* stage[MAX_RANKS];     // peer pointers: [num_parties][n] staging on (potential) global owners
  uint32_t* flags[MAX_RANKS];  // peer pointers to flag pads
  const float* grad_mc;        // multicast address spanning the party's grad arenas (nullptr -> P2P loads)
  float* param_mc;             // multicast address spanning all ranks' param arenas (nullptr -> P2P stores)
  float* w;                    // global-owner master weights (local HBM), s0/s1 optimizer state
  float* s0;
  float* s1;
  float* lock_and_steps;       // unused in sync mode
  long long n;                 // arena elements (multiple of TILE)
  int tiles;
  int num_keys;
  const int* tile_key;         // [tiles]
  const int* key_tiles;        // [num_keys] tiles per key
  const int* tile_owner;       // [tiles] global-PS owner rank of each tile (MultiGPS sharding rules, arena.py)
  const unsigned char* tile_active;  // [tiles] or nullptr: only keys pushed this round take part
  const float2* tile_mult;     // per-tile (lr_mult, wd_mult) or nullptr
  int* key_done;               // [num_keys] cumulative completion counters on this rank (global owner side)
  int* state;                  // [0]=epoch completed, [1]=CTA completion counter, [2]=optimizer step t
  OptHyper h;
  float push_scale;            // the script-level  grad / num_samples
  int defer_pull_wait;
  int param_ready_off;         // uint32 offset of param_ready[num_keys] in the flag pad
  int ready_off;               // uint32 offset of grad_ready[MAX_RANKS] (per channel: every kernel family has its own epoch)
  int arrived_off;             // uint32 offset of arrived[num_parties][tiles]
  int zero_grad;               // fuse zero_grad: clear this rank's gradient arena once every reader is done with it
  // ---- LL ("low latency") protocol buffers: 8-byte {value, epoch} packets, no flags and no fences on the critical path
  float* ll_a[MAX_RANKS];      // peer pointers: [party_size][2n]  gradients pushed by party members to a tile's party owner
  float* ll_b[MAX_RANKS];      // peer pointers: [num_parties][2n] party aggregates pushed to a tile's global owner
  float* ll_c[MAX_RANKS];      // peer pointers: [2n]              fresh parameters pushed by the global owner to every rank
  float* ll_c_mc;              // multicast address of ll_c (nullptr -> one P2P store per rank)
  const unsigned char* tile_fmt;  // [tiles] wire format per tile (0 fp32, 1 fp16, 2 Bi-Sparse between the tiers) or nullptr = fp32
  float* bsc_u;                // Bi-Sparse momentum / accumulation state of the party owner (arena-sized, local HBM)
  float* bsc_v;
  int bsc_k;                   // packets per tile and party  (= floor(1024 * threshold), >= 1)
  const int* tile_order;       // DGT on the fabric: tiles are served in contribution order (most important first); nullptr = index order
  float* dgt_contrib;          // [tiles] EMA of mean |aggregated gradient| per tile, maintained by the tile's global owner (nullptr = off)
  float dgt_alpha;             // EMA factor (DGT_CONTRIBUTION_ALPHA)
  int ll_party_mode;           // 1: the party is the whole universe of this launch (HFA local round): the tile's party owner is also its
                               //    "global" owner, results go to the party members only, no optimizer
  // ---- direct protocol (hips_fsa_direct_kernel): gradients go straight to the rank(s) that apply the update
  float* ll_d[MAX_RANKS];      // peer pointers: [world][2n]  per-sender gradient packet slots
  float* ll_d_mc;              // multicast address of ll_d (replicated mode: one multimem.st reaches every rank)
  float* ll_e[MAX_RANKS];      // peer pointers: [2n]         fresh parameters from the tile's owner (sharded mode)
  float* ll_e_mc;              // multicast address of ll_e
  int direct_replicate;        // 1: EVERY rank reduces and applies every active tile on its own replica of the server state (one hop);
                               // 0: the tile's global owner does and pushes the result back (two hops)
  int channel_id;              // 0..7, folded into the packet epoch so that channels can never mistake each other's packets
  int list_tiles;              // entries of tile_list
  const int* tile_list;        // [list_tiles] the active tiles of a channel, ascending, or nullptr (single rank: CTA i serves tile_list[i])
};
// The instance of a fabric kernel (template <bool SCHED, bool EXT>) for a parameter block: the scheduled-lr instance when the block has a
// schedule (step_lr<SCHED>), and the one with the later optimizer kinds compiled in only for those kinds (opt_apply4<EXT>).
#define GX_FAB_INSTANCE(kern, p)                                                                                      \
  ((p).h.sched.kind != SCHED_NONE ? ((p).h.kind > OPT_DCASGD ? kern<true, true> : kern<true, false>)                  \
                                  : ((p).h.kind > OPT_DCASGD ? kern<false, true> : kern<false, false>))
// parallel/fabric.py's _FabricParams mirrors this block and asserts the same size (FABRIC_PARAMS_BYTES); kernel parameters are limited to 4 KB
static_assert(sizeof(FabricParams) == 1672 && offsetof(FabricParams, h) == 728, "FabricParams layout (parallel/fabric.py)");

__device__ __forceinline__ void wait_flag_ge(const uint32_t* p, uint32_t v) {
  while (ld_acquire_sys(p) < v) { __nanosleep(20); }
}

__device__ __forceinline__ float4 f4_add(float4 a, float4 b) { return make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w); }
__device__ __forceinline__ float4 f4_scale(float4 a, float s) { return make_float4(a.x * s, a.y * s, a.z * s, a.w * s); }

// ---- per-tile server update, in two steps so that callers can issue the state loads before they wait for the aggregate
struct TileState {
  float4 W, A, B;    // master weights and optimizer state of this thread's float4 of the tile
  float lr, wd;      // after the tile's (lr_mult, wd_mult)
};
__device__ __forceinline__ TileState tile_state_load(const FabricParams& p, int t, long long off, float lr_t) {
  TileState s;
  s.lr = lr_t; s.wd = p.h.wd;
  if (p.tile_mult) { const float2 mm = __ldg(p.tile_mult + t); s.lr *= mm.x; s.wd *= mm.y; }
  s.W = *reinterpret_cast<float4*>(p.w + off);
  s.A = p.s0 ? *reinterpret_cast<float4*>(p.s0 + off) : make_float4(0, 0, 0, 0);
  s.B = p.s1 ? *reinterpret_cast<float4*>(p.s1 + off) : make_float4(0, 0, 0, 0);
  return s;
}
// optimizer step on `agg`, state stored back; returns the fresh weights
template <bool EXT>
__device__ __forceinline__ float4 tile_state_apply(const FabricParams& p, long long off, TileState& s, float4 agg) {
  opt_apply4<EXT>(s.W, agg, s.A, s.B, p.h, s.lr, s.wd);
  *reinterpret_cast<float4*>(p.w + off) = s.W;
  if (p.s0) *reinterpret_cast<float4*>(p.s0 + off) = s.A;
  if (p.s1) *reinterpret_cast<float4*>(p.s1 + off) = s.B;
  return s.W;
}

// DGT contribution of tile t (kv_app.h:853-876 EvalMsgContribution): EMA of the mean |aggregated gradient| — ranks the tiles for the next
// re-ordering (important first) and decides which tiles keep full precision (HipsFabric.dgt_rerank).  All FAB_THREADS threads call it.
__device__ __forceinline__ void dgt_update_contrib(const FabricParams& p, int t, float4 agg, float* s_red) {
  float a = fabsf(agg.x) + fabsf(agg.y) + fabsf(agg.z) + fabsf(agg.w);
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) a += __shfl_xor_sync(0xffffffffu, a, d);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = a;
  __syncthreads();
  if (threadIdx.x == 0) {
    float sum = 0.f;
#pragma unroll
    for (int i = 0; i < FAB_THREADS / 32; ++i) sum += s_red[i];
    const float mean = sum * (1.f / TILE), old = p.dgt_contrib[t];
    p.dgt_contrib[t] = old == 0.f ? mean : p.dgt_alpha * old + (1.f - p.dgt_alpha) * mean;
  }
}

// ------------------------------------------------------------------------------------------------------------------ LL protocol
// The flag protocol above costs one fence.acq_rel.sys per hand-off and tools/fabric_probe.py measures 2.4-7 us for each of them on
// NVSwitch (three on the critical path of a two-tier step).  For latency-bound models the LL variant below trades 2x bytes for zero
// fences: every 16-byte store carries {v0, epoch, v1, epoch}; each 8-byte half is written atomically, so the receiver simply polls the
// packet until both epochs match (the scheme NCCL's LL protocol relies on).  The epoch grows by one per step, packets never need clearing.
// Data flow per tile:  every rank --push--> party owner --aggregate--> global owner --Adam + push--> every rank --unpack--> param arena.
// A sender overwrites a packet of step e only in step e+1, which it enters after it has unpacked ALL parameters of step e, and those
// were produced after every packet of step e had been consumed => no extra credit/ack traffic is required in dist_sync.
__device__ __forceinline__ void ll_store(float* dst, float4 v, uint32_t epoch) {
  const float f = __uint_as_float(epoch);
  asm volatile("st.relaxed.sys.global.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(dst), "f"(v.x), "f"(f), "f"(v.y), "f"(f) : "memory");
  asm volatile("st.relaxed.sys.global.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(dst + 4), "f"(v.z), "f"(f), "f"(v.w), "f"(f) : "memory");
}
__device__ __forceinline__ void ll_store_mc(float* mc, float4 v, uint32_t epoch) {
  const float f = __uint_as_float(epoch);
  asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(mc), "f"(v.x), "f"(f), "f"(v.y), "f"(f) : "memory");
  asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(mc + 4), "f"(v.z), "f"(f), "f"(v.w), "f"(f) : "memory");
}
// Poll a (local) packet pair until both halves carry `epoch`.  Bounded: a protocol bug must not hang the GPU (state[5] reports it).
__device__ __forceinline__ float4 ll_load(const float* src, uint32_t epoch, int* err) {
  float4 a, b;
  for (long long spin = 0;; ++spin) {
    asm volatile("ld.relaxed.sys.global.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(a.x), "=f"(a.y), "=f"(a.z), "=f"(a.w) : "l"(src) : "memory");
    asm volatile("ld.relaxed.sys.global.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(b.x), "=f"(b.y), "=f"(b.z), "=f"(b.w) : "l"(src + 4) : "memory");
    if (__float_as_uint(a.y) == epoch && __float_as_uint(a.w) == epoch && __float_as_uint(b.y) == epoch && __float_as_uint(b.w) == epoch) break;
    if (spin > (1ll << 24)) { *err = 1; break; }
  }
  return make_float4(a.x, a.z, b.x, b.z);
}

// single 16-byte packet {a, epoch, b, epoch}
__device__ __forceinline__ void ll_store1(float* dst, float a, float b, uint32_t epoch) {
  const float f = __uint_as_float(epoch);
  asm volatile("st.relaxed.sys.global.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(dst), "f"(a), "f"(f), "f"(b), "f"(f) : "memory");
}
__device__ __forceinline__ void ll_store1_mc(float* mc, float a, float b, uint32_t epoch) {
  const float f = __uint_as_float(epoch);
  asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(mc), "f"(a), "f"(f), "f"(b), "f"(f) : "memory");
}
__device__ __forceinline__ float2 ll_load1(const float* src, uint32_t epoch, int* err) {
  float4 a;
  for (long long spin = 0;; ++spin) {
    asm volatile("ld.relaxed.sys.global.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(a.x), "=f"(a.y), "=f"(a.z), "=f"(a.w) : "l"(src) : "memory");
    if (__float_as_uint(a.y) == epoch && __float_as_uint(a.w) == epoch) break;
    if (spin > (1ll << 24)) { *err = 1; break; }
  }
  return make_float2(a.x, a.z);
}
__device__ __forceinline__ float pack_h2(float lo, float hi) {
  const __half2 h = __floats2half2_rn(lo, hi);
  return __uint_as_float(*reinterpret_cast<const uint32_t*>(&h));
}
__device__ __forceinline__ float2 unpack_h2(float f) {
  const uint32_t u = __float_as_uint(f);
  return __half22float2(*reinterpret_cast<const __half2*>(&u));
}
// Wire formats of a tile (FabricParams::tile_fmt): the reference's FP16 / MPQ accelerators cast at script level and Bi-Sparse runs on the
// local server's CPU; here the cast / top-k / scale are fused into the collective kernel itself.
constexpr int FMT_F32 = 0;   // {v0,e,v1,e}{v2,e,v3,e}
constexpr int FMT_F16 = 1;   // {h0h1,e,h2h3,e}: half the bytes on every hop (gradients and parameters), fp32 master weights on the owner
constexpr int FMT_BSC = 2;   // Bi-Sparse between the tiers: k {value, e, index, e} packets per tile instead of 1024 values
constexpr int FMT_F8 = 3;    // block-scaled fp8 gradients: e4m3 with one fp32 scale per 128 values (a warp), 8 values per packet => 1/4 of the
                             // fp32 bytes on the two gradient hops; parameters of such tiles return as fp16
__device__ __forceinline__ int fmt_of(const FabricParams& p, int t) { return p.tile_fmt ? (int)p.tile_fmt[t] : FMT_F32; }
// format of a tile's dense gradient packets: Bi-Sparse tiles travel as fp32 wherever their gradients go dense
__device__ __forceinline__ int grad_fmt(int f) { return (f == FMT_F16 || f == FMT_F8) ? f : FMT_F32; }

// ---- block-scaled fp8 (warp-collective: all 32 lanes of a warp call these together; a lane owns 4 consecutive values)
__device__ __forceinline__ uint32_t pack_f8x4(float4 v, float inv) {
  const uint32_t lo = __nv_cvt_float2_to_fp8x2(make_float2(v.x * inv, v.y * inv), __NV_SATFINITE, __NV_E4M3);
  const uint32_t hi = __nv_cvt_float2_to_fp8x2(make_float2(v.z * inv, v.w * inv), __NV_SATFINITE, __NV_E4M3);
  return lo | (hi << 16);
}
__device__ __forceinline__ float4 unpack_f8x4(uint32_t q, float scale) {
  const __half2_raw a = __nv_cvt_fp8x2_to_halfraw2(static_cast<__nv_fp8x2_storage_t>(q & 0xffffu), __NV_E4M3);
  const __half2_raw b = __nv_cvt_fp8x2_to_halfraw2(static_cast<__nv_fp8x2_storage_t>(q >> 16), __NV_E4M3);
  const float2 fa = __half22float2(*reinterpret_cast<const __half2*>(&a)), fb = __half22float2(*reinterpret_cast<const __half2*>(&b));
  return make_float4(fa.x * scale, fa.y * scale, fb.x * scale, fb.y * scale);
}
// even lanes write {own 4 values, neighbour's 4 values} as one packet into their slot, lane 1 writes the warp's scale into its (otherwise
// unused) slot; `mc` selects the multicast store
__device__ __forceinline__ void ll_send_f8(float* dst, bool mc, float4 v, uint32_t epoch) {
  float amax = fmaxf(fmaxf(fabsf(v.x), fabsf(v.y)), fmaxf(fabsf(v.z), fabsf(v.w)));
#pragma unroll
  for (int d = 16; d > 0; d >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, d));
  const float scale = fmaxf(amax, 1e-30f) * (1.f / 448.f);
  const uint32_t q = pack_f8x4(v, 1.f / scale);
  const uint32_t qn = __shfl_down_sync(0xffffffffu, q, 1);
  const int lane = threadIdx.x & 31;
  if ((lane & 1) == 0) { if (mc) ll_store1_mc(dst, __uint_as_float(q), __uint_as_float(qn), epoch); else ll_store1(dst, __uint_as_float(q), __uint_as_float(qn), epoch); }
  else if (lane == 1) { if (mc) ll_store1_mc(dst, scale, 0.f, epoch); else ll_store1(dst, scale, 0.f, epoch); }
}
__device__ __forceinline__ float4 ll_recv_f8(const float* src, uint32_t epoch, int* err) {
  const int lane = threadIdx.x & 31;
  float2 pk = make_float2(0.f, 0.f);
  if ((lane & 1) == 0 || lane == 1) pk = ll_load1(src, epoch, err);
  const float scale = __shfl_sync(0xffffffffu, pk.x, 1);
  const uint32_t from_prev = __shfl_up_sync(0xffffffffu, __float_as_uint(pk.y), 1);
  const uint32_t q = (lane & 1) == 0 ? __float_as_uint(pk.x) : from_prev;
  return unpack_f8x4(q, scale);
}

// dense value of one thread (4 floats) -> its 32-byte packet region
__device__ __forceinline__ void ll_send_dense(float* dst, float4 v, int fmt, uint32_t epoch) {
  if (fmt == FMT_F8) ll_send_f8(dst, false, v, epoch);
  else if (fmt == FMT_F16) ll_store1(dst, pack_h2(v.x, v.y), pack_h2(v.z, v.w), epoch);
  else ll_store(dst, v, epoch);
}
__device__ __forceinline__ void ll_send_dense_mc(float* mc, float4 v, int fmt, uint32_t epoch) {
  if (fmt == FMT_F8) ll_send_f8(mc, true, v, epoch);
  else if (fmt == FMT_F16) ll_store1_mc(mc, pack_h2(v.x, v.y), pack_h2(v.z, v.w), epoch);
  else ll_store_mc(mc, v, epoch);
}
__device__ __forceinline__ float4 ll_recv_dense(const float* src, int fmt, uint32_t epoch, int* err) {
  if (fmt == FMT_F8) return ll_recv_f8(src, epoch, err);
  if (fmt == FMT_F16) {
    const float2 pk = ll_load1(src, epoch, err);
    const float2 a = unpack_h2(pk.x), b = unpack_h2(pk.y);
    return make_float4(a.x, a.y, b.x, b.y);
  }
  return ll_load(src, epoch, err);
}

// ------------------------------------------------------------------------------------------------------------------ direct protocol
// replicated mode: this rank's gradient float4 `v` at arena offset `off` into its own slot on every rank (one multicast store, or one per rank)
__device__ __forceinline__ void direct_send_all(const FabricParams& p, long long off, float4 v, int f, uint32_t epoch) {
  const long long slot = (long long)p.rank * 2 * p.n + 2 * off;
  if (p.ll_d_mc != nullptr) ll_send_dense_mc(p.ll_d_mc + slot, v, f, epoch);
  else for (int r = 0; r < p.world; ++r) ll_send_dense(p.ll_d[r] + slot, v, f, epoch);
}
// the aggregate of every rank's packets at `off`, summed in the hierarchy's order: inside each party, push_scale, then across parties
__device__ __forceinline__ float4 direct_recv_sum(const FabricParams& p, long long off, int f, uint32_t epoch, int* err) {
  const int S = p.party_size;
  const long long n2 = 2 * p.n;
  const float* in = p.ll_d[p.rank] + 2 * off;
  float4 agg = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int g = 0; g < p.num_parties; ++g) {
    float4 ps = ll_recv_dense(in + (long long)(g * S) * n2, f, epoch, err);
    for (int j = 1; j < S; ++j) ps = f4_add(ps, ll_recv_dense(in + (long long)(g * S + j) * n2, f, epoch, err));
    ps = f4_scale(ps, p.push_scale);
    agg = g == 0 ? ps : f4_add(agg, ps);
  }
  return agg;
}

}  // namespace gx
