// HiPS data plane on NVSwitch: the two communication-bound hot paths of the reference fused into in-kernel collectives.
//
// Reference path per key per step (SURVEY §3.3): worker D2H copy -> ZMQ push -> local server CPU `+=` over NumWorkers
// (kvstore_dist_server.h:1277-1321) -> ZMQ push to the global server -> CPU sum over parties + Python optimizer on the server
// main thread (:1298-1319, :535-559) -> ack -> local server pulls (:899-936) -> workers pull (:1705-1763) -> H2D copy.
//
// Here one kernel per step, launched by every rank (one process per GPU), no NCCL / host transport on the path:
//   phase A  every rank publishes "my gradient arena is complete" to its party (system-scope release flags)
//   phase B  LOCAL PS TIER  = tile-sharded reduction inside the party: the owner of a tile pulls the tile from all party members
//            with `multimem.ld_reduce` (in-switch NVLS reduction) or P2P `ld.global` loads, applies the 1/num_samples scale that the
//            scripts apply before push, and stores the party aggregate into the global-PS owner's staging slot (P2P `st.global`).
//   phase C  GLOBAL PS TIER = the tile's global owner waits for all parties, sums the staged aggregates and runs the partitioned
//            optimizer (SGD / Adam / DCASGD; master weights + state live in that rank's HBM), then broadcasts the new tile to every
//            worker's parameter arena with `multimem.st` (NVLS multicast) or P2P stores and releases a per-key ready flag.
//   phase D  workers wait for the per-key flags.
// MixedSync (dist_async) is one-sided: the party's tile owner takes a per-tile system-scope lock in the global owner's HBM and
// applies its party's update there directly (reference: DataHandleAsyncDefault kvstore_dist_server.h:1519-1611).
// HFA / party-level sync use hips_party_allreduce (local tier only).
//
// Flag protocol: every cross-rank flag carries the (monotonically increasing) epoch; writers do  stores -> bar.sync -> fence.sys ->
// st.release.sys, readers spin with ld.acquire.sys.  All CTAs of the launch are co-resident (grid <= #SMs), phases are ordered
// A < B < C < D inside every CTA and each phase only waits on flags produced by strictly earlier phases => no cyclic wait.
#include <cuda_fp16.h>
#include "hips_ll.cuh"

namespace gx {

// Global-owner side of one tile: optimizer + broadcast + per-key completion/flag.  `agg` is this thread's float4 of the summed gradient.
template <bool EXT>
__device__ __forceinline__ void global_apply_tile(const FabricParams& p, int t, float4 agg, uint32_t epoch, float lr_t) {
  const long long off = (long long)t * TILE + threadIdx.x * 4;
  TileState s = tile_state_load(p, t, off, lr_t);
  const float4 W = tile_state_apply<EXT>(p, off, s, agg);
  if (p.world == 1) {  // degenerate single-rank HiPS: the arena optimizer, no cross-GPU traffic, flags or fences
    *reinterpret_cast<float4*>(p.param[0] + off) = W;
    return;
  }
  // pull/broadcast: NVLS multicast store or P2P stores into every worker's parameter arena
  if (p.param_mc != nullptr) {
    multimem_st_f4(p.param_mc + off, W);
  } else {
    for (int r = 0; r < p.world; ++r) st_f4_sys(p.param[r] + off, W);
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    fence_sys();
    const int key = p.tile_key[t];
    const int c = atomicAdd(p.key_done + key, 1) + 1;
    if (c == p.key_tiles[key]) {  // last tile of this key for this round: reset the counter, release the key
      p.key_done[key] = 0;
      fence_sys();
      for (int r = 0; r < p.world; ++r) st_release_sys(p.flags[r] + p.param_ready_off + key, epoch);
    }
  }
}

// Single rank: both server tiers collapse into the fused arena optimizer.  No peer ever spins on this launch, so the grid need not be
// co-resident: one tile per CTA, grid-stride beyond the grid.  A channel passes its active tiles as `tile_list` and launches one CTA per
// entry (CTA i serves tile_list[i]); otherwise CTA i serves tile i, skipping those `tile_active` excludes.  A kernel of its own, apart from
// the multi-rank one, so that its register count is its own: its CTAs are meant to become resident beside the grid that produces the
// gradients (the convolution backward wave, the dense weight gradients) and to have staged their tile when that grid ends.
template <bool SCHED, bool EXT>
__global__ void __launch_bounds__(FAB_THREADS, 4) hips_fsa_step_single_kernel(const FabricParams p) {
  const volatile int* state = p.state;
  const bool dbg = state[3] != 0 && blockIdx.x == 0 && threadIdx.x == 0;
  unsigned long long* stamps = reinterpret_cast<unsigned long long*>(p.state + 8);
  auto stamp = [&](int i) { if (dbg) { unsigned long long t; asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t)); stamps[i] = t; } };
  const bool listed = p.tile_list != nullptr;
  const int count = listed ? p.list_tiles : p.tiles;
  auto tile_of = [&](int i) { return listed ? __ldg(p.tile_list + i) : i; };
  auto prefetch_l2 = [](const float* q) { asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(q), "r"(TILE * 4) : "memory"); };

  // Before the grid dependency resolves, i.e. while the grid that writes the gradients still runs, this CTA stages its first tile:
  //   - into registers: the tile index and its (lr_mult, wd_mult), which only the host writes (when the channel is declared and the arena
  //     laid out), and the step size of the optimizer step that the state words announce;
  //   - into L2 (bulk prefetch): the tile's master weights and optimizer state, and the state words.
  // No kernel of a training step writes these except the previous launch on the same state block.  That launch may still be running here
  // when it is the grid this one depends on (one channel launched twice back to back), so the weights, optimizer state and state words are
  // loaded into registers only after the wait, from L2, and the early step size is kept only if the step word has not moved.  After the
  // wait only L2 is read: those, and the gradient that the grid just waited for wrote.
  const int i0 = blockIdx.x;
  const int t0 = i0 < count ? tile_of(i0) : 0;
  const float2 mult0 = (p.tile_mult != nullptr && i0 < count) ? __ldg(p.tile_mult + t0) : make_float2(1.f, 1.f);
  if (threadIdx.x == 0) {
    asm volatile("prefetch.global.L2 [%0];" ::"l"(p.state) : "memory");
    if (i0 < count) {
      const long long base = (long long)t0 * TILE;
      prefetch_l2(p.w + base);
      if (p.s0) prefetch_l2(p.s0 + base);
      if (p.s1) prefetch_l2(p.s1 + base);
    }
  }
  const int opt_early = state[2] + 1;
  const float lr_early = step_lr<SCHED>(p.h, opt_early);
  gx::pdl_wait();
  gx::pdl_launch();
  stamp(0);
  const int round = state[0];
  const int opt_t = state[2] + 1;
  const float lr_t = opt_t == opt_early ? lr_early : step_lr<SCHED>(p.h, opt_t);
  for (int i = i0; i < count; i += gridDim.x) {
    const int t = i == i0 ? t0 : tile_of(i);
    if (!listed && p.tile_active != nullptr && !p.tile_active[t]) continue;
    const float2 mm = i == i0 ? mult0 : (p.tile_mult != nullptr ? __ldg(p.tile_mult + t) : make_float2(1.f, 1.f));
    const long long off = (long long)t * TILE + threadIdx.x * 4;
    float* g = p.grad[0] + off;
    const float4 G = __ldcg(reinterpret_cast<const float4*>(g));
    TileState s;
    s.lr = lr_t * mm.x; s.wd = p.h.wd * mm.y;
    s.W = *reinterpret_cast<const float4*>(p.w + off);
    s.A = p.s0 ? *reinterpret_cast<const float4*>(p.s0 + off) : make_float4(0, 0, 0, 0);
    s.B = p.s1 ? *reinterpret_cast<const float4*>(p.s1 + off) : make_float4(0, 0, 0, 0);
    const float4 W = tile_state_apply<EXT>(p, off, s, f4_scale(G, p.push_scale));
    if (p.zero_grad) *reinterpret_cast<float4*>(g) = make_float4(0.f, 0.f, 0.f, 0.f);
    *reinterpret_cast<float4*>(p.param[0] + off) = W;
  }
  // bookkeeping: the state words are read by the next launch on this block after its own grid dependency, so a relaxed counter is enough
  if (threadIdx.x == 0) {
    const int done = atomicAdd(p.state + 1, 1);
    if (done == (int)gridDim.x - 1) { p.state[1] = 0; p.state[2] = opt_t; p.state[0] = round + 1; }
  }
  stamp(5);
}

// Multi-rank flag ("bulk") protocol; a single rank runs hips_fsa_step_single_kernel (gx_hips_fsa_step picks it).
template <bool SCHED, bool EXT>
__global__ void __launch_bounds__(FAB_THREADS, 1) hips_fsa_step_kernel(const FabricParams p) {
  gx::pdl_wait();
  gx::pdl_launch();
  const bool dbg = p.state[3] != 0 && blockIdx.x == 0 && threadIdx.x == 0;
  unsigned long long* stamps = reinterpret_cast<unsigned long long*>(p.state + 8);
  auto stamp = [&](int i) { if (dbg) { unsigned long long t; asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t)); stamps[i] = t; } };
  stamp(0);
  const uint32_t epoch = (uint32_t)(*reinterpret_cast<volatile int*>(p.state)) + 1u;
  const int opt_t = (*reinterpret_cast<volatile int*>(p.state + 2)) + 1;
  __shared__ float s_lr;
  if (threadIdx.x == 0) s_lr = step_lr<SCHED>(p.h, opt_t);
  __syncthreads();
  const float lr_t = s_lr;
  const int S = p.party_size, P = p.num_parties;
  const int party_base = p.party * S;
  uint32_t* my_flags = p.flags[p.rank];

  // ---------------- phase A: publish gradient-ready to the party
  if (p.world > 1 && blockIdx.x == 0 && threadIdx.x < S) {
    fence_sys();
    st_release_sys(p.flags[party_base + threadIdx.x] + p.ready_off + p.rank, epoch);
  }

  stamp(1);
  // ---------------- phase B: local PS tier (party reduction of owned tiles)
  bool waited_party = false;
  for (int t = blockIdx.x; t < p.tiles; t += gridDim.x) {
    if (t % S != p.local) continue;
    if (p.tile_active != nullptr && !p.tile_active[t]) continue;
    if (!waited_party && p.world > 1) {
      if (threadIdx.x < S) wait_flag_ge(my_flags + p.ready_off + party_base + threadIdx.x, epoch);
      __syncthreads();
      waited_party = true;
      stamp(6);
    }
    const long long off = (long long)t * TILE + threadIdx.x * 4;
    float4 acc;
    if (p.grad_mc != nullptr && S > 1) {
      acc = multimem_ld_reduce_f4(p.grad_mc + off);
    } else {
      acc = (S == 1) ? *reinterpret_cast<const float4*>(p.grad[p.rank] + off) : ld_f4_sys(p.grad[party_base] + off);
      for (int j = 1; j < S; ++j) acc = f4_add(acc, ld_f4_sys(p.grad[party_base + j] + off));
    }
    acc = f4_scale(acc, p.push_scale);
    if (dbg && acc.x == 123.456f) stamps[20] = 1;  // (debug) force the loads to retire before the stamp
    stamp(7);
    if (p.zero_grad && p.world == 1) *reinterpret_cast<float4*>(p.grad[p.rank] + off) = make_float4(0.f, 0.f, 0.f, 0.f);
    const int owner = p.tile_owner[t];
    if (P == 1 && owner == p.rank) {
      global_apply_tile<EXT>(p, t, acc, epoch, lr_t);  // both tiers collapse: stay in registers
      stamp(8);
    } else {
      st_f4_sys(p.stage[owner] + (long long)p.party * p.n + off, acc);
      __syncthreads();
      if (threadIdx.x == 0) {
        fence_sys();
        st_release_sys(p.flags[owner] + p.arrived_off + p.party * p.tiles + t, epoch);
      }
      stamp(8);
    }
  }

  stamp(2);
  // ---------------- phase C: global PS tier (tiles this rank owns globally)
  for (int t = blockIdx.x; t < p.tiles; t += gridDim.x) {
    if (p.tile_owner[t] != p.rank) continue;
    if (p.tile_active != nullptr && !p.tile_active[t]) continue;
    if (P == 1 && (t % S) == p.local) continue;  // already applied in phase B
    if (threadIdx.x < P) wait_flag_ge(my_flags + p.arrived_off + threadIdx.x * p.tiles + t, epoch);
    __syncthreads();
    stamp(9);
    const long long off = (long long)t * TILE + threadIdx.x * 4;
    float4 acc = ld_f4_sys(p.stage[p.rank] + off);
    for (int g = 1; g < P; ++g) acc = f4_add(acc, ld_f4_sys(p.stage[p.rank] + (long long)g * p.n + off));
    global_apply_tile<EXT>(p, t, acc, epoch, lr_t);
    stamp(10);
  }

  stamp(3);
  // ---------------- phase D: wait for the broadcast (unless deferred to the consuming GEMM)
  if (p.world > 1 && !p.defer_pull_wait && blockIdx.x == 0) {
    for (int t = threadIdx.x; t < p.tiles; t += blockDim.x)
      if (p.tile_active == nullptr || p.tile_active[t]) wait_flag_ge(my_flags + p.param_ready_off + p.tile_key[t], epoch);
  }

  stamp(4);
  // ---------------- fused zero_grad (multi-rank): a key's ready flag implies that every tile of it was reduced by its owner, i.e. nobody
  // will read this rank's gradients of that key again this round
  if (p.zero_grad && p.world > 1 && !p.defer_pull_wait) {
    for (int t = blockIdx.x; t < p.tiles; t += gridDim.x) {
      if (p.tile_active != nullptr && !p.tile_active[t]) continue;
      if (threadIdx.x == 0) wait_flag_ge(my_flags + p.param_ready_off + p.tile_key[t], epoch);
      __syncthreads();
      *reinterpret_cast<float4*>(p.grad[p.rank] + (long long)t * TILE + threadIdx.x * 4) = make_float4(0.f, 0.f, 0.f, 0.f);
    }
  }

  stamp(5);
  // ---------------- epoch / optimizer step bookkeeping (last CTA to finish publishes the new epoch)
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    const int done = atomicAdd(p.state + 1, 1);
    if (done == (int)gridDim.x - 1) {
      p.state[1] = 0;
      p.state[2] = opt_t;
      p.state[0] = (int)epoch;
      __threadfence();
    }
  }
}



// exclusive block scan of one int per thread (FAB_THREADS threads); s_w: >= 8 ints of scratch
__device__ __forceinline__ int block_excl_scan(int c, int* s_w, int& total) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  int incl = c;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) { const int n = __shfl_up_sync(0xffffffffu, incl, d); if (lane >= d) incl += n; }
  __syncthreads();
  if (lane == 31) s_w[w] = incl;
  __syncthreads();
  int base = 0; total = 0;
#pragma unroll
  for (int i = 0; i < FAB_THREADS / 32; ++i) { const int x = s_w[i]; if (i < w) base += x; total += x; }
  return base + incl - c;
}

// k-th largest of the 1024 keys of a tile (4 per thread), 8-bit radix select, 4 passes.  Returns the key; `ties` = how many keys equal to
// it belong to the top-k (they are taken in index order).  s_hist: 256 ints, s_w: 10 ints.
__device__ __forceinline__ uint32_t block_kth_largest(const uint32_t (&a)[4], int k, int* s_hist, int* s_w, int& ties) {
  uint32_t prefix = 0, mask = 0;
  int remaining = k;
  for (int shift = 24; shift >= 0; shift -= 8) {
    __syncthreads();
    s_hist[threadIdx.x] = 0;
    __syncthreads();
#pragma unroll
    for (int i = 0; i < 4; ++i) if ((a[i] & mask) == prefix) atomicAdd(&s_hist[(a[i] >> shift) & 255u], 1);
    __syncthreads();
    const int h = s_hist[255 - threadIdx.x];      // thread i owns bin 255-i: the exclusive scan counts the candidates in higher bins
    int tot;
    const int above = block_excl_scan(h, s_w, tot);
    if (above < remaining && above + h >= remaining) { s_w[8] = 255 - (int)threadIdx.x; s_w[9] = remaining - above; }
    __syncthreads();
    prefix |= (uint32_t)s_w[8] << shift;
    mask |= 255u << shift;
    remaining = s_w[9];
  }
  ties = remaining;
  return prefix;
}

template <bool SCHED, bool EXT>
__global__ void __launch_bounds__(FAB_THREADS, 2) hips_fsa_ll_kernel(const FabricParams p) {
  gx::pdl_wait();
  gx::pdl_launch();
  const bool dbg = p.state[3] != 0 && blockIdx.x == 0 && threadIdx.x == 0;
  unsigned long long* stamps = reinterpret_cast<unsigned long long*>(p.state + 8);
  auto stamp = [&](int i) { if (dbg) { unsigned long long t; asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t)); stamps[i] = t; } };
  stamp(0);
  __shared__ float s_tile[TILE];
  __shared__ int s_hist[FAB_THREADS];
  __shared__ int s_w[16];
  __shared__ float s_red[FAB_THREADS / 32];
  const uint32_t epoch = (uint32_t)(*reinterpret_cast<volatile int*>(p.state)) + 1u;
  const int opt_t = (*reinterpret_cast<volatile int*>(p.state + 2)) + 1;
  const float lr_t = step_lr<SCHED>(p.h, opt_t);
  const int S = p.party_size, P = p.ll_party_mode ? 1 : p.num_parties;
  const int party_base = p.party * S;
  const int slot = p.ll_party_mode ? 0 : p.party;                       // this party's packet slot on a global owner
  const int bc_lo = p.ll_party_mode ? party_base : 0, bc_n = p.ll_party_mode ? S : p.world;   // who receives the result
  float* const bc_mc = p.ll_party_mode ? nullptr : p.ll_c_mc;
  auto owner_of = [&](int t) -> int { return p.ll_party_mode ? party_base + t % S : p.tile_owner[t]; };
  const long long n2 = 2 * p.n;
  const int K = p.bsc_k;
  int* err = p.state + 5;

  // ---- phase 1: push my gradient tiles to their party owners (tiles I own myself are read in place in phase 2).  Inside a party the
  //      transport is dense (reference: worker -> local server is never sparsified), fp16 tiles travel as halves.
  for (int ti = blockIdx.x; ti < p.tiles; ti += gridDim.x) {
    const int t = p.tile_order ? p.tile_order[ti] : ti;   // DGT: important tiles first
    if (t % S == p.local) continue;
    if (p.tile_active != nullptr && !p.tile_active[t]) continue;
    const long long off = (long long)t * TILE + threadIdx.x * 4;
    float* g = p.grad[p.rank] + off;
    const float4 v = *reinterpret_cast<const float4*>(g);
    if (p.zero_grad) *reinterpret_cast<float4*>(g) = make_float4(0.f, 0.f, 0.f, 0.f);
    ll_send_dense(p.ll_a[party_base + t % S] + (long long)p.local * n2 + 2 * off, v, grad_fmt(fmt_of(p, t)), epoch);
  }
  stamp(1);
  // ---- phase 2: LOCAL PS TIER: the party owner sums the party's gradients of its tiles and forwards the aggregate to the global owner
  for (int ti = blockIdx.x; ti < p.tiles; ti += gridDim.x) {
    const int t = p.tile_order ? p.tile_order[ti] : ti;   // DGT: important tiles first
    if (t % S != p.local) continue;
    if (p.tile_active != nullptr && !p.tile_active[t]) continue;
    const int fmt = fmt_of(p, t);
    const long long off = (long long)t * TILE + threadIdx.x * 4;
    float* g = p.grad[p.rank] + off;
    float4 acc = *reinterpret_cast<const float4*>(g);
    if (p.zero_grad) *reinterpret_cast<float4*>(g) = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int j = 0; j < S; ++j) {
      if (j == p.local) continue;
      acc = f4_add(acc, ll_recv_dense(p.ll_a[p.rank] + (long long)j * n2 + 2 * off, grad_fmt(fmt), epoch, err));
    }
    acc = f4_scale(acc, p.push_scale);
    float* dst = p.ll_b[owner_of(t)] + (long long)slot * n2;
    if (fmt != FMT_BSC) {
      ll_send_dense(dst + 2 * off, acc, fmt, epoch);
      continue;
    }
    // Bi-Sparse (gradient_compression.cc:191-269 BSCompress, re-designed per 1024-value tile): momentum correction u = 0.9u + g, v += u;
    // the k largest |v| of the tile are sent as (value, index) packets in index order and their residual state is cleared.
    float4 U = *reinterpret_cast<float4*>(p.bsc_u + off), V = *reinterpret_cast<float4*>(p.bsc_v + off);
    U = f4_add(f4_scale(U, 0.9f), acc);
    V = f4_add(V, U);
    float vv[4] = {V.x, V.y, V.z, V.w}, uu[4] = {U.x, U.y, U.z, U.w};
    uint32_t a[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) a[i] = __float_as_uint(fabsf(vv[i]));
    int ties;
    const uint32_t T = block_kth_largest(a, K, s_hist, s_w, ties);
    int c_eq = 0;
#pragma unroll
    for (int i = 0; i < 4; ++i) c_eq += (a[i] == T);
    int tot;
    int eq_rank = block_excl_scan(c_eq, s_w, tot);
    bool take[4];
    int c_take = 0;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      take[i] = a[i] > T;
      if (a[i] == T) { take[i] = eq_rank < ties; ++eq_rank; }
      c_take += take[i];
    }
    int pos = block_excl_scan(c_take, s_w, tot);   // tot == K
    float* pk = dst + 2 * (long long)t * TILE;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      if (take[i]) {
        ll_store1(pk + 4 * pos, vv[i], (float)(threadIdx.x * 4 + i), epoch);
        ++pos; vv[i] = 0.f; uu[i] = 0.f;
      }
    }
    *reinterpret_cast<float4*>(p.bsc_u + off) = make_float4(uu[0], uu[1], uu[2], uu[3]);
    *reinterpret_cast<float4*>(p.bsc_v + off) = make_float4(vv[0], vv[1], vv[2], vv[3]);
  }
  stamp(2);
  // ---- phase 3: GLOBAL PS TIER: the global owner sums the parties' aggregates, runs the optimizer on its shard and pushes the result
  for (int ti = blockIdx.x; ti < p.tiles; ti += gridDim.x) {
    const int t = p.tile_order ? p.tile_order[ti] : ti;   // DGT: important tiles first
    if (owner_of(t) != p.rank) continue;
    if (p.tile_active != nullptr && !p.tile_active[t]) continue;
    const int fmt = fmt_of(p, t);
    const long long off = (long long)t * TILE + threadIdx.x * 4;
    TileState s = tile_state_load(p, t, off, lr_t);   // issued before the poll: the state loads overlap the wait
    float4 agg;
    if (fmt != FMT_BSC) {
      agg = ll_recv_dense(p.ll_b[p.rank] + 2 * off, fmt, epoch, err);
      for (int g = 1; g < P; ++g) agg = f4_add(agg, ll_recv_dense(p.ll_b[p.rank] + (long long)g * n2 + 2 * off, fmt, epoch, err));
    } else {  // BSCDecompress (:310-336) of every party's packets + sum, in shared memory
      __syncthreads();
      *reinterpret_cast<float4*>(s_tile + threadIdx.x * 4) = make_float4(0.f, 0.f, 0.f, 0.f);
      __syncthreads();
      for (int g = 0; g < P; ++g)
        for (int j = threadIdx.x; j < K; j += FAB_THREADS) {
          const float2 e = ll_load1(p.ll_b[p.rank] + (long long)g * n2 + 2 * (long long)t * TILE + 4 * j, epoch, err);
          const int idx = (int)e.y;
          if (idx >= 0 && idx < TILE) atomicAdd(s_tile + idx, e.x);
        }
      __syncthreads();
      agg = *reinterpret_cast<const float4*>(s_tile + threadIdx.x * 4);
    }
    if (p.dgt_contrib != nullptr) dgt_update_contrib(p, t, agg, s_red);
    const float4 W = tile_state_apply<EXT>(p, off, s, agg);
    if (fmt == FMT_BSC && p.h.kind < 0) {
      // BSCPullCompress (:271-308): the aggregated gradient goes back sparse — its non-zeros in index order, at most P*K of them
      const float ww[4] = {W.x, W.y, W.z, W.w};
      int c = 0;
#pragma unroll
      for (int i = 0; i < 4; ++i) c += (ww[i] != 0.f);
      int tot;
      int pos = block_excl_scan(c, s_w, tot);
      const long long base = 2 * (long long)t * TILE;
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        if (ww[i] != 0.f) {
          if (bc_mc != nullptr) ll_store1_mc(bc_mc + base + 4 * pos, ww[i], (float)(threadIdx.x * 4 + i), epoch);
          else for (int r = bc_lo; r < bc_lo + bc_n; ++r) ll_store1(p.ll_c[r] + base + 4 * pos, ww[i], (float)(threadIdx.x * 4 + i), epoch);
          ++pos;
        }
      }
      for (int j = tot + threadIdx.x; j < P * K; j += FAB_THREADS) {   // padding packets: index -1
        if (bc_mc != nullptr) ll_store1_mc(bc_mc + base + 4 * j, 0.f, -1.f, epoch);
        else for (int r = bc_lo; r < bc_lo + bc_n; ++r) ll_store1(p.ll_c[r] + base + 4 * j, 0.f, -1.f, epoch);
      }
    } else {
      const int bf = (fmt == FMT_F16 || fmt == FMT_F8) ? FMT_F16 : FMT_F32;   // parameters of fp8 tiles return as fp16
      if (bc_mc != nullptr) ll_send_dense_mc(bc_mc + 2 * off, W, bf, epoch);
      else for (int r = bc_lo; r < bc_lo + bc_n; ++r) ll_send_dense(p.ll_c[r] + 2 * off, W, bf, epoch);
    }
  }
  stamp(3);
  // ---- phase 4: pull: unpack the fresh parameters into the (plain fp32) parameter arena the forward pass reads
  for (int ti = blockIdx.x; ti < p.tiles; ti += gridDim.x) {
    const int t = p.tile_order ? p.tile_order[ti] : ti;   // DGT: important tiles first
    if (p.tile_active != nullptr && !p.tile_active[t]) continue;
    const int fmt = fmt_of(p, t);
    const long long off = (long long)t * TILE + threadIdx.x * 4;
    if (fmt == FMT_BSC && p.h.kind < 0) {   // BSCDecompress on the worker side: zero + scatter
      __syncthreads();
      *reinterpret_cast<float4*>(p.param[p.rank] + off) = make_float4(0.f, 0.f, 0.f, 0.f);
      __syncthreads();
      for (int j = threadIdx.x; j < P * K; j += FAB_THREADS) {
        const float2 e = ll_load1(p.ll_c[p.rank] + 2 * (long long)t * TILE + 4 * j, epoch, err);
        const int idx = (int)e.y;
        if (idx >= 0 && idx < TILE) p.param[p.rank][(long long)t * TILE + idx] = e.x;
      }
    } else {
      *reinterpret_cast<float4*>(p.param[p.rank] + off) = ll_recv_dense(p.ll_c[p.rank] + 2 * off, (fmt == FMT_F16 || fmt == FMT_F8) ? FMT_F16 : FMT_F32, epoch, err);
    }
  }
  stamp(4);
  // bookkeeping: the state words are only read by the NEXT launch (kernel boundary orders them), so a relaxed counter is enough —
  // a __threadfence here would wait for every outstanding remote store of this CTA (~2 us)
  if (threadIdx.x == 0) {
    const int done = atomicAdd(p.state + 1, 1);
    if (done == (int)gridDim.x - 1) {
      p.state[1] = 0;
      p.state[2] = opt_t;
      p.state[0] = (int)epoch;
    }
  }
  stamp(5);
}

// ------------------------------------------------------------------------------------------------------------------ direct protocol
// The LL kernel above walks the reference's hierarchy hop by hop (worker -> party owner -> global owner -> everybody: three dependent NVLink
// hops).  On an NVSwitch every rank reaches every other rank at full bandwidth, so the two server tiers can live on the SAME rank without
// changing what is computed: each gradient tile goes straight to the rank that applies the update, which sums it in the hierarchy's order
// (inside each party first, `push_scale` on the party aggregate, then across parties — bit-identical on every rank that does it) and runs
// the optimizer.  Two modes per launch ("channel"):
//   sharded     (direct_replicate = 0): the tile's global owner (tile_owner, all ranks by default) reduces, updates its shard of the master
//               weights / optimizer state and multicasts the fresh tile: TWO hops, 1/world of the optimizer work per rank.
//   replicated  (direct_replicate = 1): every rank receives every gradient tile (one multimem.st per sender) and applies the update to its own
//               replica of the server state: ONE hop, no result traffic.  Meant for the few small keys whose gradients are produced LAST in
//               the backward pass (conv0/conv1 of the demo CNN: 13 tiles) — their exchange cannot overlap compute, so it must be short.
// A training step launches one channel per key group as soon as that group's gradients are complete (HipsCNNTrainStep: the dense keys'
// sharded channel runs on a side stream underneath the convolution backward pass; the conv keys' replicated channel is the only exposed
// communication).  Reference for the ordering idea: per-key push with priority = -index (examples/cnn.py:121-125, kvstore_dist.h:565-625).
// Every channel owns its state block (epoch, CTA counter, optimizer step) and stamps its id into the packet epoch.
template <bool SCHED, bool EXT>
__global__ void __launch_bounds__(FAB_THREADS, 2) hips_fsa_direct_kernel(const FabricParams p) {
  // Before the grid dependency resolves (i.e. while the kernel that produces the gradients is still running): walk this CTA's tiles once and
  // pull everything that does NOT depend on that kernel towards L2 — the tile metadata, the optimizer state and master weights of the tiles
  // this rank applies, and the lines of the gradient tiles themselves (their contents arrive later; the lines are then already resident).
  // After a cold start (bench.py flushes L2 between steps) this takes a chain of DRAM round trips off the exchange's critical path.
  {
    auto pf = [](const void* q) { asm volatile("prefetch.global.L2 [%0];" ::"l"(q)); };
    if (threadIdx.x == 0) pf(p.state);
    for (int ti = blockIdx.x; ti < p.tiles; ti += gridDim.x) {
      const int t = p.tile_order ? p.tile_order[ti] : ti;
      if (p.tile_active != nullptr && !p.tile_active[t]) continue;
      const long long off = (long long)t * TILE + threadIdx.x * 4;
      if ((threadIdx.x & 7) == 0) {                      // one prefetch per 128-byte line
        pf(p.grad[p.rank] + off);
        if (p.direct_replicate != 0 || p.tile_owner[t] == p.rank) {
          pf(p.w + off);
          if (p.s0) pf(p.s0 + off);
          if (p.s1) pf(p.s1 + off);
        }
      }
    }
  }
  gx::pdl_wait();
  gx::pdl_launch();
  const bool dbg = p.state[3] != 0 && blockIdx.x == 0 && threadIdx.x == 0;
  unsigned long long* stamps = reinterpret_cast<unsigned long long*>(p.state + 8);
  auto stamp = [&](int i) { if (dbg) { unsigned long long t; asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t)); stamps[i] = t; } };
  stamp(0);
  __shared__ float s_red[FAB_THREADS / 32];
  const uint32_t round = (uint32_t)(*reinterpret_cast<volatile int*>(p.state)) + 1u;
  const uint32_t epoch = (round << 3) | (uint32_t)(p.channel_id & 7);
  const int opt_t = (*reinterpret_cast<volatile int*>(p.state + 2)) + 1;
  const float lr_t = step_lr<SCHED>(p.h, opt_t);
  const bool rep = p.direct_replicate != 0;
  int* err = p.state + 5;

  // ---- phase 1: push my gradient tiles to the rank(s) that apply them (my own slot included: the reducer reads all slots the same way)
  for (int ti = blockIdx.x; ti < p.tiles; ti += gridDim.x) {
    const int t = p.tile_order ? p.tile_order[ti] : ti;
    if (p.tile_active != nullptr && !p.tile_active[t]) continue;
    const long long off = (long long)t * TILE + threadIdx.x * 4;
    float* g = p.grad[p.rank] + off;
    const float4 v = *reinterpret_cast<const float4*>(g);
    if (p.zero_grad) *reinterpret_cast<float4*>(g) = make_float4(0.f, 0.f, 0.f, 0.f);
    const int f = grad_fmt(fmt_of(p, t));
    if (rep) direct_send_all(p, off, v, f, epoch);
    else ll_send_dense(p.ll_d[p.tile_owner[t]] + (long long)p.rank * 2 * p.n + 2 * off, v, f, epoch);
  }
  stamp(1);
  // ---- phase 2: both server tiers on the applying rank: party sums, scale, sum over parties, optimizer
  for (int ti = blockIdx.x; ti < p.tiles; ti += gridDim.x) {
    const int t = p.tile_order ? p.tile_order[ti] : ti;
    if (p.tile_active != nullptr && !p.tile_active[t]) continue;
    if (!rep && p.tile_owner[t] != p.rank) continue;
    const int f = grad_fmt(fmt_of(p, t));
    const long long off = (long long)t * TILE + threadIdx.x * 4;
    TileState s = tile_state_load(p, t, off, lr_t);   // issued before the polls: the state loads overlap the wait
    const float4 agg = direct_recv_sum(p, off, f, epoch, err);
    if (p.dgt_contrib != nullptr && (!rep || p.tile_owner[t] == p.rank)) dgt_update_contrib(p, t, agg, s_red);
    const float4 W = tile_state_apply<EXT>(p, off, s, agg);
    if (rep) {
      *reinterpret_cast<float4*>(p.param[p.rank] + off) = W;   // the pull is a local store: every rank holds the fresh replica
    } else {
      const int bf = f == FMT_F32 ? FMT_F32 : FMT_F16;          // parameters of fp16 / fp8 keys return as halves
      if (p.ll_e_mc != nullptr) ll_send_dense_mc(p.ll_e_mc + 2 * off, W, bf, epoch);
      else for (int r = 0; r < p.world; ++r) ll_send_dense(p.ll_e[r] + 2 * off, W, bf, epoch);
    }
  }
  stamp(2);
  // ---- phase 3 (sharded mode): pull = unpack the owners' packets into the parameter arena
  if (!rep) {
    for (int ti = blockIdx.x; ti < p.tiles; ti += gridDim.x) {
      const int t = p.tile_order ? p.tile_order[ti] : ti;
      if (p.tile_active != nullptr && !p.tile_active[t]) continue;
      const long long off = (long long)t * TILE + threadIdx.x * 4;
      const int bf = grad_fmt(fmt_of(p, t)) == FMT_F32 ? FMT_F32 : FMT_F16;
      *reinterpret_cast<float4*>(p.param[p.rank] + off) = ll_recv_dense(p.ll_e[p.rank] + 2 * off, bf, epoch, err);
    }
  }
  stamp(4);
  if (threadIdx.x == 0) {
    const int done = atomicAdd(p.state + 1, 1);
    if (done == (int)gridDim.x - 1) {
      p.state[1] = 0;
      p.state[2] = opt_t;
      p.state[0] = (int)round;
    }
  }
  stamp(5);
}

// One-sided MixedSync: the party's tile owner applies its aggregate directly on the global owner's HBM under a per-tile lock.
// locks live in the global owner's flag pad at `lock_off` (uint32 per tile), per-tile optimizer step counts right after them.
template <bool SCHED, bool EXT>
__global__ void __launch_bounds__(FAB_THREADS, 1) hips_async_step_kernel(const FabricParams p, float* const* w_peer, float* const* s0_peer,
                                                                          float* const* s1_peer, int lock_off, int step_off) {
  gx::pdl_wait();
  gx::pdl_launch();
  const uint32_t epoch = (uint32_t)(*reinterpret_cast<volatile int*>(p.state)) + 1u;
  const int S = p.party_size;
  const int party_base = p.party * S;
  uint32_t* my_flags = p.flags[p.rank];
  __shared__ int s_step;
  if (blockIdx.x == 0 && threadIdx.x < S) {
    fence_sys();
    st_release_sys(p.flags[party_base + threadIdx.x] + p.ready_off + p.rank, epoch);
  }
  bool waited_party = false;
  for (int t = blockIdx.x; t < p.tiles; t += gridDim.x) {
    if (t % S != p.local) continue;
    if (p.tile_active != nullptr && !p.tile_active[t]) continue;
    if (!waited_party) {
      if (threadIdx.x < S) wait_flag_ge(my_flags + p.ready_off + party_base + threadIdx.x, epoch);
      __syncthreads();
      waited_party = true;
    }
    const long long off = (long long)t * TILE + threadIdx.x * 4;
    float4 acc;
    if (p.grad_mc != nullptr && S > 1) acc = multimem_ld_reduce_f4(p.grad_mc + off);
    else {
      acc = (S == 1) ? *reinterpret_cast<const float4*>(p.grad[p.rank] + off) : ld_f4_sys(p.grad[party_base] + off);
      for (int j = 1; j < S; ++j) acc = f4_add(acc, ld_f4_sys(p.grad[party_base + j] + off));
    }
    acc = f4_scale(acc, p.push_scale);
    const int owner = p.tile_owner[t];
    uint32_t* lock = p.flags[owner] + lock_off + t;
    uint32_t* stepc = p.flags[owner] + step_off + t;
    if (threadIdx.x == 0) {
      while (atomicCAS_system(lock, 0u, 1u) != 0u) { __nanosleep(40); }
      fence_sys();
      s_step = (int)ld_relaxed_sys(stepc) + 1;
    }
    __syncthreads();
    float lr = step_lr<SCHED>(p.h, s_step), wd = p.h.wd;
    if (p.tile_mult) { const float2 mm = __ldg(p.tile_mult + t); lr *= mm.x; wd *= mm.y; }
    float* wp = w_peer[owner] + off;
    float4 W = ld_f4_sys(wp);
    float4 A = s0_peer[owner] ? ld_f4_sys(s0_peer[owner] + off) : make_float4(0, 0, 0, 0);
    float4 B = s1_peer[owner] ? ld_f4_sys(s1_peer[owner] + off) : make_float4(0, 0, 0, 0);
    opt_apply4<EXT>(W, acc, A, B, p.h, lr, wd);
    st_f4_sys(wp, W);
    if (s0_peer[owner]) st_f4_sys(s0_peer[owner] + off, A);
    if (s1_peer[owner]) st_f4_sys(s1_peer[owner] + off, B);
    // pull for the own party only (other parties see this update when they next push)
    for (int j = 0; j < S; ++j) st_f4_sys(p.param[party_base + j] + off, W);
    __syncthreads();
    if (threadIdx.x == 0) {
      fence_sys();
      asm volatile("st.relaxed.sys.global.u32 [%0], %1;" ::"l"(stepc), "r"((uint32_t)s_step) : "memory");
      fence_sys();
      st_release_sys(lock, 0u);
      for (int j = 0; j < S; ++j) red_add_release_sys(p.flags[party_base + j] + p.param_ready_off + p.tile_key[t], 1u);
    }
    __syncthreads();
  }
  // wait until every tile of every key has been delivered to this rank by its party's owners (cumulative counters)
  if (blockIdx.x == 0) {
    for (int k = threadIdx.x; k < p.num_keys; k += blockDim.x) wait_flag_ge(my_flags + p.param_ready_off + k, epoch * (uint32_t)p.key_tiles[k]);
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    const int done = atomicAdd(p.state + 1, 1);
    if (done == (int)gridDim.x - 1) { p.state[1] = 0; p.state[0] = (int)epoch; __threadfence(); }
  }
}

// Local tier only: out[party members] = scale * sum_{party} src   (HFA local synchronisation, party-level all-reduce)
//   mode 0: write the result into every party member's `dst` arena; mode 1: only into the owner's `dst` (reduce-scatter)
__global__ void __launch_bounds__(FAB_THREADS, 1) hips_party_allreduce_kernel(const FabricParams p, float* const* src_peer, float* const* dst_peer,
                                                                               float scale, int mode, int flag_off) {
  gx::pdl_wait();
  gx::pdl_launch();
  const uint32_t epoch = (uint32_t)(*reinterpret_cast<volatile int*>(p.state)) + 1u;
  const int S = p.party_size, party_base = p.party * S;
  uint32_t* my_flags = p.flags[p.rank];
  if (blockIdx.x == 0 && threadIdx.x < S) {
    fence_sys();
    st_release_sys(p.flags[party_base + threadIdx.x] + p.ready_off + p.rank, epoch);
  }
  bool waited = false;
  int mine = 0;
  for (int t = blockIdx.x; t < p.tiles; t += gridDim.x) {
    if (t % S != p.local) continue;
    if (!waited) {
      if (threadIdx.x < S) wait_flag_ge(my_flags + p.ready_off + party_base + threadIdx.x, epoch);
      __syncthreads();
      waited = true;
    }
    const long long off = (long long)t * TILE + threadIdx.x * 4;
    float4 acc = (S == 1) ? *reinterpret_cast<const float4*>(src_peer[p.rank] + off) : ld_f4_sys(src_peer[party_base] + off);
    for (int j = 1; j < S; ++j) acc = f4_add(acc, ld_f4_sys(src_peer[party_base + j] + off));
    acc = f4_scale(acc, scale);
    if (mode == 0) for (int j = 0; j < S; ++j) st_f4_sys(dst_peer[party_base + j] + off, acc);
    else *reinterpret_cast<float4*>(dst_peer[p.rank] + off) = acc;
    ++mine;
  }
  __syncthreads();
  if (threadIdx.x == 0 && mine > 0 && mode == 0) {
    fence_sys();
    for (int j = 0; j < S; ++j) red_add_release_sys(p.flags[party_base + j] + flag_off, (uint32_t)mine);
  }
  if (mode == 0 && blockIdx.x == 0 && threadIdx.x == 0) wait_flag_ge(my_flags + flag_off, epoch * (uint32_t)p.tiles);
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    const int done = atomicAdd(p.state + 1, 1);
    if (done == (int)gridDim.x - 1) { p.state[1] = 0; p.state[0] = (int)epoch; __threadfence(); }
  }
}

// Whole-world flag barrier (two-tier HiPS barrier collapses to one hop on NVSwitch): counter at flag offset `off`.
__global__ void fabric_barrier_kernel(uint32_t* const* flags, int world, int rank, int off, int* state) {
  gx::pdl_wait();
  gx::pdl_launch();
  if (threadIdx.x == 0) {
    const uint32_t e = (uint32_t)(*reinterpret_cast<volatile int*>(state)) + 1u;
    fence_sys();
    for (int r = 0; r < world; ++r) red_add_release_sys(flags[r] + off, 1u);
    wait_flag_ge(flags[rank] + off, e * (uint32_t)world);
    *state = (int)e;
  }
}


// Fabric micro-probe (tools/fabric_probe.py): latency of every primitive the fused kernels are built from, measured by thread 0 of
// CTA 0 with %globaltimer (ns) while the whole grid performs the same access on its own 4 KB tile (so queueing is included).
//   out[2k], out[2k+1] = first / second measurement of primitive k
__device__ __forceinline__ unsigned long long gtime() { unsigned long long t; asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t)::"memory"); return t; }
__device__ __forceinline__ void consume(float v) {  // a store cannot issue before its operand arrived, and the timer read is ordered after it
  __shared__ float sink[FAB_THREADS];
  asm volatile("st.volatile.shared.f32 [%0], %1;" ::"r"((uint32_t)__cvta_generic_to_shared(sink + threadIdx.x)), "f"(v) : "memory");
}

__global__ void __launch_bounds__(FAB_THREADS, 1) fabric_probe_kernel(float* local, float* peer, float* mc, uint32_t* peer_flag,
                                                                      unsigned long long* out, int tiles) {
  const bool rec = blockIdx.x == 0 && threadIdx.x == 0;
  const long long off0 = (long long)(blockIdx.x % tiles) * TILE + threadIdx.x * 4;
  const long long off1 = (long long)((blockIdx.x + gridDim.x) % tiles) * TILE + threadIdx.x * 4;
  unsigned long long t0;
  float4 v;
  for (int rep = 0; rep < 2; ++rep) {
    const long long off = rep ? off1 : off0;
    int k = 0;
    auto done = [&]() { if (rec) out[2 * k + rep] = gtime() - t0; ++k; __syncthreads(); };
    // 0 local weak load
    t0 = gtime(); asm volatile("ld.global.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(local + off) : "memory"); consume(v.x); done();
    // 1 local ld.relaxed.sys
    t0 = gtime(); v = ld_f4_sys(local + off); consume(v.x); done();
    // 2 peer weak load (L1-cacheable)
    t0 = gtime(); asm volatile("ld.global.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(peer + off) : "memory"); consume(v.x); done();
    // 3 peer ld.relaxed.sys
    t0 = gtime(); v = ld_f4_sys(peer + off); consume(v.x); done();
    // 4 multimem.ld_reduce
    if (mc) { t0 = gtime(); v = multimem_ld_reduce_f4(mc + off); consume(v.x); } else t0 = gtime();
    done();
    // 5 peer store + fence.sys
    t0 = gtime(); st_f4_sys(peer + off, v); fence_sys(); done();
    // 6 multimem.st + fence.sys
    t0 = gtime(); if (mc) { multimem_st_f4(mc + off, v); fence_sys(); } done();
    // 7 fence.sys with nothing outstanding
    t0 = gtime(); fence_sys(); done();
    // 8 peer store, __syncthreads, ONE fence by thread 0, release flag store (the tile hand-off idiom)
    t0 = gtime(); st_f4_sys(peer + off, v); __syncthreads(); if (threadIdx.x == 0) { fence_sys(); st_release_sys(peer_flag + blockIdx.x, 1u); } done();
    // 9 local acquire load of a flag
    t0 = gtime(); { uint32_t f = ld_acquire_sys(peer_flag + 4096 + blockIdx.x); consume(__uint_as_float(f)); } done();
    // 10 local store + __threadfence
    t0 = gtime(); *reinterpret_cast<float4*>(local + off) = v; __threadfence(); done();
  }
}

}  // namespace gx

using namespace gx;

GX_API int gx_fabric_params_size() { return (int)sizeof(FabricParams); }

// `params` is a host copy of FabricParams (assembled by geomx_b200/parallel/fabric.py through ctypes).
GX_API int gx_hips_fsa_step(const void* params, int grid, cudaStream_t s) {
  FabricParams p = *reinterpret_cast<const FabricParams*>(params);
  if (grid < 1) grid = 1;
  if (p.world == 1) launch_pdl(GX_FAB_INSTANCE(hips_fsa_step_single_kernel, p), dim3(grid), dim3(FAB_THREADS), 0, s, p);
  else launch_pdl(GX_FAB_INSTANCE(hips_fsa_step_kernel, p), dim3(grid), dim3(FAB_THREADS), 0, s, p);
  return GX_CHECK_LAUNCH();
}
// During stream capture: the node just captured on `s` keeps a programmatic edge only from its first dependency (the launch before it on
// its own stream); its edges from the streams it joined become full dependencies.  Measured on an H100: with a programmatic edge from the
// dense-chain tail, the dense keys' channel resolved its grid dependency about 1 us after the convolution backward grid that follows the
// tail on the main stream ended (21.5 us into the step), 2.4 us after its own predecessors had; with a full edge, 0.5 us after
// dense_wgrad ended (19.7 us).  Returns the number of edges changed (0 outside a capture), -1 on an error.
GX_API int gx_capture_demote_joined_edges(cudaStream_t s) {
  cudaStreamCaptureStatus st;
  cudaGraph_t g = nullptr;
  const cudaGraphNode_t* deps = nullptr;
  size_t n = 0;
  if (cudaStreamGetCaptureInfo(s, &st, nullptr, &g, &deps, &n) != cudaSuccess || st != cudaStreamCaptureStatusActive || n != 1) {
    cudaGetLastError();
    return 0;
  }
  cudaGraphNode_t node = deps[0];
  size_t m = 0;
  if (cudaGraphNodeGetDependencies_v2(node, nullptr, nullptr, &m) != cudaSuccess || m < 2) return 0;
  cudaGraphNode_t from[8];
  cudaGraphEdgeData ed[8];
  if (m > 8 || cudaGraphNodeGetDependencies_v2(node, from, ed, &m) != cudaSuccess) return -1;
  int changed = 0;
  for (size_t i = 1; i < m; ++i) {
    if (ed[i].type != cudaGraphDependencyTypeProgrammatic) continue;
    cudaGraphEdgeData full = {};
    if (cudaGraphRemoveDependencies_v2(g, &from[i], &node, &ed[i], 1) != cudaSuccess ||
        cudaGraphAddDependencies_v2(g, &from[i], &node, &full, 1) != cudaSuccess)
      return -1;
    ++changed;
  }
  return changed;
}

// Largest co-resident grid of the fused kernels (they spin on each other: every CTA of a launch must be resident).
GX_API int gx_hips_max_grid() {
  int dev = 0, sms = 0, occ = 1 << 30;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  // every instance of each: constant and scheduled lr, with and without the later optimizer kinds
  for (const void* k : {(const void*)hips_fsa_ll_kernel<false, false>, (const void*)hips_fsa_ll_kernel<true, false>,
                        (const void*)hips_fsa_ll_kernel<false, true>, (const void*)hips_fsa_ll_kernel<true, true>,
                        (const void*)hips_fsa_step_kernel<false, false>, (const void*)hips_fsa_step_kernel<true, false>,
                        (const void*)hips_fsa_step_kernel<false, true>, (const void*)hips_fsa_step_kernel<true, true>}) {
    int o = 0;
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&o, k, FAB_THREADS, 0);
    occ = o < occ ? o : occ;
  }
  return sms * (occ < 1 ? 1 : (occ > 2 ? 2 : occ));
}
GX_API int gx_hips_fsa_ll_step(const void* params, int grid, cudaStream_t s) {
  FabricParams p = *reinterpret_cast<const FabricParams*>(params);
  if (grid < 1) grid = 1;
  launch_pdl(GX_FAB_INSTANCE(hips_fsa_ll_kernel, p), dim3(grid), dim3(FAB_THREADS), 0, s, p);
  return GX_CHECK_LAUNCH();
}
GX_API int gx_hips_fsa_direct_step(const void* params, int grid, cudaStream_t s) {
  FabricParams p = *reinterpret_cast<const FabricParams*>(params);
  if (grid < 1) grid = 1;
  launch_pdl(GX_FAB_INSTANCE(hips_fsa_direct_kernel, p), dim3(grid), dim3(FAB_THREADS), 0, s,
             p);
  return GX_CHECK_LAUNCH();
}
GX_API int gx_hips_async_step(const void* params, float* const* w_peer, float* const* s0_peer, float* const* s1_peer, int lock_off, int step_off,
                              int grid, cudaStream_t s) {
  FabricParams p = *reinterpret_cast<const FabricParams*>(params);
  launch_pdl(GX_FAB_INSTANCE(hips_async_step_kernel, p), dim3(grid), dim3(FAB_THREADS), 0, s, p,
             w_peer, s0_peer, s1_peer, lock_off, step_off);
  return GX_CHECK_LAUNCH();
}
GX_API int gx_hips_party_allreduce(const void* params, float* const* src_peer, float* const* dst_peer, float scale, int mode, int flag_off, int grid,
                                   cudaStream_t s) {
  FabricParams p = *reinterpret_cast<const FabricParams*>(params);
  launch_pdl(hips_party_allreduce_kernel, dim3(grid), dim3(FAB_THREADS), 0, s, p, src_peer, dst_peer, scale, mode, flag_off);
  return GX_CHECK_LAUNCH();
}
GX_API int gx_fabric_barrier(uint32_t* const* flags_dev, int world, int rank, int off, int* state, cudaStream_t s) {
  launch_pdl(fabric_barrier_kernel, dim3(1), dim3(32), 0, s, flags_dev, world, rank, off, state);
  return GX_CHECK_LAUNCH();
}

GX_API int gx_fabric_probe(float* local, float* peer, float* mc, uint32_t* peer_flag, unsigned long long* out, int tiles, int grid, cudaStream_t s) {
  fabric_probe_kernel<<<grid, FAB_THREADS, 0, s>>>(local, peer, mc, peer_flag, out, tiles);
  return GX_CHECK_LAUNCH();
}
