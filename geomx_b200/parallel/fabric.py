"""HiPS fabric: topology, symmetric HBM heap and the fused push/pull kernels' host side.

One process per GPU (``torchrun``); ``torch.distributed`` is used ONLY for rendezvous, symmetric-memory handle exchange and init-time
broadcasts ("plumbing", SURVEY §5.8).  The per-step data path is ``gx_hips_fsa_step`` / ``gx_hips_async_step`` /
``gx_hips_party_allreduce`` (``csrc/kernels/hips_fabric.cu``): in-kernel P2P + NVLS multimem collectives, no NCCL call.

Roles (reference ``3rdparty/ps-lite/src/postoffice.cc:18-58`` and scripts ``scripts/gpu/run_vanilla_hips.sh``) become rank attributes:
party ``g`` = ranks ``[g*S, (g+1)*S)`` (S = workers per party); the *local server* of a party is the set of tile owners inside it; the
*global servers* are ``num_gs`` ranks (default: rank 0; MultiGPS: ranks ``0, S, 2S, …`` round-robin) whose HBM holds master weights and
optimizer state; the *master worker* role (init keys, set optimizer) is folded into rank 0; schedulers disappear.
"""
from __future__ import annotations

import ctypes
import os

import numpy as np
import torch

from ..base import MXNetError, getenv_int
from ..ops import native
from ..ops._native_api import OPT_KINDS, OptHyper, pack_hyper
from .arena import ArenaLayout

MAX_RANKS = 16


# ------------------------------------------------------------------------------------------------------------ topology
class Topology:
    def __init__(self, world=1, rank=0, num_parties=1, num_gs=1):
        if world % num_parties:
            raise MXNetError("world size %d is not divisible by the number of parties %d" % (world, num_parties))
        if world > MAX_RANKS:
            raise MXNetError("fabric supports up to %d ranks per NVSwitch domain" % MAX_RANKS)
        self.world, self.rank, self.num_parties = world, rank, num_parties
        self.party_size = world // num_parties
        self.party, self.local = rank // self.party_size, rank % self.party_size
        # num_gs = 0 ("auto", the fabric default): EVERY rank is a global server and ownership is sharded tile by tile, so the server-side
        # optimizer work and the result traffic are spread over the whole box.  num_gs >= 1 (DMLC_NUM_GLOBAL_SERVER given explicitly) keeps the
        # reference's placement: that many server ranks, small keys hashed / big keys partitioned (kvstore_dist_server.h:1770-1810).
        self.tile_sharded = int(num_gs) <= 0
        self.num_gs = world if self.tile_sharded else max(1, min(num_gs, world))
        # global servers: spread over parties first (rank 0, S, 2S, ... then 1, S+1, ...)
        order = [p * self.party_size + l for l in range(self.party_size) for p in range(num_parties)]
        self.gs_ranks = order[:self.num_gs]

    @staticmethod
    def from_env():
        world = getenv_int("WORLD_SIZE", 1); rank = getenv_int("RANK", 0)
        # default: the two-tier layout of the reference's demo (2 parties) whenever the world splits evenly
        parties = getenv_int("GEOMX_NUM_PARTIES", 0) or getenv_int("DMLC_NUM_GLOBAL_WORKER", 0) or (2 if (world >= 2 and world % 2 == 0) else 1)
        if world % parties:
            parties = 1
        return Topology(world, rank, parties, getenv_int("DMLC_NUM_GLOBAL_SERVER", 0))

    @property
    def num_workers(self): return self.party_size          # per party  (kv.num_workers)
    @property
    def num_all_workers(self): return self.world           # kv.num_all_workers
    @property
    def is_global_server(self): return self.rank in self.gs_ranks
    def party_ranks(self, g=None):
        g = self.party if g is None else g
        return list(range(g * self.party_size, (g + 1) * self.party_size))


def global_tile_owners(topo, layout, protocol, bigarray_bound=1000000):
    """World rank that plays global server for every 1024-float tile of ``layout`` (int32 array of ``layout.total // 1024`` entries).

    * ``topo.tile_sharded`` (``DMLC_NUM_GLOBAL_SERVER`` unset) and a packet protocol: tile ``ti`` -> rank ``((ti // S) % P) * S + ti % S`` —
      balanced over all ranks, and the owner is the tile's party owner inside its own party (the 3-hop LL kernel keeps one inter-tier hop local);
    * ``tile_sharded`` with the flag ("bulk") protocol: its per-key ready flags need ONE owner per key -> whole keys, largest first onto the
      least loaded rank;
    * explicit ``num_gs``: the reference's placement over ``topo.gs_ranks`` (small keys hashed, big keys partitioned,
      kvstore_dist_server.h:1770-1810)."""
    T = layout.total // 1024
    if topo.tile_sharded and protocol == "ll":
        ti = np.arange(T)
        return (((ti // topo.party_size) % topo.num_parties) * topo.party_size + ti % topo.party_size).astype(np.int32)
    if topo.tile_sharded:
        load = np.zeros(topo.world, dtype=np.int64)
        owners = np.zeros(T, dtype=np.int32)
        for sl in sorted(layout.slots, key=lambda s: -s.tiles):
            r = int(np.argmin(load))
            load[r] += sl.tiles
            owners[sl.offset // 1024: sl.offset // 1024 + sl.tiles] = r
        return owners
    owner_idx = layout.global_owner_index(topo.num_gs, bigarray_bound)
    return np.array([topo.gs_ranks[i] for i in owner_idx], dtype=np.int32)


def held_tiles(owners, replicated, rank):
    """Tiles whose server state ``rank`` holds: those it owns, and every tile in ``replicated`` (each rank updates its own replica of those:
    a single rank, or a one-hop replicated channel).  ``replicated``: bool per tile or None."""
    held = np.asarray(owners) == rank
    return held if replicated is None else held | np.asarray(replicated, dtype=bool)


def gather_tile_state(per_rank, owners, replicated=None):
    """One piece of server state as a full array, from every rank's copy of it: tile ``t`` from its owner ``owners[t]``, a replicated tile
    from rank 0's replica.  ``per_rank[r]``: rank r's array, tile-major with the same number of values per tile (1024 for an arena, 1 for a
    per-tile word).  Host-only, so that any topology can be simulated."""
    owners = np.asarray(owners)
    src = owners if replicated is None else np.where(np.asarray(replicated, dtype=bool), 0, owners)
    T = len(src)
    out = np.array(per_rank[0], copy=True).reshape(T, -1)
    for r in np.unique(src):
        sel = src == r
        out[sel] = np.asarray(per_rank[int(r)]).reshape(T, -1)[sel]
    return out.reshape(np.shape(per_rank[0]))


def scatter_tile_state(full, per_rank, owners, replicated=None):
    """Inverse of :func:`gather_tile_state`: write ``full`` into the arrays of ``per_rank`` (a dict rank -> array, updated in place) on the
    tiles that rank holds (:func:`held_tiles`); the other tiles keep their values.  Returns ``per_rank``."""
    T = len(owners)
    src = np.asarray(full).reshape(T, -1)
    for r, arr in per_rank.items():
        sel = held_tiles(owners, replicated, r)
        arr.reshape(T, -1)[sel] = src[sel]
    return per_rank


# ------------------------------------------------------------------------------------------------------------ symmetric heap
class SymmetricBuffer:
    """A tensor allocated at the same size on every rank of ``group`` with peer-mapped pointers (+ multicast address if NVLS)."""

    def __init__(self, tensor, peer_ptrs, multicast_ptr=0, keepalive=None):
        self.tensor, self.peer_ptrs, self.multicast_ptr, self._keep = tensor, list(peer_ptrs), int(multicast_ptr or 0), keepalive


class SymmetricHeap:
    """Allocation + handle exchange.  Preferred backend: ``torch.distributed._symmetric_memory`` (CUDA VMM + fabric/posix handles,
    multicast objects when the driver supports NVLS).  Fallback: legacy CUDA IPC handles exchanged over the store (P2P only)."""

    def __init__(self, topo: Topology, device):
        self.topo, self.device = topo, device
        self.backend = "local" if topo.world == 1 else None
        self._groups = {}

    def _group(self, ranks):
        import torch.distributed as dist
        key = tuple(ranks)
        if key == tuple(range(self.topo.world)):
            return dist.group.WORLD
        if key not in self._groups:
            # new_group is collective over the world: create every party group in the same order on all ranks
            for g in range(self.topo.num_parties):
                pr = tuple(self.topo.party_ranks(g))
                if pr not in self._groups:
                    self._groups[pr] = dist.new_group(list(pr))
        return self._groups[key]

    def alloc(self, numel, dtype, ranks=None, zero=True):
        """Collective over ``ranks`` (default: world).  Returns SymmetricBuffer whose peer_ptrs are indexed by GLOBAL rank (0 if absent)."""
        topo = self.topo
        if topo.world == 1:
            t = torch.zeros(numel, dtype=dtype, device=self.device) if zero else torch.empty(numel, dtype=dtype, device=self.device)
            return SymmetricBuffer(t, [t.data_ptr()] + [0] * (MAX_RANKS - 1))
        import torch.distributed as dist
        ranks = list(range(topo.world)) if ranks is None else list(ranks)
        if ranks == [topo.rank]:      # a party of one: nothing to map (and symmetric-memory multicast cannot be exported for one rank)
            t = torch.zeros(numel, dtype=dtype, device=self.device)
            ptrs = [0] * MAX_RANKS
            ptrs[topo.rank] = t.data_ptr()
            return SymmetricBuffer(t, ptrs)
        group = self._group(ranks)
        ptrs = [0] * MAX_RANKS
        if self.backend in (None, "symm_mem"):
            try:
                import torch.distributed._symmetric_memory as symm
                t = symm.empty(numel, dtype=dtype, device=self.device)
                hdl = symm.rendezvous(t, group=group)
                if zero:
                    t.zero_()
                for i, r in enumerate(ranks):
                    ptrs[r] = int(hdl.buffer_ptrs[i])
                mc = int(getattr(hdl, "multicast_ptr", 0) or 0)
                self.backend = "symm_mem"
                torch.cuda.synchronize(); dist.barrier(group=group)
                return SymmetricBuffer(t, ptrs, mc, hdl)
            except Exception as e:  # pragma: no cover - depends on driver support
                if self.backend == "symm_mem":
                    raise
                if os.environ.get("GEOMX_VERBOSE"):
                    print("[geomx] symmetric_memory unavailable (%r); falling back to CUDA IPC" % (e,))
                self.backend = "cuda_ipc"
        # legacy CUDA IPC: cudaMalloc'd storage shared through torch's IPC handle
        t = torch.zeros(numel, dtype=dtype, device=self.device)
        handle = t.untyped_storage()._share_cuda_()
        gathered = [None] * len(ranks)
        dist.all_gather_object(gathered, handle, group=group)
        keep = []
        me = ranks.index(topo.rank)
        for i, r in enumerate(ranks):
            if i == me:
                ptrs[r] = t.data_ptr()
                continue
            h = gathered[i]
            st = torch.UntypedStorage._new_shared_cuda(*h)
            peer = torch.empty(0, dtype=dtype, device=st.device).set_(st)
            keep.append(peer)
            ptrs[r] = peer.data_ptr() + 0
        torch.cuda.synchronize(); dist.barrier(group=group)
        return SymmetricBuffer(t, ptrs, 0, keep)


# ------------------------------------------------------------------------------------------------------------ kernel parameter block
_OptHyperF = OptHyper      # the optimizer block inside _FabricParams (one definition, in ops/_native_api.py)


class _FabricParams(ctypes.Structure):
    _fields_ = [
        ("world", ctypes.c_int), ("rank", ctypes.c_int), ("party_size", ctypes.c_int), ("num_parties", ctypes.c_int),
        ("party", ctypes.c_int), ("local", ctypes.c_int), ("num_gs", ctypes.c_int), ("gs_rank", ctypes.c_int * MAX_RANKS),
        ("grad", ctypes.c_void_p * MAX_RANKS), ("param", ctypes.c_void_p * MAX_RANKS), ("stage", ctypes.c_void_p * MAX_RANKS),
        ("flags", ctypes.c_void_p * MAX_RANKS),
        ("grad_mc", ctypes.c_void_p), ("param_mc", ctypes.c_void_p), ("w", ctypes.c_void_p), ("s0", ctypes.c_void_p),
        ("s1", ctypes.c_void_p), ("lock_and_steps", ctypes.c_void_p),
        ("n", ctypes.c_longlong), ("tiles", ctypes.c_int), ("num_keys", ctypes.c_int),
        ("tile_key", ctypes.c_void_p), ("key_tiles", ctypes.c_void_p), ("tile_owner", ctypes.c_void_p), ("tile_active", ctypes.c_void_p),
        ("tile_mult", ctypes.c_void_p), ("key_done", ctypes.c_void_p), ("state", ctypes.c_void_p),
        ("h", _OptHyperF), ("push_scale", ctypes.c_float), ("defer_pull_wait", ctypes.c_int), ("param_ready_off", ctypes.c_int),
        ("ready_off", ctypes.c_int), ("arrived_off", ctypes.c_int), ("zero_grad", ctypes.c_int),
        ("ll_a", ctypes.c_void_p * MAX_RANKS), ("ll_b", ctypes.c_void_p * MAX_RANKS), ("ll_c", ctypes.c_void_p * MAX_RANKS),
        ("ll_c_mc", ctypes.c_void_p),
        ("tile_fmt", ctypes.c_void_p), ("bsc_u", ctypes.c_void_p), ("bsc_v", ctypes.c_void_p), ("bsc_k", ctypes.c_int),
        ("tile_order", ctypes.c_void_p), ("dgt_contrib", ctypes.c_void_p), ("dgt_alpha", ctypes.c_float),
        ("ll_party_mode", ctypes.c_int),
        ("ll_d", ctypes.c_void_p * MAX_RANKS), ("ll_d_mc", ctypes.c_void_p), ("ll_e", ctypes.c_void_p * MAX_RANKS), ("ll_e_mc", ctypes.c_void_p),
        ("direct_replicate", ctypes.c_int), ("channel_id", ctypes.c_int), ("list_tiles", ctypes.c_int), ("tile_list", ctypes.c_void_p),
    ]


# the block is passed by value as a kernel parameter, and CUDA limits those to 4 KB.  hips_ll.cuh static_asserts the same size and offset.
FABRIC_PARAMS_BYTES, FABRIC_PARAMS_H_OFFSET = 1672, 728
assert ctypes.sizeof(_FabricParams) == FABRIC_PARAMS_BYTES <= 4096 and _FabricParams.h.offset == FABRIC_PARAMS_H_OFFSET


def dgt_num_important(sorted_contrib, k, adaptive=False, k_min=0.2):
    """Size of the important set given the contributions in DESCENDING order.  Fixed mode: ``round(k * n)`` tiles (reference semantics of
    ``DMLC_K``, kv_app.h:987-994).  Adaptive mode: the shortest prefix whose contributions sum to ``k`` of the total, at least
    ``k_min * n`` tiles."""
    n = int(sorted_contrib.numel())
    if n == 0:
        return 0
    if not adaptive:
        return max(1, int(round(k * n)))
    c = sorted_contrib.double()           # the total in the precision of the running sum: a tile below fp32 resolution still counts
    total = float(c.sum())
    if total <= 0.0:
        return max(1, int(round(k_min * n)))
    cum = torch.cumsum(c, 0) / total
    need = int(torch.searchsorted(cum, torch.tensor([k - 1e-12], dtype=cum.dtype, device=cum.device))[0]) + 1
    return max(1, min(n, max(need, int(round(k_min * n)))))


class HipsFabric:
    """Owns the symmetric arenas of one model replica and launches the fused HiPS kernels.

    ``layout``: :class:`ArenaLayout`; ``opt_spec``: ``Optimizer.spec()`` dict or None (server stores aggregated gradients)."""

    def __init__(self, layout: ArenaLayout, topo: Topology | None = None, device=None, opt_spec=None, use_multicast=True, loopback=False):
        """``loopback``: with a single rank, still run the multi-rank packet kernels (push to the own slot, poll it back) instead of the
        collapsed arena-optimizer path — a one-GPU exercise of exactly the code that runs between GPUs (smoke tests, launch census)."""
        native.require()
        self.layout = layout
        self.topo = topo or Topology.from_env()
        self.device = device or torch.device("cuda", torch.cuda.current_device())
        t = self.topo
        self.heap = SymmetricHeap(t, self.device)
        n, T, K, P = layout.total, layout.num_tiles, len(layout.slots), t.num_parties
        self.n, self.tiles, self.num_keys = n, T, K
        # --- symmetric buffers ------------------------------------------------------------------------------------
        self.param = self.heap.alloc(n, torch.float32)                                  # world: pull target + forward operand
        self.grad = self.heap.alloc(n, torch.float32, ranks=t.party_ranks())            # party: local-tier reduction source
        self.stage = self.heap.alloc(P * n, torch.float32)                              # world: per-party aggregates on global owners
        # flag pad layout (uint32 words): one region per kernel family so that each keeps its own epoch
        off = 0
        self.off = {}
        for name, size in (("fsa_ready", MAX_RANKS), ("fsa_arrived", P * T), ("fsa_param_ready", K),
                           ("async_ready", MAX_RANKS), ("async_param_ready", K), ("async_lock", T), ("async_step", T),
                           ("par_ready", MAX_RANKS), ("par_done", 4), ("barrier", 4)):
            self.off[name] = off
            off += (size + 15) // 16 * 16
        self.flags = self.heap.alloc(off, torch.int32)
        # LL protocol (latency-bound arenas): {value, epoch} packet buffers — 2x the arena per sender slot, no fences on the critical path.
        # Bandwidth-bound arenas (> GEOMX_LL_MAX_BYTES) keep the flag ("bulk") protocol whose fences amortise over many tiles per CTA.
        ll_max = getenv_int("GEOMX_LL_MAX_BYTES", 64 << 20)
        proto = os.environ.get("GEOMX_FABRIC_PROTOCOL", "auto")
        self.loopback = bool(loopback) and t.world == 1
        self.protocol = "bulk" if ((t.world == 1 and not self.loopback) or proto == "bulk" or (proto == "auto" and 4 * n > ll_max)) else "ll"
        if self.protocol == "ll":
            self.ll_a = self.heap.alloc(t.party_size * 2 * n, torch.float32)
            self.ll_b = self.heap.alloc(P * 2 * n, torch.float32)
            self.ll_c = self.heap.alloc(2 * n, torch.float32)
        else:
            self.ll_a = self.ll_b = self.ll_c = None
        # direct protocol (hips_fsa_direct_kernel): per-sender gradient slots + a result buffer; world x the arena, so only for small arenas
        self.ll_d = self.ll_e = None
        if self.protocol == "ll" and os.environ.get("GEOMX_FABRIC_DIRECT", "1") == "1" and 8 * n * t.world <= getenv_int("GEOMX_DIRECT_MAX_BYTES", 256 << 20):
            self.ll_d = self.heap.alloc(t.world * 2 * n, torch.float32)
            self.ll_e = self.heap.alloc(2 * n, torch.float32)
        self.channels = {}            # name -> dict(id, mask, replicate, grid)
        # --- global-owner state (private HBM) ---------------------------------------------------------------------
        self.w = torch.zeros(n, dtype=torch.float32, device=self.device)
        self.s0 = torch.zeros(n, dtype=torch.float32, device=self.device)
        self.s1 = torch.zeros(n, dtype=torch.float32, device=self.device)
        dev = self.device
        self.tile_key = torch.from_numpy(layout.tile_key()).to(dev)
        self.key_tiles = torch.from_numpy(layout.key_tiles()).to(dev)
        self.tile_owner_np = global_tile_owners(t, layout, self.protocol, getenv_int("MXNET_KVSTORE_BIGARRAY_BOUND", 1000000))
        self.tile_owner = torch.from_numpy(self.tile_owner_np).to(dev)
        self.tile_mult = torch.from_numpy(layout.tile_mult()).to(dev)
        self.tile_active = torch.ones(T, dtype=torch.uint8, device=dev)
        self.key_done = torch.zeros(K, dtype=torch.int32, device=dev)
        self.state = {k: torch.zeros(64, dtype=torch.int32, device=dev) for k in ("fsa", "async", "party", "barrier")}
        self.use_multicast = use_multicast and bool(self.param.multicast_ptr) and os.environ.get("GEOMX_NO_MULTICAST", "0") != "1"
        self.opt_spec = None
        self.push_scale = 1.0
        self.tile_fmt = None            # per-tile wire format (LL protocol): 0 fp32, 1 fp16, 2 Bi-Sparse between the tiers, 3 block-scaled fp8
        self.tile_order = self.dgt_contrib = None     # DGT on the fabric (enable_dgt)
        self.dgt_k, self.dgt_alpha, self._dgt_base_fmt = 1.0, 0.3, None
        self.bsc_u = self.bsc_v = None
        self.bsc_k = 0
        # one CTA per tile while the launch stays co-resident (the kernels spin on each other); grid-stride beyond that.  The LL kernel's
        # phases are one round each when grid >= tiles; the bulk protocol keeps <= 132 CTAs (its per-tile fences contend at higher counts)
        self.grid = max(1, min(T, int(native.require().gx_hips_max_grid()) if self.protocol == "ll" else 132))
        if t.world == 1 and not self.loopback:
            self.grid = max(1, min(T, 4096))     # nothing spins on a single rank: one tile per CTA, no co-residency requirement
        self._params_cache = {}
        self._peer_tables = {}
        self.set_optimizer(opt_spec)

    # -- views ----------------------------------------------------------------------------------------------------------
    def param_view(self, i): return self.layout.view(self.param.tensor, i)
    def grad_view(self, i): return self.layout.view(self.grad.tensor, i)

    def set_optimizer(self, spec):
        self.opt_spec = spec
        self._params_cache.clear()

    FMT_F32, FMT_F16, FMT_BSC, FMT_F8 = 0, 1, 2, 3

    def set_wire_formats(self, key_formats=None, bsc_threshold=0.01):
        """Per-key wire format of the fused step: ``{key_index: 'fp32'|'fp16'|'bsc'}`` (missing keys: fp32), or None for all-fp32.

        fp16 = the reference's FP16 / MPQ transports (script-level ``astype('float16')``, examples/cnn_fp16.py:115, cnn_mpq.py:122) fused
        into the push kernel: gradients and parameters cross NVLink as halves, master weights stay fp32 on the global owner.
        fp8  = block-scaled fp8 gradients (e4m3, one fp32 scale per 128 values, 8 values per packet) on both gradient hops; the parameters of
        such keys return as fp16.
        bsc  = Bi-Sparse between the tiers (gradient_compression.cc:191-336), re-designed per 1024-value tile: the party owner keeps the
        momentum-corrected residual, sends the ``k = floor(1024*threshold)`` largest entries as (value, index) packets; without a server
        optimizer the aggregate returns sparse as well (BSCPullCompress)."""
        self._params_cache.clear()
        for ch in self.channels.values():
            ch.pop("direct_ok", None)
        if not key_formats:
            self.tile_fmt = None
            return
        if self.protocol != "ll":
            raise RuntimeError("wire formats need the LL protocol (world > 1 and arena <= GEOMX_LL_MAX_BYTES)")
        code = {"fp32": 0, "fp16": 1, "bsc": 2, "fp8": 3}
        fmt = np.zeros(self.tiles, dtype=np.uint8)
        for i, f in key_formats.items():
            sl = self.layout.slots[i]
            fmt[sl.offset // 1024: sl.offset // 1024 + sl.tiles] = code[f]
        if (fmt == 2).any():
            k = max(1, int(1024 * float(bsc_threshold)))
            if k * self.topo.num_parties > 512:
                raise RuntimeError("Bi-Sparse threshold too large for the packet buffers: floor(1024*thr)*num_parties must be <= 512")
            self.bsc_k = k
            if self.bsc_u is None:
                self.bsc_u = torch.zeros(self.n, dtype=torch.float32, device=self.device)
                self.bsc_v = torch.zeros(self.n, dtype=torch.float32, device=self.device)
        new = torch.from_numpy(fmt).to(self.device)
        if self.tile_fmt is not None and self.tile_fmt.shape == new.shape:
            self.tile_fmt.copy_(new)              # in place: a captured CUDA graph holds this pointer
        else:
            self.tile_fmt = new

    # -- DGT on the fabric ---------------------------------------------------------------------------------------------------------
    def enable_dgt(self, k=None, alpha=None):
        """Differential gradient transmission mapped onto NVSwitch (reference: kv_app.h:842-1022, van.cc:707-824): the global owner of a
        tile keeps the EMA of its mean |aggregated gradient| (in-kernel); ``dgt_rerank()`` turns these contributions into (a) the order in
        which the fused kernel serves the tiles — important first — and (b) the wire precision: the top ``k`` fraction keeps its format, the
        rest travels as block-scaled fp8 (the reference's 4-bit encode of unimportant blocks, ENABLE_DGT=3)."""
        if self.protocol != "ll":
            raise RuntimeError("DGT on the fabric needs the LL protocol")
        self.dgt_k = float(os.environ.get("DMLC_K", 0.8)) if k is None else float(k)
        # ADAPTIVE_K_FLAG=1 (parsed but unused by the reference, kv_app.h:844-848): K is read as a share of the total CONTRIBUTION instead of
        # a share of the tiles — the important set is the shortest prefix of the ranking that carries K of the contribution mass, never
        # smaller than DMLC_K_MIN of the tiles.  Concentrated gradients then send few tiles at full precision, flat ones many.
        self.dgt_adaptive = bool(int(os.environ.get("ADAPTIVE_K_FLAG", 0)))
        self.dgt_k_min = float(os.environ.get("DMLC_K_MIN", 0.2))
        self.dgt_alpha = float(os.environ.get("DGT_CONTRIBUTION_ALPHA", 0.3)) if alpha is None else float(alpha)
        if self.dgt_contrib is None:
            self.dgt_contrib = torch.zeros(self.tiles, dtype=torch.float32, device=self.device)
            self.tile_order = torch.arange(self.tiles, dtype=torch.int32, device=self.device)
        if self.tile_fmt is None:
            self.tile_fmt = torch.zeros(self.tiles, dtype=torch.uint8, device=self.device)
        self._dgt_base_fmt = self.tile_fmt.clone()
        self._params_cache.clear()

    def dgt_rerank(self):
        """Collective (all ranks): gather every owner's contributions, re-rank the tiles, demote the unimportant ones to fp8.  Off the hot
        path (call every few dozen steps); everything is updated in place so captured graphs pick the new order up."""
        assert self.dgt_contrib is not None, "enable_dgt() first"
        c = self.dgt_contrib.clone()
        owned = torch.from_numpy(self.tile_owner_np == self.topo.rank).to(self.device)
        c = torch.where(owned, c, torch.zeros_like(c))
        if self.topo.world > 1:
            import torch.distributed as dist
            dist.all_reduce(c)
        order = torch.argsort(c, descending=True, stable=True)
        self.tile_order.copy_(order.to(torch.int32))
        n_imp = dgt_num_important(c[order], self.dgt_k, getattr(self, "dgt_adaptive", False), getattr(self, "dgt_k_min", 0.2))
        self.dgt_num_important = n_imp
        fmt = self._dgt_base_fmt.clone()
        unimportant = order[n_imp:]
        dense = (fmt[unimportant] == 0) | (fmt[unimportant] == 1)          # Bi-Sparse tiles keep their own format
        fmt[unimportant[dense]] = 3
        self.tile_fmt.copy_(fmt)
        return c

    def set_push_scale(self, s):
        self.push_scale = float(s)
        self._params_cache.clear()

    def load_master_from_param(self):
        """Global owners adopt the (already broadcast) parameter arena as master weights — the `init` handshake."""
        self.w.copy_(self.param.tensor)
        self.init_dcasgd_previous_weight()

    def init_dcasgd_previous_weight(self):
        """DCASGD's previous weight (state slot ``s1``) starts as the current master weight, as the reference's ``create_state`` makes it
        (``(mom, weight.copy())``); a zero start would add ``lamda * g^2 * w`` to the first update."""
        if self.opt_spec is not None and OPT_KINDS[self.opt_spec["name"]].s1_is_weight:
            self.s1.copy_(self.w)

    # -- parameter block ------------------------------------------------------------------------------------------------
    def _hyper(self):
        # the schedule, if any, is evaluated by the kernels at their step count; without one the lr is constant
        return pack_hyper(self.opt_spec)

    def _block(self, channel, masked=False, zero_grad=False):
        if channel in self.channels:
            return self._channel_block(channel, zero_grad)
        key = (channel, masked, zero_grad)
        if key in self._params_cache:
            return self._params_cache[key]
        t = self.topo
        p = _FabricParams()
        p.world, p.rank, p.party_size, p.num_parties, p.party, p.local = t.world, t.rank, t.party_size, t.num_parties, t.party, t.local
        p.num_gs = t.num_gs
        for i, r in enumerate(t.gs_ranks):
            p.gs_rank[i] = r
        for r in range(MAX_RANKS):
            p.grad[r] = self.grad.peer_ptrs[r] or None
            p.param[r] = self.param.peer_ptrs[r] or None
            p.stage[r] = self.stage.peer_ptrs[r] or None
            p.flags[r] = self.flags.peer_ptrs[r] or None
            if self.ll_a is not None:
                p.ll_a[r] = self.ll_a.peer_ptrs[r] or None
                p.ll_b[r] = self.ll_b.peer_ptrs[r] or None
                p.ll_c[r] = self.ll_c.peer_ptrs[r] or None
            if self.ll_d is not None:
                p.ll_d[r] = self.ll_d.peer_ptrs[r] or None
                p.ll_e[r] = self.ll_e.peer_ptrs[r] or None
        p.tile_order = self.tile_order.data_ptr() if self.tile_order is not None else None
        p.dgt_contrib = self.dgt_contrib.data_ptr() if self.dgt_contrib is not None else None
        p.dgt_alpha = float(self.dgt_alpha)
        mc_ok = self.use_multicast and os.environ.get("GEOMX_LL_MULTICAST", "1") == "1"
        p.ll_d_mc = (self.ll_d.multicast_ptr or None) if (self.ll_d is not None and mc_ok) else None
        p.ll_e_mc = (self.ll_e.multicast_ptr or None) if (self.ll_e is not None and mc_ok) else None
        p.ll_c_mc = (self.ll_c.multicast_ptr or None) if (self.ll_a is not None and self.use_multicast and os.environ.get("GEOMX_LL_MULTICAST", "1") == "1") else None
        p.tile_fmt = self.tile_fmt.data_ptr() if self.tile_fmt is not None else None
        p.bsc_u = self.bsc_u.data_ptr() if self.bsc_u is not None else None
        p.bsc_v = self.bsc_v.data_ptr() if self.bsc_v is not None else None
        p.bsc_k = int(self.bsc_k)
        p.grad_mc = (self.grad.multicast_ptr or None) if self.use_multicast else None
        p.param_mc = (self.param.multicast_ptr or None) if self.use_multicast else None
        p.w, p.s0, p.s1 = self.w.data_ptr(), self.s0.data_ptr(), self.s1.data_ptr()
        p.n, p.tiles, p.num_keys = self.n, self.tiles, self.num_keys
        p.tile_key, p.key_tiles, p.tile_owner = self.tile_key.data_ptr(), self.key_tiles.data_ptr(), self.tile_owner.data_ptr()
        p.tile_active = self.tile_active.data_ptr() if masked else None
        p.tile_mult = self.tile_mult.data_ptr()
        p.key_done = self.key_done.data_ptr()
        p.state = self.state[channel].data_ptr()
        p.h = self._hyper()
        p.push_scale = self.push_scale
        p.defer_pull_wait = 0
        p.zero_grad = int(zero_grad)
        pre = {"fsa": "fsa", "async": "async", "party": "par"}[channel]
        p.ready_off = self.off[pre + "_ready"]
        p.arrived_off = self.off["fsa_arrived"]
        p.param_ready_off = self.off.get(pre + "_param_ready", self.off["fsa_param_ready"])
        assert ctypes.sizeof(p) == native.require().gx_fabric_params_size(), "FabricParams layout mismatch"
        self._params_cache[key] = p
        return p

    # -- channels (direct protocol) ---------------------------------------------------------------------------------------------
    def add_channel(self, name, key_indices, replicate=False, grid=None):
        """Declare a key group that is exchanged by its own launch (``channel_step(name)``), typically as soon as the backward pass has
        produced that group's gradients.  ``replicate=True`` selects the one-hop mode (every rank applies the update to its own replica of the
        server state — for the small keys whose exchange cannot overlap compute); otherwise the two-hop sharded mode.  Each channel has its own
        epoch / optimizer-step state, so channels of one step may run concurrently on different streams."""
        if name in self.channels or name in self.state:
            raise ValueError("channel %r exists" % name)
        if len(self.channels) >= 7:
            raise ValueError("at most 7 channels")
        mask = np.zeros(self.tiles, dtype=np.uint8)
        for i in key_indices:
            sl = self.layout.slots[i]
            mask[sl.offset // 1024: sl.offset // 1024 + sl.tiles] = 1
        active = int(mask.sum())
        self.state[name] = torch.zeros(64, dtype=torch.int32, device=self.device)
        self.state[name][2] = int(self.state["fsa"][2].item())        # optimizer step t continues
        self.channels[name] = {"id": len(self.channels) + 1, "mask": torch.from_numpy(mask).to(self.device), "replicate": bool(replicate),
                               "keys": list(key_indices), "tiles": active,
                               "list": torch.from_numpy(np.flatnonzero(mask).astype(np.int32)).to(self.device),
                               "grid": int(grid) if grid else max(1, min(active, int(native.require().gx_hips_max_grid()) // 2))}
        self._params_cache.clear()
        return self.channels[name]

    def _channel_formats_direct_ok(self, ch):
        """Bi-Sparse needs the party aggregate (3-hop kernel).  Cached per channel: the check reads device memory, which is not allowed while a
        CUDA graph is being captured (the first, eager warm-up step fills the cache; set_wire_formats invalidates it)."""
        if "direct_ok" not in ch:
            ch["direct_ok"] = self.tile_fmt is None or not bool(((self.tile_fmt == 2) & (ch["mask"] != 0)).any().item())
        return ch["direct_ok"]

    def _channel_block(self, name, zero_grad):
        key = ("channel", name, zero_grad)
        if key in self._params_cache:
            return self._params_cache[key]
        ch = self.channels[name]
        base = self._block("fsa", False, zero_grad)
        p = _FabricParams.from_buffer_copy(base)
        p.tile_active = ch["mask"].data_ptr()
        p.tile_list, p.list_tiles = ch["list"].data_ptr(), ch["tiles"]
        p.state = self.state[name].data_ptr()
        p.direct_replicate = int(ch["replicate"])
        if ch["replicate"] and os.environ.get("GEOMX_REPL_MULTICAST", "1") != "1":
            p.ll_d_mc = None      # one-hop mode with unicast stores: own packets stay local instead of making the round trip through the switch
        p.channel_id = ch["id"]
        self._params_cache[key] = p
        return p

    def channel_step(self, name, zero_grad=False):
        """Exchange one channel's keys: push -> (both server tiers on the applying rank) -> optimizer -> pull, one launch."""
        ch = self.channels[name]
        p = self._channel_block(name, zero_grad)
        lib = native.require()
        if self.topo.world == 1 and not self.loopback:
            rc = lib.gx_hips_fsa_step(ctypes.byref(p), ch["tiles"], self._stream())       # single rank: the fused arena optimizer, a CTA per tile
        elif self.ll_d is not None and self._channel_formats_direct_ok(ch):
            rc = lib.gx_hips_fsa_direct_step(ctypes.byref(p), ch["grid"], self._stream())
        elif self.protocol == "ll":
            rc = lib.gx_hips_fsa_ll_step(ctypes.byref(p), self.grid, self._stream())      # 3-hop hierarchy walk (Bi-Sparse between the tiers)
        else:
            rc = lib.gx_hips_fsa_step(ctypes.byref(p), self.grid, self._stream())
        native.launch_count += 1
        if rc:
            raise RuntimeError("channel_step(%s) failed rc=%d" % (name, rc))

    def channel_fused_args(self, name, zero_grad=False):
        """For compute kernels that perform a replicated channel's exchange in their own tail (cnn_bwd_exchange_kernel): the channel's
        parameter block, its tile list and tile count — or ``None`` when the channel needs a launch of its own (sharded mode, Bi-Sparse
        tiles, DGT bookkeeping, or a multi-rank job without the direct-protocol buffers).  Whether a step uses a capable channel this way
        is the step's choice."""
        ch = self.channels[name]
        single = self.topo.world == 1 and not self.loopback
        if not ch["replicate"] or self.dgt_contrib is not None:
            return None
        if not single and (self.ll_d is None or not self._channel_formats_direct_ok(ch)):
            return None
        return self._channel_block(name, zero_grad), ch["list"], ch["tiles"]

    @property
    def opt_step(self):
        """Optimizer step count t (identical on every channel that has run the same number of rounds)."""
        names = list(self.channels) or ["fsa"]
        return max(int(self.state[n][2].item()) for n in names)

    def set_opt_step(self, t):
        for n in ["fsa"] + list(self.channels):
            self.state[n][2] = int(t)

    # -- checkpoints ----------------------------------------------------------------------------------------------------
    def replicated_tiles(self):
        """bool per tile: every rank keeps its own replica of the tile's server state (a single rank, or a one-hop replicated channel)."""
        if self.topo.world == 1:
            return np.ones(self.tiles, dtype=bool)
        rep = np.zeros(self.tiles, dtype=bool)
        for ch in self.channels.values():
            if ch["replicate"]:
                rep |= self._key_tile_mask(ch["keys"])
        return rep

    def _key_tile_mask(self, keys):
        mask = np.zeros(self.tiles, dtype=bool)
        for i in keys:
            sl = self.layout.slots[i]
            mask[sl.offset // 1024: sl.offset // 1024 + sl.tiles] = True
        return mask

    def tile_step_words(self):
        """Per tile, the state whose optimizer step word counts the tile's dist_sync updates: its channel's, else the one exchange's."""
        words = np.array(["fsa"] * self.tiles, dtype=object)
        for name, ch in self.channels.items():
            words[self._key_tile_mask(ch["keys"])] = name
        return words

    def gather_ranks(self, t):
        """Host (numpy) copies of the local tensor ``t`` of every rank, in rank order (collective over the world)."""
        t = t.contiguous()
        if self.topo.world == 1:
            return [t.cpu().numpy()]
        import torch.distributed as dist
        out = [torch.empty_like(t) for _ in range(self.topo.world)]
        dist.all_gather(out, t)
        return [o.cpu().numpy() for o in out]

    def export_state(self, async_counts=False):
        """Collective over the world: the server state as full host arrays in arena order, whoever holds each tile (the owner of a sharded
        tile, rank 0's replica of a replicated one).  ``w`` / ``s0`` / ``s1``: float32 [n]; ``step``: int32 [tiles], the update count of
        each tile — the step word of its exchange (dist_sync), or with ``async_counts`` the one-sided update's per-tile count.  With DGT
        ``dgt_contrib`` (from the owners, as ``dgt_rerank`` reads it), ``tile_order`` and ``tile_fmt``; with Bi-Sparse the party owners'
        residuals ``bsc_u`` / ``bsc_v`` of every rank, float32 [world, n].  Protocol state (epochs, counters, flags) is not part of it."""
        owners, rep = self.tile_owner_np, self.replicated_tiles()
        out = {k: gather_tile_state(self.gather_ranks(getattr(self, k)), owners, rep) for k in ("w", "s0", "s1")}
        if async_counts:
            a = self.off["async_step"]
            out["step"] = gather_tile_state(self.gather_ranks(self.flags.tensor[a:a + self.tiles]), owners)
        else:
            words = self.tile_step_words()
            out["step"] = np.array([int(self.state[n][2].item()) for n in words], dtype=np.int32)
        if self.dgt_contrib is not None:
            out["dgt_contrib"] = gather_tile_state(self.gather_ranks(self.dgt_contrib), owners)
            out["tile_order"] = self.tile_order.cpu().numpy()
            out["tile_fmt"] = self.tile_fmt.cpu().numpy()
        if self.bsc_u is not None:
            out["bsc_u"] = np.stack(self.gather_ranks(self.bsc_u))
            out["bsc_v"] = np.stack(self.gather_ranks(self.bsc_v))
        return out

    def import_state(self, state, async_counts=False):
        """Inverse of :meth:`export_state`, on every rank with the same ``state``: each rank copies the tiles it holds into its buffers in
        place (captured graphs stay valid); the optimizer step words are set, the protocol state is left as it is.  A tile's step word is
        shared by its channel, so every tile of a channel must carry the same count (``ValueError`` otherwise, before anything is written)."""
        owners, rep, me, T = self.tile_owner_np, self.replicated_tiles(), self.topo.rank, self.tiles
        step = np.asarray(state.get("step", np.zeros(T, dtype=np.int32)))
        words = None
        if not async_counts:
            words = {}
            for n, w in zip(self.tile_step_words(), step.tolist()):
                if words.setdefault(n, w) != w:
                    raise ValueError("step: the keys exchanged together (%s) were saved with different update counts" % n)

        def put(dev, full, replicated):
            local = dev.cpu().numpy()
            scatter_tile_state(np.asarray(full), {me: local}, owners, replicated)
            dev.copy_(torch.from_numpy(local))

        for k in ("w", "s0", "s1"):
            if k in state:
                put(getattr(self, k), state[k], rep)
        if async_counts:
            a = self.off["async_step"]
            put(self.flags.tensor[a:a + T], step, None)
        elif "step" in state:
            for n, w in words.items():
                self.state[n][2] = w
            if "fsa" not in words:
                self.state["fsa"][2] = int(step.max())
        if self.dgt_contrib is not None:
            put(self.dgt_contrib, state["dgt_contrib"], None)
            self.tile_order.copy_(torch.from_numpy(np.asarray(state["tile_order"])))
            self.tile_fmt.copy_(torch.from_numpy(np.asarray(state["tile_fmt"])))
        if self.bsc_u is not None:
            self.bsc_u.copy_(torch.from_numpy(np.asarray(state["bsc_u"])[me]))
            self.bsc_v.copy_(torch.from_numpy(np.asarray(state["bsc_v"])[me]))

    def _peer_table(self, name, ptrs):
        if name not in self._peer_tables:
            arr = np.array([int(x or 0) for x in ptrs], dtype=np.int64)
            self._peer_tables[name] = torch.from_numpy(arr).to(self.device)
        return self._peer_tables[name]

    def _stream(self):
        return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)

    # -- kernels --------------------------------------------------------------------------------------------------------
    def fsa_step(self, masked=False, zero_grad=False):
        """dist_sync: party reduce -> global reduce + optimizer -> broadcast (one launch); optionally clears the gradient arena for the next step."""
        p = self._block("fsa", masked, zero_grad)
        lib = native.require()
        if self.protocol == "ll":
            rc = lib.gx_hips_fsa_ll_step(ctypes.byref(p), self.grid, self._stream())
        else:
            rc = lib.gx_hips_fsa_step(ctypes.byref(p), self.grid, self._stream())
        native.launch_count += 1
        if rc:
            raise RuntimeError("gx_hips_fsa_step failed rc=%d" % rc)

    def check_protocol_errors(self):
        """True if a bounded LL poll ever gave up (a protocol bug or a dead peer) — state word 5 of every dist_sync channel."""
        return any(bool(int(self.state[n][5].item())) for n in ["fsa"] + list(self.channels))

    def async_step(self):
        """dist_async (MixedSync): one-sided update of the global owner's HBM under per-tile locks."""
        p = self._block("async")
        if "w_peer" not in self._peer_tables and self.topo.world > 1:
            self._exchange_state_peers()
        wp = self._peer_table("w_peer", [self.w.data_ptr()] + [0] * (MAX_RANKS - 1))
        s0 = self._peer_table("s0_peer", [self.s0.data_ptr()] + [0] * (MAX_RANKS - 1))
        s1 = self._peer_table("s1_peer", [self.s1.data_ptr()] + [0] * (MAX_RANKS - 1))
        rc = native.require().gx_hips_async_step(ctypes.byref(p), ctypes.c_void_p(wp.data_ptr()), ctypes.c_void_p(s0.data_ptr()),
                                                 ctypes.c_void_p(s1.data_ptr()), self.off["async_lock"], self.off["async_step"], self.grid, self._stream())
        native.launch_count += 1
        if rc:
            raise RuntimeError("gx_hips_async_step failed rc=%d" % rc)

    def _exchange_state_peers(self):
        """Async mode needs the global owners' master/state arenas peer-mapped: re-home them in symmetric memory."""
        for name in ("w", "s0", "s1"):
            buf = self.heap.alloc(self.n, torch.float32)
            buf.tensor.copy_(getattr(self, name))
            setattr(self, name, buf.tensor)
            setattr(self, "_sym_" + name, buf)
            self._peer_tables[name + "_peer"] = torch.from_numpy(np.array(buf.peer_ptrs, dtype=np.int64)).to(self.device)
        self._params_cache.clear()

    def party_allreduce(self, src: SymmetricBuffer, dst: SymmetricBuffer, scale=1.0, reduce_scatter=False):
        """Local tier only (HFA local synchronisation / generic party all-reduce)."""
        if self.protocol == "ll" and src is self.grad and dst is self.param and not reduce_scatter:
            # latency-bound arenas: the LL kernel in party mode (push to the tile's party owner, sum, push to the party) — two one-way hops,
            # no fences; it shares the packet buffers and therefore the epoch counter of the dist_sync channel
            key = ("fsa-party", float(scale))
            p = self._params_cache.get(key)
            if p is None:
                base = self._block("fsa", False, False)
                p = _FabricParams.from_buffer_copy(base)
                p.ll_party_mode = 1
                p.h.kind = -1
                p.push_scale = float(scale)
                p.tile_fmt = None
                p.dgt_contrib = None
                self._params_cache[key] = p
            rc = native.require().gx_hips_fsa_ll_step(ctypes.byref(p), self.grid, self._stream())
            native.launch_count += 1
            if rc:
                raise RuntimeError("gx_hips_fsa_ll_step (party mode) failed rc=%d" % rc)
            return
        p = self._block("party")
        sp = self._peer_table("par_src_%d" % id(src), src.peer_ptrs)
        dp = self._peer_table("par_dst_%d" % id(dst), dst.peer_ptrs)
        rc = native.require().gx_hips_party_allreduce(ctypes.byref(p), ctypes.c_void_p(sp.data_ptr()), ctypes.c_void_p(dp.data_ptr()), float(scale),
                                                      1 if reduce_scatter else 0, self.off["par_done"], self.grid, self._stream())
        native.launch_count += 1
        if rc:
            raise RuntimeError("gx_hips_party_allreduce failed rc=%d" % rc)

    def barrier(self):
        """Device-side whole-world flag barrier (the two-tier HiPS barrier is one NVSwitch hop)."""
        fl = self._peer_table("flags_peer", self.flags.peer_ptrs)
        rc = native.require().gx_fabric_barrier(ctypes.c_void_p(fl.data_ptr()), self.topo.world, self.topo.rank, self.off["barrier"],
                                                ctypes.c_void_p(self.state["barrier"].data_ptr()), self._stream())
        native.launch_count += 1
        if rc:
            raise RuntimeError("gx_fabric_barrier failed rc=%d" % rc)

