"""``mx.kv.create('dist_sync' | 'dist_async')`` on the NVSwitch fabric — the per-key KVStore API over the fused HiPS kernels.

Selected by ``kvstore.dist.create_dist`` when the process was started by ``torchrun`` (``RANK``/``WORLD_SIZE``) or stand-alone without any
``DMLC_*`` parameter-server environment.  Semantics follow ``python/mxnet/kvstore.py`` + ``src/kvstore/kvstore_dist.h``:

* ``init``   — keys are registered in call order; on the first data operation the keys are laid out in ONE flat symmetric arena
               (``parallel/arena.py``), rank 0's values win (``InitImpl`` :308-322) and fp32 arrays passed to ``init`` are re-homed onto the arena
               so later pulls into them are zero-copy.
* ``push``   — queues the (summed) value into the gradient arena; ``pull`` registers its targets.  Nothing is launched until a pulled
               array is read or ``mx.nd.waitall()`` runs — then ONE ``gx_hips_fsa_step`` (or ``gx_hips_async_step``) launch serves every queued
               key; keys that were not pushed this round are masked out (``tile_active``).  When the script passes priorities
               (``priority=-idx``, examples/cnn.py:121-125) — or sets ``ENABLE_P3=1`` — the kernel walks the tiles of high-priority keys first
               (``tile_order``), which is what P3 / the engine's priority queue achieve on the TCP path.
* optimizers — the specs of SGD / Adam / DCASGD / NAG / Signum / RMSProp / AdaGrad / AdaDelta / Ftrl run natively on the global-PS shard
               inside the exchange kernel; any other ``mx.optimizer`` object
               (or one with an lr_scheduler / per-parameter multipliers) is executed by the Python updater on the aggregated gradient, identically
               on every rank — the same arithmetic the reference's server-side pickled optimizer performs (kvstore.py:452-499).
* TSEngine   — ``ENABLE_INTRA_TS`` / ``ENABLE_INTER_TS`` select an overlay for heterogeneous TCP links; NVSwitch is uniform, so they are
               rejected here instead of being silently ignored.
* roles      — ``rank`` / ``num_workers`` are party-local, ``num_all_workers`` is the world size; there is no separate master-worker process:
               ``is_master_worker`` is False everywhere and ``configures_servers`` is True on world rank 0, whose ``set_optimizer`` /
               ``set_gradient_compression`` calls are broadcast to all ranks when the arena is finalised (the reference ships them to the servers
               through ``kController`` / ``kSetGradientCompression``).
* HFA        — ``MXNET_KVSTORE_USE_HFA=1``: rounds with ``local_iters % K2 != 0`` only run the party-level all-reduce
               (``gx_hips_party_allreduce``); global rounds average the party averages (``milestone + Σ(avg_g − milestone)/P`` with identical
               milestones) through the FSA kernel without an optimizer.
"""
from __future__ import annotations

import os

import numpy as np
import torch

from ..base import MXNetError, getenv_int
from ..kvstore.base import KVStoreBase
from .arena import ArenaLayout
from .fabric import HipsFabric, Topology


def _ensure_process_group(device):
    import torch.distributed as dist
    world = getenv_int("WORLD_SIZE", 1)
    if world > 1 and not dist.is_initialized():
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        os.environ.setdefault("MASTER_PORT", "29500")
        if device.type == "cuda":
            dist.init_process_group("nccl", device_id=device)
        else:
            dist.init_process_group("gloo")
    return world


class KVStoreFabric(KVStoreBase):
    def __init__(self, kv_type="dist_sync"):
        super().__init__(kv_type)
        if not torch.cuda.is_available():
            raise MXNetError("the NVSwitch fabric KVStore needs CUDA devices; use the DMLC_* environment for the TCP parameter-server path")
        local = getenv_int("LOCAL_RANK", 0)
        torch.cuda.set_device(local)
        self._device = torch.device("cuda", local)
        _ensure_process_group(self._device)
        self._topo = Topology.from_env()
        self._sync = "async" not in kv_type
        self._keys, self._init_vals = [], {}
        self._fabric = None
        self._opt_spec = None
        self._pushed, self._pulls = set(), []
        self._hfa = getenv_int("MXNET_KVSTORE_USE_HFA", 0) != 0
        self._hfa_k2 = max(1, getenv_int("MXNET_KVSTORE_HFA_K2", 1))
        self._local_iters = 0
        self._key_index = {}
        self._fp16_keys, self._wire_formats = set(), {}
        self._host_optimizer, self._host_updater, self._host_w = None, None, None
        self._priorities_seen = getenv_int("ENABLE_P3", 0) != 0        # P3 = priority-ordered propagation: on the fabric, priority tile order
        self._order_sig = None
        if (getenv_int("ENABLE_INTRA_TS", 0) or getenv_int("ENABLE_INTER_TS", 0)) and not getenv_int("GEOMX_FABRIC_IGNORE_TS", 0):
            raise MXNetError("ENABLE_INTRA_TS / ENABLE_INTER_TS (TSEngine) schedule peer-to-peer merges over heterogeneous TCP links "
                             "(3rdparty/ps-lite/src/van.cc:1174-1504); the NVSwitch fabric is uniform and reduces in one fused kernel, so the "
                             "overlay does not exist here.  Unset them, use the DMLC_* TCP launch for TSEngine, or set GEOMX_FABRIC_IGNORE_TS=1.")

    # -- identity ---------------------------------------------------------------------------------------------------------------
    @property
    def rank(self): return self._topo.local
    @property
    def num_workers(self): return self._topo.party_size
    @property
    def num_all_workers(self): return self._topo.world
    @property
    def is_master_worker(self): return False
    @property
    def configures_servers(self): return self._topo.rank == 0
    @property
    def fabric(self):
        self._finalize()
        return self._fabric

    # -- configuration (rank 0 decides, broadcast at finalize) ---------------------------------------------------------------------
    def set_optimizer(self, optimizer):
        spec = optimizer.spec()
        native_ok = spec is not None and optimizer.spec_is_static() and os.environ.get("GEOMX_PY_UPDATER", "0") != "1"
        self._optimizer = optimizer
        if native_ok:
            self._opt_spec, self._host_optimizer = spec, None
        else:
            # no (complete) native spec: the fused kernel only aggregates, the optimizer object runs on the aggregate on every rank
            if self._fabric is not None and self._host_w is None:
                raise MXNetError("switching to a Python-executed optimizer needs set_optimizer before the first push/pull")
            self._opt_spec, self._host_optimizer = None, optimizer
        if self._fabric is not None:
            self._fabric.set_optimizer(self._opt_spec)
            self._fabric.init_dcasgd_previous_weight()      # the reference's servers create the new optimizer's state from the current weight
            if self._host_optimizer is not None:
                from .. import optimizer as opt
                self._host_updater = opt.get_updater(self._host_optimizer)

    def _set_gradient_compression(self, params):
        t = params.get("type", "none")
        if t == "2bit":
            # 2-bit with error feedback (gradient_compression-inl.h:40-127): quantised by the native kernel before the push; see _push
            self._twobit_thr = float(params.get("threshold", 0.5))
            self._twobit_res = {}
        # 'bsc': the party aggregate is sparsified between the tiers inside the fused kernel (HipsFabric.set_wire_formats)
        if self._fabric is not None:
            self._apply_wire_formats()

    def _apply_wire_formats(self):
        """Map the reference's accelerators onto per-key wire formats of the fused step: Bi-Sparse for keys >= MXNET_KVSTORE_SIZE_LOWER_BOUND
        when ``set_gradient_compression({'type':'bsc'})`` was issued (kvstore_dist_server.h:841-878), fp16 for keys the script pushes as
        float16 (examples/cnn_fp16.py, cnn_mpq.py)."""
        f = self._fabric
        if f is None or f.protocol != "ll":
            return
        comp = self._compression or {}
        fmts = {}
        if comp.get("type") == "bsc":
            bound = getenv_int("MXNET_KVSTORE_SIZE_LOWER_BOUND", 200000)
            for i, (_, shape) in enumerate(self._keys):
                if int(np.prod(shape)) >= bound:
                    fmts[i] = "bsc"
        low = "fp8" if getenv_int("GEOMX_WIRE_FP8", 0) else "fp16"      # GEOMX_WIRE_FP8=1: block-scaled fp8 gradients for the keys pushed as float16
        for i in self._fp16_keys:
            fmts.setdefault(i, low)
        if fmts != self._wire_formats:
            f.set_wire_formats(fmts, float(comp.get("threshold", 0.01)))
            self._wire_formats = fmts
            if f.dgt_contrib is not None:
                f._dgt_base_fmt = f.tile_fmt.clone() if f.tile_fmt is not None else None

    # -- data ---------------------------------------------------------------------------------------------------------------------
    def _init(self, key, value):
        if self._fabric is not None:
            raise MXNetError("all keys must be initialised before the first push/pull on the fabric KVStore")
        if key in self._key_index:
            raise MXNetError("duplicate init of key %s" % key)
        self._key_index[key] = len(self._keys)
        self._keys.append((key, tuple(value.shape)))
        self._init_vals[key] = value

    def _finalize(self):
        if self._fabric is not None or getattr(self, "_finalizing", False):
            return
        self._finalizing = True
        topo = self._topo
        if topo.world > 1:
            import torch.distributed as dist
            cfg = [self._opt_spec, self._compression, self._host_optimizer] if topo.rank == 0 else [None, None, None]
            dist.broadcast_object_list(cfg, src=0)
            self._opt_spec, self._compression, self._host_optimizer = cfg
            if (self._compression or {}).get("type") == "2bit" and not hasattr(self, "_twobit_thr"):
                self._twobit_thr, self._twobit_res = float(self._compression.get("threshold", 0.5)), {}
        layout = ArenaLayout.build(self._keys)
        f = HipsFabric(layout, topo, self._device, self._opt_spec)
        for i, (key, _) in enumerate(self._keys):
            v = self._init_vals[key]
            f.param_view(i).copy_(v._data.detach().to(self._device))      # raw tensor: `_t` would run the pending-pull hook (re-entrancy)
        if topo.world > 1:
            import torch.distributed as dist
            dist.broadcast(f.param.tensor, src=0)
            torch.cuda.synchronize(); dist.barrier()
        f.load_master_from_param()
        for i, (key, _) in enumerate(self._keys):
            v = self._init_vals[key]
            if v._data.dtype == torch.float32 and v._data.is_cuda:
                had_grad = v._grad is not None
                v._data = f.param_view(i)                 # zero-copy pull target from now on
                if had_grad:
                    v._data.requires_grad_(True)
        self._init_vals = None
        self._fabric = f
        self._finalizing = False
        if self._host_optimizer is not None:
            from .. import optimizer as opt
            self._host_updater = opt.get_updater(self._host_optimizer)
            self._host_w = f.param.tensor.clone()        # the weights: the fabric's parameter arena carries the aggregated gradient in this mode
        self._apply_wire_formats()
        if getenv_int("ENABLE_DGT", 0) and f.protocol == "ll":
            # DGT on NVSwitch: contribution-ranked tile order + fp8 for the unimportant (1 - DMLC_K) fraction, re-ranked every few rounds
            f.enable_dgt()
            self._dgt_every, self._dgt_round = max(1, getenv_int("GEOMX_DGT_RERANK_EVERY", 16)), 0

    def _push(self, key, vals, priority):
        self._finalize()
        i = self._key_index[key]
        g = self._fabric.grad_view(i)
        if vals[0]._t.dtype == torch.float16 and i not in self._fp16_keys:
            self._fp16_keys.add(i)                    # the script casts this key to fp16 (FP16 / MPQ): halves on the wire from now on
            self._apply_wire_formats()
        g.copy_(vals[0]._t.detach().reshape(g.shape))
        for v in vals[1:]:
            g.add_(v._t.detach().reshape(g.shape).to(g.device))
        if getattr(self, "_twobit_thr", None) is not None and g.dtype == torch.float32:
            # 2-bit gradient compression: residual += grad; every element becomes +thr / -thr / 0, the remainder stays in the residual for
            # the next round (quantize_2bit / dequantize_2bit kernels of csrc/kernels/compress.cu, bit-exact reference packing)
            from ..ops import native
            flat = g.reshape(-1)
            res = self._twobit_res.setdefault(i, torch.zeros_like(flat))
            packed = torch.empty((flat.numel() + 15) // 16, dtype=torch.int32, device=flat.device)
            native.quantize_2bit(flat, res, packed, self._twobit_thr)
            native.dequantize_2bit(packed, flat, self._twobit_thr)
        self._pushed.add(i)
        if priority != 0:
            self._priorities_seen = True
        self._fabric.layout.slots[i].priority = priority

    def _pull(self, key, outs, priority):
        # lazy, and NOT finalising: the reference's scripts interleave `kv.init(i, w); kv.pull(i, w)` key by key (examples/cnn.py:89-96), so
        # the arena can only be laid out when a pulled array is first read (or pushed to) — by then every key has been initialised
        if key not in self._key_index:
            raise MXNetError("key %s has not been initialised" % key)
        self._pulls.append((self._key_index[key], outs))
        for o in outs:
            o._pending = self.flush

    def flush(self):
        if not self._pushed and not self._pulls:
            return
        self._finalize()
        f = self._fabric
        pulls, self._pulls = self._pulls, []
        for _, outs in pulls:
            for o in outs:
                o._pending = None
        if self._pushed:
            nkeys = len(self._keys)
            full = len(self._pushed) == nkeys
            if not full:
                mask = torch.zeros(f.tiles, dtype=torch.uint8)
                for i in self._pushed:
                    s = f.layout.slots[i]
                    mask[s.offset // 1024: s.offset // 1024 + s.tiles] = 1
                f.tile_active.copy_(mask.to(f.device))
            if self._priorities_seen and f.dgt_contrib is None and f.protocol == "ll":
                self._apply_priority_order()
            if self._hfa:
                self._flush_hfa(full)
            elif self._sync:
                f.fsa_step(masked=not full)
                if self._host_updater is not None:
                    self._run_host_optimizer()
                if f.dgt_contrib is not None and full:
                    self._dgt_round += 1
                    if self._dgt_round % self._dgt_every == 0:
                        f.dgt_rerank()
            else:
                if not full:
                    raise MXNetError("dist_async on the fabric needs every key pushed each round")
                f.async_step()
            self._pushed.clear()
            f.grad.tensor.zero_()
        for i, outs in pulls:
            src = f.param_view(i)
            for o in outs:
                tgt = o._data
                if tgt.data_ptr() == src.data_ptr():
                    continue
                (tgt.detach() if tgt.requires_grad else tgt).copy_(src.reshape(tgt.shape), non_blocking=True)

    def _apply_priority_order(self):
        """Tiles of high-priority keys first (the reference pushes with priority = -index so that the layers the next forward pass needs first
        are exchanged first, examples/cnn.py:121-125 / kvstore_dist.h:565-625 / P3 van.cc:847-860).  The order lives in a device array the
        kernels read through ``tile_order``; it is rewritten only when the priorities change."""
        f = self._fabric
        slots = f.layout.slots
        sig = tuple(getattr(s, "priority", 0) for s in slots)
        if sig == self._order_sig:
            return
        keys = sorted(range(len(slots)), key=lambda i: (-sig[i], i))
        order = np.concatenate([np.arange(slots[i].offset // 1024, slots[i].offset // 1024 + slots[i].tiles) for i in keys]).astype(np.int32)
        if order.size < f.tiles:                                   # padding tiles (if any) keep their place at the end
            rest = np.setdiff1d(np.arange(f.tiles, dtype=np.int32), order)
            order = np.concatenate([order, rest]).astype(np.int32)
        if f.tile_order is None:
            f.tile_order = torch.from_numpy(order).to(f.device)
            f._params_cache.clear()
        else:
            f.tile_order.copy_(torch.from_numpy(order).to(f.device))
        self._order_sig = sig

    def _run_host_optimizer(self):
        """Python-executed optimizer (no complete native spec): the exchange left the aggregated gradient of every pushed key in the
        parameter arena; apply the optimizer object to the rank-local weight copy (identical on all ranks) and publish the weights."""
        from ..ndarray import NDArray
        f = self._fabric
        for i in sorted(self._pushed):
            w = f.layout.view(self._host_w, i)
            agg = f.param_view(i)
            self._host_updater(i, NDArray(agg.clone()), NDArray(w))
            agg.copy_(w)

    def _row_sparse_pull(self, key, outs, row_ids, priority):
        """Rows of a key from the (already exchanged) parameter arena: unique row ids (CUB radix sort + select, csrc/kernels/sparse_ops.cu) and
        a row gather — kvstore_dist.h PullRowSparse_ :660-702 without the wire."""
        from ..ndarray.sparse import RowSparseNDArray, _gather
        from ..kvstore.utils import unique_rows
        if key not in self._key_index:
            raise MXNetError("key %s has not been initialised" % key)
        self.flush()
        self._finalize()
        src = self._fabric.param_view(self._key_index[key])
        src2d = src.reshape(src.shape[0], -1)
        for o, ids in zip(outs, row_ids):
            rows = unique_rows(ids._t.to(src.device))
            picked = _gather(src2d.contiguous(), rows).reshape((rows.numel(),) + tuple(src.shape[1:]))
            if isinstance(o, RowSparseNDArray):
                dev = o.data._t.device
                o._set_rows(picked.to(dev), rows.to(dev))
                o._shape = tuple(src.shape)
            else:
                tgt = o._t
                tgt.zero_()
                tgt[rows.to(tgt.device)] = picked.to(tgt.device)

    def _flush_hfa(self, full):
        f, topo = self._fabric, self._topo
        if not full:
            raise MXNetError("HFA synchronisation pushes every key (examples/cnn_hfa.py)")
        self._local_iters += 1
        if self._local_iters % self._hfa_k2 != 0:
            f.party_allreduce(f.grad, f.param, scale=1.0)
        else:
            spec, scale = f.opt_spec, f.push_scale
            f.set_optimizer(None); f.set_push_scale(1.0 / topo.num_parties)
            f.fsa_step()
            f.set_optimizer(spec); f.set_push_scale(scale)

    def _barrier(self):
        self.flush()
        if self._fabric is not None:
            self._fabric.barrier()
        elif self._topo.world > 1:
            import torch.distributed as dist
            dist.barrier()

    def save_optimizer_states(self, fname, dump_optimizer=False):
        """Global-PS shard state (master weights + optimizer moments + step) of this rank — checkpointable, unlike the reference's servers."""
        self._finalize(); self.flush()
        f = self._fabric
        torch.cuda.synchronize()
        torch.save({"w": f.w.cpu(), "s0": f.s0.cpu(), "s1": f.s1.cpu(), "state": {k: v.cpu() for k, v in f.state.items()},
                    "spec": f.opt_spec, "local_iters": self._local_iters}, "%s.rank%d" % (fname, self._topo.rank))

    def load_optimizer_states(self, fname):
        self._finalize()
        f = self._fabric
        d = torch.load("%s.rank%d" % (fname, self._topo.rank), weights_only=False)
        f.w.copy_(d["w"]); f.s0.copy_(d["s0"]); f.s1.copy_(d["s1"])
        f.state["fsa"][2] = d["state"]["fsa"][2]          # optimizer step t (epochs keep running)
        self._local_iters = d.get("local_iters", 0)
        if d.get("spec") is not None:
            f.set_optimizer(d["spec"])

    def get_num_dead_node(self, node_id=0, timeout=60):
        return 0
