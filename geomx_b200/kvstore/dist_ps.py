"""``dist_*`` KVStore over the native HiPS transport (multi-process / multi-host / CPU path).

Parity: ``python/mxnet/kvstore.py`` on top of ``KVStoreDist`` (``src/kvstore/kvstore_dist.h``): push stages the (locally reduced) value
into a pinned host buffer (``comm_buf_``), ships it with ``ZPush``; pull receives into a pinned buffer and fans it out to the device
copies (``comm_->Broadcast``); ``set_optimizer`` pickles the optimizer to the servers (``kController``) — here an optimizer with a native
spec is shipped *declaratively* (``kSetOptimizerSpec``) and executed by the C++ server without Python; ``set_gradient_compression``
(2bit worker-side, bsc server-side), ``_barrier``, ``_send_command_to_servers``, ``num_dead_node``; server profiler commands.
Asynchrony: pushes are issued immediately (non-blocking), pulls are queued and resolved at the first read of a target array or at
``mx.nd.waitall()`` — the lazy equivalent of the reference's engine-variable ordering, so all keys' rounds overlap.
"""
from __future__ import annotations

import pickle

import torch

from .. import runtime
from ..base import MXNetError
from ..ndarray import NDArray
from .base import KVStoreBase

_DT = {torch.float32: 0, torch.float64: 1, torch.float16: 2, torch.uint8: 3, torch.int32: 4, torch.int8: 5, torch.int64: 6, torch.bfloat16: 12}

CMD_CONTROLLER, CMD_MULTI_PRECISION, CMD_STOP, CMD_SYNC, CMD_SYNC_GLOBAL, CMD_COMPRESSION, CMD_PROFILER, CMD_OPT_SPEC, CMD_SAVE, CMD_LOAD = range(10)


def _pinned(numel, dtype):
    """Staging buffer of the PS client: a block of the native host pool (page-locked when CUDA is present; csrc/runtime/storage.h)."""
    try:
        from ..storage import pinned_empty
        return pinned_empty(numel, dtype)
    except Exception:
        pass
    t = torch.empty(numel, dtype=dtype)
    if torch.cuda.is_available():
        try:
            t = t.pin_memory()
        except RuntimeError:
            pass
    return t


# the kinds the C++ host server executes from a spec (csrc/hips/server_optim.h, ServerOptSpec::valid); it aborts on any other name, so the
# other native kinds ship the pickled optimizer like any Python optimizer
HOST_SERVER_KINDS = ("sgd", "adam", "dcasgd")


def spec_to_string(spec):
    return ";".join("%s=%s" % (k, v) for k, v in spec.items() if k != "multi_precision")


class KVStoreDist(KVStoreBase):
    def __init__(self, kv_type="dist_sync"):
        super().__init__(kv_type)
        self._C = runtime.C()
        self._kv = self._C.KVStoreDist(kv_type)
        self._is_worker = self._C.is_worker_node()
        self._send_buf, self._recv_buf, self._push_handle = {}, {}, {}
        self._pulls = []
        self._rows_keep = {}
        self._key_type = None
        self._next_str_key = 0
        self._closed = False
        if self._is_worker:
            from .. import profiler
            profiler.set_kvstore_handle(self)

    # -- identity ---------------------------------------------------------------------------------------------------------------
    @property
    def rank(self): return self._kv.rank if self._is_worker else 0
    @property
    def num_workers(self): return self._kv.num_workers
    @property
    def num_all_workers(self): return self._kv.num_all_workers
    @property
    def is_master_worker(self): return self._kv.is_master_worker
    @property
    def is_recovery(self):
        """True when this worker replaced a dead one (it skipped the start-up barriers and key initialisation)."""
        return bool(self._kv.is_recovery)

    def _key(self, k):
        kt = str if isinstance(k, str) else int
        if self._key_type is None:
            self._key_type = kt
        elif self._key_type is not kt:
            raise MXNetError("inconsistent key types: mixing str and int keys is not allowed")
        if kt is str:
            if k not in self._str_key_map:
                self._str_key_map[k] = self._next_str_key; self._next_str_key += 1
            return self._str_key_map[k]
        return int(k)

    # -- data --------------------------------------------------------------------------------------------------------------------
    def _stage(self, key, vals):
        """reduce the per-device values of one key and stage them in the key's pinned send buffer"""
        t0 = vals[0]._t.detach()
        buf = self._send_buf.get(key)
        if buf is None or buf.numel() != t0.numel() or buf.dtype != t0.dtype:
            buf = _pinned(t0.numel(), t0.dtype); self._send_buf[key] = buf
        h = self._push_handle.pop(key, None)
        if h is not None:
            self._kv.wait(h)               # the previous push of this key still reads the buffer
        if len(vals) == 1:
            buf.copy_(t0.reshape(-1), non_blocking=False)
        else:
            acc = t0.reshape(-1).clone()
            for v in vals[1:]:
                acc.add_(v._t.detach().reshape(-1).to(acc.device))
            buf.copy_(acc)
        return buf

    def _init(self, key, value):
        buf = self._stage(key, [value])
        self._kv.init(key, buf.data_ptr(), buf.numel(), _DT[buf.dtype])

    def _push(self, key, vals, priority):
        buf = self._stage(key, vals)
        self._push_handle[key] = self._kv.push(key, buf.data_ptr(), buf.numel(), _DT[buf.dtype], int(priority))

    def _pull(self, key, outs, priority):
        self._pulls.append((key, outs, int(priority)))
        for o in outs:
            o._pending = self.flush

    def flush(self):
        if not self._pulls:
            return
        pulls, self._pulls = self._pulls, []
        pulls.sort(key=lambda p: -p[2])       # higher priority first (MXNet: larger = earlier)
        issued = []
        for key, outs, prio in pulls:
            for o in outs:
                o._pending = None
            t0 = outs[0]._data
            if len(outs) == 1 and t0.device.type == "cpu" and t0.is_contiguous() and not t0.requires_grad:
                buf = t0                               # host target: the response is written straight into it (no staging copy)
            else:
                buf = self._recv_buf.get(key)
                if buf is None or buf.numel() != t0.numel() or buf.dtype != t0.dtype:
                    buf = _pinned(t0.numel(), t0.dtype); self._recv_buf[key] = buf
            h = self._kv.pull(key, buf.data_ptr(), buf.numel(), _DT[buf.dtype], prio)
            self._push_handle.pop(key, None)
            issued.append((h, buf, outs))
        for h, buf, outs in issued:
            self._kv.wait(h)
            for o in outs:
                tgt = o._data
                if tgt is buf:
                    continue
                (tgt.detach() if tgt.requires_grad else tgt).copy_(buf.view(tgt.shape), non_blocking=True)

    def _push_row_sparse(self, key, vals, priority):
        """Only the non-zero rows travel (kvstore_dist.h PushRowSparse :628-657); several device copies are summed first."""
        from ..ndarray import sparse
        acc = None
        for v in vals:
            v = v if isinstance(v, sparse.RowSparseNDArray) else sparse.cast_storage(v, "row_sparse")
            acc = v if acc is None else sparse.add(acc, v)
        ids = acc.indices._t.long().cpu().contiguous()
        rows = acc.data._t.float().cpu().contiguous()
        row_len = 1
        for d in acc.shape[1:]:
            row_len *= int(d)
        h = self._push_handle.pop(key, None)
        if h is not None:
            self._kv.wait(h)
        self._rows_keep[key] = (ids, rows)
        self._push_handle[key] = self._kv.push_rows(key, ids.data_ptr(), ids.numel(), rows.data_ptr(), row_len, int(priority))

    def _row_sparse_pull(self, key, outs, row_ids, priority):
        """Sends the unique row ids, receives exactly those rows (kvstore_dist.h PullRowSparse_ :660-702)."""
        from ..ndarray.sparse import RowSparseNDArray
        from .utils import unique_rows
        self.flush()
        for o, ids in zip(outs, row_ids):
            rows = unique_rows(ids._t).cpu().contiguous()
            shape = o.shape
            row_len = 1
            for d in shape[1:]:
                row_len *= int(d)
            buf = _pinned(max(1, rows.numel() * row_len), torch.float32)
            h = self._kv.pull_rows(key, rows.data_ptr(), rows.numel(), buf.data_ptr(), row_len, int(priority))
            self._push_handle.pop(key, None)
            self._kv.wait(h)
            picked = buf[:rows.numel() * row_len].view((rows.numel(),) + tuple(shape[1:]))
            if isinstance(o, RowSparseNDArray):
                dev = o.data._t.device
                o._set_rows(picked.to(dev).clone(), rows.to(dev))
            else:
                tgt = o._data
                tgt.zero_()
                tgt[rows.to(tgt.device)] = picked.to(tgt.device).to(tgt.dtype)

    # -- configuration ----------------------------------------------------------------------------------------------------------
    def set_optimizer(self, optimizer):
        if not self._is_worker:
            return super().set_optimizer(optimizer)      # on a server: install the python updater (controller path)
        if self.rank == 0:
            spec = optimizer.spec()
            import os
            # the declarative spec carries one scalar lr / wd: an lr_scheduler or per-parameter multipliers (e.g. wd_mult = 0 on biases) need the
            # optimizer object itself on the server, which is what the reference always ships (kvstore.py:452-499)
            if (spec is not None and spec["name"] in HOST_SERVER_KINDS and optimizer.spec_is_static()
                    and os.environ.get("GEOMX_PY_UPDATER", "0") != "1"):
                self._kv.send_command_to_servers(CMD_OPT_SPEC, spec_to_string(spec))
            else:
                self._kv.send_command_to_servers(CMD_CONTROLLER, pickle.dumps(optimizer, 0).decode("latin1"))
            if optimizer.multi_precision:
                self._kv.send_command_to_servers(CMD_MULTI_PRECISION, "")
        self._optimizer = optimizer

    def _set_gradient_compression(self, params):
        self._kv.set_gradient_compression(params.get("type", "none"), float(params.get("threshold", 0.5)))

    def _barrier(self):
        self.flush(); self._kv.barrier()

    def _send_command_to_servers(self, head, body):
        self._kv.send_command_to_servers(int(head), str(body))

    def get_num_dead_node(self, node_id=7, timeout=60):
        return self._kv.num_dead_node(node_id, timeout)

    def set_server_profiler_command(self, which, params):
        self._kv.send_command_to_servers(CMD_PROFILER, "%s%d" % (params, which))

    def save_optimizer_states(self, fname, dump_optimizer=False):
        """Server-side state checkpoint (optimizer moments, HFA milestones, compression residuals) — not possible in the reference."""
        if self.rank == 0:
            self._kv.send_command_to_servers(CMD_SAVE, fname)

    def load_optimizer_states(self, fname):
        if self.rank == 0:
            self._kv.send_command_to_servers(CMD_LOAD, fname)

    # -- server / scheduler role ----------------------------------------------------------------------------------------------------
    def run_server(self, controller):
        kv = self

        class _Upd:
            def __call__(_self, key, grad, weight):
                if kv._updater is None:      # no optimizer on the server: store the aggregate (reference ApplyUpdates without updater_)
                    weight[...] = grad
                    return
                kv._updater(key, NDArray(torch.from_numpy(grad)), NDArray(torch.from_numpy(weight)))

        def ctrl(head, body):
            controller(head, body.decode("latin1").encode("latin1") if isinstance(body, bytes) else body)

        self._kv.run_server(ctrl, _Upd())

    def close(self):
        if not self._closed:
            self._closed = True
            if self._is_worker:
                self.flush()
            self._kv.shutdown()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
