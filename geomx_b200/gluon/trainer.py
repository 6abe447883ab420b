"""``gluon.Trainer`` — applies an optimizer to a set of Parameters, optionally through a KVStore.

Public behaviour follows the reference (``python/mxnet/gluon/trainer.py:27-434``): constructor arguments (``params`` dict/list, ``optimizer``
name or instance, ``kvstore`` name / instance / None, ``update_on_kvstore``, ``compression_params``), ``step`` (``rescale_grad = scale /
batch_size``), ``allreduce_grads`` + ``update`` for the split form, ``save_states`` / ``load_states`` (pickled updater states incl. the
optimizer), ``learning_rate`` / ``set_learning_rate``; dist kvstores default to updating on the server, async ones require it.

Internals are this framework's own: the kvstore decision is resolved once into a :class:`_SyncPlan` (``none`` / ``reduce`` / ``server``), every
public entry point goes through :meth:`_ready`, and parameters whose shape was still deferred when the plan was bound are registered with the
store as soon as they materialise.  On CUDA with a native-spec optimizer (SGD / momentum / Adam) and no kvstore, the whole parameter set is
updated by ONE multi-tensor fused kernel launch (``ops.native.multi_tensor_update``) instead of one launch per parameter (the reference runs
three mshadow passes per Adam parameter).
"""
from __future__ import annotations

import torch

from .. import optimizer as opt
from .parameter import Parameter, ParameterDict

__all__ = ["Trainer"]


class _SyncPlan:
    """How gradients / weights travel: ``none`` (local update), ``reduce`` (kvstore sums gradients, workers update), ``server`` (kvstore
    applies the optimizer, workers pull weights)."""

    __slots__ = ("store", "mode")

    def __init__(self, store=None, mode="none"):
        self.store, self.mode = store, mode

    @staticmethod
    def resolve(kvstore, update_on_kvstore, num_contexts):
        from .. import kvstore as kvs
        single_device_local = isinstance(kvstore, str) and num_contexts == 1 and "dist" not in kvstore
        if kvstore is None or single_device_local:
            return _SyncPlan()
        store = kvs.create(kvstore) if isinstance(kvstore, str) else kvstore
        distributed = "dist" in store.type
        on_server = distributed if update_on_kvstore is None else bool(update_on_kvstore)
        if distributed and "async" in store.type and not on_server:
            raise ValueError("Please set update_on_kvstore to true when training in async mode.")
        return _SyncPlan(store, "server" if on_server else "reduce")


class Trainer:
    def __init__(self, params, optimizer, optimizer_params=None, kvstore="device", compression_params=None, update_on_kvstore=None):
        if isinstance(params, (dict, ParameterDict)):
            params = list(params.values())
        if not isinstance(params, (list, tuple)) or not all(isinstance(p, Parameter) for p in params):
            raise ValueError("First argument must be a list or dict of Parameters, got %s." % type(params))
        self._params = list(params)
        self._index = {p.name: i for i, p in enumerate(self._params)}
        for p in self._params:
            p._trainer = self
        self._contexts = self._common_contexts()
        optimizer_params = dict(optimizer_params or {})
        self._scale = float(optimizer_params.get("rescale_grad", 1.0))
        if isinstance(optimizer, opt.Optimizer):
            if optimizer_params:
                raise ValueError("optimizer_params must be None if optimizer is an instance of Optimizer instead of str")
            self._optimizer = optimizer
            self._optimizer.param_dict = dict(enumerate(self._params))
        else:
            self._optimizer = opt.create(optimizer, param_dict=dict(enumerate(self._params)), **optimizer_params)
        self._updaters = [opt.get_updater(self._optimizer) for _ in self._contexts]
        self._request = (kvstore, update_on_kvstore, compression_params)
        self._plan = None            # bound lazily: parameters may not be initialised yet
        self._unregistered = list(self._params)

    # -- compatibility views used around the code base -----------------------------------------------------------------------------
    @property
    def _kvstore(self):
        return self._plan.store if self._plan else None

    @property
    def _update_on_kvstore(self):
        return None if self._plan is None or self._plan.store is None else self._plan.mode == "server"

    @property
    def _kv_initialized(self):
        return self._plan is not None

    def _common_contexts(self):
        seen = None
        for p in self._params:
            ctx = p.list_ctx()
            if seen is not None and ctx != seen:
                raise ValueError("All Parameters must live on the same set of contexts: %s is on %s, earlier ones on %s" % (p.name, ctx, seen))
            seen = ctx
        return seen or []

    def _reset_kvstore(self):
        """Forget the bound store (parameters were re-initialised): everything is registered again on the next step."""
        if self._plan and self._plan.store is not None and "dist" in self._plan.store.type:
            raise RuntimeError("Cannot reset distributed KVStore.")
        self._plan = None
        self._unregistered = list(self._params)

    def _ready(self):
        """Bind the sync plan on first use and register every parameter that has materialised since."""
        if self._plan is None:
            kvstore, update_on_kvstore, compression = self._request
            plan = _SyncPlan.resolve(kvstore, update_on_kvstore, len(self._contexts))
            if plan.store is not None:
                if compression:
                    plan.store.set_gradient_compression(compression)
                if plan.mode == "server":
                    plan.store.set_optimizer(self._optimizer)
            self._plan = plan
        if not self._unregistered:
            return
        store, later = self._plan.store, []
        for p in self._unregistered:
            if p._deferred_init:
                later.append(p)
            elif store is not None:
                i = self._index[p.name]
                store.init(i, p.list_data()[0])
                store.pull(i, p.list_data(), priority=-i)      # every replica starts from the value the store holds (rank 0's)
        self._unregistered = later

    def _trainable(self):
        return [(i, p) for i, p in enumerate(self._params) if p.grad_req != "null"]

    # -- public API -----------------------------------------------------------------------------------------------------------------
    @property
    def learning_rate(self):
        return self._optimizer.learning_rate

    @property
    def optimizer(self):
        return self._optimizer

    def set_learning_rate(self, lr):
        self._optimizer.set_learning_rate(lr)

    def _set_rescale(self, batch_size):
        scale = self._scale / batch_size
        plan = self._plan
        if plan is not None and plan.mode == "server" and "dist" in plan.store.type and self._optimizer.rescale_grad != scale:
            # the optimizer object already lives on the servers: a new normalisation factor would silently not apply there
            raise UserWarning("Possible change in the `batch_size` from previous `step` detected. Optimizer gradient normalizing factor "
                              "will not change w.r.t new batch_size when update_on_kvstore=True and when distributed kvstore is used.")
        self._optimizer.rescale_grad = scale

    def step(self, batch_size, ignore_stale_grad=False):
        """One optimisation step: gradients are summed over devices / workers, then weights are updated (``rescale_grad = scale/batch_size``)."""
        self._set_rescale(batch_size)
        self._ready()
        self._exchange()
        self._apply(ignore_stale_grad)

    def allreduce_grads(self):
        self._ready()
        if self._plan.mode == "server":
            raise AssertionError("allreduce_grads() when parameters are updated on kvstore is not supported. "
                                 "Try setting `update_on_kvstore` to False when creating trainer.")
        self._exchange()

    def update(self, batch_size, ignore_stale_grad=False):
        self._ready()
        if self._plan.mode == "server":
            raise AssertionError("update() when parameters are updated on kvstore is not supported. "
                                 "Try setting `update_on_kvstore` to False when creating trainer.")
        self._set_rescale(batch_size)
        self._apply(ignore_stale_grad)

    def _exchange(self):
        plan = self._plan
        if plan.store is None:
            return
        for i, p in self._trainable():
            plan.store.push(i, p.list_grad(), priority=-i)
            if plan.mode == "reduce":
                plan.store.pull(i, p.list_grad(), priority=-i)

    def _apply(self, ignore_stale_grad=False):
        plan = self._plan
        if plan.mode == "server":
            for i, p in self._trainable():
                plan.store.pull(i, p.list_data(), priority=-i)
            return
        if self._fused_update():
            return
        for i, p in self._trainable():
            for updater, weight, grad in zip(self._updaters, p.list_data(), p.list_grad()):
                updater(i, grad, weight)

    def _fused_update(self):
        """One multi-tensor launch for the whole parameter set when a native spec exists (CUDA, fp32, one context, no scheduler)."""
        from ..ops import native
        if len(self._contexts) != 1 or not native.available():
            return False
        if self._optimizer.lr_scheduler is not None:
            return False
        spec = self._optimizer.spec()
        if spec is None or spec["name"] not in native.OPT_KINDS:
            return False
        ws, gs, idxs = [], [], []
        for i, p in self._trainable():
            w, g = p.list_data()[0]._t, p.list_grad()[0]._t
            if not (w.is_cuda and w.dtype == torch.float32 and g.dtype == torch.float32):
                return False
            ws.append(w.detach()); gs.append(g); idxs.append(i)
        return True if not ws else native.multi_tensor_update(self._optimizer, self._updaters[0], idxs, ws, gs)

    def _row_sparse_pull(self, parameter, out, row_id):
        """Refresh the rows ``row_id`` of a row_sparse parameter from the store before they are read (server-side updates only)."""
        self._ready()
        if self._plan.mode == "server":
            i = self._index[parameter.name]
            self._plan.store.row_sparse_pull(i, out=out, row_ids=row_id, priority=-i)

    # -- optimizer state ------------------------------------------------------------------------------------------------------------
    def save_states(self, fname):
        self._ready()
        if self._plan.mode == "server":
            if self._unregistered:
                raise AssertionError("Cannot save trainer states when some parameters are not yet initialized in kvstore.")
            self._plan.store.save_optimizer_states(fname, dump_optimizer=True)
        else:
            with open(fname, "wb") as f:
                f.write(self._updaters[0].get_states(dump_optimizer=True))

    def load_states(self, fname):
        self._ready()
        if self._plan.mode == "server":
            store = self._plan.store
            store.load_optimizer_states(fname)
            # a dist worker has no local updater (the states live on the servers): keep this side's optimizer object
            local = getattr(store, "_updater", None)
            if local is not None and getattr(local, "optimizer", None) is not None:
                self._optimizer = local.optimizer
        else:
            with open(fname, "rb") as f:
                blob = f.read()
            for updater in self._updaters:
                updater.set_states(blob)
                updater.optimizer = self._updaters[0].optimizer
            self._optimizer = self._updaters[0].optimizer
        self._optimizer.param_dict = dict(enumerate(self._params))
