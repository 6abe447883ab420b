"""The reference's demo model (``examples/cnn.py:56-64``) and its H100 training engine.

``build_cnn()`` returns the Gluon network exactly as the reference scripts declare it:
``Conv2D(16,k5,relu) → MaxPool2 → Conv2D(32,k5,relu) → MaxPool2 → Dense(256,relu) → Dense(128,relu) → Dense(10)`` (178 762 parameters).

``HipsCNNTrainStep`` is the flagship hot path: one *training step* = forward + backward of that network for a per-worker batch
plus the HiPS push/pull of all 10 keys (``dist_sync``: party aggregation → global aggregation + optimizer → broadcast), captured ONCE
into a CUDA graph and replayed per step.  At the reference's batch size (32 per worker) the step is 5-6 hand-written sm_90a launches:

  cnn_fwd      conv0+bias+ReLU+pool → conv1+bias+ReLU+pool → dense0 → dense1 → classifier → softmax-CE, and the data gradients dz4 and
               dz3, fp32 FMA, the conv0 map never leaves shared memory; clusters of two images, whose 8 CTAs exchange a2, a3 and a4
               (cnn_fwd_dense0_kernel, csrc/kernels/cnn_direct.cu)
  mlp_chain    da2 = dz3 · W0, one 16-CTA cluster (dense_tail_kernel, csrc/kernels/mlp_chain.cu).  With look-ahead the forward kernel stops
               at a3 and the cluster kernel runs the chain from a3 to da2.
  dense_wgrad  the three dense weight gradients and bias gradients, on a parallel branch: in the dense channel's step on the
               high-priority stream when there is one, otherwise on the side stream, joined before the exchange   (csrc/kernels/mlp_chain.cu).
               When the forward kernel has computed dz3 it has stored everything this kernel reads, so its branch forks right after the
               forward kernel, beside mlp_chain; the dense channel behind it also waits for mlp_chain, which reads the W0 it writes,
               through a full graph edge (a programmatic one from mlp_chain made it wait for cnn_bwd_all too).
  cnn_bwd_all  conv1 data gradient + pool/ReLU routing + conv0 weight gradient ‖ conv1 weight gradient, one grid      (csrc/kernels/cnn_direct.cu)
  exchange     one LL kernel for all keys after the backward pass (several ranks), or key-group channels: the dense keys' exchange on
               a high-priority stream underneath cnn_bwd_all, the conv keys' one-hop exchange after it (one rank / GEOMX_STEP_OVERLAP=1)
                                                                                                                      (csrc/kernels/hips_fabric.cu)

Without the direct convolutions (odd batches, ``GEOMX_DIRECT_CONV=0``) the cluster kernel starts from a2 and computes dense0 itself
(mlp_chain_kernel).  Larger batches (and ``GEOMX_DIRECT_CONV=0`` / ``GEOMX_FUSED_MLP=0``) use the generic kernels: direct conv0 + im2col, wgmma GEMMs with fused
bias / ReLU / max-pool / mask / column-sum epilogues (3xTF32 = fp32-accurate by default), weight-gradient GEMMs on a parallel graph branch.
With one rank and one party both PS tiers collapse into the arena optimizer inside the exchange kernels.

Which of these kernel paths a step takes is decided once, when the engine is constructed: ``step_path()`` maps the batch size, the
engine's arguments and the step switches (``STEP_SWITCHES``, read from the environment at that moment) to a ``StepPath`` record, and
``_steps()`` binds the launches of that record.  Changing a switch afterwards does not change the engine; construct a new one.

The reference runs the same step as ~200 engine ops (per-image im2col+SGEMM) + 20 ZMQ round trips (SURVEY §3.3-3.4).
The public API a user calls is ``step(X_host, y_host, sample_weight=None) -> loss`` (H2D of the batch from pinned memory, graph replay, D2H of
the loss), for any 1 <= n <= B rows: a short or sample-weighted batch runs the weighted instance of the kernel that produces the dlogits,
which scales row i by its coefficient w_i * B / n (0 for the padding rows), in graphs of its own.

The engine also scores its live weights: ``evaluate(X, y) -> (mean_loss, accuracy)`` (``evaluate_async`` returns a handle) and
``predict(X) -> logits`` run the whole forward pass of any number of images, the per-sample softmax-CE and the arg-max as ONE launch
(cnn_eval_kernel, csrc/kernels/cnn_direct.cu: the forward kernel's clusters of two images, extended by dense1 and the classifier), on
buffers of their own, ordered on the current stream after the steps enqueued before it.
"""
from __future__ import annotations

import copy
import os
from typing import NamedTuple

import numpy as np
import torch

from .. import gluon, initializer
from ..context import Context
from ..ndarray import NDArray
from ..ops import native
from ..parallel.arena import ArenaLayout
from ..parallel.fabric import HipsFabric, Topology

__all__ = ["build_cnn", "CNN_PARAM_SHAPES", "HipsCNNTrainStep", "StepPath", "step_path", "STEP_SWITCHES"]

CNN_PARAM_SHAPES = [(16, 1, 5, 5), (16,), (32, 16, 5, 5), (32,), (256, 512), (256,), (128, 256), (128,), (10, 128), (10,)]
# the structural names that ``net.save_parameters`` gives the parameters of build_cnn() (the index of the layer in the Sequential)
CNN_PARAM_NAMES = ["0.weight", "0.bias", "2.weight", "2.bias", "4.weight", "4.bias", "5.weight", "5.bias", "6.weight", "6.bias"]
# version of the file that HipsCNNTrainStep.save_states writes
CHECKPOINT_VERSION = 1
# checkpoint meta fields that must equal the loading engine's: the optimizer kind, update mode, sync mode and the accelerator set
_MUST_MATCH = ("meta:opt_kind", "meta:update", "meta:mode", "meta:hfa", "meta:wire_formats", "meta:bsc_threshold", "meta:dgt")

# The environment variables that select the training step's kernel path; HipsCNNTrainStep reads them once, when it is constructed.
STEP_SWITCHES = ("GEOMX_STEP_OVERLAP", "GEOMX_STEP_EXCHANGE", "GEOMX_FUSED_MLP", "GEOMX_DIRECT_CONV", "GEOMX_CNN_BWD_ONE_LAUNCH",
                 "GEOMX_NO_POOL_FUSION", "GEOMX_FUSED_EXCHANGE", "GEOMX_E2E_DIRECT_INPUT")

# Names of the step's launches that more than one stage or caller refers to (tests, tools and bench.py key on the names).
DIRECT_FWD = "conv0+conv1 fwd (direct, relu+pool fused)"
GEMM_FWD = ("conv0+relu+pool+im2col", "conv1 gemm (bias,relu,maxpool fused)")
MLP = "mlp chain fwd+bwd (cluster)"
DENSE_WGRAD = "dense weight gradients"
DENSE_KV = "hips push+opt+pull (dense keys, overlapped)"
ONE_GRID = "conv bwd: conv1 wgrad + dgrad + conv0 wgrad (direct, one grid)"
FUSED_BWD = "conv bwd (one grid) + conv-key exchange in its tail"
EXCH = "hips push+opt+pull"
LOCAL = "local optimizer (fused arena Adam)"


class StepPath(NamedTuple):
    """The kernel path of one engine's training step (see :func:`step_path`)."""
    direct_conv: bool       # convolutions: direct fp32 kernels (True) or im2col + wgmma GEMMs
    pool_fusion: bool       # GEMM convolutions: conv1's max-pool in the GEMM epilogue (where the kernel can express it)
    dense: str              # where the dense chain's cluster kernel starts: 'a2' (mlp_chain), 'a3' (dense_tail; the forward kernel computes
                            # dense0), 'dz3' (dense_tail from dz3; the forward kernel also runs the head), or 'gemm' (seven GEMM / head launches)
    wgrad: str | None       # the cluster path's dense weight gradients: 'side' stream or 'comm' stream (in the dense channel's step)
    bwd: str                # convolution backward: 'one_grid', 'exchange_tail' (one grid, conv keys' exchange in its tail), 'two_launch', 'gemm'
    exchange: str           # the exchange: 'fsa', 'async', 'conv' (channel), 'all' (single channel), 'local_opt' (HFA: local optimizer only)
    local_tail: bool        # update='local': the arena optimizer applies the exchanged aggregate after the exchange
    overlap: bool           # key-group channels: the dense keys' exchange on the comm stream underneath the convolution backward
    single: str | None      # the one direct-protocol channel of all keys ('all') when not overlapping
    n_fwd: int              # leading launches that need only the batch and the weights (a look-ahead launch runs them for the next batch)
    lookahead: bool
    lookahead_join: str     # how a look-ahead launch joins before the next batch's forward launches: 'join' (side) or 'join_comm' (side + comm)
    direct_input: bool      # the host pipeline captures one graph per input buffer instead of copying staging -> input


def step_path(B, *, mode="dist_sync", hfa=False, update="server", lookahead=False, world=1, direct_protocol=False, conv_tail_capable=False,
              env=None):
    """Choose the training step's kernel path from plain values: the per-worker batch ``B``, the engine's ``mode`` / ``hfa`` / ``update`` /
    ``lookahead``, the number of ranks, whether the fabric has the direct-protocol buffers, whether the conv keys' channel can run in a
    compute kernel's tail, and the step switches in ``env`` (a mapping of :data:`STEP_SWITCHES` names to strings; missing = default)."""
    env = env or {}
    on = lambda k, default: env.get(k, default) == "1"
    sync = mode == "dist_sync" and not hfa
    # One rank -> channels (their exchange is local arithmetic); several ranks -> one exchange after the backward pass (the overlapped
    # two-hop channel's polling slows the backward pass down, and at 8 ranks it outlasts the pass it hides behind).  Hence the default.
    overlap = sync and on("GEOMX_STEP_OVERLAP", "1" if world == 1 else "0") and (world == 1 or direct_protocol)
    single = "all" if (sync and not overlap and world > 1 and direct_protocol
                       and env.get("GEOMX_STEP_EXCHANGE", "ll") in ("sharded", "replicated")) else None
    lookahead = bool(lookahead) and sync
    fused_mlp = B <= 32 and on("GEOMX_FUSED_MLP", "1")
    # small-batch regime: both convolutions forward / backward as direct fp32-FMA kernels (csrc/kernels/cnn_direct.cu) instead of im2col +
    # wgmma GEMMs; their conv1 weight-gradient body splits the batch in halves, so odd batches and batches > 64 use the GEMMs
    direct_conv = B <= 64 and B % 2 == 0 and on("GEOMX_DIRECT_CONV", "1")
    # even B <= 32: dense0 is row-separable, so the forward kernel computes a3 on its 128 SMs; in the classic step it also runs the chain
    # down to dz3.  A look-ahead launch ends with the NEXT batch's forward kernel, which would overwrite this batch's loss and logits before
    # the host reads them: it keeps the forward kernel that stops at a3.
    if not fused_mlp:
        dense = "gemm"
    elif not direct_conv:
        dense = "a2"
    else:
        dense = "a3" if lookahead else "dz3"
    if not direct_conv:
        bwd = "gemm"
    elif not on("GEOMX_CNN_BWD_ONE_LAUNCH", "1"):
        bwd = "two_launch"
    elif overlap and conv_tail_capable and on("GEOMX_FUSED_EXCHANGE", "0"):
        bwd = "exchange_tail"
    else:
        bwd = "one_grid"
    if overlap:
        exchange = "conv"
    elif single:
        exchange = single
    elif hfa:
        exchange = "local_opt"
    else:
        exchange = "async" if mode == "dist_async" else "fsa"
    return StepPath(
        direct_conv=direct_conv, pool_fusion=not on("GEOMX_NO_POOL_FUSION", "0"), dense=dense,
        # the dense channel reads these gradients: with one, they are issued in its comm-stream step.  A look-ahead launch ends with the
        # next batch's forward convolutions, which overwrite the x this kernel reads: it keeps them on the side stream, joined before those
        wgrad=None if dense == "gemm" else ("comm" if overlap and not lookahead else "side"),
        bwd=bwd, exchange=exchange, local_tail=update == "local" and not hfa, overlap=overlap, single=single,
        n_fwd=1 if direct_conv else 2, lookahead=lookahead,
        # the next batch's forward convolutions overwrite a2 (and a3), which the side branch may still be reading; a forward kernel that
        # also computes dense0 reads W0 / b0, which the dense keys' exchange (comm) updates
        lookahead_join="join_comm" if dense in ("a3", "dz3") else "join",
        direct_input=not lookahead and on("GEOMX_E2E_DIRECT_INPUT", "1"))


def build_cnn():
    net = gluon.nn.Sequential()
    net.add(gluon.nn.Conv2D(channels=16, kernel_size=5, activation="relu"), gluon.nn.MaxPool2D(pool_size=2, strides=2),
            gluon.nn.Conv2D(channels=32, kernel_size=5, activation="relu"), gluon.nn.MaxPool2D(pool_size=2, strides=2),
            gluon.nn.Dense(256, activation="relu"), gluon.nn.Dense(128, activation="relu"), gluon.nn.Dense(10))
    return net


def _pack(arrays):
    """The bytes of ``arrays``, one after the other (one broadcast of a whole checkpoint)."""
    return np.concatenate([np.ascontiguousarray(a).reshape(-1).view(np.uint8) for a in arrays])


def _unpack(buf, layout):
    """Inverse of :func:`_pack`: ``layout`` lists (name, shape, dtype) in packing order; returns name -> array."""
    out, o = {}, 0
    for name, shape, dt in layout:
        n = int(np.prod(shape)) * np.dtype(dt).itemsize
        out[name] = buf[o:o + n].view(dt).reshape(shape).copy()
        o += n
    return out


class LossHandle:
    """Result of ``HipsCNNTrainStep.step_async``: the per-sample losses of one step in pinned host memory + the event that guards them.
    For a batch of ``n`` rows with sample weights ``w`` (``None``: unweighted), ``wait()`` returns the ``n`` values ``w_i * loss_i`` and
    ``item()`` their mean over ``n``, as Gluon's losses weight them."""

    __slots__ = ("_host", "_event", "_n", "_w")

    def __init__(self, host, event, n=None, w=None):
        self._host, self._event, self._n, self._w = host, event, n, w

    def _values(self):
        if self._n is None or (self._w is None and self._n == self._host.numel()):
            return self._host
        v = self._host[:self._n]
        return v if self._w is None else v * self._w

    def wait(self):
        if self._event is not None:
            self._event.synchronize()
        return None if self._host is None else self._values()

    def item(self):
        if self._host is None:          # look-ahead engine, first call: no step has finished yet
            return float("nan")
        self._event.synchronize()
        v = self._values()
        return float(v.sum()) / v.numel()

    asscalar = item


class EvalHandle:
    """Result of ``HipsCNNTrainStep.evaluate_async``: the fp64 loss sum and the count of correct samples in pinned host memory + the event
    that guards them.  ``wait()`` / ``item()`` synchronise on that event and return ``(mean_loss, accuracy)``."""

    __slots__ = ("_host", "_event", "_n")

    def __init__(self, host, event, n):
        self._host, self._event, self._n = host, event, n

    def wait(self):
        self._event.synchronize()
        return float(self._host[0]) / self._n, float(self._host[1]) / self._n

    item = wait


def _key_mults(optimizer, net):
    """Per-key ``(lr_mult, wd_mult)`` of the demo CNN's ten keys, resolved as ``Optimizer._get_lr`` / ``_get_wd`` resolve them for index
    ``i``: the ``Parameter`` of ``net`` (what ``gluon.Trainer`` hands over through ``param_dict``) or the optimizer's ``param_dict``, then
    ``optimizer.lr_mult`` / ``wd_mult`` by index, then by ``idx2name``."""
    params = dict(optimizer.param_dict)
    if net is not None:
        params = dict(enumerate(net.collect_params().values()))
    out = []
    for i in range(len(CNN_PARAM_SHAPES)):
        if i in params:
            out.append((float(params[i].lr_mult), float(params[i].wd_mult)))
            continue
        m = []
        for table in (optimizer.lr_mult, optimizer.wd_mult):
            if i in table:
                m.append(float(table[i]))
            elif i in optimizer.idx2name:
                m.append(float(table.get(optimizer.idx2name[i], 1.0)))
            else:
                m.append(1.0)
        out.append(tuple(m))
    return out


_NATIVE_OPTIMIZERS = "SGD, Adam, DCASGD, NAG, Signum, RMSProp (centered=False), AdaGrad, AdaDelta, Ftrl"
# why the other optimizers of the library do not run in the update kernels
_NOT_NATIVE = {
    "RMSProp(centered=True)": "centered RMSProp keeps three state arrays, the kernels two",
    "FTML": "it keeps three state arrays, the kernels two",
    "Nadam": "its momentum schedule is one scalar shared by all keys and advanced once per key update",
    "Adamax": "m / u is 0 / 0 wherever every gradient so far was exactly 0, where the reference writes NaN",
    "SGLD": "it needs a device random-number generator",
    "LBSGD": "it has its own warm-up strategy",
}


class HipsCNNTrainStep:
    """Graph-captured training step of the demo CNN on the HiPS fabric (SGD, Adam, DCASGD, NAG, Signum, RMSProp, AdaGrad, AdaDelta, Ftrl).

    Parameters
    ----------
    net : Gluon network from :func:`build_cnn` (initialised; its parameters are re-homed into the symmetric arena so
          ``net(x)`` / ``save_parameters`` keep working on the live weights) or ``None`` (Xavier init here).
    batch_size : per-worker batch (reference default 32).
    optimizer : ``mx.optimizer.Optimizer`` with a native spec — SGD, Adam, DCASGD, NAG, Signum, RMSProp (``centered=False``), AdaGrad,
          AdaDelta or Ftrl — runs on the global-PS shard (or on every worker with local updates).  Centered RMSProp, FTML, Nadam, Adamax,
          SGLD and LBSGD raise ``ValueError`` with the reason.  Honoured in full:
          its ``lr_scheduler`` (Factor / MultiFactor / Poly / Cosine, with warm-up) is evaluated by the update kernels from the device step
          count, so every replay of the captured step takes the scheduled rate; per-key ``lr_mult`` / ``wd_mult`` (from ``net``'s
          Parameters, else the optimizer's tables) scale each key's update; the step count starts at ``begin_num_update``.  An optimizer
          whose schedule cannot run on the device (any other scheduler, or a subclass that changes a schedule's values) raises
          ``ValueError`` here.  ``set_learning_rate`` changes a constant rate between steps; ``learning_rate`` is the rate of the next update.
    topo : :class:`Topology` (default: from ``WORLD_SIZE`` / ``RANK`` / ``GEOMX_NUM_PARTIES`` / ``DMLC_NUM_GLOBAL_SERVER``).

    ``save_states`` / ``load_states`` checkpoint and resume the whole training state (one ``mx.nd.save`` file, keyed by parameter, so a
    run may resume with another batch size or number of ranks).
    """

    def __init__(self, net=None, batch_size=32, optimizer=None, topo=None, device=None, use_graph=True,
                 use_multicast=True, mode="dist_sync", fused_zero_grad=True, wire_dtype="fp32", dgt=False, dgt_rerank_every=32,
                 update="server", bsc_threshold=None, size_lower_bound=None, hfa=None, loopback=False, lookahead=False):
        """``update='server'`` (examples/cnn.py): the optimizer runs on the global-PS shard inside the exchange kernel.  ``update='local'``
        (examples/cnn_bsc.py / cnn_fp16.py / cnn_mpq.py): the kvstore only aggregates gradients (``set_optimizer`` is not called on it), every
        worker applies its own Adam to the pulled aggregate — one fused arena-optimizer launch.  ``bsc_threshold``: Bi-Sparse between the tiers
        for keys >= ``size_lower_bound`` elements.  ``hfa=(K1, K2)`` (examples/cnn_hfa.py): local Adam on the own gradient every step, party
        average of the weights every K1 steps, global average every K1*K2 steps (reference milestone algebra, kvstore_dist_server.h:959-972).

        ``lookahead=True`` software-pipelines consecutive steps: the launch made by ``step(X[k+1], y[k+1])`` starts at the classifier head of
        batch k (whose convolutions already ran), exchanges the dense keys underneath the convolution backward pass, the conv-key exchange AND
        the forward convolutions of batch k+1, and returns the loss of batch k (``nan`` on the first call; ``flush()`` trains the last batch).
        The arithmetic and its order are unchanged — batch k+1's convolutions still read the conv weights updated by batch k, its head the
        dense weights updated by batch k — only the place where the step is cut into launches moves, so that the two-hop exchange of the
        660 KB dense keys has ~25 us of independent work to hide behind instead of ~9.  (Where the forward kernel also computes dense0, even
        batches <= 32, it reads W0 and so waits for the dense keys' exchange.)"""
        native.require()
        from .. import optimizer as opt
        self.B = B = int(batch_size)
        self.device = device or torch.device("cuda", torch.cuda.current_device())
        self.topo = topo or Topology.from_env()
        self.mode = mode
        self.hfa = tuple(int(v) for v in hfa) if hfa else None
        self.update = "local" if (update == "local" or self.hfa) else "server"
        self.fused_zero_grad = fused_zero_grad   # False keeps the gradients readable after a step (tests / debugging): memset instead
        optimizer = optimizer or opt.Adam(learning_rate=0.01)
        spec = optimizer.spec()
        if spec is None:
            name = type(optimizer).__name__
            why = _NOT_NATIVE.get(name + ("(centered=True)" if getattr(optimizer, "centered", False) else ""), "it has no native spec")
            raise ValueError("optimizer %s cannot run in the update kernels: %s.  Supported: %s" % (name, why, _NATIVE_OPTIMIZERS))
        sched = optimizer.lr_scheduler
        if sched is not None:
            if not hasattr(sched, "device_spec"):
                raise ValueError("lr_scheduler %s cannot run on the device: only Factor / MultiFactor / Poly / Cosine schedules can"
                                 % type(sched).__name__)
            # raises ValueError for a schedule the kernels cannot evaluate.  The base lr is the scheduler's own, as Optimizer._get_lr
            # applies it (the two differ only when the scheduler was attached after the optimizer was made); the engine keeps a copy of the
            # scheduler as it was given, so that `learning_rate` reports what the kernels apply
            spec = dict(spec, lr=float(sched.base_lr), lr_schedule=sched.device_spec())
            sched = copy.copy(sched)
        self.optimizer = optimizer
        self._sched = sched
        self._lr = float(spec["lr"])
        self.layout = ArenaLayout.build(list(enumerate(CNN_PARAM_SHAPES)), mults=_key_mults(optimizer, net))
        self._local_spec = spec if self.update == "local" else None
        self._local_packed = (None, None)      # (spec, OptHyper): _local_opt packs self._local_spec again only when it was replaced
        self.fabric = HipsFabric(self.layout, self.topo, self.device, None if self.update == "local" else spec, use_multicast=use_multicast,
                                 loopback=loopback)
        # the script-level `grad / num_samples`, folded into the push kernel; with local updates the aggregate is also averaged over the workers
        self.fabric.set_push_scale(1.0 / B if self.update == "server" else 1.0 / (B * self.topo.world))
        from ..base import getenv_int
        lower = int(size_lower_bound) if size_lower_bound is not None else getenv_int("MXNET_KVSTORE_SIZE_LOWER_BOUND", 200000)
        fmts = {}
        if wire_dtype in ("fp16", "mpq", "fp8") and self.fabric.protocol == "ll":
            # FP16: every key as halves on the wire (examples/cnn_fp16.py); MPQ: only the keys above MXNET_KVSTORE_SIZE_LOWER_BOUND (cnn_mpq.py:52)
            bound = lower if wire_dtype == "mpq" else 0
            fmts = {i: ("fp8" if wire_dtype == "fp8" else "fp16") for i, sl in enumerate(self.layout.slots) if sl.numel >= bound}
        if bsc_threshold and self.fabric.protocol == "ll":
            fmts.update({i: "bsc" for i, sl in enumerate(self.layout.slots) if sl.numel >= lower})
        self._bsc_threshold = float(bsc_threshold or 0.01) if "bsc" in fmts.values() else 0.0
        if fmts:
            self.fabric.set_wire_formats(fmts, bsc_threshold=float(bsc_threshold or 0.01))
        self._dgt_every = 0
        if dgt and self.fabric.protocol == "ll":
            self.fabric.enable_dgt()
            self._dgt_every = max(1, int(dgt_rerank_every))
        f = self.fabric
        # Key groups ("channels") of the step: the dense keys' gradients are complete long before the convolution backward pass ends, so their
        # exchange runs underneath it on its own stream (two-hop, optimizer sharded over all ranks); the conv keys come last and use the
        # one-hop replicated mode — the only communication left on the critical path (reference ordering: push(idx, priority=-idx),
        # examples/cnn.py:121-125).  GEOMX_STEP_OVERLAP=0 selects the single fused exchange at the end of the step, =1 the channels.
        # The step switches are read here, once: the engine's kernel path does not change after construction.
        env = {k: os.environ[k] for k in STEP_SWITCHES if k in os.environ}
        choose = lambda tail_capable: step_path(B, mode=mode, hfa=bool(self.hfa), update=self.update, lookahead=lookahead, world=self.topo.world,
                                                direct_protocol=f.ll_d is not None, conv_tail_capable=tail_capable, env=env)
        path = choose(False)
        if path.overlap:
            f.add_channel("dense", [4, 5, 6, 7, 8, 9], replicate=False, grid=int(os.environ.get("GEOMX_DENSE_CHANNEL_GRID", 40)) or None)
            f.add_channel("conv", [0, 1, 2, 3], replicate=True)
        if path.single:
            # GEOMX_STEP_OVERLAP=0: ONE exchange of all keys after the backward pass.  GEOMX_STEP_EXCHANGE picks its protocol: `ll` (three-hop
            # hierarchy walk), `sharded` / `replicated` (direct protocol, two hops / one hop)
            f.add_channel(path.single, list(range(10)), replicate=env.get("GEOMX_STEP_EXCHANGE") == "replicated")
        self.P = [f.param_view(i) for i in range(10)]
        self.G = [f.grad_view(i) for i in range(10)]
        if self.update == "local":
            # worker-local weights + optimizer state: the fabric's parameter arena only receives the aggregated gradient (or, with HFA, the
            # averaged weights) in this mode
            n_el = self.layout.total
            self.Wl = torch.zeros(n_el, dtype=torch.float32, device=self.device)
            self.s0l, self.s1l = torch.zeros_like(self.Wl), torch.zeros_like(self.Wl)
            self.opt_state = torch.zeros(4, dtype=torch.int32, device=self.device)
            self.P = [self.layout.view(self.Wl, i) for i in range(10)]
        # resumed training: the device step count (schedule and Adam's bias correction) continues from begin_num_update, as the
        # optimizer's own per-index count does
        begin = int(optimizer.begin_num_update)
        if begin:
            if self.update == "local":
                self.opt_state[0] = begin
            elif mode == "dist_async":
                f.flags.tensor[f.off["async_step"]: f.off["async_step"] + f.tiles] = begin      # the one-sided update counts per tile
            else:
                f.set_opt_step(begin)
        self._init_params(net)
        dev, f32 = self.device, torch.float32
        e = lambda *s, dt=f32: torch.empty(*s, dtype=dt, device=dev)
        # the batch lives in ONE device buffer [x | label | coef] so that the per-step staging -> compute hand-over is a single D2D copy.
        # coef [B] is the per-row gradient coefficient of a short or sample-weighted batch (see step_async); only weighted steps read it
        self.xin = e(B * 28 * 28 + 2 * B)
        self.x, self.lc = self.xin[:B * 784].view(B, 1, 28, 28), self.xin[B * 784:]
        self.label, self.coef = self.lc[:B], self.lc[B:]
        self.a1, self.idx1 = e(B, 16, 12, 12), e(B, 16, 12, 12, dt=torch.uint8)
        self.col1 = e(B * 64, 400)
        self.z2 = e(B, 32, 8, 8)
        self.a2, self.idx2 = e(B, 32, 4, 4), e(B, 32, 4, 4, dt=torch.uint8)
        self.a3, self.a4 = e(B, 256), e(B, 128)
        self.loss, self.logits = e(B), e(B, 10)
        self.dz4, self.dz3, self.da2 = e(B, 128), e(B, 256), e(B, 512)
        self.dl = e(B, 16)          # dlogits, classes padded to 16 (cluster kernel -> dense weight-gradient kernel)
        self.dz2rows, self.dcol1, self.da1 = e(B * 64, 32), e(B * 64, 400), e(B, 16, 12, 12)
        self.loss_host = torch.empty(B, dtype=f32).pin_memory()
        # look-ahead: the head of the launch belongs to the PREVIOUS batch, whose labels and coefficients must outlive the arrival of the next
        # batch in `xin`
        self.lc_cur = torch.empty_like(self.lc) if path.lookahead else self.lc
        self.label_cur, self.coef_cur = self.lc_cur[:B], self.lc_cur[B:]
        self.x_cur = torch.empty_like(self.x) if path.lookahead else self.x        # ... and so must its images (conv0's weight gradient reads them)
        self._primed_batch = (False, B, None)   # look-ahead: (weighted, n, host weights) of the primed batch, whose loss the next launch reports
        self._primed = False
        self._warmed = False        # capture() has run its two eager warm-up steps
        self.graph = None
        self._graph_alt = None
        self._graph_w = {}          # weighted steps: input buffer -> graph, captured on first use
        self._xbufs = [self.xin, None]
        self._side = torch.cuda.Stream(device=self.device)
        # the exchange branch gets a high-priority stream: its (few) CTAs must become resident at once on every rank — they poll each other —
        # instead of queueing behind the convolution-backward CTAs that are launched at the same time
        self._comm = torch.cuda.Stream(device=self.device, priority=-1)
        self.use_graph = use_graph
        self.steps_done = 0
        self.kernels_per_step = 0
        self._ev = None             # evaluate / predict buffers (never shared with the step), grown to the largest N seen
        # whether the conv keys' exchange can run in the backward grid's tail is a property of their channel.  Asked last: the answer
        # allocates the channel's tile list, which would otherwise shift the step's buffers in the allocator.
        if path.overlap and f.channel_fused_args("conv") is not None:
            path = choose(True)
        self.path = path
        self.direct_conv, self.overlap, self.single, self.lookahead = path.direct_conv, path.overlap, path.single, path.lookahead
        self.fused_mlp, self.fused_exchange = path.dense != "gemm", path.bwd == "exchange_tail"
        self._fwd_dense0, self._fwd_head, self._n_fwd = path.dense in ("a3", "dz3"), path.dense == "dz3", path.n_fwd

    # ------------------------------------------------------------------------------------------------------------
    def _init_params(self, net):
        f, topo = self.fabric, self.topo
        if net is not None:
            params = list(net.collect_params().values())
            assert [tuple(p.shape) for p in params] == CNN_PARAM_SHAPES, "network does not match the demo CNN"
            for i, p in enumerate(params):
                f.param_view(i).copy_(p.data()._t.detach().to(self.device))
        else:
            init = initializer.Xavier()
            for i, shape in enumerate(CNN_PARAM_SHAPES):
                host = torch.zeros(shape)
                init(initializer.InitDesc("w%d_%s" % (i, "weight" if len(shape) > 1 else "bias")), host)
                f.param_view(i).copy_(host.to(self.device))
        if topo.world > 1:
            import torch.distributed as dist
            dist.broadcast(f.param.tensor, src=0)      # `init`: rank-0 (master worker) value wins, then barrier
            torch.cuda.synchronize()
            dist.barrier()
        f.load_master_from_param()
        if self.update == "local":
            self.Wl.copy_(f.param.tensor)
            if native.OPT_KINDS[self._local_spec["name"]].s1_is_weight:
                self.s1l.copy_(self.Wl)      # DCASGD's previous weight starts as the initial weight (reference create_state)
        if net is not None:  # re-home the Gluon parameters onto the live arena (zero-copy pull)
            for i, p in enumerate(net.collect_params().values()):
                d = p.data()
                d._data = self.P[i]
                d._ctx_hint = Context("gpu", self.device.index or 0)
                if p.grad_req != "null":
                    d.attach_grad(p.grad_req)
        self.net = net

    # ------------------------------------------------------------------------------------------------------------
    def _local_opt(self, grad_tensor, zero=None):
        """update='local': the worker's arena optimizer (spec ``self._local_spec``) applied to ``grad_tensor``; ``zero`` is cleared."""
        sp, h = self._local_packed
        if sp is not self._local_spec:
            sp = self._local_spec
            # HFA applies the optimizer to the worker's own gradient arena, a sum over the batch: the reference's cnn_hfa.py steps the trainer
            # with `trainer.step(num_samples)`, i.e. rescale_grad / B.  The pulled aggregate of the other local mode is already averaged.
            h = native.pack_hyper(dict(sp, rescale_grad=sp["rescale_grad"] / self.B) if self.hfa else sp)
            self._local_packed = (sp, h)
        native.arena_opt_h(h, self.Wl, grad_tensor, self.s0l, self.s1l, self.layout.total, self.fabric.tile_mult, self.opt_state, zero)

    def _steps(self, weighted=False):
        """The training step of ``self.path`` as an ordered list of (name, stream, launch); `stream` is 'main', 'side' (parallel graph branch
        for weight gradients), 'comm' (a key group's exchange on the high-priority stream), 'join' (main, after the side branch) or 'join_comm'
        (main, after the side branch and the comm stream).  The launches look their kernels, buffers and parameter blocks up when they run.
        ``weighted``: the kernel that produces the dlogits scales row b by ``coef_cur[b]`` (its weighted instance); the launches are the same."""
        n, path = native, self.path
        B, P, G, f = self.B, self.P, self.G, self.fabric
        a2f = self.a2.view(B, 512)
        Wc1, Gc1 = P[2].view(32, 400), G[2].view(32, 400)
        # look-ahead: the forward launch carries the labels and coefficients of its batch to where the next launch's head reads them
        carry = (self.lc, self.lc_cur) if path.lookahead else None
        w = self.coef_cur if weighted else None

        # forward convolutions (the part a look-ahead launch runs for the NEXT batch)
        if path.dense in ("a3", "dz3"):
            def conv_fwd():
                head = dict(wd1=P[6], bd1=P[7], wd2=P[8], bd2=P[9], label=self.label_cur, loss=self.loss, logits=self.logits, a4=self.a4,
                            dz4=self.dz4, dz3=self.dz3, dl=self.dl, weight=w) if path.dense == "dz3" else {}
                if not n.cnn_fwd_dense0(self.x, P[0], P[1], P[2], P[3], P[4], P[5], self.a1, self.idx1, self.a2, self.idx2, self.a3, carry=carry,
                                        x_keep=self.x_cur if path.lookahead else None, **head):
                    raise RuntimeError("cnn_fwd_dense0 does not cover batch %d" % B)
            fwd = [(DIRECT_FWD, "main", conv_fwd)]
        elif path.direct_conv:
            fwd = [(DIRECT_FWD, "main", lambda: n.cnn_fwd(self.x, P[0], P[1], P[2], P[3], self.a1, self.idx1, self.a2, self.idx2, carry=carry,
                                                          x_keep=self.x_cur if path.lookahead else None))]
        else:
            def conv1_fwd():
                # bias + ReLU + 2x2 max-pool in the GEMM epilogue (only the pooled map and its arg-max leave the SM); the two-kernel form is
                # the fallback for geometries the in-warp pooling cannot express
                if not (path.pool_fusion and n.gemm_pool(self.col1, Wc1, self.a2, self.idx2, 8, 8, bias=P[3], relu=True)):
                    n.gemm(self.col1, Wc1, self.z2, bias=P[3], relu=True, store_nchw_hw=64)
                    n.maxpool2x2_fwd(self.z2, self.a2, self.idx2)
                if path.lookahead:
                    self.lc_cur.copy_(self.lc); self.x_cur.copy_(self.x)
            fwd = [(GEMM_FWD[0], "main", lambda: n.conv_relu_pool_im2col_fwd(self.x, P[0], P[1], self.a1, self.idx1, self.col1, 5, 5)),
                   (GEMM_FWD[1], "main", conv1_fwd)]

        # dense chain: forward and backward down to da2, the input of the convolution backward pass
        wgrad = lambda: n.dense_wgrad(a2f, self.a3, self.a4, self.dz4, self.dz3, self.dl, G[4], G[5], G[6], G[7], G[8], G[9])
        if path.dense == "gemm":
            dense = [
                ("dense0 gemm", "main", lambda: n.gemm(a2f, P[4], self.a3, bias=P[5], relu=True)),
                ("dense1 gemm", "main", lambda: n.gemm(self.a3, P[6], self.a4, bias=P[7], relu=True)),
                ("head fwd+bwd", "main", lambda: n.head_fwd_bwd(self.a4, P[8], P[9], self.label_cur, self.loss, self.logits, G[8], G[9], self.dz4, G[7],
                                                                True, weight=w)),
                ("dW1 gemm", "side", lambda: n.gemm(self.dz4, self.a3, G[6], a_mn=True, b_mn=True)),
                ("dz3 gemm (mask,colsum)", "main", lambda: n.gemm(self.dz4, P[6], self.dz3, b_mn=True, mask=self.a3, colsum=G[5])),
                ("dW0 gemm", "side", lambda: n.gemm(self.dz3, a2f, G[4], a_mn=True, b_mn=True)),
                ("da2 gemm", "main", lambda: n.gemm(self.dz3, P[4], self.da2, b_mn=True)),
            ]
        elif path.dense == "a2":
            # dense0 -> dense1 -> classifier -> softmax-CE forward and backward: one cluster launch for the data path (what the convolution
            # backward pass waits for) and one weight-gradient launch on a parallel branch, instead of the seven above
            dense = [(MLP, "main", lambda: n.mlp_chain_data(a2f, P[4], P[5], P[6], P[7], P[8], P[9], self.label_cur, self.loss, self.logits,
                                                            self.da2, self.a3, self.a4, self.dz4, self.dz3, self.dl, weight=w))]
        else:
            dense = [(MLP, "main", lambda: n.dense_tail(self.a3, P[4], P[6], P[7], P[8], P[9], self.label_cur, self.loss, self.logits, self.da2,
                                                        self.a4, self.dz4, self.dz3, self.dl, from_dz3=path.dense == "dz3",
                                                        weight=w if path.dense == "a3" else None))]
        if path.wgrad == "side":
            dense.append((DENSE_WGRAD, "side", wgrad))

        # the dense keys' exchange on the comm stream; the dense weight gradients go in the same step when they are issued there (only a
        # programmatic edge separates the two)
        dense_kv = lambda: f.channel_step("dense", zero_grad=self.fused_zero_grad)
        if path.wgrad == "comm":
            def wgrad_kv(tail=None):
                # tail: the stream of the dense chain's data path, when the comm branch forked before it (see _body).  The exchange writes
                # W0, which that path reads, so it waits for it; the weight gradients do not
                wgrad()
                if tail is not None:
                    torch.cuda.current_stream().wait_stream(tail)
                dense_kv()
                if tail is not None:
                    # in a captured graph the edge from the tail becomes a full one; only the edge from the weight gradients stays
                    # programmatic (see gx_capture_demote_joined_edges)
                    n.capture_demote_joined_edges()
            comm = [(DENSE_WGRAD + " + " + DENSE_KV, "comm", wgrad_kv)]
        else:
            comm = [(DENSE_KV, "comm", dense_kv)] if path.overlap else []

        # convolution backward
        if path.bwd == "exchange_tail":
            # both backward jobs in one heterogeneous grid, and the conv keys' exchange in its tail (the CTAs that finish last serve one tile each)
            def bwd_exchange():
                fused = f.channel_fused_args("conv", zero_grad=self.fused_zero_grad)
                if fused is None:
                    raise RuntimeError("the conv keys' channel can no longer run in the backward grid's tail")
                n.cnn_bwd_exchange(self.x_cur, P[2], self.a1, self.idx1, self.a2, self.idx2, self.da2, G[0], G[1], G[2], G[3], *fused)
            bwd = [(FUSED_BWD, "main", bwd_exchange)]
        elif path.bwd == "one_grid":
            # both backward jobs in one heterogeneous grid: no side-stream fork / join around the convolution backward
            bwd = [(ONE_GRID, "main", lambda: n.cnn_bwd_all(self.x_cur, P[2], self.a1, self.idx1, self.a2, self.idx2, self.da2, G[0], G[1], G[2],
                                                            G[3]))]
        elif path.bwd == "two_launch":
            bwd = [("conv1 wgrad (direct, sparse)", "side", lambda: n.cnn_wgrad1(self.a1, self.a2, self.idx2, self.da2, G[2], G[3])),
                   ("conv1 dgrad + conv0 wgrad (direct)", "main", lambda: n.cnn_bwd(self.x_cur, P[2], self.a1, self.idx1, self.a2, self.idx2,
                                                                                    self.da2, G[0], G[1]))]
        else:
            bwd = [
                ("pool+relu bwd -> rows", "main", lambda: n.pool_relu_bwd_rows(self.da2.view(B, 32, 4, 4), self.a2, self.idx2, self.dz2rows, G[3])),
                ("dWc1 gemm (split-K)", "side", lambda: n.gemm(self.dz2rows, self.col1, Gc1, a_mn=True, b_mn=True, split_k=16, accumulate=True)),
                ("dcol1 gemm", "main", lambda: n.gemm(self.dz2rows, Wc1, self.dcol1, b_mn=True)),
                ("conv0 wgrad + col2im", "main", lambda: n.conv_relu_pool_wgrad_col2im(self.x_cur, self.dcol1, self.a1, self.idx1, G[0], G[1],
                                                                                       CNN_PARAM_SHAPES[0], 5, 5)),
            ]

        # the exchange, after the backward pass and the side branch (unless it runs in the backward grid's tail)
        if path.bwd == "exchange_tail":
            exchange = []
        elif path.exchange in ("conv", "all"):
            exchange = [(EXCH, "join", lambda: f.channel_step(path.exchange, zero_grad=self.fused_zero_grad))]
        elif path.exchange == "local_opt":
            # HFA: no exchange inside the step; the optimizer consumes (and clears) the worker's own gradient arena
            exchange = [(EXCH, "join", lambda: self._local_opt(f.grad.tensor, f.grad.tensor if self.fused_zero_grad else None))]
        elif path.exchange == "async":
            exchange = [(EXCH, "join", lambda: (f.async_step(), f.grad.tensor.zero_() if self.fused_zero_grad else None))]
        else:
            exchange = [(EXCH, "join", lambda: f.fsa_step(zero_grad=self.fused_zero_grad))]

        # update='local': the exchange delivered the aggregated gradient into the fabric's parameter arena; one arena-optimizer launch applies it
        tail = [(LOCAL, "main", lambda: self._local_opt(f.param.tensor))] if path.local_tail else []
        return fwd + dense + comm + bwd + exchange + tail

    def _body(self, stop_after=None, part="all", weighted=False):
        """Issue the step (``part='all'``), only its forward convolutions (``'fwd'``), everything after them (``'rest'``), or the look-ahead
        rotation ``rest(batch k) + fwd(batch k+1)`` (``'rotated'``); ``weighted`` as in :meth:`_steps`."""
        before = native.launch_count
        f = self.fabric
        # the gradient arena is cleared by the previous step's HiPS kernel (fused zero_grad) unless gradients must stay readable
        if not self.fused_zero_grad:
            f.grad.tensor.zero_()
        main, side, comm = torch.cuda.current_stream(), self._side, self._comm
        forked = comm_forked = False
        steps = self._steps(weighted)
        nf, join = self.path.n_fwd, self.path.lookahead_join
        rotated = steps[nf:] + [(name, join if where == "main" else where, fn) for name, where, fn in steps[:nf]]
        steps = {"all": steps, "fwd": steps[:nf], "rest": steps[nf:], "rotated": rotated}[part]
        # from dz3, the forward launches store everything the dense weight gradients read (a2, a3, a4, dz4, dz3, dl) and the tail only
        # turns dz3 into da2: the comm branch forks right after the forward launches, and its exchange joins the tail (see _steps)
        early = part == "all" and self.path.wgrad == "comm" and self.path.dense == "dz3"
        for i, (name, where, fn) in enumerate(steps):
            if stop_after is not None and i >= stop_after:
                break
            if early and i == nf:
                comm.wait_stream(main); comm_forked = True
            if where == "side":      # weight-gradient GEMMs leave the critical path: parallel branch of the captured graph
                side.wait_stream(main)
                with torch.cuda.stream(side):
                    fn()
                forked = True
            elif where == "comm":    # a key group's exchange: third branch, after everything issued so far on main and side (or `early`)
                if not early:
                    comm.wait_stream(main)
                if forked:           # (a stream that has no work of this step yet must not be waited on: it is not part of a graph capture)
                    comm.wait_stream(side)
                with torch.cuda.stream(comm):
                    fn(tail=main) if early else fn()
                comm_forked = True
            else:
                if where in ("join", "join_comm") and forked:
                    main.wait_stream(side); forked = False
                if where == "join_comm" and comm_forked:
                    main.wait_stream(comm); comm_forked = False
                fn()
        if forked:
            main.wait_stream(side)
        if comm_forked:
            main.wait_stream(comm)
        if part in ("all", "rotated"):
            self.kernels_per_step = native.launch_count - before

    def capture(self, weighted=False):
        """Warm up (2 eager steps on a side stream) and capture the step into a CUDA graph.  After ``set_learning_rate`` dropped the graphs,
        only the capture runs: the warm-up steps are real updates and happen once per engine (``weighted``: on the batch in the input buffer
        with its coefficients, see :meth:`_steps`)."""
        if self.graph is not None or not self.use_graph:
            return
        if not self._warmed:
            s = torch.cuda.Stream()
            s.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s):
                for _ in range(2):
                    self._body(weighted=weighted)
                    self.steps_done += 1
            torch.cuda.current_stream().wait_stream(s)
            torch.cuda.synchronize()
            if self._dgt_every:
                self.fabric.dgt_rerank()      # first ranking now: the collective's lazy communicator set-up belongs to the warm-up, not to a timed step
            if self.topo.world > 1:
                import torch.distributed as dist
                dist.barrier()
            self._warmed = True
        if self.lookahead:
            self._prime()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            self._body(part="rotated" if self.lookahead else "all")
        self.graph = g
        self._graph_alt = None
        self._graph_w = {}

    # learning rate ---------------------------------------------------------------------------------------------------
    @property
    def opt_step(self):
        """Number of optimizer updates applied so far (``begin_num_update`` included): the device step count that the schedule and
        Adam's bias correction read.  Reading it synchronises with the device."""
        if self.update == "local":
            return int(self.opt_state[0])
        f = self.fabric
        if self.mode == "dist_async" and not self.hfa:
            return int(f.flags.tensor[f.off["async_step"]: f.off["async_step"] + f.tiles].max())
        return f.opt_step

    @property
    def learning_rate(self):
        """The learning rate of the next update, before Adam's bias correction and the per-key ``lr_mult``: the schedule at
        ``opt_step + 1``, or the constant lr."""
        return self._sched(self.opt_step + 1) if self._sched is not None else self._lr

    def set_learning_rate(self, lr):
        """Set the constant learning rate of the following updates, as ``Optimizer.set_learning_rate`` / ``Trainer.set_learning_rate``
        do (raises ``UserWarning`` when the optimizer has an ``lr_scheduler``: the schedule owns the rate).

        The lr is part of the kernels' parameter blocks, which a captured graph holds: this waits for the device, drops the captured graphs
        and lets the next step capture them again, without the warm-up steps of the first capture (a look-ahead engine keeps its primed
        batch).  Several ranks: every rank calls it with the same value before the same step, as every worker calls its own
        ``Trainer.set_learning_rate`` in the reference; in the replicated channels each rank updates its own replica of the server state
        with the lr it was given."""
        if self._sched is not None:
            raise UserWarning("LRScheduler of the optimizer has already been defined.")
        self.optimizer.set_learning_rate(lr)
        self._lr = float(lr)
        torch.cuda.synchronize(self.device)
        if self.update == "local":
            self._local_spec = dict(self._local_spec, lr=self._lr)
        else:
            self.fabric.set_optimizer(dict(self.fabric.opt_spec, lr=self._lr))
        self.graph = None
        self._graph_alt = None
        self._graph_w = {}

    def _prime(self):
        """Look-ahead: run the forward convolutions of the batch in ``self.x`` so that the next launch can start at the classifier head."""
        if not self._primed:
            self._body(part="fwd")
            self._primed = True

    def flush(self):
        """Look-ahead: train on the batch whose convolutions are already done (the last one enqueued) and return its mean loss."""
        if not (self.lookahead and self._primed):
            return None
        weighted, n, w = self._primed_batch
        self._body(part="rest", weighted=weighted)
        self._primed = False
        self._primed_batch = (False, self.B, None)
        self.steps_done += 1
        if not weighted:
            return float(self.loss.mean())
        loss = self.loss[:n].cpu()
        return float((loss if w is None else loss * w).sum()) / n

    # checkpoints -----------------------------------------------------------------------------------------------------
    def save_states(self, fname):
        """Save the whole training state to ``fname``, as ``gluon.Trainer.save_states`` does for the generic path: waits for the steps
        already enqueued and writes the state after the last completed update.  One ``mx.nd.save`` file (the ``.params`` format, no
        pickle): the live weights under the names ``net.save_parameters`` writes for :func:`build_cnn` (so
        ``build_cnn().load_parameters(fname, ignore_extra=True)`` loads them), and per parameter ``master:`` / ``s0:`` / ``s1:`` /
        ``step:`` (the master weight, both optimizer state slots and the update count: one per key, one per tile with ``dist_async``; with
        ``update='local'`` the worker's own), ``bsc_u:`` / ``bsc_v:`` (Bi-Sparse residuals of every rank), ``dgt_contrib:`` / ``dgt_fmt:``
        and ``dgt:order`` (the DGT ranking), ``batch:x`` / ``batch:label`` (a look-ahead engine's primed batch, one row per rank) and
        ``batch:weight`` (its gradient coefficients ``w_i * B / n``, 0 for padding rows; written only when a rank's primed batch was short or
        weighted, an absent entry meaning all ones), and a ``meta:`` block.  The state is keyed by parameter, whichever rank holds it; what belongs to a worker (HFA's state, the primed
        batches) has one row per rank.

        Several ranks: collective, every rank calls it; rank 0 writes the file, and every rank raises if that fails."""
        state = self._ckpt_state(with_batch=True)
        err = None
        if self.topo.rank == 0:
            try:
                from .. import ndarray as nd
                nd.save(fname, {k: NDArray(torch.from_numpy(np.ascontiguousarray(v))) for k, v in state.items()})
            except Exception as e:                          # the other ranks must learn of it instead of waiting
                err = e
        if self.topo.world > 1:
            import torch.distributed as dist
            status = torch.tensor([err is None], dtype=torch.int32, device=self.device)
            dist.broadcast(status, src=0)
            if err is None and not bool(status[0]):
                raise RuntimeError("%s: rank 0 could not write the checkpoint" % fname)
        if err is not None:
            raise err

    def load_states(self, fname):
        """Resume from a :meth:`save_states` file.  Copies into the engine's buffers in place: the captured CUDA graphs stay valid (an engine
        that has not captured yet runs its warm-up and capture first, so that the warm-up updates do not land on the loaded state).  When
        the file's constant lr differs from the engine's, it is applied through :meth:`set_learning_rate`, which drops the graphs.  A
        look-ahead engine with the saver's batch size, world size and parties primes each rank's own saved batch again; any other engine
        does not train on the saved batches and warns (``flush()`` before saving avoids that).  A restored short or weighted batch trains with
        its saved coefficients; the loss the next step reports for it is the mean over ``B`` of ``coef_i * loss_i``, which equals the mean over
        its ``n`` rows of ``w_i * loss_i``.

        The saving and the loading engine may differ in batch size, world size, parties, global servers and look-ahead; the optimizer kind,
        ``update``, ``mode``, HFA and the accelerators (wire formats, Bi-Sparse, DGT) must match, and HFA and Bi-Sparse also need the same
        world and party count.  A mismatch, or a missing, mis-shaped or mis-typed entry, raises ``ValueError`` naming it before anything
        on the device is written.  Protocol state (packet epochs, counters, ready flags) is not restored.

        Several ranks: collective, every rank calls it; only rank 0 reads the file and broadcasts its contents."""
        torch.cuda.synchronize(self.device)
        meta, layout = self._ckpt_meta(), self._ckpt_layout()
        batch = [("batch:x", (self.topo.world, self.B, 1, 28, 28), np.dtype(np.float32)),
                 ("batch:label", (self.topo.world, self.B), np.dtype(np.float32))]
        data, err, use_batch, use_weight = None, None, False, False
        if self.topo.rank == 0:
            try:
                data = self._ckpt_read(fname, meta, layout)
                use_batch, use_weight = "batch:x" in data, "batch:weight" in data
            except Exception as e:                          # other ranks must not wait for a payload that never comes
                err = e
        if self.topo.world > 1:
            import torch.distributed as dist
            status = torch.tensor([err is None, use_batch, use_weight], dtype=torch.int32, device=self.device)
            dist.broadcast(status, src=0)
            if err is None and not bool(status[0]):
                raise ValueError("%s: the checkpoint was refused on rank 0" % fname)
            use_batch, use_weight = bool(status[1]), bool(status[2])
        if err is not None:
            raise err
        if use_weight:
            batch.append(("batch:weight", (self.topo.world, self.B), np.dtype(np.float32)))
        order = [(n, s, dt) for n, (s, dt) in layout.items()] + (batch if use_batch else [])
        if self.topo.world > 1:
            buf = _pack([data[n] for n, _, _ in order]) if self.topo.rank == 0 else \
                np.empty(sum(int(np.prod(s)) * dt.itemsize for _, s, dt in order), dtype=np.uint8)
            t = torch.from_numpy(buf).to(self.device)
            dist.broadcast(t, src=0)
            data = _unpack(t.cpu().numpy(), order)
        lr = float(data["meta:lr"][0])
        if self._sched is None and lr != self._lr:
            self.set_learning_rate(lr)
        if self.use_graph and not self._warmed:
            self.xin.zero_()
            self.capture()
        self._ckpt_apply(data)
        self._primed = False
        self._primed_batch = (False, self.B, None)
        if use_batch:
            self.x.copy_(torch.from_numpy(data["batch:x"][self.topo.rank]))
            self.label.copy_(torch.from_numpy(data["batch:label"][self.topo.rank]))
            c = data["batch:weight"][self.topo.rank] if use_weight else None
            weighted = c is not None and not bool((c == 1).all())
            if weighted:
                self.coef.copy_(torch.from_numpy(c))
            self._prime()
            self._primed_batch = (weighted, self.B, torch.from_numpy(c.copy()) if weighted else None)
        torch.cuda.synchronize(self.device)

    def _ckpt_meta(self):
        f, t = self.fabric, self.topo
        spec = self._local_spec if self.update == "local" else f.opt_spec
        base = f._dgt_base_fmt if f.dgt_contrib is not None else f.tile_fmt
        i32 = lambda *v: np.array(v, dtype=np.int32)
        return {
            "meta:version": i32(CHECKPOINT_VERSION),
            "meta:opt_kind": i32(native.OPT_KINDS[spec["name"]].code),
            "meta:update": i32(self.update == "local"),
            "meta:mode": i32(self.mode == "dist_async"),
            "meta:hfa": i32(*(self.hfa or (0, 0))),
            "meta:wire_formats": base.cpu().numpy() if base is not None else np.zeros(f.tiles, dtype=np.uint8),
            "meta:bsc_threshold": np.array([self._bsc_threshold], dtype=np.float64),
            "meta:dgt": i32(f.dgt_contrib is not None),
            "meta:topology": i32(t.world, t.num_parties, 0 if t.tile_sharded else t.num_gs),
            "meta:steps_done": np.array([self.steps_done], dtype=np.int64),
            "meta:lr": np.array([self._lr], dtype=np.float64),
        }

    def _ckpt_layout(self):
        """name -> (shape, dtype) of every entry this engine reads from a checkpoint, meta block first (the primed batch aside)."""
        f32, i32 = np.dtype(np.float32), np.dtype(np.int32)
        out = {n: (v.shape, v.dtype) for n, v in self._ckpt_meta().items()}
        f, world = self.fabric, self.topo.world
        row = (world,) if self.hfa else ()
        for i, n in enumerate(CNN_PARAM_NAMES):
            out[n] = (CNN_PARAM_SHAPES[i], f32)
        for i, n in enumerate(CNN_PARAM_NAMES):
            sl = self.layout.slots[i]
            for p in ("master:", "s0:", "s1:"):
                out[p + n] = (row + CNN_PARAM_SHAPES[i], f32)
            if self.update == "local":
                out["step:" + n] = ((world if self.hfa else 1,), i32)
            else:
                out["step:" + n] = ((sl.tiles if self.mode == "dist_async" else 1,), i32)
            if f.bsc_u is not None:
                out["bsc_u:" + n] = out["bsc_v:" + n] = ((world, sl.tiles * 1024), f32)
            if f.dgt_contrib is not None:
                out["dgt_contrib:" + n] = ((sl.tiles,), f32)
                out["dgt_fmt:" + n] = ((sl.tiles,), np.dtype(np.uint8))
        if f.dgt_contrib is not None:
            out["dgt:order"] = ((f.tiles,), i32)
        return out

    def _ckpt_state(self, with_batch):
        """Collective: this engine's state as checkpoint entries (name -> host array), the values of rank 0 where ranks differ."""
        torch.cuda.synchronize(self.device)
        f, L, T = self.fabric, self.layout, self.fabric.tiles
        out = self._ckpt_meta()
        for i, n in enumerate(CNN_PARAM_NAMES):
            out[n] = self.P[i].detach().cpu().numpy()
        per_tile = self.update == "server" and self.mode == "dist_async"
        fs = f.export_state(async_counts=per_tile)
        if self.update == "local":
            # the worker's own optimizer: identical on every rank, except with HFA, where each worker trains on its own gradient
            ranks = (lambda x: np.stack(f.gather_ranks(x))) if self.hfa else (lambda x: x.cpu().numpy())
            fs["w"], fs["s0"], fs["s1"] = ranks(self.Wl), ranks(self.s0l), ranks(self.s1l)
            count = ranks(self.opt_state[:1])
        for i, n in enumerate(CNN_PARAM_NAMES):
            sl = L.slots[i]
            a, t0 = sl.offset, sl.offset // 1024
            shape = CNN_PARAM_SHAPES[i]
            for k, name in (("w", "master:"), ("s0", "s0:"), ("s1", "s1:")):
                v = fs[k][..., a:a + sl.numel]
                out[name + n] = v.reshape(v.shape[:-1] + shape)
            if self.update == "local":
                out["step:" + n] = count.reshape(-1)
            else:
                out["step:" + n] = fs["step"][t0:t0 + (sl.tiles if per_tile else 1)]
            if "bsc_u" in fs:
                out["bsc_u:" + n] = fs["bsc_u"][:, a:a + sl.tiles * 1024]
                out["bsc_v:" + n] = fs["bsc_v"][:, a:a + sl.tiles * 1024]
            if "dgt_contrib" in fs:
                out["dgt_contrib:" + n] = fs["dgt_contrib"][t0:t0 + sl.tiles]
                out["dgt_fmt:" + n] = fs["tile_fmt"][t0:t0 + sl.tiles]
        if "tile_order" in fs:
            out["dgt:order"] = fs["tile_order"]
        # a look-ahead engine is primed on every rank or on none (the ranks make the same calls); each rank primed its own batch
        if with_batch and self.lookahead and self._primed:
            out["batch:x"] = np.stack(f.gather_ranks(self.x_cur))
            out["batch:label"] = np.stack(f.gather_ranks(self.label_cur))
            coef = self.coef_cur if self._primed_batch[0] else torch.ones_like(self.coef_cur)
            coef = np.stack(f.gather_ranks(coef))
            if not (coef == 1).all():
                out["batch:weight"] = coef
        return out

    def _ckpt_read(self, fname, meta, layout):
        """Read and check a checkpoint against this engine's meta block ``meta`` and its entry layout ``layout`` (name -> (shape, dtype)):
        name -> host array, ``ValueError`` for anything malformed or mismatched.  The file is untrusted input."""
        from .. import ndarray as nd
        try:
            raw = nd.load(fname)
        except OSError:
            raise
        except Exception as e:          # the parser's errors on a damaged or foreign file (MXNetError, struct / decoding errors)
            raise ValueError("%s is not a readable NDArray file: %s" % (fname, e)) from e
        if not isinstance(raw, dict):
            raise ValueError("%s holds unnamed arrays, not a training-engine checkpoint" % fname)
        got = {}
        for k, v in raw.items():
            try:
                got[k] = v.asnumpy()
            except Exception as e:
                raise ValueError("checkpoint entry %r cannot be read: %s" % (k, e)) from e

        def entry(name):
            shape, dtype = layout[name]
            if name not in got:
                raise ValueError("checkpoint entry %r is missing" % name)
            have = got[name]
            if have.dtype != dtype or have.shape != tuple(shape):
                raise ValueError("checkpoint entry %r is %s %s; this engine needs %s %s" % (name, have.dtype, have.shape, dtype, tuple(shape)))
            return have

        v = entry("meta:version")
        if int(v[0]) != CHECKPOINT_VERSION:
            raise ValueError("meta:version: unknown checkpoint format version %d (this engine reads %d)" % (int(v[0]), CHECKPOINT_VERSION))
        for n in meta:
            entry(n)
        for n in _MUST_MATCH:
            if not np.array_equal(got[n], meta[n]):
                raise ValueError("%s: the checkpoint has %s, this engine %s" % (n, got[n].tolist(), meta[n].tolist()))
        same_ranks = np.array_equal(got["meta:topology"][:2], meta["meta:topology"][:2])
        if (self.hfa or self._bsc_threshold) and not same_ranks:
            # HFA state belongs to each worker, Bi-Sparse residuals to each party owner: the same ranks must take them up again
            raise ValueError("meta:topology: HFA / Bi-Sparse state was saved by %d ranks in %d parties, this engine has %d in %d"
                             % tuple(got["meta:topology"][:2].tolist() + meta["meta:topology"][:2].tolist()))
        if int(got["meta:steps_done"][0]) < 0:
            raise ValueError("meta:steps_done: negative step count %d" % int(got["meta:steps_done"][0]))
        lr = float(got["meta:lr"][0])
        if self._sched is not None and lr != self._lr:
            raise ValueError("meta:lr: the checkpoint's lr %g differs from the base lr %g of this engine's lr_scheduler" % (lr, self._lr))
        if not np.isfinite(lr):
            raise ValueError("meta:lr: %g is not a learning rate" % lr)
        out = {n: entry(n) for n in layout}
        if self.update == "server" and self.mode != "dist_async":
            # the keys exchanged together share one optimizer step word: they must carry one count
            words = self.fabric.tile_step_words()
            first = {}
            for i, n in enumerate(CNN_PARAM_NAMES):
                w = words[self.layout.slots[i].offset // 1024]
                m, c = first.setdefault(w, (n, int(out["step:" + n][0])))
                if int(out["step:" + n][0]) != c:
                    raise ValueError("step:%s: %d updates, but step:%s, exchanged with it, has %d" % (n, int(out["step:" + n][0]), m, c))
        if "dgt:order" in layout:
            if not np.array_equal(np.sort(out["dgt:order"]), np.arange(self.fabric.tiles)):
                raise ValueError("dgt:order: not a permutation of the %d tiles" % self.fabric.tiles)
            base = meta["meta:wire_formats"]
            for i, n in enumerate(CNN_PARAM_NAMES):
                t0 = self.layout.slots[i].offset // 1024
                fmt, b = out["dgt_fmt:" + n], base[t0:t0 + len(out["dgt_fmt:" + n])]
                if not np.where(b == self.fabric.FMT_BSC, fmt == b, (fmt == b) | (fmt == self.fabric.FMT_F8)).all():
                    raise ValueError("dgt_fmt:%s: formats other than the base format or its fp8 demotion" % n)
        if "batch:weight" in got and "batch:x" not in got:
            raise ValueError("batch:weight without the primed batch batch:x / batch:label it belongs to")
        if "batch:x" in got or "batch:label" in got:
            x, y = got.get("batch:x"), got.get("batch:label")
            if x is None or y is None or x.dtype != np.float32 or y.dtype != np.float32 or x.ndim != 5 or x.shape[2:] != (1, 28, 28) \
                    or y.shape != x.shape[:2] or x.shape[0] != int(got["meta:topology"][0]):
                raise ValueError("batch:x / batch:label: not one batch of (B, 1, 28, 28) fp32 images and B fp32 labels per saving rank")
            wt = got.get("batch:weight")
            if wt is not None and (wt.dtype != np.float32 or wt.shape != y.shape):
                raise ValueError("batch:weight: not one fp32 gradient coefficient per row of batch:label")
            if self.lookahead and same_ranks and x.shape[1] == self.B:
                out["batch:x"], out["batch:label"] = x, y
                if wt is not None:
                    out["batch:weight"] = wt
            else:
                import warnings
                warnings.warn("%s holds the primed batches of %d ranks of batch size %d, which this engine does not train on (it restores "
                              "them only with lookahead=True and the same batch size, world size and parties)" % (fname, x.shape[0], x.shape[1]))
        return out

    def _ckpt_apply(self, data):
        """Write the checked entries ``data`` into this engine's buffers, in place."""
        f, L, me = self.fabric, self.layout, self.topo.rank
        fs = {k: np.zeros(f.n, dtype=np.float32) for k in ("w", "s0", "s1")}
        per_tile = self.update == "server" and self.mode == "dist_async"
        step = np.zeros(f.tiles, dtype=np.int32)
        if "dgt:order" in data:
            fs["dgt_contrib"], fs["tile_fmt"] = np.zeros(f.tiles, dtype=np.float32), np.zeros(f.tiles, dtype=np.uint8)
            fs["tile_order"] = data["dgt:order"]
        if f.bsc_u is not None:
            fs["bsc_u"], fs["bsc_v"] = (np.zeros((self.topo.world, f.n), dtype=np.float32) for _ in range(2))
        row = (lambda v: v[me]) if self.hfa else (lambda v: v)
        for i, n in enumerate(CNN_PARAM_NAMES):
            sl = L.slots[i]
            a, t0 = sl.offset, sl.offset // 1024
            for k, name in (("w", "master:"), ("s0", "s0:"), ("s1", "s1:")):
                fs[k][a:a + sl.numel] = row(data[name + n]).reshape(-1)
            step[t0:t0 + sl.tiles] = row(data["step:" + n])
            if "bsc_u" in fs:
                fs["bsc_u"][:, a:a + sl.tiles * 1024] = data["bsc_u:" + n]
                fs["bsc_v"][:, a:a + sl.tiles * 1024] = data["bsc_v:" + n]
            if "dgt_contrib" in fs:
                fs["dgt_contrib"][t0:t0 + sl.tiles] = data["dgt_contrib:" + n]
                fs["tile_fmt"][t0:t0 + sl.tiles] = data["dgt_fmt:" + n]
        if self.update == "local":
            wl = {k: torch.from_numpy(fs.pop(k)).to(self.device) for k in ("w", "s0", "s1")}
            f.import_state(fs)
            self.Wl.copy_(wl["w"]); self.s0l.copy_(wl["s0"]); self.s1l.copy_(wl["s1"])
            self.opt_state[0] = int(step[0])
        else:
            fs["step"] = step
            f.import_state(fs, async_counts=per_tile)
            for i, n in enumerate(CNN_PARAM_NAMES):
                self.P[i].copy_(torch.from_numpy(data[n]))
        self.steps_done = int(data["meta:steps_done"][0])

    def _bind_input(self, k):
        """Point the step at input buffer ``k`` (0 = ``self.xin``; 1 = the second staging buffer of the host pipeline).  Only matters while
        launches are being issued or captured: a captured graph keeps the buffer it was captured with."""
        buf = self._xbufs[k]
        B = self.B
        self.xin, self.x, self.lc = buf, buf[:B * 784].view(B, 1, 28, 28), buf[B * 784:]
        self.label, self.coef = self.lc[:B], self.lc[B:]
        if not self.lookahead:
            self.x_cur, self.lc_cur, self.label_cur, self.coef_cur = self.x, self.lc, self.label, self.coef

    def _alt_graph(self):
        """The same step captured on input buffer 1: the host pipeline alternates between the two graphs, so a batch is consumed where the
        H2D copy put it (no staging -> compute copy on the critical path of the step)."""
        if self._graph_alt is None:
            self._bind_input(1)
            try:
                s = torch.cuda.Stream()
                s.wait_stream(torch.cuda.current_stream())
                g = torch.cuda.CUDAGraph()
                with torch.cuda.stream(s):
                    with torch.cuda.graph(g, stream=s):
                        self._body()
                torch.cuda.current_stream().wait_stream(s)
            finally:
                self._bind_input(0)
            self._graph_alt = g
        return self._graph_alt

    def _weighted_graph(self, k):
        """The step with the weighted instances of its dlogits kernel (see :meth:`_steps`), captured on input buffer ``k`` on first use, as
        :meth:`_alt_graph` does: no warm-up steps, nothing collective.  The unweighted graphs stay as they are.  The capture is relaxed: it
        may be the first launch of a weighted kernel, whose one-time set-up (shared-memory size, cluster occupancy) runs then."""
        g = self._graph_w.get(k)
        if g is None:
            self._bind_input(k)
            try:
                s = torch.cuda.Stream()
                s.wait_stream(torch.cuda.current_stream())
                g = torch.cuda.CUDAGraph()
                with torch.cuda.stream(s):
                    with torch.cuda.graph(g, stream=s, capture_error_mode="relaxed"):
                        self._body(part="rotated" if self.lookahead else "all", weighted=True)
                torch.cuda.current_stream().wait_stream(s)
            finally:
                self._bind_input(0)
            self._graph_w[k] = g
        return g

    def run_device(self, buf=0, weighted=False):
        """One step on whatever is currently in input buffer ``buf`` (0: ``self.x`` / ``self.label``; device-only, used by the kernel-time
        bench and by the host pipeline).  ``weighted``: the step scales the gradient of row b by ``coef[b]`` of its input buffer (with
        look-ahead, of the primed batch, carried to ``coef_cur``)."""
        # DGT: re-rank before every step whose count of steps already taken (graph warm-up steps included) is a positive multiple of
        # dgt_rerank_every, eager or graphed; capture() also ranks once after its warm-up.  Outside any captured graph: the order and the
        # formats are updated in place
        if self._dgt_every and self.steps_done and self.steps_done % self._dgt_every == 0:
            self.fabric.dgt_rerank()
        if self.use_graph:
            if self.graph is None:
                self.capture(weighted)
            if self.lookahead:
                self._prime()
            if weighted:
                self._weighted_graph(buf).replay()
            else:
                (self._alt_graph() if buf == 1 else self.graph).replay()
        elif buf == 1:
            self._bind_input(1)
            try:
                self._body(weighted=weighted)
            finally:
                self._bind_input(0)
        elif self.lookahead:
            self._prime()
            self._body(part="rotated", weighted=weighted)
        else:
            self._body(weighted=weighted)
        self.steps_done += 1
        if self.hfa and self.steps_done % self.hfa[0] == 0:
            self._hfa_sync(global_round=(self.steps_done // self.hfa[0]) % self.hfa[1] == 0)

    def _hfa_sync(self, global_round):
        """Average the workers' weights inside the party (every K1 steps) or over the whole job (every K1*K2 steps).  Outside the captured
        step: the party round is ONE launch of the party all-reduce kernel, the global round one launch of the fused exchange without an
        optimizer (push_scale 1/parties turns the sum of party means into their mean)."""
        f, topo = self.fabric, self.topo
        if topo.world == 1:
            return
        f.grad.tensor.copy_(self.Wl).mul_(1.0 / topo.party_size)
        if global_round:
            scale = f.push_scale
            f.set_push_scale(1.0 / topo.num_parties)
            f.fsa_step()
            f.set_push_scale(scale)
        else:
            f.party_allreduce(f.grad, f.param, scale=1.0)
        self.Wl.copy_(f.param.tensor)
        f.grad.tensor.zero_()

    def _pipeline(self):
        if not hasattr(self, "_pl"):
            dev, B = self.device, self.B
            # direct mode: the two H2D targets ARE the step's two input buffers (one captured graph each); look-ahead steps keep the
            # single-graph form with a staging -> compute copy
            if self.path.direct_input:
                self._xbufs[1] = torch.empty_like(self.xin)
                stage = [self._xbufs[0], self._xbufs[1]]
            else:
                stage = [torch.empty_like(self.xin) for _ in range(2)]
            self._pl = {
                "h2d": torch.cuda.Stream(device=dev), "d2h": torch.cuda.Stream(device=dev), "stage": stage,
                "sx": [s[:B * 784].view(B, 1, 28, 28) for s in stage], "sy": [s[B * 784:B * 785] for s in stage],
                "sc": [s[B * 785:] for s in stage],
                # what the staging -> compute copy of an unweighted step covers: the images and labels, not the coefficients
                "xl": self.xin[:B * 785], "stage_xl": [s[:B * 785] for s in stage],
                "ready": [torch.cuda.Event() for _ in range(2)], "done": [torch.cuda.Event() for _ in range(2)],
                "ring": [(torch.empty_like(self.loss, device="cpu").pin_memory(), torch.cuda.Event()) for _ in range(4)], "n": 0, "last_loss": None,
            }
        return self._pl

    def _coefficients(self, dst, w, n):
        """Write the gradient coefficients of a batch of ``n`` rows into ``dst`` [B] on the current stream: ``w_i * B / n`` for the real rows
        (``w_i = 1`` when ``w`` is None), 0 for the padding rows.  With the push scale 1 / B the step then contributes
        ``(1/n) * sum_i w_i * grad_i``, the reference loop's ``grad / num_samples`` of a weighted loss."""
        B = self.B
        if w is not None and w.is_cuda:
            dst[n:].zero_()
            dst[:n].copy_(w.reshape(n), non_blocking=True)
            dst[:n].mul_(B / n)
            return
        c = torch.zeros(B, dtype=torch.float32)
        if w is None:
            c[:n] = B / n
        else:
            c[:n] = w.reshape(n).float() * (B / n)
        dst.copy_(c.pin_memory(), non_blocking=True)

    def step_async(self, X, y, sample_weight=None):
        """Public API: enqueue one training step and return a :class:`LossHandle` without waiting for the GPU (the MXNet engine's contract:
        an op returns at once, ``asscalar()`` synchronises).  ``X`` (n,1,28,28) or (n,784) and ``y`` (n,), ``1 <= n <= B``, are host tensors /
        NDArrays (pinned → async H2D) or device tensors; so is ``sample_weight`` (n,) when given.

        A batch of ``n`` rows with weights ``w`` (``w_i = 1`` without ``sample_weight``) contributes the gradient ``(1/n) * sum_i w_i grad_i``
        in every update mode, as the reference loop's ``loss_fn(net(X), y, sample_weight).backward(); kv.push(idx, grad / n)`` does; the
        last, short batch of an epoch (``DataLoader(..., last_batch='keep')``) trains on its own rows.  The step pads the batch to ``B`` rows
        with zero images of label 0 and gives each row the coefficient ``w_i * B / n`` (0 for the padding rows), which the kernel producing
        the dlogits applies.  The handle reports ``w_i * loss_i`` of the ``n`` rows.  A full batch without weights runs exactly the step it
        ran before weights existed.  Ranks may pass different ``n`` and weights in the same step.  ``n`` outside ``[1, B]`` or ``y`` /
        ``sample_weight`` of another length raise ``ValueError`` before anything is enqueued; weights are not checked for finiteness.

        Three streams: the batch is copied host→device on a copy stream into one of the step's TWO input buffers (overlapping the previous
        step's compute); the compute stream replays the graph that was captured on that buffer (two graphs of the same step, alternating —
        no staging→compute copy; ``GEOMX_E2E_DIRECT_INPUT=0`` and look-ahead steps use one graph plus a device-to-device copy), and the
        per-sample loss goes device→host on a third stream into a pinned ring slot; ``handle.item()`` waits for exactly that copy.  A
        training loop therefore launches step i+1 before it reads the loss of step i.  Weighted and short steps replay graphs of their own,
        captured on first use."""
        X = X._t if isinstance(X, NDArray) else X
        y = y._t if isinstance(y, NDArray) else y
        w = sample_weight._t if isinstance(sample_weight, NDArray) else sample_weight
        B = self.B
        n = int(X.shape[0]) if X.dim() > 0 else 0
        if not 1 <= n <= B or X.numel() != n * 784:
            raise ValueError("X must be (n, 1, 28, 28) or (n, 784) with 1 <= n <= %d (the batch size), got %s" % (B, tuple(X.shape)))
        if y.numel() != n:
            raise ValueError("y must hold one label per image: %d labels for %d images" % (y.numel(), n))
        if w is not None and w.numel() != n:
            raise ValueError("sample_weight must hold one weight per image: %d weights for %d images" % (w.numel(), n))
        weighted = w is not None or n < B
        pl = self._pipeline()
        i = pl["n"]; b = i % 2
        pl["n"] = i + 1
        main = torch.cuda.current_stream()
        # a short batch fills the first n rows of the input buffer and clears the rest; a full one is copied as it always was
        if X.is_cuda:
            if n < B:
                self.x[:n].copy_(X.reshape(n, 1, 28, 28), non_blocking=True)
                self.label[:n].copy_(y.reshape(n), non_blocking=True)
                self.x[n:].zero_(); self.label[n:].zero_()
            else:
                self.x.copy_(X.reshape(self.x.shape), non_blocking=True)
                self.label.copy_(y.reshape(self.label.shape), non_blocking=True)
            if weighted:
                self._coefficients(self.coef, w, n)
        else:
            h2d = pl["h2d"]
            if i >= 2:
                h2d.wait_event(pl["done"][b])              # staging buffer b was handed over by step i-2
            if w is not None and w.is_cuda:
                h2d.wait_stream(main)                      # the weights come from work on the compute stream
            with torch.cuda.stream(h2d):
                if n < B:
                    pl["sx"][b][:n].copy_(X.reshape(n, 1, 28, 28), non_blocking=True)
                    pl["sy"][b][:n].copy_(y.reshape(n), non_blocking=True)
                    pl["sx"][b][n:].zero_(); pl["sy"][b][n:].zero_()
                else:
                    pl["sx"][b].copy_(X.reshape(self.x.shape), non_blocking=True)
                    pl["sy"][b].copy_(y.reshape(self.label.shape), non_blocking=True)
                if weighted:
                    self._coefficients(pl["sc"][b], w, n)
                pl["ready"][b].record(h2d)
            main.wait_event(pl["ready"][b])
            if not self.path.direct_input:
                if weighted:
                    self.xin.copy_(pl["stage"][b], non_blocking=True)
                else:
                    pl["xl"].copy_(pl["stage_xl"][b], non_blocking=True)
        w_host = None
        if w is not None:
            # the weights the loss is reported with (a host copy, taken in stream order when they live on the device)
            if w.is_cuda:
                w_host = torch.empty(n, dtype=torch.float32).pin_memory()
                w_host.copy_(w.reshape(n), non_blocking=True)
            else:
                w_host = w.reshape(n).float().clone()
        if pl["last_loss"] is not None:
            main.wait_event(pl["last_loss"])                # the loss buffer of the previous step has been read out
        if self.lookahead and not self._primed:
            # first batch of a look-ahead run: only its convolutions can run yet (after the graph warm-up, which also uses this batch);
            # there is no finished step to report
            if self.use_graph and self.graph is None:
                self.capture(weighted)
            self._prime()
            self._primed_batch = (weighted, n, w_host)
            pl["done"][b].record(main)
            return LossHandle(None, None)
        if self.lookahead:
            # the launch trains the primed batch (its head runs now) and primes this one
            (run_weighted, ln, lw), self._primed_batch = self._primed_batch, (weighted, n, w_host)
        else:
            run_weighted, ln, lw = weighted, n, w_host
        self.run_device(buf=b if (not X.is_cuda and self.path.direct_input) else 0, weighted=run_weighted)
        pl["done"][b].record(main)
        host, ev = pl["ring"][i % 4]
        d2h = pl["d2h"]
        d2h.wait_event(pl["done"][b])
        with torch.cuda.stream(d2h):
            host.copy_(self.loss, non_blocking=True)
            ev.record(d2h)
        pl["last_loss"] = ev
        return LossHandle(host, ev, ln, lw)

    def step(self, X, y, sample_weight=None):
        """Public API: one training step; returns the mean (weighted) loss as a Python float (forces the D2H read of the per-sample loss).
        Arguments as in :meth:`step_async`."""
        return self.step_async(X, y, sample_weight).item()

    # evaluation -----------------------------------------------------------------------------------------------------
    def _eval_launch(self, X, y, want_logits=False):
        """Stage ``X`` (and ``y``) and issue the one-launch forward pass of the live weights (``native.cnn_eval``) on the current stream.
        Returns N, the logits (a new tensor, or None), the per-sample loss and the correct flags (None without ``y``)."""
        X = X._t if isinstance(X, NDArray) else X
        y = y._t if isinstance(y, NDArray) else y
        N = int(X.shape[0]) if X.dim() > 0 else 0
        if N < 1 or X.numel() != N * 784:
            raise ValueError("X must be (N, 1, 28, 28) or (N, 784) with N >= 1, got %s" % (tuple(X.shape),))
        if y is not None and y.numel() != N:
            raise ValueError("y must hold one label per image: %d labels for %d images" % (y.numel(), N))
        ev = self._ev
        if ev is None or ev["cap"] < N:
            e = lambda n, dt=torch.float32: torch.empty(n, dtype=dt, device=self.device)
            ev = self._ev = {"cap": N, "x": e(N * 784), "label": e(N), "loss": e(N), "pred": e(N, torch.int32), "correct": e(N, torch.int32)}

        def staged(t, buf):          # CUDA fp32 contiguous: used in place; anything else is copied (async from pinned memory) and converted
            if t.is_cuda and t.device == self.device and t.dtype == torch.float32 and t.is_contiguous():
                return t
            return buf.copy_(t.reshape(buf.shape), non_blocking=True)

        x = staged(X, ev["x"][:N * 784].view(N, 1, 28, 28))
        label = None if y is None else staged(y, ev["label"][:N])
        loss, correct = (None, None) if y is None else (ev["loss"][:N], ev["correct"][:N])
        logits = torch.empty(N, 10, dtype=torch.float32, device=self.device) if want_logits else None
        native.cnn_eval(x, *self.P, label, logits, loss, ev["pred"][:N], correct)
        return N, logits, loss, correct

    def evaluate_async(self, X, y):
        """Public API: score the **live** weights (``self.P``: the fabric's parameter arena with ``update='server'``, the worker's own
        ``Wl`` with ``update='local'`` / HFA) on ``X`` (N,1,28,28) or (N,784) and labels ``y`` (N,), float or int, for any N >= 1, and return
        an :class:`EvalHandle` without waiting for the GPU.  ``X`` / ``y`` may be host tensors (pinned: async H2D), CUDA tensors (used in
        place when contiguous fp32) or NDArrays.

        The whole forward pass, per-sample softmax-CE loss and arg-max run as ONE kernel launch (``cnn_eval_kernel``) on the current stream,
        so it sees the weights after every step enqueued before it: with ``lookahead=True`` the weights after the last completed update (the
        next batch's convolutions, already run, do not change them); the overlapped exchange channels are joined into that stream within the
        step.  Evaluation has buffers of its own and writes nothing the training step reads.  A label that is not an integer in [0, 10)
        scores a NaN loss and counts as wrong.  The totals are summed from the per-sample results in a fixed order: the loss in fp64, the
        correct samples as an exact integer count.  Rank-local: each rank scores what it is given."""
        if y is None:
            raise ValueError("evaluate needs labels; predict(X) gives the logits alone")
        N, _, loss, correct = self._eval_launch(X, y)
        tot = torch.stack((loss.double().sum(), correct.sum().double()))
        host = torch.empty(2, dtype=torch.float64).pin_memory()
        host.copy_(tot, non_blocking=True)
        event = torch.cuda.Event()
        event.record()
        return EvalHandle(host, event, N)

    def evaluate(self, X, y):
        """Public API: ``evaluate_async(X, y).item()`` — ``(mean_loss, accuracy)`` of the live weights as Python floats."""
        return self.evaluate_async(X, y).item()

    def predict(self, X):
        """Public API: logits [N, 10] (a new CUDA tensor) of the live weights for ``X`` (N,1,28,28) or (N,784); one launch on the current
        stream, ordered after the steps enqueued before it, as in :meth:`evaluate_async`."""
        return self._eval_launch(X, None, want_logits=True)[1]

    # reference semantics helpers ------------------------------------------------------------------------------------
    def params_numpy(self):
        return [p.detach().cpu().numpy().copy() for p in self.P]

    def h2d_bytes_per_step(self):
        return self.x.numel() * 4 + self.label.numel() * 4

    def d2h_bytes_per_step(self):
        return self.loss.numel() * 4
