"""The one-rank exchange (``hips_fsa_step_single_kernel``) against the fp64 update reference of ``tests/_update_ref.py``.

A channel launch runs one CTA per active tile and stages the tile before its grid dependency resolves: the tile index, its multipliers and
the step size into registers, the master weights, optimizer state and state words into L2.  These tests show that nothing of that staging
can be stale:

  1. two channels, launched back to back in a captured graph after the copy that writes their gradients, over several replays: keys with
     (lr_mult, wd_mult) other than 1, a constant and a scheduled lr, with and without the fused gradient clearing;
  2. one channel launched twice back to back (the second launch depends on the first, which writes everything the second one stages);
  3. a new lr (``set_optimizer``, what ``HipsCNNTrainStep.set_learning_rate`` calls) and restored server state (``import_state``, what
     ``load_states`` calls) between steps.
"""
import numpy as np
import pytest
import torch

from geomx_b200 import lr_scheduler as S

import _update_ref as R
from _cnn_ref import cleanup, dev, nat  # noqa: F401  (nat: fixture)
from _update_harness import FAB_SPECS, KEY_MULTS, KEY_SIZES, PUSH_SCALE, _fab_grads, _fab_init, _fabric, clean_env  # noqa: F401

pytestmark = pytest.mark.gpu

TOL = R.DISP_TOL
CHANNELS = {"a": [0, 2, 4], "b": [1, 3, 5]}       # 1 + 1 + 5 tiles and 1 + 2 + 69 tiles


def _sched(base):
    """Linear warm-up over 2 updates, then a halving at update 4: every update of a 6-update run has its own lr."""
    return S.MultiFactorScheduler(step=[4], factor=0.5, base_lr=base, warmup_steps=2, warmup_begin_lr=base / 10)


def _fp32_sched(sched):
    d = sched.device_spec()
    f32 = lambda x: float(np.float32(x))
    return S.MultiFactorScheduler(d["milestones"], f32(d["factor"]), f32(sched.base_lr), warmup_steps=d["warmup_steps"],
                                  warmup_begin_lr=f32(d["warmup_begin_lr"]), warmup_mode=d["warmup_mode"])


def _check(f, W0, ref, stores, keys=None):
    keys = range(len(KEY_SIZES)) if keys is None else keys
    W = [f.layout.view(f.w, i) for i in keys]
    e_w = R.displacement_err(W, [W0[i] for i in keys], [ref.w[i] for i in keys], stores=stores)
    e_s0 = max(R.rel(f.layout.view(f.s0, i), ref.s0[i]) for i in keys)
    e_s1 = max(R.rel(f.layout.view(f.s1, i), ref.s1[i]) for i in keys) if ref.h["kind"] != "sgd" else 0.0
    assert all(torch.equal(f.param_view(i), f.layout.view(f.w, i)) for i in keys), "parameter arena differs from the master weights"
    return max(e_w, e_s0, e_s1)


@pytest.mark.parametrize("zero_grad", [False, True], ids=["keep-grad", "zero-grad"])
@pytest.mark.parametrize("sched", [False, True], ids=["const-lr", "sched-lr"])
@pytest.mark.parametrize("kind", ["sgd", "adam"])
def test_two_channels_captured(nat, clean_env, kind, sched, zero_grad):
    spec = dict(FAB_SPECS[kind])
    sch = _sched(spec["lr"]) if sched else None
    f = _fabric(dict(spec, lr_schedule=sch.device_spec()) if sched else spec, False)
    try:
        assert f.topo.world == 1 and not f.loopback
        g = torch.Generator().manual_seed(7 + 2 * sched + zero_grad + len(kind))
        W0 = _fab_init(f, g)
        for name, keys in CHANNELS.items():
            ch = f.add_channel(name, keys, replicate=True)
            assert ch["list"].tolist() == torch.nonzero(ch["mask"]).flatten().tolist()
        src = torch.zeros_like(f.grad.tensor)
        ref = R.UpdateRef(spec, W0, mults=KEY_MULTS, push_scale=PUSH_SCALE)
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.stream(s), torch.cuda.graph(graph):
            f.grad.tensor.copy_(src)
            f.channel_step("a", zero_grad=zero_grad)
            f.channel_step("b", zero_grad=zero_grad)
        torch.cuda.synchronize()
        ref_sched = _fp32_sched(sch) if sched else None
        for k in range(1, 7):
            grads = _fab_grads(g)
            for i, x in enumerate(grads):
                f.layout.view(src, i).copy_(x)
            graph.replay()
            torch.cuda.synchronize()
            if sched:
                ref.h["lr"] = ref_sched(k)
            ref.step(grads)
            assert all(int(f.state[n][2]) == k and int(f.state[n][0]) == k and int(f.state[n][1]) == 0 for n in CHANNELS)
            cleared = all(bool((f.grad_view(i) == 0).all()) for i in range(len(KEY_SIZES)))
            kept = all(torch.equal(f.grad_view(i).cpu(), x) for i, x in enumerate(grads))
            assert (cleared and not kept) if zero_grad else kept
            e = _check(f, W0, ref, stores=k)
            assert e < TOL, (k, e)
        print("\n  two channels %s %s %s: %.1e" % (kind, "sched" if sched else "const", "zero" if zero_grad else "keep", e))
    finally:
        del f
        cleanup()


@pytest.mark.parametrize("graph", [False, True], ids=["eager", "graph"])
@pytest.mark.parametrize("kind", ["sgd", "adam", "dcasgd"])
def test_same_channel_back_to_back(nat, clean_env, kind, graph):
    """The same channel twice in a row on the same gradient: the second launch depends on the first, which writes the master weights,
    optimizer state and step words that the second one stages before its grid dependency resolves."""
    spec = FAB_SPECS[kind]
    f = _fabric(spec, False)
    try:
        g = torch.Generator().manual_seed(40 + len(kind) + graph)
        W0 = _fab_init(f, g)
        f.add_channel("c", list(range(len(KEY_SIZES))), replicate=True)
        ref = R.UpdateRef(spec, W0, mults=KEY_MULTS, push_scale=PUSH_SCALE)
        twice = lambda: (f.channel_step("c"), f.channel_step("c"))
        cg = None
        if graph:
            s = torch.cuda.Stream()
            s.wait_stream(torch.cuda.current_stream())
            cg = torch.cuda.CUDAGraph()
            with torch.cuda.stream(s), torch.cuda.graph(cg):
                twice()
            torch.cuda.synchronize()
        for k in range(1, 4):
            grads = _fab_grads(g)
            for i, x in enumerate(grads):
                f.grad_view(i).copy_(x)
            torch.cuda.synchronize()
            cg.replay() if graph else twice()
            torch.cuda.synchronize()
            ref.step(grads)
            ref.step(grads)
            assert int(f.state["c"][2]) == 2 * k and f.opt_step == 2 * k
            e = _check(f, W0, ref, stores=2 * k)
            assert e < TOL, (k, e)
        print("\n  back to back %s %s: %.1e" % (kind, "graph" if graph else "eager", e))
    finally:
        del f
        cleanup()


@pytest.mark.parametrize("kind", ["sgd", "adam"])
def test_lr_and_state_changes_between_steps(nat, clean_env, kind):
    """Steps 1-2, a new lr, steps 3-4, the server state saved after step 2 restored, steps 5-6 (replaying from step 3 on, at the new lr):
    the launches must stage the lr and the state the host set, not what the previous launch left."""
    spec = dict(FAB_SPECS[kind])
    f = _fabric(spec, False)
    try:
        g = torch.Generator().manual_seed(70 + len(kind))
        W0 = _fab_init(f, g)
        f.add_channel("a", CHANNELS["a"], replicate=True)
        f.add_channel("b", CHANNELS["b"], replicate=True)
        ref = R.UpdateRef(spec, W0, mults=KEY_MULTS, push_scale=PUSH_SCALE)
        stores = 0

        def step(grads):
            nonlocal stores
            for i, x in enumerate(grads):
                f.grad_view(i).copy_(x)
            f.channel_step("a")
            f.channel_step("b")
            torch.cuda.synchronize()
            ref.step(grads)
            stores += 1
            e = _check(f, W0, ref, stores)
            assert e < TOL, (stores, e)

        for _ in range(2):
            step(_fab_grads(g))
        saved, saved_ref = f.export_state(), [[t.clone() for t in ts] for ts in (ref.w, ref.s0, ref.s1)] + [list(ref.t)]
        new_lr = spec["lr"] * 0.3
        f.set_optimizer(dict(spec, lr=new_lr))
        ref.h["lr"] = float(np.float32(new_lr))
        later = [_fab_grads(g) for _ in range(2)]
        for grads in later:
            step(grads)
        f.import_state(saved)
        ref.w, ref.s0, ref.s1, ref.t = saved_ref
        assert f.opt_step == 2
        for grads in later:
            step(grads)
        assert f.opt_step == 4
    finally:
        del f
        cleanup()
