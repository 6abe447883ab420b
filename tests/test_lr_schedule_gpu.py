"""Learning-rate schedules evaluated on the device (``sched_lr`` / ``step_lr`` in ``csrc/kernels/optim.cuh``) against the Python schedules
of ``lr_scheduler.py`` and the fp64 update reference of ``tests/_update_ref.py``:

  1. the device schedule itself, every step 1..600 of every class, through ``arena_opt`` (SGD, g = 1, w zeroed: w = -lr_t);
  2. ``arena_opt`` with Adam, SGD-momentum and DCASGD under a schedule;
  3. fabric rounds under a schedule on every exchange path;
  4. training-engine cases under a schedule, advanced with the engine's own gradients, with the mutations a schedule bug would produce;
  5. per-key multipliers and the resume offset ``begin_num_update``;
  6. ``HipsCNNTrainStep.set_learning_rate`` on captured graphs, a look-ahead engine and the two-graph input path;
  7. the refusal of a schedule the device cannot evaluate.
"""
import numpy as np
import pytest
import torch

import geomx_b200 as mx
from geomx_b200 import lr_scheduler as S

import _update_ref as R
from _cnn_ref import cleanup, dev, nat  # noqa: F401  (nat: fixture)
from _update_harness import (ENGINE_CASES, FAB_PATHS, FAB_SPECS, KEY_MULTS, KEY_SIZES, MIXED_FMTS, PUSH_SCALE, TOL, _batches,  # noqa: F401
                             _clip_for, _engine_ref, _fab_grads, _fab_init, _fabric, _snapshot, clean_env, half_ulps)

pytestmark = pytest.mark.gpu
f32 = lambda x: float(np.float32(x))


def _fp32_copy(sched):
    """The same schedule with every hyper-parameter rounded to fp32, as the kernels receive it (evaluated in fp64 by Python)."""
    d = sched.device_spec()
    wu = dict(warmup_steps=d["warmup_steps"], warmup_begin_lr=f32(d["warmup_begin_lr"]), warmup_mode=d["warmup_mode"])
    base = f32(sched.base_lr)
    if d["kind"] == "factor":
        return S.FactorScheduler(d["step"], f32(d["factor"]), f32(d["stop_factor_lr"]), base, **wu)
    if d["kind"] == "multifactor":
        return S.MultiFactorScheduler(d["milestones"], f32(d["factor"]), base, **wu)
    if d["kind"] == "poly":
        return S.PolyScheduler(d["max_update"], base, f32(d["pwr"]), f32(d["final_lr"]), **wu)
    return S.CosineScheduler(d["max_update"], base, f32(d["final_lr"]), **wu)


# ============================================================================================================ 1. the schedule itself
WU = [dict(warmup_steps=40, warmup_begin_lr=0.003, warmup_mode="linear"), dict(warmup_steps=25, warmup_begin_lr=0.004, warmup_mode="constant")]
SCHEDULES = {
    "factor": lambda wu: S.FactorScheduler(step=30, factor=0.8, stop_factor_lr=0.002, base_lr=0.1, **wu),       # stop binds from k = 18
    "factor-nostop": lambda wu: S.FactorScheduler(step=7, factor=0.97, stop_factor_lr=1e-9, base_lr=0.05, **wu),
    "multifactor": lambda wu: S.MultiFactorScheduler(step=[41, 100, 101, 250, 599], factor=0.45, base_lr=0.1, **wu),
    "poly": lambda wu: S.PolyScheduler(max_update=400, base_lr=0.1, pwr=2, final_lr=0.001, **wu),
    "poly-sqrt": lambda wu: S.PolyScheduler(max_update=550, base_lr=0.1, pwr=0.5, final_lr=0.0, **wu),
    "cosine": lambda wu: S.CosineScheduler(max_update=500, base_lr=0.1, final_lr=0.0, **wu),
    "cosine-final": lambda wu: S.CosineScheduler(max_update=333, base_lr=0.02, final_lr=0.002, **wu),
}


def _device_lrs(nat, sched, t0, count):
    """lr_t of updates t0+1 .. t0+count as the device evaluates it: one 1024-float tile, SGD without momentum, wd 0, rescale 1, g = 1 and w
    zeroed before every launch, so that the launch leaves w = -lr_t."""
    d = sched.device_spec()
    w = torch.zeros(1024, device=dev())
    g = torch.ones(1024, device=dev())
    step_state = torch.tensor([t0, 0], dtype=torch.int32, device=dev())
    out = torch.empty(count, device=dev())
    for i in range(count):
        w.zero_()
        nat.arena_opt("sgd", w, g, None, None, 1024, None, f32(sched.base_lr), 0.0, 1.0, -1.0, 0.0, 0.9, 0.999, 1e-8, 0.04, step_state,
                      schedule=d)
        out[i:i + 1].copy_(w[:1])
    torch.cuda.synchronize()
    assert int(step_state[0]) == t0 + count
    return (-out).double().cpu()


@pytest.mark.parametrize("wu", [0, 1], ids=["linear-warmup", "constant-warmup"])
@pytest.mark.parametrize("name", list(SCHEDULES))
def test_device_schedule_every_step(nat, name, wu):
    """Every update t = 1..600 (warm-up end, factor steps, milestones, max_update and beyond inside the range), and 300 updates from
    t = 100 001 (a resumed run): |lr_dev - lr_fp64| <= 1e-6 lr_fp64.  A boundary off by one step moves lr by far more."""
    sched = SCHEDULES[name](WU[wu])
    ref = _fp32_copy(sched)
    for t0, count in ((0, 600), (100000, 300)):
        got = _device_lrs(nat, sched, t0, count)
        want = torch.tensor([ref(t) for t in range(t0 + 1, t0 + count + 1)], dtype=torch.float64)
        err = (got - want).abs()
        bad = torch.nonzero(err > 1e-6 * want.abs()).flatten()
        assert bad.numel() == 0, [(t0 + 1 + int(i), float(got[i]), float(want[i])) for i in bad[:5]]
        # the schedule really varies inside the range (so that an off-by-one would show)
        if t0 == 0:
            assert float(want.max()) > 1.5 * float(want.min()), name
    shifted = torch.tensor([ref(t) for t in range(0, 600)], dtype=torch.float64)        # a device evaluating the schedule at t - 1
    assert bool(((_device_lrs(nat, sched, 0, 600) - shifted).abs() > 1e-6 * shifted.abs()).any())


def test_device_schedule_stop_factor_binds(nat):
    sched = SCHEDULES["factor"](WU[0])
    got = _device_lrs(nat, sched, 0, 600)
    assert float(got[-1]) == f32(0.002) and float(got[550]) == f32(0.002)         # t = 541 on: 0.1 * 0.8^18 < 0.002
    assert float(got[500]) > 1.3 * f32(0.002)


# ============================================================================================================ 2. arena_opt under a schedule
ARENA_SPECS = {
    "adam": dict(name="adam", lr=0.01, wd=0.02, rescale_grad=0.5, clip_gradient=0.3, beta1=0.9, beta2=0.999, epsilon=1e-8),
    "sgd": dict(name="sgd", lr=0.1, wd=0.02, rescale_grad=0.5, clip_gradient=0.3, momentum=0.9),
    "dcasgd": dict(name="dcasgd", lr=0.1, wd=0.02, rescale_grad=0.5, clip_gradient=0.3, momentum=0.9, lamda=5.0),
}


def _ms(base):
    """Linear warm-up over 3 updates, then two milestones: every update of an 8-update run has its own lr."""
    return S.MultiFactorScheduler(step=[4, 6], factor=0.5, base_lr=base, warmup_steps=3, warmup_begin_lr=base / 10)


@pytest.mark.parametrize("kind", ["sgd", "adam", "dcasgd"])
def test_arena_opt_scheduled(nat, kind):
    spec = ARENA_SPECS[kind]
    sched = _ms(spec["lr"])
    ref_sched = _fp32_copy(sched)
    h = R.hyper(spec)
    g = torch.Generator().manual_seed(11 + len(kind))
    tiles = 5
    n = tiles * 1024
    tm = torch.stack([0.25 + 2 * torch.rand(tiles, generator=g), 2 * torch.rand(tiles, generator=g)], 1).float()
    lm, wm = tm[:, 0].double().repeat_interleave(1024), tm[:, 1].double().repeat_interleave(1024)
    w0 = torch.randn(n, generator=g) * 0.1
    w, s0 = w0.to(dev()), torch.zeros(n, device=dev())
    s1 = w0.clone().to(dev()) if kind == "dcasgd" else torch.zeros(n, device=dev())
    rw, rs0, rs1 = w0.double(), torch.zeros(n, dtype=torch.float64), s1.double().cpu()
    step_state = torch.zeros(2, dtype=torch.int32, device=dev())
    for t in range(1, 9):
        gr = torch.randn(n, generator=g)
        nat.arena_opt(kind, w, gr.to(dev()), s0, s1, n, tm.to(dev()), h["lr"], h["wd"], h["rescale"], h["clip"], h["momentum"], h["beta1"],
                      h["beta2"], h["eps"], h["lamda"], step_state, schedule=sched.device_spec())
        R.update(dict(h, lr=ref_sched(t)), rw, gr.double(), rs0, rs1, t, lm, wm)
        torch.cuda.synchronize()
        e = R.displacement_err([w], [w0], [rw], stores=t)
        assert e < TOL, (kind, t, e)
    print("\n  arena_opt %s scheduled: %.1e" % (kind, e))


# ============================================================================================================ 3. fabric rounds
@pytest.mark.parametrize("kind", ["sgd", "adam"])
@pytest.mark.parametrize("path,loopback,fmts", FAB_PATHS, ids=["%s%s" % (p, "-lp" if lb else "") + ("-fp16fp8" if f else "")
                                                              for p, lb, f in FAB_PATHS])
def test_fabric_rounds_scheduled(nat, clean_env, path, loopback, fmts, kind):
    """Eight rounds across the end of warm-up and two milestones; the reference takes the scheduled lr of each round."""
    spec = dict(FAB_SPECS[kind])
    sched = _ms(spec["lr"])
    ref_sched = _fp32_copy(sched)
    f = _fabric(dict(spec, lr_schedule=sched.device_spec()), loopback, fmts)
    try:
        g = torch.Generator().manual_seed(500 + 10 * len(kind) + 2 * loopback + (fmts is None))
        W0 = _fab_init(f, g)
        if path in ("sharded", "replicated", "direct-sharded", "direct-replicated"):
            f.add_channel("c", list(range(len(KEY_SIZES))), replicate=path.endswith("replicated"))
            run = lambda: f.channel_step("c")
        else:
            run = lambda: f.fsa_step()
        ref = R.UpdateRef(spec, W0, mults=KEY_MULTS, push_scale=PUSH_SCALE, fmts=fmts, round_after_scale=path == "ll")
        for k in range(1, 9):
            grads = _fab_grads(g)
            for i, x in enumerate(grads):
                f.grad_view(i).copy_(x)
            run()
            torch.cuda.synchronize()
            ref.h["lr"] = ref_sched(k)
            ref.step(grads)
            assert f.opt_step == k and not f.check_protocol_errors()
            W = [f.layout.view(f.w, i) for i in range(len(KEY_SIZES))]
            e_w = R.displacement_err(W, W0, ref.w, stores=k)
            assert e_w < TOL, (k, e_w)
            if fmts is not None and loopback and path != "direct-replicated":
                P = [f.param_view(i) for i in range(len(KEY_SIZES))]
                assert max(half_ulps(P[i], ref.w[i]) if fm != "fp32" else 0.0 for i, fm in enumerate(fmts)) <= 2.0
        print("\n  %-18s %-4s scheduled  w %.1e" % (path + ("-lp" if loopback else ""), kind, e_w))
    finally:
        del f
        cleanup()


# ============================================================================================================ 4. engine cases
ENGINE_SCHED_CASES = ["A-adam-graph", "C-adam", "single-adam", "loopback-ov0-adam", "loopback-ov1-sgd", "async-adam", "local-adam", "hfa-sgd"]


def _case_opt(kind, sched_fn, **extra):
    s = dict(R.CASE_SPECS[kind])
    kw = dict(learning_rate=s["lr"], wd=s["wd"], rescale_grad=s["rescale_grad"], lr_scheduler=sched_fn(s["lr"]), **extra)
    if kind == "adam":
        return mx.optimizer.Adam(**kw)
    if kind == "sgd":
        return mx.optimizer.SGD(momentum=s["momentum"], **kw)
    return mx.optimizer.DCASGD(momentum=s["momentum"], lamda=s["lamda"], **kw)


def _engine_sched_run(name, clean_env, optimizer, steps=6, seed=0, net=None):
    """An engine case of test_update_paths_gpu.ENGINE_CASES with ``optimizer``; gradients kept readable; a graph case is captured once and
    its warm-up undone.  Returns (engine, P0, per-step gradient sums, per-step (params, master), spec with the case's clip)."""
    B, env, kind, kw, graph, want, attrs = ENGINE_CASES[name]
    for k, v in env.items():
        clean_env.setenv(k, v)
    from geomx_b200.parallel import Topology
    torch.manual_seed(1234 + seed)
    batches = _batches(B, steps, 99 + seed)
    loop = kw.get("loopback", False)
    eng = mx.models.HipsCNNTrainStep(net=net, batch_size=B, optimizer=optimizer, topo=Topology(1, 0, 1, 0 if loop else 1), use_graph=graph,
                                     fused_zero_grad=False, **kw)
    # a schedule changes nothing in the step's path: the same launches on the same streams as the constant-lr case
    assert [(n, s) for n, s, _ in eng._steps()] == want, (name, eng._steps())
    for a, v in attrs.items():
        assert getattr(eng, a) == v, (name, a, getattr(eng, a))
    P0 = [p.clone() for p in eng.P]
    spec = dict(R.CASE_SPECS[kind], lr=optimizer.lr, wd=optimizer.wd)
    spec["clip_gradient"] = _clip_for(P0, *batches[0], B, spec["rescale_grad"])
    if eng.update == "local":
        eng._local_spec = dict(eng._local_spec, clip_gradient=spec["clip_gradient"])
    else:
        eng.fabric.set_optimizer(dict(eng.fabric.opt_spec, clip_gradient=spec["clip_gradient"]))
    t0 = eng.opt_step
    if graph:
        eng.x.copy_(batches[0][0]); eng.label.copy_(batches[0][1])
        snap = _snapshot(eng)
        eng.capture()
        torch.cuda.synchronize()
        for t, v in snap:
            t.copy_(v)
        eng.fabric.set_opt_step(t0)
    grads, hist = [], []
    master = eng.Wl if eng.update == "local" else eng.fabric.w
    for X, y in batches:
        eng.x.copy_(X); eng.label.copy_(y)
        eng.graph.replay() if graph else eng._body()
        torch.cuda.synchronize()
        grads.append([x.detach().cpu().clone() for x in eng.G])
        hist.append(([p.detach().cpu().clone() for p in eng.P], [eng.layout.view(master, i).cpu().clone() for i in range(10)]))
    assert eng.opt_step == t0 + steps, (eng.opt_step, t0, steps)
    return eng, P0, grads, hist, spec


def _replay(eng, P0, spec, grads, lr_of, t0=0, mults=None):
    ref = _engine_ref(eng, P0, spec)
    if mults is not None:
        ref.mults = list(mults)
    ref.t = [t0] * 10
    out = []
    for k, gs in enumerate(grads, 1):
        ref.h["lr"] = lr_of(t0 + k)
        ref.step(gs)
        out.append([w.clone() for w in ref.w])
    return out


def _check_hist(name, eng, P0, hist, refs):
    half = [i for i in range(10) if eng.fabric.tile_fmt is not None and int(eng.fabric.tile_fmt[eng.layout.slots[i].offset // 1024]) != 0]
    worst = 0.0
    for k, ((P, M), rw) in enumerate(zip(hist, refs), 1):
        exact = [i for i in range(10) if i not in half]
        e = max(R.displacement_err(M, P0, rw, stores=k),
                R.displacement_err([P[i] for i in exact], [P0[i] for i in exact], [rw[i] for i in exact], stores=k))
        assert e < TOL, (name, k, e)
        worst = max(worst, e)
    return worst


def _sched_engine(base):
    """Linear warm-up over 3 updates, milestones after updates 4 and 5: each of six updates has its own lr."""
    return S.MultiFactorScheduler(step=[4, 5], factor=0.5, base_lr=base, warmup_steps=3, warmup_begin_lr=base / 10)


@pytest.mark.parametrize("name", ENGINE_SCHED_CASES)
def test_engine_schedule_matches_fp64(nat, clean_env, name):
    kind = ENGINE_CASES[name][2]
    opt = _case_opt(kind, _sched_engine)
    eng, P0, grads, hist, spec = _engine_sched_run(name, clean_env, opt)
    try:
        ref_sched = _fp32_copy(opt.lr_scheduler)
        worst = _check_hist(name, eng, P0, hist, _replay(eng, P0, spec, grads, ref_sched))
        good = _replay(eng, P0, spec, grads, ref_sched)[-1]
        no_wu = S.MultiFactorScheduler(step=[4, 5], factor=0.5, base_lr=ref_sched.base_lr)
        muts = {"t-1": lambda t: ref_sched(t - 1), "t+1": lambda t: ref_sched(t + 1), "constant": lambda t: ref_sched.base_lr,
                "no-warmup": no_wu}
        far = {m: R.displacement_err(_replay(eng, P0, spec, grads, fn)[-1], P0, good) for m, fn in muts.items()}
        print("\n  %-18s scheduled  %.1e  | mutations: %s" % (name, worst, "  ".join("%s %.1e" % kv for kv in far.items())))
        assert all(e > 10 * TOL for e in far.values()), far
        assert eng.learning_rate == opt.lr_scheduler(eng.opt_step + 1)
    finally:
        del eng
        cleanup()


# ============================================================================================================ 5. multipliers, resume offset
def test_engine_multipliers_and_resume_offset(nat, clean_env):
    net = mx.models.build_cnn()
    net.initialize(init=mx.init.Xavier(), ctx=mx.gpu(0))
    net(mx.nd.array(torch.zeros(1, 1, 28, 28), ctx=mx.gpu(0)))
    params = list(net.collect_params().values())
    params[0].lr_mult = 0.5
    for p in params[1::2]:
        p.wd_mult = 0.0
    mults = [(0.5 if i == 0 else 1.0, 0.0 if i % 2 else 1.0) for i in range(10)]
    sched = lambda base: S.FactorScheduler(step=100, factor=0.5, base_lr=base)       # t = 101 is the first update of the halved rate
    opt = _case_opt("adam", sched, begin_num_update=100)
    eng, P0, grads, hist, spec = _engine_sched_run("A-adam-graph", clean_env, opt, net=net)
    try:
        assert spec["wd"] > 0
        ref_sched = _fp32_copy(opt.lr_scheduler)
        worst = _check_hist("mults", eng, P0, hist, _replay(eng, P0, spec, grads, ref_sched, t0=100, mults=mults))
        good = _replay(eng, P0, spec, grads, ref_sched, t0=100, mults=mults)[-1]
        far = {"mults ignored": R.displacement_err(_replay(eng, P0, spec, grads, ref_sched, t0=100)[-1], P0, good),
               "t from 0": R.displacement_err(_replay(eng, P0, spec, grads, ref_sched, t0=0, mults=mults)[-1], P0, good)}
        print("\n  multipliers + begin_num_update=100: %.1e  | %s" % (worst, "  ".join("%s %.1e" % kv for kv in far.items())))
        assert all(e > 10 * TOL for e in far.values()), far
        assert eng.opt_step == 106
    finally:
        del eng
        cleanup()


# ============================================================================================================ 6. set_learning_rate
@pytest.mark.parametrize("how", ["graph", "lookahead", "step_async"])
def test_set_learning_rate(nat, clean_env, how):
    """Three steps at lr 0.01, ``set_learning_rate(0.003)``, three more: the updates after the call use the new rate, the step count
    advances by one per step (no warm-up steps ran again), the weights match the reference."""
    from geomx_b200.parallel import Topology
    torch.manual_seed(4321)
    B = 32
    opt = mx.optimizer.Adam(learning_rate=0.01, wd=0.05)
    eng = mx.models.HipsCNNTrainStep(batch_size=B, optimizer=opt, topo=Topology(1, 0, 1, 1), use_graph=True, fused_zero_grad=False,
                                     lookahead=how == "lookahead")
    try:
        batches = _batches(B, 7, 7)
        P0 = [p.clone() for p in eng.P]
        eng.x.copy_(batches[0][0]); eng.label.copy_(batches[0][1])
        snap = _snapshot(eng)
        eng.capture()
        torch.cuda.synchronize()
        for t, v in snap:
            t.copy_(v)
        eng.fabric.set_opt_step(0)
        spec = dict(R.CASE_SPECS["adam"], lr=0.01, wd=0.05, clip_gradient=-1.0)
        grads, hist, lrs = [], [], []
        for k, (X, y) in enumerate(batches[1:], 1):
            if k == 4:
                eng.set_learning_rate(0.003)
                assert eng.graph is None and eng._graph_alt is None and eng.learning_rate == 0.003
            lrs.append(eng.learning_rate)
            if how == "step_async":
                h = eng.step_async(X.cpu().pin_memory(), y.cpu().pin_memory())
                h.wait()
            else:
                eng.step(X, y)
            torch.cuda.synchronize()
            assert eng.opt_step == k, (how, k, eng.opt_step)
            grads.append([x.detach().cpu().clone() for x in eng.G])
            hist.append(([p.detach().cpu().clone() for p in eng.P], [eng.layout.view(eng.fabric.w, i).cpu().clone() for i in range(10)]))
        assert lrs == [0.01] * 3 + [0.003] * 3
        if how == "step_async":
            assert eng._graph_alt is not None          # the second input buffer's graph was captured again after the call
        f32lr = lambda t: f32(0.01) if t <= 3 else f32(0.003)
        worst = _check_hist(how, eng, P0, hist, _replay(eng, P0, spec, grads, f32lr))
        good = _replay(eng, P0, spec, grads, f32lr)[-1]
        stale = R.displacement_err(_replay(eng, P0, spec, grads, lambda t: f32(0.01))[-1], P0, good)
        print("\n  set_learning_rate %-10s %.1e  (old rate kept: %.1e)" % (how, worst, stale))
        assert stale > 10 * TOL
        sched_opt = mx.optimizer.Adam(learning_rate=0.01, lr_scheduler=S.FactorScheduler(step=10, factor=0.5))
        sched_eng = mx.models.HipsCNNTrainStep(batch_size=B, optimizer=sched_opt, topo=Topology(1, 0, 1, 1), use_graph=False)
        with pytest.raises(UserWarning):
            sched_eng.set_learning_rate(0.1)
        del sched_eng
    finally:
        del eng
        cleanup()


# ============================================================================================================ 7. refusal
def test_engine_refuses_custom_schedule(nat, clean_env):
    from geomx_b200.parallel import Topology

    class Halving(S.LRScheduler):
        def decayed(self, num_update):
            return self.base_lr / 2 ** (num_update // 10)

    class Nudged(S.CosineScheduler):
        def __call__(self, num_update):
            return super().__call__(num_update) * 0.9

    class Stretched(S.PolyScheduler):
        @property
        def max_steps(self):
            return 2 * self.max_update

    for sched in (Halving(), Nudged(max_update=100), Stretched(max_update=100), lambda t: 0.01):
        opt = mx.optimizer.SGD(learning_rate=0.1)
        opt.lr_scheduler = sched
        with pytest.raises(ValueError):
            mx.models.HipsCNNTrainStep(batch_size=32, optimizer=opt, topo=Topology(1, 0, 1, 1), use_graph=False)
    cleanup()


def test_engine_schedule_base_lr_is_the_schedulers(nat, clean_env):
    """A scheduler attached after the optimizer was made keeps its own base_lr, as ``Optimizer._get_lr`` applies it: the kernels get that
    base, and ``learning_rate`` reports the rate they apply (from the engine's copy of the scheduler)."""
    from geomx_b200.parallel import Topology
    opt = mx.optimizer.SGD(learning_rate=0.1)
    sched = S.FactorScheduler(step=2, factor=0.5, base_lr=0.02, warmup_steps=1, warmup_begin_lr=0.005)
    opt.lr_scheduler = sched
    for update in ("server", "local"):
        eng = mx.models.HipsCNNTrainStep(batch_size=32, optimizer=opt, topo=Topology(1, 0, 1, 1), use_graph=False, update=update)
        spec = eng._local_spec if update == "local" else eng.fabric.opt_spec
        assert spec["lr"] == 0.02 and spec["lr_schedule"] == sched.device_spec()
        assert eng.learning_rate == sched(1) == 0.02
        sched.base_lr = 0.5                      # the engine evaluates the schedule it was given, not later edits of the object
        assert eng.learning_rate == 0.02
        sched.base_lr = 0.02
        with pytest.raises(UserWarning):
            eng.set_learning_rate(0.1)
        del eng
    cleanup()
