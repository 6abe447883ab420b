"""NAG, Signum (with and without momentum), RMSProp, AdaGrad, AdaDelta and Ftrl on every update path, against the fp64 rules of
``tests/_optim_ref.py`` over five or more steps: the kernels of ``optim.cu`` called directly, the fabric on its own over the paths of
``test_update_paths_gpu.py``, the training engine on its kernel paths (with the reference advanced by the engine's own gradient sums, and each
kind's plausible-bug mutations shown to land outside the tolerance), ``mx.kv.create('dist_sync')``, the Trainer's fused multi-tensor update,
and a short training run per kind.

Signum takes the sign of its momentum.  Where the fp64 momentum lies within fp32 rounding of zero an fp32 kernel may take the other sign;
the reference marks those elements (``UpdateRef.sign_ambiguous``) and the checks take the reference's value there, and count them.
"""
import ctypes

import pytest
import torch

import geomx_b200 as mx
from geomx_b200.models.cnn import LOCAL

import _optim_ref as R
from _cnn_ref import cleanup, dev, nat  # noqa: F401  (nat: fixture)
from _update_harness import (A, C, FAB_PATHS, KEY_MULTS, KEY_SIZES, ONE, PUSH_SCALE, TOL, _batches, _clip_for, _fab_grads,  # noqa: F401
                             _fab_init, _fabric, _padding_zero, _snapshot, clean_env, half_ulps)

pytestmark = pytest.mark.gpu

O = mx.optimizer
KINDS = ["nag", "signum", "signsgd", "rmsprop", "adagrad", "adadelta", "ftrl"]

# hyper-parameters of the kernel and fabric cases: clip cuts part of the gradients (rescale 0.5 for the kernels, 2 with the fabric's
# 1/32 push scale), wd, momentum and the kinds' own parameters are active
_OWN = {
    "nag": dict(name="nag", lr=0.1, momentum=0.9),
    "signum": dict(name="signum", lr=0.01, momentum=0.9, wd_lh=0.05),
    "signsgd": dict(name="signum", lr=0.01, momentum=0.0, wd_lh=0.05),
    "rmsprop": dict(name="rmsprop", lr=0.01, gamma1=0.9, epsilon=1e-8, clip_weights=0.3),
    "adagrad": dict(name="adagrad", lr=0.1, epsilon=1e-7),
    "adadelta": dict(name="adadelta", lr=1.0, rho=0.9, epsilon=1e-5),
    "ftrl": dict(name="ftrl", lr=0.1, lamda1=0.01, beta=1.0),
}
KSPECS = {k: dict(v, wd=0.02, rescale_grad=0.5, clip_gradient=0.3) for k, v in _OWN.items()}
FSPECS = {k: dict(v, wd=0.02, rescale_grad=2.0, clip_gradient=0.02) for k, v in _OWN.items()}


def _take_ambiguous(ws, ref):
    """``ws`` with the reference's weights where Signum's sign was within rounding (see the module docstring); and how many there were."""
    out = [torch.where(a.reshape(w.shape).to(w.device), r.reshape(w.shape).to(w.device, torch.float32), w) if a.any() else w
           for w, r, a in zip(ws, ref.w, ref.sign_ambiguous)]
    return out, sum(int(a.sum()) for a in ref.sign_ambiguous)


def _sched():
    return mx.lr_scheduler.FactorScheduler(step=2, factor=0.7)


# ============================================================================================================ a. optim.cu kernels
@pytest.mark.parametrize("scheduled", [False, True], ids=["const", "sched"])
@pytest.mark.parametrize("kind", KINDS)
def test_arena_opt(nat, kind, scheduled):
    """Fused arena optimizer through the packed entry point: a distinct (lr_mult, wd_mult) per tile, the device step counter, ``g_zero``
    cleared; with ``scheduled`` a factor schedule evaluated from the device step count.  Six launches at two arena sizes."""
    spec = dict(KSPECS[kind])
    sched = _sched()
    if scheduled:
        sched.base_lr = spec["lr"]
        spec["lr_schedule"] = sched.device_spec()
    hp = nat.pack_hyper(spec)
    h = R.hyper(spec)
    g = torch.Generator().manual_seed(17 + len(kind))
    step_state = torch.zeros(2, dtype=torch.int32, device=dev())
    t = 0
    for tiles in (5, 1300):
        n = tiles * 1024
        tm = torch.stack([0.25 + 2 * torch.rand(tiles, generator=g), 2 * torch.rand(tiles, generator=g)], 1).float()
        lm, wm = tm[:, 0].double().repeat_interleave(1024), tm[:, 1].double().repeat_interleave(1024)
        w0 = torch.randn(n, generator=g) * 0.1
        w, s0, s1 = w0.to(dev()), torch.zeros(n, device=dev()), torch.zeros(n, device=dev())
        ref = R.UpdateRef(None, [w0])
        ref.h = h
        for _ in range(3):
            gr = torch.randn(n, generator=g)
            gd = gr.to(dev())
            nat.arena_opt_h(hp, w, gd, s0, s1, n, tm.to(dev()), step_state, gd)
            torch.cuda.synchronize()
            t += 1
            assert int(step_state[0]) == t and int(step_state[1]) == 0
            assert bool((gd == 0).all())
            hk = dict(h, lr=float(sched(t)) if scheduled else h["lr"])
            amb = R.update(hk, ref.w[0], gr.double(), ref.s0[0], ref.s1[0], t, lm, wm)
            if amb is not None:
                ref.sign_ambiguous[0] |= amb
            (wc,), n_amb = _take_ambiguous([w.cpu()], ref)
            e = (R.displacement_err([wc], [w0], ref.w, stores=3), R.rel(s0, ref.s0[0]), R.rel(s1, ref.s1[0]))
            print("\n  arena_opt %-8s %s tiles %4d t=%d  dw %.1e s0 %.1e s1 %.1e  sign-ambiguous %d" % ((kind, "sched" if scheduled else "const",
                                                                                                      tiles, t) + e + (n_amb,)))
            assert max(e) < TOL and n_amb < 1e-4 * n, (e, n_amb)


@pytest.mark.parametrize("n", [1, 1023, 500003])
@pytest.mark.parametrize("kind", KINDS)
def test_single_opt(nat, kind, n):
    spec = KSPECS[kind]
    hp, h = nat.pack_hyper(spec), R.hyper(spec)
    g = torch.Generator().manual_seed(n + 3 * len(kind))
    w0 = torch.randn(n, generator=g) * 0.1
    w, s0, s1 = w0.to(dev()), torch.zeros(n, device=dev()), torch.zeros(n, device=dev())
    ref = R.UpdateRef(None, [w0])
    ref.h = h
    for t in range(1, 6):
        gr = torch.randn(n, generator=g)
        nat.single_opt_h(hp, w, gr.to(dev()), s0, s1, h["lr"])
        amb = R.update(h, ref.w[0], gr.double(), ref.s0[0], ref.s1[0], t)
        if amb is not None:
            ref.sign_ambiguous[0] |= amb
    torch.cuda.synchronize()
    (wc,), n_amb = _take_ambiguous([w.cpu()], ref)
    e = (R.displacement_err([wc], [w0], ref.w, stores=5), R.rel(s0, ref.s0[0]), R.rel(s1, ref.s1[0]))
    assert max(e) < TOL and n_amb <= max(1, 1e-4 * n), (e, n_amb)


@pytest.mark.parametrize("kind", KINDS)
def test_multi_tensor_opt(nat, kind):
    spec = KSPECS[kind]
    hp, h = nat.pack_hyper(spec), R.hyper(spec)
    g = torch.Generator().manual_seed(41 + len(kind))
    sizes = [1, 3, 1000, 16385, 70000]
    mults = [(0.5, 2.0), (2.0, 0.0), (1.0, 1.5), (0.25, 3.0), (1.5, 0.5)]
    w0 = [torch.randn(n, generator=g) * 0.1 for n in sizes]
    ws = [w.to(dev()) for w in w0]
    s0 = [torch.zeros(n, device=dev()) for n in sizes]
    s1 = [torch.zeros(n, device=dev()) for n in sizes]
    ref = R.UpdateRef(None, w0, mults=mults)
    ref.h = h
    for t in range(1, 6):
        grads = [torch.randn(n, generator=g) for n in sizes]
        gd = [x.to(dev()) for x in grads]
        arr = (nat._TensorEntry * len(sizes))()
        for j in range(len(sizes)):
            arr[j] = nat._TensorEntry(ws[j].data_ptr(), gd[j].data_ptr(), s0[j].data_ptr(), s1[j].data_ptr(), sizes[j], *mults[j])
        table = torch.frombuffer(bytearray(bytes(arr)), dtype=torch.uint8).to(dev())
        assert nat._lib().gx_multi_tensor_opt_h(ctypes.byref(hp), ctypes.c_void_p(table.data_ptr()), len(sizes), max(sizes), h["lr"],
                                                nat._s()) == 0
        torch.cuda.synchronize()
        for j in range(len(sizes)):
            amb = R.update(h, ref.w[j], grads[j].double(), ref.s0[j], ref.s1[j], t, *mults[j])
            if amb is not None:
                ref.sign_ambiguous[j] |= amb
    wc, n_amb = _take_ambiguous([w.cpu() for w in ws], ref)
    e = R.displacement_err(wc, w0, ref.w, stores=5)
    e_s = max(max(R.rel(a, b) for a, b in zip(s0, ref.s0)), max(R.rel(a, b) for a, b in zip(s1, ref.s1)))
    assert e < TOL and e_s < TOL and n_amb <= 10, (e, e_s, n_amb)


# ============================================================================================================ b. the fabric on its own
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("path,loopback,fmts", FAB_PATHS, ids=["%s%s" % (p, "-lp" if lb else "") + ("-fp16fp8" if f else "")
                                                              for p, lb, f in FAB_PATHS])
def test_fabric_rounds(nat, clean_env, path, loopback, fmts, kind):
    """Five rounds of one fabric path: master weights, both state slots, the parameter arena and the zero padding against the reference."""
    spec = FSPECS[kind]
    f = _fabric(spec, loopback, fmts)
    try:
        g = torch.Generator().manual_seed(100 * [p[0] for p in FAB_PATHS].index(path) + 7 * len(kind) + (fmts is None) + 2 * loopback)
        W0 = _fab_init(f, g)
        if path in ("sharded", "replicated", "direct-sharded", "direct-replicated"):
            f.add_channel("c", list(range(len(KEY_SIZES))), replicate=path.endswith("replicated"))
            run = lambda: f.channel_step("c")
        else:
            run = lambda: f.fsa_step()
        ref = R.UpdateRef(spec, W0, mults=KEY_MULTS, push_scale=PUSH_SCALE, fmts=fmts, round_after_scale=path == "ll")
        exact_param = not loopback or path == "direct-replicated" or fmts is None
        for k in range(1, 6):
            grads = _fab_grads(g)
            for i, x in enumerate(grads):
                f.grad_view(i).copy_(x)
            run()
            torch.cuda.synchronize()
            ref.step(grads)
            assert f.opt_step == k and not f.check_protocol_errors()
            W, n_amb = _take_ambiguous([f.layout.view(f.w, i) for i in range(len(KEY_SIZES))], ref)
            e_w = R.displacement_err(W, W0, ref.w, stores=k)
            e_s0 = max(R.rel(f.layout.view(f.s0, i), ref.s0[i]) for i in range(len(KEY_SIZES)))
            e_s1 = max(R.rel(f.layout.view(f.s1, i), ref.s1[i]) for i in range(len(KEY_SIZES)))
            P = [f.param_view(i) for i in range(len(KEY_SIZES))]
            Wm = [f.layout.view(f.w, i) for i in range(len(KEY_SIZES))]
            if exact_param:
                assert all(torch.equal(p, w) for p, w in zip(P, Wm)), "parameter arena differs from the master weights"
            else:
                assert all(torch.equal(P[i], Wm[i].half().float()) for i, fm in enumerate(fmts) if fm != "fp32"), "fp16 pull != fp16(master)"
                f32 = [i for i, fm in enumerate(fmts) if fm == "fp32"]
                Pa, _ = _take_ambiguous(P, ref)
                e_p = R.displacement_err([Pa[i] for i in f32], [W0[i] for i in f32], [ref.w[i] for i in f32], stores=k)
                assert e_p < TOL, (k, e_p)
            _padding_zero(f)
            if k == 5:
                print("\n  %-18s %-8s %s  w %.1e s0 %.1e s1 %.1e  sign-ambiguous %d" % (path + ("-lp" if loopback else ""), kind,
                                                                                      "fp16/fp8" if fmts else "fp32    ", e_w, e_s0, e_s1, n_amb))
            assert e_w < TOL and e_s0 < TOL and e_s1 < TOL and n_amb <= 10, (k, e_w, e_s0, e_s1, n_amb)
    finally:
        del f
        cleanup()


# ============================================================================================================ c. the engine
# optimizer objects of the engine cases: settings under which the demo CNN trains (the smoke test) and the kinds' terms matter
def _engine_opt(kind, clip=None, **extra):
    kw = dict(wd=0.01, rescale_grad=1.0, clip_gradient=clip, **extra)
    return {
        "nag": lambda: O.NAG(learning_rate=0.02, momentum=0.9, **kw),
        "signum": lambda: O.Signum(learning_rate=0.001, momentum=0.9, wd_lh=0.01, **kw),
        "signsgd": lambda: O.Signum(learning_rate=0.001, momentum=0.0, **kw),
        "rmsprop": lambda: O.RMSProp(learning_rate=0.001, gamma1=0.9, epsilon=1e-8, clip_weights=0.5, **kw),
        "adagrad": lambda: O.AdaGrad(learning_rate=0.01, eps=1e-7, **kw),
        "adadelta": lambda: O.AdaDelta(rho=0.9, epsilon=1e-5, **kw),
        "ftrl": lambda: O.Ftrl(learning_rate=0.01, lamda1=1e-5, beta=1e-6, **kw),
    }[kind]()


# name -> (B, env, kind, engine kwargs, graph, the step's (launch, stream) list)
ENGINE_CASES = {**{"A-" + k: (32, {}, k, {}, False, A) for k in KINDS},
                "A-rmsprop-graph": (32, {}, "rmsprop", {}, True, A),
                "C-nag": (32, {"GEOMX_FUSED_EXCHANGE": "1"}, "nag", {}, False, C),
                "single-adagrad": (32, {"GEOMX_STEP_OVERLAP": "0"}, "adagrad", {}, False, ONE),
                "loopback-ov1-ftrl": (32, {"GEOMX_STEP_OVERLAP": "1"}, "ftrl", dict(loopback=True), False, A),
                "loopback-ov0-signum": (32, {"GEOMX_STEP_OVERLAP": "0"}, "signum", dict(loopback=True), False, ONE),
                "async-adadelta": (32, {}, "adadelta", dict(mode="dist_async"), False, ONE),
                "local-rmsprop": (32, {}, "rmsprop", dict(update="local"), False, A + [(LOCAL, "main")]),
                "hfa-nag": (32, {}, "nag", dict(hfa=(2, 2)), False, ONE)}


def _engine_run(name, clean_env, steps=6):
    B, env, kind, kw, graph, want = ENGINE_CASES[name]
    for k, v in env.items():
        clean_env.setenv(k, v)
    from geomx_b200.parallel import Topology
    torch.manual_seed(4321)
    batches = _batches(B, steps, 199)
    loop = kw.get("loopback", False)
    eng = mx.models.HipsCNNTrainStep(batch_size=B, optimizer=_engine_opt(kind), topo=Topology(1, 0, 1, 0 if loop else 1), use_graph=graph,
                                     fused_zero_grad=False, **kw)
    P0 = [p.clone() for p in eng.P]
    spec = dict(_engine_opt(kind).spec(), clip_gradient=_clip_for(P0, *batches[0], B, 1.0))
    if eng.update == "local":
        eng._local_spec = dict(eng._local_spec, clip_gradient=spec["clip_gradient"])
    else:
        eng.fabric.set_optimizer(dict(eng.fabric.opt_spec, clip_gradient=spec["clip_gradient"]))
    assert [(n, s) for n, s, _ in eng._steps()] == want, name
    if graph:
        eng.x.copy_(batches[0][0]); eng.label.copy_(batches[0][1])
        snap = _snapshot(eng)
        eng.capture()
        torch.cuda.synchronize()
        for t, v in snap:
            t.copy_(v)
        eng.fabric.set_opt_step(0)
    grads, hist = [], []
    master = eng.Wl if eng.update == "local" else eng.fabric.w
    for X, y in batches:
        eng.x.copy_(X); eng.label.copy_(y)
        eng.graph.replay() if graph else eng._body()
        torch.cuda.synchronize()
        grads.append([x.detach().cpu().clone() for x in eng.G])
        hist.append(([p.detach().cpu().clone() for p in eng.P], [eng.layout.view(master, i).cpu().clone() for i in range(10)]))
    return eng, P0, grads, spec, hist


def _engine_ref(eng, P0, spec, mutation=None):
    # HFA applies the optimizer to the worker's own gradient sum (rescale_grad / B inside the update); the other modes push-scale by 1/B
    after = eng.fabric.loopback and not eng.overlap
    return R.UpdateRef(spec, P0, push_scale=1.0 / eng.B, round_after_scale=after, mutation=mutation)


@pytest.mark.parametrize("name", list(ENGINE_CASES))
def test_engine_update_matches_fp64(nat, clean_env, name):
    eng, P0, grads, spec, hist = _engine_run(name, clean_env)
    try:
        f = eng.fabric
        steps = len(grads)
        if eng.update == "local":
            assert int(eng.opt_state[0]) == steps
        elif eng.mode == "dist_async":
            counts = f.flags.tensor[f.off["async_step"]: f.off["async_step"] + f.tiles]
            assert bool((counts == steps).all())
        else:
            assert f.opt_step == steps
        assert not f.check_protocol_errors()
        ref = _engine_ref(eng, P0, spec)
        worst, amb = [0.0, 0.0], 0
        for k, (gs, (P, M)) in enumerate(zip(grads, hist), 1):
            ref.step(gs)
            Mx, amb = _take_ambiguous(M, ref)
            Px, _ = _take_ambiguous(P, ref)
            e = (R.displacement_err(Mx, P0, ref.w, stores=k), R.displacement_err(Px, P0, ref.w, stores=k))
            worst = [max(a, b) for a, b in zip(worst, e)]
            assert e[0] < TOL and e[1] < TOL, (name, k, e)
        assert amb <= 20, amb
        muts = {}
        for m in R.relevant_mutations(spec, push_scale=1.0 / eng.B):
            bad = _engine_ref(eng, P0, spec, mutation=m)
            for gs in grads:
                bad.step(gs)
            muts[m] = R.displacement_err(bad.w, P0, ref.w)
        print("\n  %-20s master %.1e  params %.1e  sign-ambiguous %d | mutations: %s" % (
            name, worst[0], worst[1], amb, "  ".join("%s %.1e" % kv for kv in muts.items())))
        assert len(muts) >= 2 and not {m: e for m, e in muts.items() if not e > 10 * TOL}, (name, muts)
    finally:
        del eng
        cleanup()


@pytest.mark.parametrize("kind", ["rmsprop", "nag", "adadelta"])
def test_engine_schedule_mults_begin(nat, clean_env, kind):
    """A factor schedule, per-key multipliers from the Gluon net's Parameters and ``begin_num_update``: the engine's update equals the
    reference advanced with the scheduled lr of each step's count (which starts after ``begin_num_update``) and each key's multipliers."""
    from geomx_b200.parallel import Topology
    net = mx.models.build_cnn()
    net.initialize(init=mx.init.Xavier(), ctx=mx.gpu(0))
    net(mx.nd.zeros((1, 1, 28, 28), ctx=mx.gpu(0)))          # completes the deferred shape inference
    params = list(net.collect_params().values())
    mults = [(0.5 + 0.25 * (i % 3), 0.0 if i % 2 else 2.0) for i in range(10)]
    for p, (lm, wm) in zip(params, mults):
        p.lr_mult, p.wd_mult = lm, wm
    sched = _sched()
    opt = _engine_opt(kind, lr_scheduler=sched, begin_num_update=3)
    eng = mx.models.HipsCNNTrainStep(net=net, batch_size=32, optimizer=opt, topo=Topology(1, 0, 1, 1), use_graph=False, fused_zero_grad=False)
    try:
        P0 = [p.clone() for p in eng.P]
        spec = opt.spec()
        ref = R.UpdateRef(spec, P0, mults=mults, push_scale=1.0 / 32)
        h = ref.h
        for k, (X, y) in enumerate(_batches(32, 5, 7), 1):
            eng.x.copy_(X); eng.label.copy_(y)
            eng._body()
            torch.cuda.synchronize()
            ref.h = dict(h, lr=float(sched(3 + k)))
            ref.step([x.detach().cpu().clone() for x in eng.G])
            e = R.displacement_err([p.cpu() for p in eng.P], P0, ref.w, stores=k)
            assert e < TOL, (k, e)
        assert eng.fabric.opt_step == 3 + 5
        print("\n  schedule + mults + begin_num_update %s: %.1e" % (kind, e))
    finally:
        del eng
        cleanup()


def test_engine_refuses_other_optimizers_with_reason(nat):
    for opt, why in ((O.RMSProp(centered=True), "three state arrays"), (O.FTML(), "three state arrays"), (O.Nadam(), "momentum schedule"),
                     (O.Adamax(), "0 / 0"), (O.SGLD(), "random-number"), (O.LBSGD(), "warm-up")):
        with pytest.raises(ValueError, match=why) as ei:
            mx.models.HipsCNNTrainStep(batch_size=32, optimizer=opt, use_graph=False)
        assert "Supported: SGD, Adam, DCASGD, NAG, Signum, RMSProp (centered=False), AdaGrad, AdaDelta, Ftrl" in str(ei.value)


@pytest.mark.parametrize("kind", KINDS)
def test_engine_trains(nat, clean_env, kind):
    """50 graph-replayed steps on a fixed set of four synthetic batches lower the mean loss over the set."""
    from geomx_b200.parallel import Topology
    torch.manual_seed(7)
    g = torch.Generator().manual_seed(8)
    batches = [(torch.rand(32, 1, 28, 28, generator=g).pin_memory(), torch.randint(0, 10, (32,), generator=g).float().pin_memory())
               for _ in range(4)]
    eng = mx.models.HipsCNNTrainStep(batch_size=32, optimizer=_engine_opt(kind), topo=Topology(1, 0, 1, 1), use_graph=True)
    try:
        losses = [eng.step(*batches[i % 4]) for i in range(52)]
        first, last = sum(losses[:4]) / 4, sum(losses[-4:]) / 4
        print("\n  %-8s loss %.4f -> %.4f" % (kind, first, last))
        assert last == last and last < first, (kind, first, last)
    finally:
        del eng
        cleanup()


# ============================================================================================================ d. KVStore and Trainer
def test_kvstore_fabric_rmsprop(nat, clean_env):
    """``mx.kv.create('dist_sync')`` with ``set_optimizer(RMSProp)`` runs the native kind; four rounds, one of them partial (masked)."""
    clean_env.delenv("WORLD_SIZE", raising=False)
    clean_env.delenv("RANK", raising=False)
    clean_env.setenv("GEOMX_FABRIC", "auto")
    from geomx_b200.models import CNN_PARAM_SHAPES
    from geomx_b200.parallel.fabric_kvstore import KVStoreFabric
    kv = mx.kv.create("dist_sync")
    assert isinstance(kv, KVStoreFabric)
    g = torch.Generator().manual_seed(13)
    W0 = [torch.randn(s, generator=g) * 0.1 for s in CNN_PARAM_SHAPES]
    for i, w in enumerate(W0):
        kv.init(i, mx.nd.array(w.to(dev()), ctx=mx.gpu(0)))
    opt = O.RMSProp(learning_rate=0.01, gamma1=0.9, wd=0.01, clip_gradient=0.05, clip_weights=0.3)
    kv.set_optimizer(opt)
    assert kv.fabric.opt_spec["name"] == "rmsprop"
    ref = R.UpdateRef(opt.spec(), W0)
    sets = [None, None, [0, 1, 4, 5, 8, 9], None]
    grads_all = R.cnn_like_grads(g, CNN_PARAM_SHAPES, len(sets), batch=1)
    outs = [mx.nd.zeros(s, ctx=mx.gpu(0)) for s in CNN_PARAM_SHAPES]
    for k, (active, grads) in enumerate(zip(sets, grads_all), 1):
        for i in (range(10) if active is None else active):
            kv.push(i, mx.nd.array(grads[i].to(dev()), ctx=mx.gpu(0)))
        for i in range(10):
            kv.pull(i, out=outs[i])
        ref.step(grads, active)
        e = R.displacement_err([o._t.detach().cpu() for o in outs], W0, ref.w, stores=k)
        assert e < TOL, (k, e)
    bad = R.UpdateRef(opt.spec(), W0, mutation="rmsprop_clip_before_wd")
    for grads, active in zip(grads_all, sets):
        bad.step(grads, active)
    e_bad = R.displacement_err(bad.w, W0, ref.w)
    print("\n  KVStore RMSProp: %.1e (clip before wd would give %.1e)" % (e, e_bad))
    assert e_bad > 10 * TOL


@pytest.mark.parametrize("kind", KINDS + ["dcasgd"])
def test_trainer_fused_matches_python_updater(nat, kind):
    """``gluon.Trainer``'s one-launch multi-tensor update against the per-parameter Python ``Updater`` on an identical net, five steps."""
    nets, trainers = [], []
    for fused in (True, False):
        torch.manual_seed(5)
        net = mx.models.build_cnn()
        net.initialize(init=mx.init.Xavier(), ctx=mx.gpu(0))
        net(mx.nd.zeros((1, 1, 28, 28), ctx=mx.gpu(0)))      # completes the deferred shape inference
        opt = O.DCASGD(learning_rate=0.05, momentum=0.9, lamda=0.5, wd=0.01, clip_gradient=0.05) if kind == "dcasgd" else \
            _engine_opt(kind, clip=0.05)
        tr = mx.gluon.Trainer(net.collect_params(), opt, kvstore=None)
        if not fused:
            tr._fused_update = lambda: False
        nets.append(net); trainers.append(tr)
    P0 = [p.data()._t.detach().cpu().clone() for p in nets[0].collect_params().values()]
    assert all(torch.equal(a, p.data()._t.cpu()) for a, p in zip(P0, nets[1].collect_params().values()))
    loss = mx.gluon.loss.SoftmaxCrossEntropyLoss()
    g = torch.Generator().manual_seed(6)
    for _ in range(5):
        X = mx.nd.array(torch.rand(16, 1, 28, 28, generator=g).to(dev()), ctx=mx.gpu(0))
        y = mx.nd.array(torch.randint(0, 10, (16,), generator=g).float().to(dev()), ctx=mx.gpu(0))
        grads = None
        for net, tr in zip(nets, trainers):
            with mx.autograd.record():
                out = loss(net(X), y)
            out.backward()
            if grads is None:          # both nets step on the gradients of the fused one (their weights differ by rounding)
                grads = [p.grad()._t.detach().clone() for p in net.collect_params().values()]
            else:
                for p, gr in zip(net.collect_params().values(), grads):
                    p.grad()._t.copy_(gr)
            tr.step(16)
    torch.cuda.synchronize()
    Pf = [p.data()._t.cpu().double() for p in nets[0].collect_params().values()]
    Pp = [p.data()._t.cpu() for p in nets[1].collect_params().values()]
    flipped = 0
    if kind == "signum":
        # the sign of a momentum within rounding of zero may differ between the two: such an element is one lr step (0.001) apart
        off = [(a.double() - b).abs() > 5e-4 for a, b in zip(Pp, Pf)]
        flipped = sum(int(o.sum()) for o in off)
        Pp = [torch.where(o, b.float(), a) for a, b, o in zip(Pp, Pf, off)]
    e = R.displacement_err(Pp, P0, Pf, stores=5)
    print("\n  Trainer fused vs Python %-8s %.1e  sign flips %d" % (kind, e, flipped))
    assert e < TOL and flipped <= 20, (e, flipped)
