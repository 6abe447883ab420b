"""What the update-path GPU tests share: the switches they clear, the synthetic fabric arena and its gradients, the engine cases with their
optimizers, batches and clip thresholds, and the tolerance.  The fp64 update reference itself is ``_update_ref.py``."""
import pytest
import torch
import torch.nn.functional as F

import geomx_b200 as mx
from geomx_b200.models.cnn import DENSE_WGRAD, DIRECT_FWD, EXCH, LOCAL, MLP, ONE_GRID, STEP_SWITCHES

import _update_ref as R
from _cnn_ref import PATHS, dev

# the step switches and the fabric's own
SWITCHES = STEP_SWITCHES + ("GEOMX_FABRIC_PROTOCOL", "GEOMX_FABRIC_DIRECT", "GEOMX_PY_UPDATER", "GEOMX_WIRE_FP8", "ENABLE_DGT", "ENABLE_P3",
                            "MXNET_KVSTORE_USE_HFA")

TOL = R.DISP_TOL


@pytest.fixture
def clean_env(monkeypatch):
    for k in SWITCHES:
        monkeypatch.delenv(k, raising=False)
    return monkeypatch


def half_ulps(p, ref_w):
    """Distance, in fp16 steps, of ``p`` (a pulled fp16 parameter, stored as fp32) from the fp64 reference weight rounded to fp16: at most
    one (the kernel rounds its fp32 master weight, which may sit on the other side of a rounding boundary)."""
    r = ref_w.double().cpu()
    p = p.double().cpu().reshape(r.shape)
    mag = torch.maximum(r.abs(), p.abs()).clamp_min(2.0 ** -14)
    ulp = torch.exp2(torch.floor(torch.log2(mag)) - 10)
    return float(((p - r.float().half().double()).abs() / ulp).max())


# ---------------------------------------------------------------------------------------------------------------- the fabric on its own
KEY_SIZES = [1, 1000, 1024, 1025, 5000, 70000]
KEY_MULTS = [(0.5, 2.0), (2.0, 0.0), (1.0, 1.5), (0.25, 1.0), (1.5, 0.5), (0.75, 3.0)]
FAB_SPECS = {
    "sgd": dict(name="sgd", lr=0.1, wd=0.02, rescale_grad=2.0, clip_gradient=0.02, momentum=0.9),
    "adam": dict(name="adam", lr=0.01, wd=0.02, rescale_grad=2.0, clip_gradient=0.02, beta1=0.9, beta2=0.999, epsilon=1e-8),
    "dcasgd": dict(name="dcasgd", lr=0.1, wd=0.02, rescale_grad=2.0, clip_gradient=0.02, momentum=0.9, lamda=40.0),
}
MIXED_FMTS = ["fp32", "fp16", "fp8", "fp16", "fp8", "fp32"]
PUSH_SCALE = 1.0 / 32


def _fabric(spec, loopback, fmts=None):
    from geomx_b200.parallel import ArenaLayout, HipsFabric, Topology
    layout = ArenaLayout.build([(i, (n,)) for i, n in enumerate(KEY_SIZES)], mults=KEY_MULTS)
    f = HipsFabric(layout, Topology(1, 0, 1, 0 if loopback else 1), dev(), spec, loopback=loopback)
    f.set_push_scale(PUSH_SCALE)
    if fmts is not None:
        f.set_wire_formats({i: m for i, m in enumerate(fmts)})
    return f


def _fab_init(f, g):
    W0 = [torch.randn(n, generator=g) * 0.1 for n in KEY_SIZES]
    for i, w in enumerate(W0):
        f.param_view(i).copy_(w)
    f.load_master_from_param()
    return W0


def _fab_grads(g):
    """Pushed sums of a batch of 32: mean gradients ~1e-2 (clip 0.02 after rescale 2 cuts the larger half), some exact zeros."""
    out = []
    for n in KEY_SIZES:
        x = torch.randn(n, generator=g) * 0.01 * 32
        x[torch.rand(n, generator=g) < 0.05] = 0.0
        out.append(x)
    return out


def _padding_zero(f):
    for sl in f.layout.slots:
        a, b = sl.offset + sl.numel, sl.offset + sl.tiles * 1024
        for t in (f.param.tensor, f.w):
            if b > a:
                assert bool((t[a:b] == 0).all()), "padding of key %d is no longer zero" % sl.key


FAB_PATHS = [("fsa", False, None), ("sharded", False, None), ("replicated", False, None),
             ("ll", True, None), ("direct-sharded", True, None), ("direct-replicated", True, None),
             ("ll", True, MIXED_FMTS), ("direct-sharded", True, MIXED_FMTS), ("direct-replicated", True, MIXED_FMTS)]


# ---------------------------------------------------------------------------------------------------------------- the engine
# the step's (launch, stream) lists: paths A, C and G of test_step_paths_gpu.py; one exchange after the backward pass; local updates
A, C, G = PATHS["A"][3], PATHS["C"][3], PATHS["G"][3]
ONE = [(DIRECT_FWD, "main"), (MLP, "main"), (DENSE_WGRAD, "side"), (ONE_GRID, "main"), (EXCH, "join")]
A_LOCAL = A + [(LOCAL, "main")]


def _opt(kind, clip=None):
    s = dict(R.CASE_SPECS[kind])
    c = s["clip_gradient"] if clip is None else clip
    kw = dict(learning_rate=s["lr"], wd=s["wd"], rescale_grad=s["rescale_grad"], clip_gradient=None if c < 0 else c)
    if kind == "adam":
        return mx.optimizer.Adam(**kw)
    if kind == "sgd":
        return mx.optimizer.SGD(momentum=s["momentum"], **kw)
    return mx.optimizer.DCASGD(momentum=s["momentum"], lamda=s["lamda"], **kw)


def _batches(B, steps, seed):
    g = torch.Generator().manual_seed(seed)
    return [(torch.rand(B, 1, 28, 28, generator=g).to(dev()), torch.randint(0, 10, (B,), generator=g).float().to(dev())) for _ in range(steps)]


def _clip_for(P0, X, y, B, rescale):
    """A clip threshold that cuts the largest ~20 % of the first step's rescaled mean gradients (fp32 autograd of the demo CNN)."""
    ps = [p.detach().clone().requires_grad_(True) for p in P0]
    h = F.max_pool2d(torch.relu(F.conv2d(X, ps[0], ps[1])), 2)
    h = F.max_pool2d(torch.relu(F.conv2d(h, ps[2], ps[3])), 2).flatten(1)
    h = torch.relu(F.linear(h, ps[4], ps[5]))
    h = torch.relu(F.linear(h, ps[6], ps[7]))
    F.cross_entropy(F.linear(h, ps[8], ps[9]), y.long(), reduction="sum").backward()
    flat = torch.cat([p.grad.reshape(-1) for p in ps]).abs() * (rescale / B)
    return float(torch.quantile(flat[flat > 0].cpu(), 0.8))


# name -> (B, env, optimizer kind, engine kwargs, graph, the step's (launch, stream) list, attribute checks)
ENGINE_CASES = {
    "A-adam": (32, {}, "adam", {}, False, A, dict(overlap=True)),
    "A-adam-graph": (32, {}, "adam", {}, True, A, dict(overlap=True)),
    "A-sgd": (32, {}, "sgd", {}, False, A, dict(overlap=True)),
    "A-dcasgd": (32, {}, "dcasgd", {}, False, A, dict(overlap=True)),
    "C-adam": (32, {"GEOMX_FUSED_EXCHANGE": "1"}, "adam", {}, False, C, dict(fused_exchange=True)),
    "G-sgd": (96, {}, "sgd", {}, False, G, dict(direct_conv=False, fused_mlp=False)),
    "single-adam": (32, {"GEOMX_STEP_OVERLAP": "0"}, "adam", {}, False, ONE, dict(overlap=False)),
    "loopback-ov1-adam": (32, {"GEOMX_STEP_OVERLAP": "1"}, "adam", dict(loopback=True), False, A, dict(overlap=True)),
    "loopback-ov1-sgd": (32, {"GEOMX_STEP_OVERLAP": "1"}, "sgd", dict(loopback=True), False, A, dict(overlap=True)),
    "loopback-ov0-adam": (32, {"GEOMX_STEP_OVERLAP": "0"}, "adam", dict(loopback=True), False, ONE, dict(overlap=False)),
    "loopback-ov0-sgd": (32, {"GEOMX_STEP_OVERLAP": "0"}, "sgd", dict(loopback=True), False, ONE, dict(overlap=False)),
    "loopback-fp16": (32, {"GEOMX_STEP_OVERLAP": "1"}, "adam", dict(loopback=True, wire_dtype="fp16"), False, A, dict(overlap=True)),
    "loopback-fp8": (32, {"GEOMX_STEP_OVERLAP": "0"}, "sgd", dict(loopback=True, wire_dtype="fp8"), False, ONE, dict(overlap=False)),
    "async-adam": (32, {}, "adam", dict(mode="dist_async"), False, ONE, dict(overlap=False, mode="dist_async")),
    "local-adam": (32, {}, "adam", dict(update="local"), False, A_LOCAL, dict(update="local")),
    "local-dcasgd": (32, {}, "dcasgd", dict(update="local"), False, A_LOCAL, dict(update="local")),
    "hfa-sgd": (32, {}, "sgd", dict(hfa=(2, 2)), False, ONE, dict(update="local", hfa=(2, 2))),
}


def _snapshot(eng):
    f = eng.fabric
    ts = [f.param.tensor, f.w, f.s0, f.s1] + ([eng.Wl, eng.s0l, eng.s1l, eng.opt_state] if eng.update == "local" else [])
    return [(t, t.clone()) for t in ts]


def _engine_ref(eng, P0, spec, mutation=None):
    """The reference of an engine case (not yet stepped): push scale 1/B, the fabric's wire formats, the exchange's rounding order."""
    fmts = None
    if eng.fabric.tile_fmt is not None:
        fmt_of = {0: "fp32", 1: "fp16", 3: "fp8"}
        fmts = [fmt_of[int(eng.fabric.tile_fmt[sl.offset // 1024])] for sl in eng.layout.slots]
    # the LL exchange (one fused exchange in loop-back) rounds the scaled aggregate; the direct-protocol channels the raw gradient
    after = eng.fabric.loopback and not eng.overlap
    return R.UpdateRef(spec, P0, push_scale=1.0 / eng.B, fmts=fmts, round_after_scale=after, mutation=mutation)
