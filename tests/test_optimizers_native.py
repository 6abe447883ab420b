"""NAG, Signum, RMSProp, AdaGrad, AdaDelta and Ftrl as the update kernels run them, checked without a GPU:

* each class's Python ``update`` (the fallback path) against the fp64 rules of ``_optim_ref.py``, written from the reference's sources,
  over several steps with rescale, clip, wd and momentum active, and with the reference's ``clip_gradient = 0`` quirk;
* ``spec()`` packed by ``pack_hyper`` into the kernels' ``OptHyper``; the classes without a native kind give None;
* the ctypes mirrors of ``OptHyper`` / ``FabricParams`` against the layout the C headers assert;
* the TCP plane ships the pickled optimizer for kinds its C++ server does not run.

The update kernels' register and spill budgets are rows of ``test_kernel_budgets.py``.
"""
import os
import pickle
import re

import numpy as np
import pytest
import torch

import geomx_b200 as mx
from geomx_b200 import build
from geomx_b200.ndarray import NDArray
from geomx_b200.ops import _native_api as api

import _optim_ref as R

O = mx.optimizer

# name -> (constructor, kwargs): clip cuts part of the gradients, wd, rescale and momentum are active
CASES = {
    "nag": (O.NAG, dict(learning_rate=0.1, momentum=0.9, wd=0.02, rescale_grad=0.5, clip_gradient=0.3)),
    "nag-nomom": (O.NAG, dict(learning_rate=0.1, momentum=0.0, wd=0.02, rescale_grad=0.5, clip_gradient=0.3)),
    "signum": (O.Signum, dict(learning_rate=0.01, momentum=0.9, wd_lh=0.05, wd=0.02, rescale_grad=0.5, clip_gradient=0.3)),
    "signsgd": (O.Signum, dict(learning_rate=0.01, momentum=0.0, wd_lh=0.05, wd=0.02, rescale_grad=0.5, clip_gradient=0.3)),
    "rmsprop": (O.RMSProp, dict(learning_rate=0.01, gamma1=0.8, epsilon=1e-6, wd=0.02, rescale_grad=0.5, clip_gradient=0.3,
                                clip_weights=0.15)),
    "adagrad": (O.AdaGrad, dict(learning_rate=0.1, eps=1e-6, wd=0.02, rescale_grad=0.5, clip_gradient=0.3)),
    "adadelta": (O.AdaDelta, dict(rho=0.8, epsilon=1e-4, wd=0.02, rescale_grad=0.5, clip_gradient=0.3)),
    "ftrl": (O.Ftrl, dict(learning_rate=0.1, lamda1=0.05, beta=0.5, wd=0.02, rescale_grad=0.5, clip_gradient=0.3)),
}


def _run_python(opt, w0, grads):
    """The class's own ``update`` on fp64 tensors, one key."""
    w = NDArray(w0.clone())
    st = opt.create_state(0, w)
    for g in grads:
        opt.update(0, w, NDArray(g.clone()), st)
    return w._t


def _run_ref(spec, w0, grads):
    h = R.hyper(spec, fp32=False)
    w, s0 = w0.clone(), torch.zeros_like(w0)
    s1 = torch.zeros_like(w0)
    for t, g in enumerate(grads, 1):
        R.update(h, w, g.clone(), s0, s1, t)
    return w


def _data(seed, n=4000, steps=6):
    g = torch.Generator().manual_seed(seed)
    w0 = torch.randn(n, generator=g, dtype=torch.float64) * 0.1
    grads = [torch.randn(n, generator=g, dtype=torch.float64) * 0.5 for _ in range(steps)]
    for x in grads:
        x[torch.rand(n, generator=g) < 0.05] = 0.0
    return w0, grads


@pytest.mark.parametrize("case", list(CASES))
def test_python_update_matches_reference_rule(case):
    cls, kw = CASES[case]
    opt = cls(**kw)
    spec = opt.spec()
    assert spec is not None and spec["name"] in R.NEW_KINDS
    w0, grads = _data(len(case))
    got, ref = _run_python(opt, w0, grads), _run_ref(spec, w0, grads)
    cut = float(((grads[0] * kw["rescale_grad"]).abs() > kw["clip_gradient"]).double().mean())
    assert 0.1 < cut < 0.9, cut
    assert R.rel(got - w0, ref - w0) < 1e-12, (case, R.rel(got - w0, ref - w0))


@pytest.mark.parametrize("case", list(CASES))
def test_clip_zero(case):
    """``clip_gradient=0``: RMSProp, Ftrl and Signum do not clip (the reference forwards the clip only when truthy); NAG, AdaGrad and
    AdaDelta clip every gradient to 0."""
    cls, kw = CASES[case]
    kw = dict(kw, clip_gradient=0.0)
    opt = cls(**kw)
    spec = opt.spec()
    w0, grads = _data(3 + len(case))
    got, ref = _run_python(opt, w0, grads), _run_ref(spec, w0, grads)
    assert R.rel(got - w0, ref - w0) < 1e-12
    off = cls(**dict(kw, clip_gradient=None))
    same_as_off = R.rel(_run_python(off, w0, grads) - w0, got - w0) < 1e-12
    assert same_as_off == (spec["name"] in R.CLIP_ZERO_OFF or case == "signsgd"), case
    h = api.pack_hyper(spec)
    assert h.clip == (-1.0 if spec["name"] in R.CLIP_ZERO_OFF else 0.0)


# -------------------------------------------------------------------------------------------------------- literal reference expressions
def _literal(case, kw, w, g, state):
    """The reference's own expressions (optimizer.py and the operators of optimizer_op-inl.h), transcribed as they stand, in numpy fp64."""
    lr, wd, rs = kw.get("learning_rate"), kw["wd"], kw["rescale_grad"]
    c = kw.get("clip_gradient")
    clip_np = lambda x: np.clip(x, -c, c)
    if case == "nag":
        grad = g * rs
        if c is not None:
            grad = clip_np(grad)
        mom = state
        mom[:] *= kw["momentum"]
        grad += wd * w
        mom[:] += grad
        grad[:] += kw["momentum"] * mom
        w[:] += -lr * grad
    elif case == "signum":                           # SignumKernel, clip_gradient forwarded only when truthy
        mu, mom = kw["momentum"], state
        cg = c if c else -1.0
        gg = np.clip(rs * g, -cg, cg) if cg >= 0 else rs * g
        mom[:] = mu * mom - (1 - mu) * wd * w - (1 - mu) * gg
        w[:] = (1. - lr * kw["wd_lh"]) * w + lr * ((mom > 0).astype(np.float64) - (mom < 0))
    elif case == "signsgd":                          # SignSGDKernel
        w[:] = (1. - lr * wd) * w - lr * ((g > 0).astype(np.float64) - (g < 0))
    elif case == "rmsprop":                          # RMSPropUpdate
        cg, cw = (c if c else -1.0), (kw["clip_weights"] if kw["clip_weights"] else -1.0)
        n = state
        grad = rs * g + wd * w
        if cg >= 0:
            n[:] = (1. - kw["gamma1"]) * np.clip(grad, -cg, cg) ** 2 + kw["gamma1"] * n
            out = w - lr * (np.clip(grad, -cg, cg) / np.sqrt(n + kw["epsilon"]))
        else:
            n[:] = (1. - kw["gamma1"]) * (grad * grad) + kw["gamma1"] * n
            out = w - lr * (grad / np.sqrt(n + kw["epsilon"]))
        w[:] = np.clip(out, -cw, cw) if cw >= 0 else out
    elif case == "adagrad":
        grad = g * rs
        if c is not None:
            grad = clip_np(grad)
        history = state
        history[:] += np.square(grad)
        div = grad / np.sqrt(history + kw["eps"])
        w[:] += (div + w * wd) * -lr
    elif case == "adadelta":
        grad = g * rs
        if c is not None:
            grad = clip_np(grad)
        acc_g, acc_delta = state
        rho, eps = kw["rho"], kw["epsilon"]
        acc_g[:] = rho * acc_g + (1. - rho) * grad * grad
        cur = np.sqrt(acc_delta + eps) / np.sqrt(acc_g + eps) * grad
        acc_delta[:] = rho * acc_delta + (1. - rho) * cur * cur
        w[:] -= cur + wd * w
    elif case == "ftrl":                             # FtrlUpdate
        cg = c if c else -1.0
        z, n = state
        grad = rs * g
        if cg >= 0:
            grad = np.clip(grad, -cg, cg)
        z += grad - (np.sqrt(n + grad ** 2) - np.sqrt(n)) * w / lr
        n += grad ** 2
        w[:] = (np.sign(z) * kw["lamda1"] - z) / ((kw["beta"] + np.sqrt(n)) / lr + wd) * (np.abs(z) > kw["lamda1"])


@pytest.mark.parametrize("clip", ["clip", "clip0", "noclip"])
@pytest.mark.parametrize("case", ["nag", "signum", "signsgd", "rmsprop", "adagrad", "adadelta", "ftrl"])
def test_python_update_matches_literal_reference(case, clip):
    cls, kw = CASES[case]
    kw = dict(kw, clip_gradient={"clip": kw["clip_gradient"], "clip0": 0.0, "noclip": None}[clip])
    opt = cls(**kw)
    w0, grads = _data(11 + len(case) + len(clip))
    got = _run_python(opt, w0, grads)
    w = w0.numpy().copy()
    z = lambda: np.zeros_like(w)
    state = {"adadelta": (z(), z()), "ftrl": (z(), z())}.get(case, z())
    for g in grads:
        _literal(case, kw, w, g.numpy().copy(), state)
    assert R.rel(got - w0, torch.from_numpy(w) - w0) < 1e-12, case


def test_rmsprop_adds_wd_before_clip():
    """RMSProp regularises and then clips: with a clip that cuts every gradient the step is lr * clip / sqrt(n + eps) whatever wd is."""
    w0 = torch.full((8,), 1.0, dtype=torch.float64)
    g = torch.full((8,), 0.001, dtype=torch.float64)
    outs = []
    for wd in (0.5, 0.9):
        opt = O.RMSProp(learning_rate=0.1, gamma1=0.0, epsilon=0.0, wd=wd, clip_gradient=0.1)
        outs.append(_run_python(opt, w0, [g]))
    assert torch.allclose(outs[0], outs[1]) and torch.allclose(outs[0], w0 - 0.1)


# -------------------------------------------------------------------------------------------------------- spec and packing
def test_spec_packs_into_opt_hyper():
    for case, (cls, kw) in CASES.items():
        spec = cls(**kw).spec()
        info = api.OPT_KINDS[spec["name"]]
        h = api.pack_hyper(spec)
        f32 = lambda x: float(np.float32(x))
        assert h.kind == info.code == api.OPT_KIND[spec["name"]]
        assert (h.lr, h.wd, h.rescale) == (f32(spec["lr"]), f32(spec["wd"]), f32(spec["rescale_grad"]))
        for field, key, _ in info.fields:
            assert getattr(h, field) == f32(spec[key]), (case, field)
        assert h.sched.kind == 0
    assert api.pack_hyper(O.RMSProp(clip_weights=0.0).spec()).clip_weights == -1.0
    assert api.pack_hyper(O.RMSProp(clip_weights=-2.0).spec()).clip_weights == -1.0
    assert [k for k, v in api.OPT_KINDS.items() if v.s1_is_weight] == ["dcasgd"]
    assert (api.OPT_KIND["sgd"], api.OPT_KIND["adam"], api.OPT_KIND["dcasgd"]) == (0, 1, 2)
    sched = O.NAG(momentum=0.9, learning_rate=0.1, lr_scheduler=mx.lr_scheduler.FactorScheduler(step=10, factor=0.5)).spec()
    assert api.pack_hyper(sched).sched.kind == api.SCHED_KIND["factor"]


def test_no_native_kind_gives_none():
    for opt in (O.RMSProp(centered=True), O.Adamax(), O.Nadam(), O.FTML(), O.SGLD(), O.LBSGD(), O.Signum(momentum=-0.5)):
        assert opt.spec() is None, type(opt).__name__


def test_state_slots_follow_create_state():
    w = NDArray(torch.zeros(5))
    for case, (cls, kw) in CASES.items():
        opt = cls(**kw)
        s0, s1 = api.state_slots(opt.create_state(0, w))
        with_mom = opt.spec()["name"] in ("nag", "signum")
        two = opt.spec()["name"] in ("adadelta", "ftrl")
        assert (s0 is not None) == (not with_mom or kw["momentum"] != 0.0), case
        assert (s1 is not None) == two, case
    s0, s1 = api.state_slots(O.DCASGD(momentum=0.0).create_state(0, NDArray(torch.ones(3))))
    assert s0 is None and bool((s1 == 1).all())


# -------------------------------------------------------------------------------------------------------- C layout
def _header(name):
    with open(os.path.join(build.CSRC, "kernels", name)) as f:
        return f.read()


def test_opt_hyper_layout_matches_c():
    src = _header("optim.cuh")
    lay = api.OPT_HYPER_LAYOUT
    assert "sizeof(LrSchedule) == %d" % lay["sched_size"] in src
    for field in ("wd_lh", "lamda1", "kind", "sched"):
        assert "offsetof(OptHyper, %s) == %d" % (field, lay[field]) in src, field
        assert getattr(api.OptHyper, field).offset == lay[field]
    assert "sizeof(OptHyper) == %d" % lay["size"] in src
    # the C struct's float fields, in order, are the mirror's
    body = re.search(r"struct OptHyper \{(.*?)\};", src, re.S).group(1)
    names = re.findall(r"(\w+)\s*[,;]", re.sub(r"//.*", "", body).replace("float", "").replace("int", "").replace("LrSchedule", ""))
    assert names == [n for n, _ in api.OptHyper._fields_], names


def test_fabric_params_size_matches_c():
    import ctypes
    from geomx_b200.parallel import fabric
    src = _header("hips_ll.cuh")
    assert "sizeof(FabricParams) == %d" % fabric.FABRIC_PARAMS_BYTES in src
    assert "offsetof(FabricParams, h) == %d" % fabric.FABRIC_PARAMS_H_OFFSET in src
    assert ctypes.sizeof(fabric._FabricParams) == fabric.FABRIC_PARAMS_BYTES <= 4096
    assert fabric._OptHyperF is api.OptHyper


# -------------------------------------------------------------------------------------------------------- TCP plane
class _StubKV:
    rank = 0

    def __init__(self):
        self.sent = []

    def send_command_to_servers(self, head, body):
        self.sent.append((head, body))


def _dist_ps_set(optimizer):
    from geomx_b200.kvstore import dist_ps
    kv = object.__new__(dist_ps.KVStoreDist)
    kv._is_worker = True
    kv._kv = _StubKV()
    kv.set_optimizer(optimizer)
    return dist_ps, kv._kv.sent


def test_dist_ps_ships_pickled_optimizer_for_kinds_the_host_server_lacks():
    dist_ps, sent = _dist_ps_set(O.RMSProp(learning_rate=0.01))
    assert [h for h, _ in sent] == [dist_ps.CMD_CONTROLLER]
    assert isinstance(pickle.loads(sent[0][1].encode("latin1")), O.RMSProp)
    for opt in (O.NAG(momentum=0.9), O.Ftrl(), O.AdaDelta(), O.AdaGrad(), O.Signum()):
        _, sent = _dist_ps_set(opt)
        assert [h for h, _ in sent] == [dist_ps.CMD_CONTROLLER], type(opt).__name__
    _, sent = _dist_ps_set(O.Adam(learning_rate=0.01))
    assert [h for h, _ in sent] == [dist_ps.CMD_OPT_SPEC] and sent[0][1].startswith("name=adam")
