"""The fp64 update reference of ``tests/_update_ref.py`` against the optimizer classes, and its mutations against the GPU tests' tolerances.

``tests/test_update_paths_gpu.py`` checks every optimizer update path of the kernels against ``_update_ref``.  This file (CPU only) shows
that the reference computes what ``geomx_b200.optimizer``'s SGD / Adam / DCASGD ``update()`` compute, and that each named mutation of it (a
plausible kernel bug) moves the result by at least 100x the tolerance the GPU tests allow, on gradient sequences of the demo CNN's
magnitudes — so those tolerances can catch each of those bugs.
"""
import pytest
import torch

import geomx_b200 as mx

import _update_ref as R

SHAPES = [(7,), (33, 5), (4, 3, 5, 5), (1,), (300,)]


def _optimizers():
    return {
        "sgd": mx.optimizer.SGD(learning_rate=0.1, momentum=0.9, wd=0.01, clip_gradient=0.02, rescale_grad=2.0),
        "sgd0": mx.optimizer.SGD(learning_rate=0.1, wd=0.01, clip_gradient=0.02, rescale_grad=0.5),
        "adam": mx.optimizer.Adam(learning_rate=0.01, wd=0.05, clip_gradient=0.02, rescale_grad=1.5),
        "dcasgd": mx.optimizer.DCASGD(learning_rate=0.1, momentum=0.9, lamda=40.0, wd=0.01, clip_gradient=0.02, rescale_grad=2.0),
        "dcasgd0": mx.optimizer.DCASGD(learning_rate=0.1, lamda=40.0, wd=0.01, clip_gradient=0.05),
    }


@pytest.mark.parametrize("name", ["sgd", "sgd0", "adam", "dcasgd", "dcasgd0"])
def test_reference_matches_optimizer_classes(name):
    """Several steps on random shapes with clip, wd, momentum, rescale and per-key multipliers all active: the reference and the optimizer
    class's ``update()`` (run in fp64 on CPU tensors) agree to fp64 rounding — weights and every state slot."""
    g = torch.Generator().manual_seed(len(name) * 17 + ord(name[-1]))
    opt = _optimizers()[name]
    mults = [(0.5 + 0.5 * i, 2.0 - 0.4 * i) for i in range(len(SHAPES))]
    opt.set_lr_mult({i: m[0] for i, m in enumerate(mults)})
    opt.set_wd_mult({i: m[1] for i, m in enumerate(mults)})
    W0 = [torch.randn(s, generator=g, dtype=torch.float64) * 0.1 for s in SHAPES]
    ws = [w.clone() for w in W0]
    states = [opt.create_state(i, w) for i, w in enumerate(ws)]
    ref = R.UpdateRef(opt.spec(), W0, mults=mults)
    ref.h = R.hyper(opt.spec(), fp32=False)        # the classes compute with the Python floats
    clipped = 0
    for k in range(5):
        grads = [torch.randn(s, generator=g, dtype=torch.float64) * 0.01 * (1 + k) for s in SHAPES]
        for i, (w, gr) in enumerate(zip(ws, grads)):
            opt.update(i, w, gr, states[i])
        clipped += sum(int((gr.abs() * opt.rescale_grad > opt.clip_gradient).sum()) for gr in grads)
        _ref_step64(ref, grads)
        for i, w in enumerate(ws):
            assert R.rel(w, ref.w[i]) < 1e-12, (name, k, i, R.rel(w, ref.w[i]))
    assert clipped > 0, "the clip threshold cut nothing"
    for i, st in enumerate(states):
        if name == "adam":
            m, v = st
            assert R.rel(m._t, ref.s0[i]) < 1e-12 and R.rel(v._t, ref.s1[i]) < 1e-12
        elif name.startswith("dcasgd"):
            mom, prev = st
            assert R.rel(prev._t, ref.s1[i]) < 1e-15
            if mom is not None:
                assert R.rel(mom._t, ref.s0[i]) < 1e-12
        elif st is not None:
            assert R.rel(st._t, ref.s0[i]) < 1e-12
    assert ref.t == [5] * len(SHAPES)


def _ref_step64(ref, grads):
    """``UpdateRef.step`` rounds the pushed gradient to the wire format (fp32 at least); for the class comparison the update itself is
    what is checked, so feed it the fp64 gradients directly."""
    for i, gr in enumerate(grads):
        ref.t[i] += 1
        lm, wm = ref.mults[i]
        R.update(ref.h, ref.w[i], gr.double() * ref.push_scale, ref.s0[i], ref.s1[i], ref.t[i], lm, wm)


def test_dcasgd_previous_weight_starts_at_the_weight():
    """The reference's DCASGD state is ``(mom, weight.copy())``: a first update from a non-zero weight has no ``lamda * g^2 * w`` term."""
    opt = mx.optimizer.DCASGD(learning_rate=0.1, lamda=10.0)
    w = torch.full((4,), 0.5, dtype=torch.float64)
    g = torch.full((4,), 0.3, dtype=torch.float64)
    st = opt.create_state(0, w)
    opt.update(0, w, g, st)
    assert torch.allclose(w, torch.full((4,), 0.5 - 0.1 * 0.3, dtype=torch.float64))
    ref = R.UpdateRef(opt.spec(), [torch.full((4,), 0.5)])
    ref.step([g.float()])
    assert R.rel(ref.w[0], w) < 1e-7
    bad = R.UpdateRef(opt.spec(), [torch.full((4,), 0.5)], mutation="dcasgd_prev_zero")
    bad.step([g.float()])
    assert R.rel(bad.w[0], w) > 1e-2


def test_fp8_wire_emulation():
    """Block-scaled e4m3: per 128-value block the largest magnitude is represented exactly (it maps to 448), every value within e4m3's
    relative step (2^-4 of the value, or the block's subnormal step), signs and zeros kept, a short last block padded."""
    g = torch.Generator().manual_seed(3)
    x = torch.randn(1000, generator=g) * torch.logspace(-4, 1, 1000)
    y = R.fp8_wire(x)
    assert y.shape == x.shape
    for b in range(0, 1000, 128):
        xb, yb = x[b:b + 128], y[b:b + 128]
        i = int(xb.abs().argmax())
        assert abs(float(yb[i]) - float(xb[i])) <= 1e-6 * abs(float(xb[i]))
        scale = float(xb.abs().max()) / 448.0
        err = (yb - xb).abs()
        assert bool((err <= xb.abs() * 2.0 ** -4 + scale * 2.0 ** -9 * 1.01).all())
    assert bool((torch.sign(y) == torch.sign(x)).all() | (y == 0).all())
    assert bool((R.fp8_wire(torch.zeros(130)) == 0).all())


CNN_SHAPES = [(16, 1, 5, 5), (16,), (32, 16, 5, 5), (32,), (256, 512), (256,), (128, 256), (128,), (10, 128), (10,)]


def test_mutations_are_far_outside_the_gpu_tolerance():
    """On synthetic gradient sequences of the CNN's magnitudes and with the GPU tests' optimizer settings, every mutation that applies to an
    optimizer moves the weights' displacement by at least 100x the GPU tests' displacement tolerance."""
    gen = torch.Generator().manual_seed(11)
    W0 = [torch.randn(s, generator=gen) * 0.1 for s in CNN_SHAPES]
    mults = [(0.5, 2.0), (2.0, 0.0), (1.0, 1.5), (0.25, 1.0), (1.5, 0.5), (1.0, 1.0), (0.75, 3.0), (1.0, 1.0), (1.25, 0.25), (1.0, 1.0)]
    grads = R.cnn_like_grads(gen, CNN_SHAPES, 6, batch=32)
    checked = []
    for kind, spec in R.CASE_SPECS.items():
        for use_mults in (False, True):
            m = mults if use_mults else None
            good = R.UpdateRef(spec, W0, mults=m, push_scale=1 / 32)
            for gs in grads:
                good.step(gs)
            for mut in R.relevant_mutations(spec, push_scale=1 / 32, mults=m):
                bad = R.UpdateRef(spec, W0, mults=m, push_scale=1 / 32, mutation=mut)
                for gs in grads:
                    bad.step(gs)
                e = R.displacement_err(bad.w, W0, good.w)
                checked.append((kind, use_mults, mut, e))
                assert e >= 100 * R.DISP_TOL, (kind, use_mults, mut, e)
    got = {m for _, _, m, _ in checked}
    assert got == set(R.MUTATIONS), set(R.MUTATIONS) - got
    for c in checked:
        print("  %-7s mults=%-5s %-20s displacement error %.2e" % c)
