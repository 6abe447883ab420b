"""The fp64 update reference of ``tests/_update_ref.py`` against the optimizer classes, and its mutations against the GPU tests' tolerances.

``tests/test_update_paths_gpu.py`` checks every optimizer update path of the kernels against ``_update_ref``.  This file (CPU only) shows
that the reference computes what ``geomx_b200.optimizer``'s SGD / Adam / DCASGD ``update()`` compute, and that each named mutation of it (a
plausible kernel bug) moves the result by at least 100x the tolerance the GPU tests allow, on gradient sequences of the demo CNN's
magnitudes — so those tolerances can catch each of those bugs.
"""
import math

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


# ---------------------------------------------------------------------------------------------------------- Bi-Sparse tiles and DGT
def test_bsc_stage_hand_made_tiles():
    """The Bi-Sparse stage on hand-made tiles: the K largest |v| go, ties at the K-th magnitude to the lowest index; sent entries are
    cleared in u and v, the rest carries over (u = 0.9u + g, v += u); the aggregate is what ``bsc_decompress`` makes of the (value, index)
    list, and the pull (``bsc_pull_compress`` of the aggregate, then zero + scatter with ``-1`` padding) returns its non-zeros."""
    from geomx_b200.kvstore import compression as gc
    g1 = torch.zeros(1024, dtype=torch.float64)
    g1[[5, 100, 700]] = 3.0
    g1[[9, 400]] = -3.0
    g1[50] = 7.0
    g1[[2, 3]] = 0.5
    K = 3
    u, v = torch.zeros(1024, dtype=torch.float64), torch.zeros(1024, dtype=torch.float64)
    agg, sels = R.bsc_round(u, v, g1, K)
    assert sels[0].tolist() == [5, 9, 50]
    zipped = torch.cat([g1[sels[0]], sels[0].double()]).float()
    assert torch.equal(agg.float(), gc.bsc_decompress(zipped, 1024))
    assert R.selection_slack(g1, sels[0], K) == 0.0
    rest = g1.clone()
    rest[sels[0]] = 0.0
    assert torch.equal(u, rest) and torch.equal(v, rest)
    # pull: the aggregate's non-zeros in index order, padded with index -1, scattered into a zeroed (here: dirty) tile
    pulled = gc.bsc_pull_compress(agg.float(), K / 1024, 1)
    assert pulled[K:].tolist() == [5.0, 9.0, 50.0]
    assert torch.equal(gc.bsc_decompress(pulled, 1024, out=torch.full((1024,), 9.0), accumulate=False), agg.float())
    # second round: momentum on what was not sent
    g2 = torch.zeros(1024, dtype=torch.float64)
    g2[700] = 1.0
    agg2, sels2 = R.bsc_round(u, v, g2, K)
    u_exp = rest * R.BSC_MOMENTUM + g2
    v_exp = rest + u_exp
    assert sels2[0].tolist() == [100, 400, 700]         # |v| = 3 + 0.9*3 (100, 400) and 3 + 0.9*3 + 1 (700)
    assert torch.equal(agg2[[100, 400, 700]], v_exp[[100, 400, 700]])
    # the mutations on the same tiles
    u, v = torch.zeros(1024, dtype=torch.float64), torch.zeros(1024, dtype=torch.float64)
    assert R.bsc_round(u, v, g1, K, mutation="bsc_ties_high_index")[1][0].tolist() == [50, 400, 700]
    u, v = torch.zeros(1024, dtype=torch.float64), torch.zeros(1024, dtype=torch.float64)
    R.bsc_round(u, v, g1, K, mutation="bsc_residual_kept")
    assert torch.equal(v, g1)
    # fewer than K non-zeros: every non-zero goes, the rest of the K packets carry zeros of the lowest indices
    u, v = torch.zeros(1024, dtype=torch.float64), torch.zeros(1024, dtype=torch.float64)
    g3 = torch.zeros(1024, dtype=torch.float64)
    g3[[600, 601]] = -2.0
    agg3, sels3 = R.bsc_round(u, v, g3, 5)
    assert sels3[0].tolist() == [0, 1, 2, 600, 601] and torch.equal(agg3, g3)
    # the slack of a selection that is not a top-K
    assert R.selection_slack(g1, torch.tensor([5, 9, 2]), K) > 0.5
    assert R.selection_slack(g1, torch.tensor([5, 9, 50, 100]), K) == float("inf")
    assert R.selection_slack(g3, torch.tensor([600]), 5) == float("inf")
    assert R.bsc_k(0.01) == 10 and R.bsc_k(1e-6) == 1 and R.bsc_k(0.5) == 512


def test_per_tile_formats_match_per_key_formats():
    """A key whose formats are given per tile computes what the per-key format computes when every tile has it; a mixed key rounds each
    tile by its own format."""
    gen = torch.Generator().manual_seed(21)
    shapes = [(3000,), (1025,)]
    W0 = [torch.randn(s, generator=gen) * 0.1 for s in shapes]
    grads = R.cnn_like_grads(gen, shapes, 3)
    spec = R.CASE_SPECS["adam"]
    for after in (False, True):
        a = R.UpdateRef(spec, W0, push_scale=1 / 32, fmts=["fp8", "fp16"], round_after_scale=after)
        b = R.UpdateRef(spec, W0, push_scale=1 / 32, fmts=[["fp8"] * 3, ["fp16"] * 2], round_after_scale=after)
        for gs in grads:
            a.step(gs)
            b.step(gs)
        assert all(torch.equal(x, y) for x, y in zip(a.w, b.w))
        assert all(torch.equal(x, y) for x, y in zip(a.params(), b.params()))
    m = R.UpdateRef(None, W0, push_scale=1 / 32, fmts=[["fp32", "fp8", "fp16"], "fp32"], round_after_scale=True)
    m.step(grads[0])
    s = grads[0][0].float() * (1 / 32)
    assert torch.equal(m.w[0][:1024], s[:1024].double())
    assert torch.equal(m.w[0][1024:2048], R.fp8_wire(s[1024:2048]).double())
    assert torch.equal(m.w[0][2048:], R.fp16_wire(s[2048:]).double())


def test_num_important_matches_the_fabric():
    """The reference's size of the important set equals ``dgt_num_important`` of the fabric, fixed and adaptive, on random and degenerate
    contributions."""
    from geomx_b200.parallel.fabric import dgt_num_important
    gen = torch.Generator().manual_seed(4)
    for n in (1, 2, 7, 100, 333):
        for c in (torch.rand(n, generator=gen) ** 4, torch.zeros(n), torch.ones(n)):
            c = c.sort(descending=True).values
            for k in (0.1, 0.5, 0.8, 1.0):
                for adaptive, k_min in ((False, 0.2), (True, 0.2), (True, 0.05), (True, 0.6)):
                    assert R.num_important(c, k, adaptive, k_min) == dgt_num_important(c, k, adaptive, k_min), (n, k, adaptive, k_min)


def _stage_case():
    """The CNN's keys, Bi-Sparse on those >= 1000 elements (the bench's ``bsc`` configuration), Adam on the aggregate; CNN-like gradient
    sums on a grid of 2^-4 so that tiles have exact ties at their K-th magnitude (as quantised gradients do)."""
    gen = torch.Generator().manual_seed(12)
    W0 = [torch.randn(s, generator=gen) * 0.1 for s in CNN_SHAPES]
    grads = [[torch.round(g / 0.0625) * 0.0625 for g in gs] for gs in R.cnn_like_grads(gen, CNN_SHAPES, 6, batch=32)]
    fmts = ["bsc" if math.prod(s) >= 1000 else "fp32" for s in CNN_SHAPES]
    return W0, grads, fmts


def test_stage_mutations_are_far_outside_the_gpu_tolerance():
    """Every Bi-Sparse mutation moves the weights' displacement (or, for the scale applied after the selection, which is linear and so only
    visible in the carried state, ``u`` / ``v``) by at least 100x the GPU tests' tolerance; so does skipping the DGT demotion."""
    W0, grads, fmts = _stage_case()
    spec = R.CASE_SPECS["adam"]
    run = lambda mut: _run(R.UpdateRef(spec, W0, push_scale=1 / 32, fmts=fmts, round_after_scale=True, mutation=mut), grads)
    good = run(None)
    out = {}
    for mut in ("bsc_no_momentum", "bsc_residual_kept", "bsc_ties_high_index", "bsc_scale_after_select"):
        bad = run(mut)
        e = R.displacement_err(bad.w, W0, good.w)
        if mut == "bsc_scale_after_select":
            assert e < 1e-6, e                   # linear: the aggregate is the same
            e = max(R.rel(b, a) for a, b in zip(good.u + good.v, bad.u + bad.v) if a.norm() > 0)
        out[mut] = e
    # DGT: fp16 keys, re-ranked after two rounds by the reference's own contribution EMA; half the tiles demoted
    fm16 = ["fp16" if math.prod(s) >= 1000 else "fp32" for s in CNN_SHAPES]
    res = {}
    for mut in (None, "dgt_no_demotion"):
        ref = R.UpdateRef(spec, W0, push_scale=1 / 32, fmts=list(fm16), round_after_scale=True, mutation=mut)
        ema = None
        for k, gs in enumerate(grads):
            ref.step(gs)
            mean = torch.cat(ref.agg).abs().view(-1, 1024).mean(1)
            ema = mean if ema is None else R.dgt_ema(ema, mean, 0.3)
            if k == 1:
                base = [f for i in range(len(W0)) for f in ref.tile_fmts(i)]
                _, n_imp, new = R.dgt_formats(base, ema, 0.5, mutation=mut)
                assert n_imp == round(0.5 * len(base))
                pos = 0
                for i in range(len(W0)):
                    T = len(ref.tile_fmts(i))
                    ref.fmts[i] = new[pos:pos + T]
                    pos += T
        res[mut] = ref
    assert any("fp8" in f for f in res[None].fmts if isinstance(f, list))
    out["dgt_no_demotion"] = R.displacement_err(res["dgt_no_demotion"].w, W0, res[None].w)
    for m, e in out.items():
        print("  %-24s %.2e" % (m, e))
    assert set(out) == set(R.STAGE_MUTATIONS)
    weak = {m: e for m, e in out.items() if not e >= 100 * R.DISP_TOL}
    assert not weak, weak


def _run(ref, grads):
    for gs in grads:
        ref.step(gs)
    return ref
