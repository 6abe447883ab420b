"""Every kernel path of the demo CNN's training step against an fp64 reference, at the batch sizes and data that select each path.

``HipsCNNTrainStep._steps()`` assembles the step from different kernel sets depending on the batch size and on environment switches:

  A  direct convolutions, one backward grid, fused dense chain    even B <= 32
  B  A with the backward as two launches                          GEOMX_CNN_BWD_ONE_LAUNCH=0
  C  A with the conv keys' exchange in the backward grid's tail   GEOMX_FUSED_EXCHANGE=1
  D  direct convolutions, dense part as wgmma GEMMs + head kernel even 32 < B <= 64, or GEOMX_FUSED_MLP=0
  E  im2col + GEMM convolutions with the max-pool in the epilogue odd B <= 31, or GEOMX_DIRECT_CONV=0
  F  E with GEMM (NCHW store) + separate max-pool kernel          GEOMX_NO_POOL_FUSION=1
  G  GEMM convolutions and GEMM dense part                        B = 33, B > 64

``tests/test_step_path.py`` checks the choice of path (``step_path``) without a GPU; this file checks that each path's launches run, in the
recorded order and on the recorded streams, and compute the step.

The reference takes the two max-pool arg-max decisions from the kernels (``idx1`` / ``idx2``): a window whose two largest candidates agree to
fp32 rounding can legitimately go either way.  Those decisions are checked separately against the fp64 first maximum, wherever the window is
not such a near-tie.  Exact ties (the zero background of the demo's images makes every conv0 window there a four-way tie) must resolve to the
first position, like torch's max-pool.

The file also tests the direct convolution kernels at their edges (list densities, batch limits, output contracts), the kernels of the GEMM
paths that the step calls but no other test does, the loss of confidently classified samples, and the split-K GEMM epilogue contract.
"""
import math

import pytest
import torch
import torch.nn.functional as F

from _cnn_ref import (CASE_IDS, CASES, GRAD_NAMES, PATHS, check_routing, conv_forward_ref, conv_params, dev, engine, images, nan,  # noqa: F401
                      nat, rel_err, route, step_params, step_reference, windows)

pytestmark = pytest.mark.gpu


# ---------------------------------------------------------------------------------------------------------------- 1. the step, per path
@pytest.mark.parametrize("data", ["rand", "patch"])
@pytest.mark.parametrize("path,B,env", CASES, ids=CASE_IDS)
def test_step_path_matches_fp64(nat, engine, path, B, env, data):
    """One training step of every kernel path: per-sample loss, logits and all 10 gradients against fp64 autograd (2e-5 relative: the
    direct convolutions are exact fp32 FMA chains, the GEMMs 3xTF32 = fp32-accurate; measured errors are printed).  A second pass on the same
    batch must give the same gradients: accumulators (column sums, conv0 bias atomics) and the fused exchange's ticket / round counters
    have to re-arm themselves.  With SGD at lr = 0 the exchange must also hand back the parameters unchanged."""
    g = torch.Generator().manual_seed(1000 * B + (7 if data == "patch" else 0) + ord(path))
    P0 = step_params(g)
    X = images(g, B, data)
    y = torch.randint(0, 10, (B,), generator=g).float().to(dev())
    eng = engine(B, env=env, use_graph=False, fused_zero_grad=False)
    for p, v in zip(eng.P, P0):
        p.copy_(v)
    eng.fabric.load_master_from_param()
    eng.x.copy_(X); eng.label.copy_(y)
    eng.z2.fill_(float("nan"))
    eng._body(); torch.cuda.synchronize()
    # the intended kernels ran (otherwise a case would quietly test another path)
    direct, fused_mlp, fused_exchange, want = PATHS[path]
    steps = [(n, s) for n, s, _ in eng._steps()]
    assert (eng.direct_conv, eng.fused_mlp, eng.fused_exchange) == (direct, fused_mlp, fused_exchange), (path, B, steps)
    assert steps == want, (path, B, steps)
    if not direct:        # the pooled conv1 GEMM leaves z2 untouched; the unfused form writes it and pools it separately
        assert bool(torch.isnan(eng.z2).all()) == (path != "F"), path
    loss, logits = eng.loss.clone(), eng.logits.clone()
    grads = [t.clone() for t in eng.G]
    loss_ref, logits_ref, grads_ref, ties = step_reference(P0, X, y, eng.idx1, eng.idx2)
    errs = {"loss": rel_err(loss, loss_ref), "logits": rel_err(logits, logits_ref)}
    errs.update({n: rel_err(a, b) for n, a, b in zip(GRAD_NAMES, grads, grads_ref)})
    print("\n  path %s B=%-2d %-5s  near-ties conv0/conv1 %d/%d, exact ties %d/%d  |  %s" % (
        path, B, data, ties[0], ties[2], ties[1], ties[3], "  ".join("%s %.1e" % kv for kv in errs.items())))
    bad = {k: v for k, v in errs.items() if not v < 2e-5}
    assert not bad, (path, B, data, bad)
    # second pass on the same batch: same result, parameters untouched
    eng._body(); torch.cuda.synchronize()
    again = [rel_err(a, b) for a, b in zip(eng.G, grads)]
    assert max(again) < 1e-6 and rel_err(eng.loss, loss) < 1e-6, (path, B, data, again)
    for i, (p, p0) in enumerate(zip(eng.P, P0)):
        assert torch.equal(p, p0), "parameter %d changed by an lr = 0 step (path %s)" % (i, path)


def test_switches_are_read_at_construction(nat, engine, monkeypatch):
    """The kernel path is chosen when the engine is constructed: step switches changed afterwards change neither the step's launches nor the
    graph that the host pipeline captures later on its second input buffer."""
    B = 32
    eng = engine(B, use_graph=True)
    g = torch.Generator().manual_seed(77)
    eng.x.copy_(images(g, B, "rand")); eng.label.copy_(torch.randint(0, 10, (B,), generator=g).float().to(dev()))
    steps = [(n, s) for n, s, _ in eng._steps()]
    assert steps == PATHS["A"][3], steps
    eng.capture(); torch.cuda.synchronize()
    assert eng.kernels_per_step == 6, eng.kernels_per_step
    for k, v in (("GEOMX_CNN_BWD_ONE_LAUNCH", "0"), ("GEOMX_FUSED_EXCHANGE", "1"), ("GEOMX_DIRECT_CONV", "0"), ("GEOMX_FUSED_MLP", "0"),
                 ("GEOMX_E2E_DIRECT_INPUT", "0")):
        monkeypatch.setenv(k, v)
    assert [(n, s) for n, s, _ in eng._steps()] == steps
    eng._pipeline()
    eng._alt_graph(); torch.cuda.synchronize()
    assert eng.kernels_per_step == 6, eng.kernels_per_step


# ---------------------------------------------------------------------------------------------------------------- 2. cnn_direct.cu at its edges
DIRECT_CASES = [(B, "rand", "default") for B in (1, 2, 3, 6, 32, 63, 64, 256)] + [(32, "patch", "posbias"), (6, "patch", "posbias")] + \
               [(8, "rand", r) for r in ("full", "empty", "dead0")]


@pytest.mark.parametrize("B,data,regime", DIRECT_CASES, ids=["B%d-%s-%s" % c for c in DIRECT_CASES])
def test_cnn_direct_kernels_at_edges(nat, B, data, regime):
    """cnn_fwd / cnn_bwd (any B) and cnn_wgrad1 / cnn_bwd_all (even B <= 64) against fp64, including their output contracts: dw0 / db0 are
    accumulated (two calls onto a non-zero start give start + 2 grad), dw1 / db1 are overwritten (NaN before)."""
    g = torch.Generator().manual_seed(B * 31 + len(regime) + len(data))
    x = images(g, B, data)
    w0, b0, w1, b1 = conv_params(g, regime)
    da2 = torch.randn(B, 32, 4, 4, generator=g).to(dev())
    a1, idx1 = nan(B, 16, 12, 12), nan(B, 16, 12, 12, dtype=torch.uint8)
    a2, idx2 = nan(B, 32, 4, 4), nan(B, 32, 4, 4, dtype=torch.uint8)
    nat.cnn_fwd(x, w0, b0, w1, b1, a1, idx1, a2, idx2)
    torch.cuda.synchronize()
    ps = [t.double().requires_grad_(True) for t in (w0, b0, w1, b1)]
    a1_ref, a2_ref, ties = conv_forward_ref(x.double(), *ps, idx1, idx2)
    (a2_ref * da2.double()).sum().backward()
    ref = {"dw0": ps[0].grad, "db0": ps[1].grad, "dw1": ps[2].grad, "db1": ps[3].grad}
    e_fwd = (rel_err(a1, a1_ref), rel_err(a2, a2_ref))
    assert e_fwd[0] < 1e-6 and e_fwd[1] < 1e-6, e_fwd
    n_lists = int((a2 > 0).sum())
    if regime == "full":
        assert n_lists == a2.numel()
    if regime == "empty":
        assert n_lists == 0
    if regime == "dead0":
        assert not bool((a1 > 0).any())
    zero_w0 = regime in ("empty", "dead0")      # no gradient reaches conv0: dw0 / db0 exactly 0, the accumulators untouched
    zero_w1 = regime == "empty"
    errs = {}

    def start(r):
        scale = float(r.abs().mean()) or 1.0
        return (torch.randn(r.shape, generator=g) * scale).to(dev())

    def check_acc(name, got, s, calls):
        if zero_w0:
            assert torch.equal(got, s), name
            assert float(ref[name].abs().max()) == 0.0, name
            errs[name] = 0.0
            return
        e = float((got.double() - s.double() - calls * ref[name]).norm() / (calls * ref[name]).norm())
        errs[name] = max(errs.get(name, 0.0), e)
        assert e < 1e-5, (name, e)

    def check_over(name, got):
        if zero_w1 or (name == "dw1" and regime == "dead0"):
            assert bool((got == 0).all()) and float(ref[name].abs().max()) == 0.0, name
            errs[name] = 0.0
            return
        e = rel_err(got, ref[name])
        errs[name] = max(errs.get(name, 0.0), e)
        assert e < 1e-5, (name, e)

    s_dw0, s_db0 = start(ref["dw0"]), start(ref["db0"])
    dw0, db0 = s_dw0.clone(), s_db0.clone()
    for _ in range(2):
        nat.cnn_bwd(x, w1, a1, idx1, a2, idx2, da2, dw0, db0)
    torch.cuda.synchronize()
    check_acc("dw0", dw0, s_dw0, 2); check_acc("db0", db0, s_db0, 2)
    if B % 2 == 0 and B <= 64:
        dw1, db1 = nan(32, 16, 5, 5), nan(32)
        for _ in range(2):
            assert nat.cnn_wgrad1(a1, a2, idx2, da2, dw1, db1)
        torch.cuda.synchronize()
        check_over("dw1", dw1); check_over("db1", db1)
        dw0, db0 = s_dw0.clone(), s_db0.clone()
        dw1, db1 = nan(32, 16, 5, 5), nan(32)
        for _ in range(2):
            nat.cnn_bwd_all(x, w1, a1, idx1, a2, idx2, da2, dw0, db0, dw1, db1)
        torch.cuda.synchronize()
        check_acc("dw0", dw0, s_dw0, 2); check_acc("db0", db0, s_db0, 2)
        check_over("dw1", dw1); check_over("db1", db1)
    print("\n  B=%-3d %-5s %-7s lists %d/%d  near-ties %d/%d exact ties %d/%d  a1 %.1e a2 %.1e  %s" % (
        B, data, regime, n_lists, a2.numel(), ties[0], ties[2], ties[1], ties[3], e_fwd[0], e_fwd[1],
        "  ".join("%s %.1e" % kv for kv in errs.items())))


@pytest.mark.parametrize("B", [3, 66])
def test_cnn_direct_batch_refusals(nat, B):
    """The conv1 weight-gradient body keeps every image's planes in shared memory and splits the batch in halves: odd B and B > 64 are
    refused, not computed wrongly."""
    t = lambda *s, dt=torch.float32: torch.zeros(*s, dtype=dt, device=dev())
    x, w1 = t(B, 1, 28, 28), t(32, 16, 5, 5)
    a1, idx1, a2, idx2 = t(B, 16, 12, 12), t(B, 16, 12, 12, dt=torch.uint8), t(B, 32, 4, 4), t(B, 32, 4, 4, dt=torch.uint8)
    da2, dw0, db0 = t(B, 32, 4, 4), t(16, 1, 5, 5), t(16)
    dw1, db1 = nan(32, 16, 5, 5), nan(32)
    assert nat.cnn_wgrad1(a1, a2, idx2, da2, dw1, db1) is False
    with pytest.raises(RuntimeError):
        nat.cnn_bwd_all(x, w1, a1, idx1, a2, idx2, da2, dw0, db0, dw1, db1)
    torch.cuda.synchronize()
    assert bool(torch.isnan(dw1).all()) and bool((dw0 == 0).all())


# ---------------------------------------------------------------------------------------------------------------- 3. the GEMM paths' own kernels
@pytest.mark.parametrize("data", ["rand", "patch"])
@pytest.mark.parametrize("B", [1, 33, 96])
def test_conv_relu_pool_im2col_fwd(nat, B, data):
    """conv0 + bias + ReLU + pool with the im2col slab of conv1 (paths E-G): pooled map and arg-max against fp64, slab == unfold(pooled)."""
    g = torch.Generator().manual_seed(40 + B)
    x = images(g, B, data)
    w0, b0, _, _ = conv_params(g, "posbias" if data == "patch" else "default")
    y, idx, col = nan(B, 16, 12, 12), nan(B, 16, 12, 12, dtype=torch.uint8), nan(B * 64, 400)
    nat.conv_relu_pool_im2col_fwd(x, w0, b0, y, idx, col, 5, 5)
    torch.cuda.synchronize()
    xd, w0d, b0d = x.double(), w0.double(), b0.double()
    z1 = F.conv2d(xd, w0d)
    ref = torch.relu(windows(z1).amax(-1) + b0d.view(1, -1, 1, 1))
    assert rel_err(y, ref) < 1e-6, rel_err(y, ref)
    near, exact = check_routing("idx", idx, z1, F.conv2d(xd.abs(), w0d.abs()), b0d)
    assert torch.equal(col, F.unfold(y, 5).transpose(1, 2).reshape(B * 64, 400))
    print("\n  B=%d %s: pooled %.1e, near-ties %d, exact ties %d" % (B, data, rel_err(y, ref), near, exact))


@pytest.mark.parametrize("B", [1, 33, 96])
def test_conv_relu_pool_wgrad_col2im(nat, B):
    """col2im of dcol1 + pool / ReLU backward + conv0 weight and bias gradient (paths E-G); dw / db are accumulated."""
    g = torch.Generator().manual_seed(50 + B)
    x = images(g, B, "rand")
    w0, b0, _, _ = conv_params(g)
    y, idx, col = nan(B, 16, 12, 12), nan(B, 16, 12, 12, dtype=torch.uint8), nan(B * 64, 400)
    nat.conv_relu_pool_im2col_fwd(x, w0, b0, y, idx, col, 5, 5)
    dcol = torch.randn(B * 64, 400, generator=g).to(dev())
    da1 = F.fold(dcol.double().reshape(B, 64, 400).transpose(1, 2), (12, 12), 5)
    dz1 = route(torch.where(y > 0, da1, torch.zeros_like(da1)), idx)
    ref_dw = torch.nn.grad.conv2d_weight(x.double(), (16, 1, 5, 5), dz1)
    ref_db = dz1.sum((0, 2, 3))
    s_dw, s_db = torch.randn(16, 1, 5, 5, generator=g).to(dev()), torch.randn(16, generator=g).to(dev())
    dw, db = s_dw.clone(), s_db.clone()
    for _ in range(2):
        nat.conv_relu_pool_wgrad_col2im(x, dcol, y, idx, dw, db, (16, 1, 5, 5), 5, 5)
    torch.cuda.synchronize()
    e_dw = rel_err(dw.double() - s_dw.double(), 2 * ref_dw)
    e_db = rel_err(db.double() - s_db.double(), 2 * ref_db)
    print("\n  B=%d: dw %.1e db %.1e" % (B, e_dw, e_db))
    assert e_dw < 1e-5 and e_db < 1e-5, (e_dw, e_db)


@pytest.mark.parametrize("B", [1, 33, 96])
def test_pool_relu_bwd_rows(nat, B):
    """Pool + ReLU backward of conv1 into pixel-major rows (the dWc1 / dcol1 GEMM operand) and the accumulated conv1 bias gradient."""
    g = torch.Generator().manual_seed(60 + B)
    dp = torch.randn(B, 32, 4, 4, generator=g).to(dev())
    pooled = torch.relu(torch.randn(B, 32, 4, 4, generator=g)).to(dev())
    idx = torch.randint(0, 4, (B, 32, 4, 4), generator=g).to(torch.uint8).to(dev())
    rows = nan(B * 64, 32)
    s_db = torch.randn(32, generator=g).to(dev())
    db = s_db.clone()
    nat.pool_relu_bwd_rows(dp, pooled, idx, rows, db)
    torch.cuda.synchronize()
    dz = route(torch.where(pooled > 0, dp, torch.zeros_like(dp)), idx)
    assert torch.equal(rows, dz.permute(0, 2, 3, 1).reshape(B * 64, 32))
    e = rel_err(db.double() - s_db.double(), dz.double().sum((0, 2, 3)))
    assert e < 1e-5, e


def head_reference(a, W, bias, label):
    ps = [t.double().requires_grad_(True) for t in (a, W, bias)]
    logits = F.linear(ps[0], ps[1], ps[2])
    loss = F.cross_entropy(logits, label.long(), reduction="none")
    loss.sum().backward()
    da = ps[0].grad * (a > 0)
    return loss.detach(), logits.detach(), ps[1].grad, ps[2].grad, da, da.sum(0)


@pytest.mark.parametrize("C", [2, 10, 32])
@pytest.mark.parametrize("B", [1, 33, 96])
def test_head_fwd_bwd(nat, B, C):
    """Classifier head of paths D and G: logits, softmax-CE loss, dW, db, the ReLU-masked input gradient and its column sum (the previous
    layer's bias gradient) against fp64."""
    K = 128
    g = torch.Generator().manual_seed(70 + B * C)
    a = torch.relu(torch.randn(B, K, generator=g)).to(dev())
    W = (torch.randn(C, K, generator=g) * 0.1).to(dev())
    bias = (torch.randn(C, generator=g) * 0.1).to(dev())
    label = torch.randint(0, C, (B,), generator=g).float().to(dev())
    outs = [nan(B), nan(B, C), nan(C, K), nan(C), nan(B, K), nan(K)]
    nat.head_fwd_bwd(a, W, bias, label, *outs, True)
    torch.cuda.synchronize()
    refs = head_reference(a, W, bias, label)
    errs = [rel_err(o, r) for o, r in zip(outs, refs)]
    print("\n  B=%d C=%d: loss %.1e logits %.1e dW %.1e db %.1e da %.1e dbias_prev %.1e" % ((B, C) + tuple(errs)))
    assert max(errs) < 1e-5, errs


def test_head_fwd_bwd_refusals(nat):
    """More than 32 classes (one warp holds a row's logits) and K not a multiple of 4 (128-bit staging loads) are refused."""
    for B, K, C in ((4, 128, 33), (4, 126, 10)):
        a, W, bias = torch.rand(B, K, device=dev()), torch.rand(C, K, device=dev()), torch.rand(C, device=dev())
        outs = [nan(B), nan(B, C), nan(C, K), nan(C), nan(B, K), nan(K)]
        with pytest.raises(RuntimeError):
            nat.head_fwd_bwd(a, W, bias, torch.zeros(B, device=dev()), *outs, True)


@pytest.mark.parametrize("C", [10, 100])
def test_softmax_ce(nat, C):
    """Warp-per-row softmax cross-entropy forward / backward; C = 100 runs each lane over several classes."""
    R = 96
    g = torch.Generator().manual_seed(80 + C)
    x = (torch.randn(R, C, generator=g) * 3).to(dev())
    label = torch.randint(0, C, (R,), generator=g).float().to(dev())
    dloss = torch.randn(R, generator=g).to(dev())
    xd = x.double().requires_grad_(True)
    loss_ref = F.cross_entropy(xd, label.long(), reduction="none")
    (loss_ref * dloss.double()).sum().backward()
    loss = nat.softmax_ce_fwd(x, label)
    dx = nat.softmax_ce_bwd(x, label, dloss)
    dx1 = nat.softmax_ce_bwd(x, label, None)          # no dloss: unit weights
    torch.cuda.synchronize()
    p = torch.softmax(xd.detach(), 1) - F.one_hot(label.long(), C).double()
    errs = (rel_err(loss, loss_ref), rel_err(dx, xd.grad), rel_err(dx1, p))
    assert max(errs) < 1e-5, errs


def confident_logits(g, B, C):
    """Logits whose label entry leads the others by margins spread evenly over [0, 20] (loss from ~2 down to ~2e-8)."""
    margin = torch.linspace(0, 20, B, dtype=torch.float64)
    z = torch.randn(B, C, generator=g, dtype=torch.float64)
    label = torch.randint(0, C, (B,), generator=g)
    others = z.masked_fill(F.one_hot(label, C).bool(), -math.inf).amax(1)
    z[torch.arange(B), label] = others + margin
    return z.float(), label.float(), margin


@pytest.mark.parametrize("kernel", ["softmax_ce_fwd", "head_fwd_bwd", "mlp_chain"])
def test_confident_loss(nat, kernel):
    """The per-sample loss of confidently classified samples is tiny (9 e^-margin), so an absolute error of a few 1e-7 in the log is a large
    relative one.  Within each band of margins the kernel's worst error against fp64 (of the kernel's own logits) must stay within 4x the worst
    error of fp32 torch on the same logits, plus 5e-8."""
    C = 10
    B = 32 if kernel == "mlp_chain" else 96
    g = torch.Generator().manual_seed(90)
    z, label, margin = confident_logits(g, B, C)
    lab = label.to(dev())
    loss = nan(B)
    if kernel == "softmax_ce_fwd":
        logits = z.to(dev())
        nat.softmax_ce_fwd(logits, lab, loss)
    elif kernel == "head_fwd_bwd":
        # a = [logits | 0 0], W = identity: the head's own logits are the given ones, exactly
        K = 12
        a = torch.zeros(B, K, device=dev()); a[:, :C] = z.to(dev())
        W = torch.zeros(C, K, device=dev()); W[:, :C] = torch.eye(C, device=dev())
        logits = nan(B, C)
        nat.head_fwd_bwd(a, W, torch.zeros(C, device=dev()), lab, loss, logits, nan(C, K), nan(C), nan(B, K),
                         nan(K), True)
    else:
        # identity weights pass x[:, :10] (shifted to positive, so the ReLUs are transparent) through both hidden layers to the logits
        x = torch.zeros(B, 512, device=dev()); x[:, :C] = (z + 40).to(dev())
        eye = lambda n, k: torch.eye(n, k, device=dev())
        w = [eye(256, 512), torch.zeros(256, device=dev()), eye(128, 256), torch.zeros(128, device=dev()), eye(C, 128), torch.zeros(C, device=dev())]
        logits = nan(B, C)
        gr = [nan(256, 512), nan(256), nan(128, 256), nan(128), nan(C, 128), nan(C), nan(B, 512)]
        assert nat.mlp_chain(x, *w, lab, loss, logits, *gr)
    torch.cuda.synchronize()
    exact = F.cross_entropy(logits.double(), lab.long(), reduction="none")
    torch32 = F.cross_entropy(logits, lab.long(), reduction="none")
    e_k = (loss.double() - exact).abs().cpu()
    e_t = (torch32.double() - exact).abs().cpu()
    for lo, hi in ((0, 4), (4, 10), (10, 20.5)):
        band = (margin >= lo) & (margin < hi)
        mk, mt = float(e_k[band].max()), float(e_t[band].max())
        print("\n  %s margins [%g, %g): kernel max abs err %.2e, fp32 torch %.2e" % (kernel, lo, hi, mk, mt))
        assert mk <= 4 * mt + 5e-8, (kernel, lo, hi, mk, mt)


# ---------------------------------------------------------------------------------------------------------------- 4. split-K GEMM contract
def test_gemm_split_k_refuses_relu(nat):
    """With split_k > 1 every split applies the epilogue to its partial sum; ReLU is not linear, so the combination is refused."""
    g = torch.Generator().manual_seed(95)
    A, B = torch.randn(64, 2048, generator=g).to(dev()), torch.randn(96, 2048, generator=g).to(dev())
    D = torch.zeros(64, 96, device=dev())
    with pytest.raises(RuntimeError):
        nat.gemm(A, B, D, relu=True, split_k=8)
    torch.cuda.synchronize()
    assert not bool(D.any())
    nat.gemm(A, B, D, relu=True)
    assert rel_err(D, torch.relu(A.double() @ B.double().t())) < 2e-6


@pytest.mark.parametrize("K", [2048, 2052])
@pytest.mark.parametrize("split_k", [2, 7, 16])
def test_gemm_split_k_bias_mask_colsum(nat, split_k, K):
    """Split-K with bias + mask + column sum into a zeroed D: the bias is added by one split only, mask and column sum are linear.  K = 2052
    leaves a short last K block, and with 7 / 16 splits a short last split."""
    M, N = 200, 72
    g = torch.Generator().manual_seed(96 + K + split_k)
    A, B = torch.randn(M, K, generator=g).to(dev()), torch.randn(N, K, generator=g).to(dev())
    bias, mask = torch.randn(N, generator=g).to(dev()), torch.randn(M, N, generator=g).to(dev())
    D, cs = torch.zeros(M, N, device=dev()), torch.zeros(N, device=dev())
    nat.gemm(A, B, D, bias=bias, mask=mask, colsum=cs, split_k=split_k)
    torch.cuda.synchronize()
    ref = (A.double() @ B.double().t() + bias.double()) * (mask > 0)
    e = (rel_err(D, ref), rel_err(cs, ref.sum(0)))
    assert max(e) < 2e-6, e
