"""GPU numerics: every hand-written sm_90a kernel against the plain PyTorch fp32 definition of the same op."""
import math

import numpy as np
import pytest
import torch

import geomx_b200 as mx

from _cnn_ref import dev, engine, nat, rel_err, step_reference  # noqa: F401  (nat, engine: fixtures)

pytestmark = pytest.mark.gpu


# ---------------------------------------------------------------------------------------------------------------- GEMM
@pytest.mark.parametrize("a_mn,b_mn", [(False, False), (False, True), (True, False), (True, True)])
@pytest.mark.parametrize("M,N,K", [(32, 256, 512), (128, 256, 32), (2048, 32, 400), (2048, 400, 32), (200, 72, 100), (256, 512, 32)])
def test_gemm_tf32_majors(nat, a_mn, b_mn, M, N, K):
    torch.manual_seed(0)
    A = torch.randn(M, K, device=dev()); B = torch.randn(N, K, device=dev())
    Am = A.t().contiguous() if a_mn else A
    Bm = B.t().contiguous() if b_mn else B
    D = torch.zeros(M, N, device=dev())
    nat.gemm(Am, Bm, D, a_mn=a_mn, b_mn=b_mn)
    ref = A.double() @ B.double().t()
    e = rel_err(D, ref)
    # default precision is 3xTF32 (hi/lo split, three wgmma per K step, accumulator added into fp32 registers every 4 K blocks):
    # fp32-SGEMM accuracy, measured against the fp64 product
    assert e < 2e-6, "3xTF32 gemm rel err %g (a_mn=%s b_mn=%s %dx%dx%d)" % (e, a_mn, b_mn, M, N, K)
    nat.set_gemm_precision("tf32")
    try:
        D.zero_(); nat.gemm(Am, Bm, D, a_mn=a_mn, b_mn=b_mn)
        e1 = rel_err(D, ref)
    finally:
        nat.set_gemm_precision("3xtf32")
    assert 1e-5 < e1 < 2e-3, "plain tf32 mode rel err %g" % e1     # the fast mode really is the 10-bit-mantissa product


def test_gemm_epilogues(nat):
    torch.manual_seed(1)
    M, N, K = 64, 96, 128
    A = torch.randn(M, K, device=dev()); B = torch.randn(N, K, device=dev()); bias = torch.randn(N, device=dev())
    mask = torch.randn(M, N, device=dev())
    ref = torch.relu(A @ B.t() + bias)
    D = torch.empty(M, N, device=dev()); nat.gemm(A, B, D, bias=bias, relu=True)
    assert rel_err(D, ref) < 2e-6
    cs = torch.zeros(N, device=dev()); D2 = torch.empty(M, N, device=dev())
    nat.gemm(A, B, D2, mask=mask, colsum=cs)
    ref2 = (A @ B.t()) * (mask > 0)
    assert rel_err(D2, ref2) < 2e-6 and rel_err(cs, ref2.sum(0)) < 2e-6
    # NCHW scatter: rows = (image, pixel), cols = channel
    n_img, hw, C = 4, 16, 24
    A3 = torch.randn(n_img * hw, K, device=dev()); B3 = torch.randn(C, K, device=dev())
    Y = torch.empty(n_img, C, 4, 4, device=dev()); nat.gemm(A3, B3, Y, store_nchw_hw=hw)
    ref3 = (A3 @ B3.t()).reshape(n_img, hw, C).permute(0, 2, 1).reshape(n_img, C, 4, 4)
    assert rel_err(Y, ref3) < 2e-6
    # split-K accumulate
    A4 = torch.randn(32, 2048, device=dev()); B4 = torch.randn(400, 2048, device=dev())
    D4 = torch.zeros(32, 400, device=dev()); nat.gemm(A4, B4, D4, split_k=16, accumulate=True)
    assert rel_err(D4, A4 @ B4.t()) < 2e-6
    # unaligned leading dimension -> CUDA-core fallback with the same contract
    A5 = torch.randn(50, 25, device=dev()); B5 = torch.randn(16, 25, device=dev()); D5 = torch.empty(50, 16, device=dev())
    nat.gemm(A5, B5, D5)
    assert rel_err(D5, A5 @ B5.t()) < 1e-5


# ---------------------------------------------------------------------------------------------------------------- ops through autograd
def _grads(fn, *inputs):
    ins = [i.clone().requires_grad_(True) for i in inputs]
    out = fn(*ins)
    g = torch.randn_like(out)
    out.backward(g)
    return out.detach(), [i.grad for i in ins], g


def test_dense_fn(nat):
    from geomx_b200.ops import functional as OF
    torch.manual_seed(2)
    x = torch.randn(32, 512, device=dev()); w = torch.randn(256, 512, device=dev()) * 0.05; b = torch.randn(256, device=dev())
    for act in (None, "relu"):
        torch.manual_seed(3)
        y, gr, g = _grads(lambda a, c, d: OF.dense(a, c, d, act), x, w, b)
        OF.use_native(False)
        torch.manual_seed(3)
        y2, gr2, _ = _grads(lambda a, c, d: OF.dense(a, c, d, act), x, w, b)
        OF.use_native(True)
        assert rel_err(y, y2) < 2e-6
        for a, c in zip(gr, gr2):
            assert rel_err(a, c) < 1e-5


@pytest.mark.parametrize("cin,cout,k,hw,stride,pad", [(16, 32, 5, 12, 1, 0), (1, 16, 5, 28, 1, 0), (8, 16, 3, 10, 2, 1)])
def test_conv_fn(nat, cin, cout, k, hw, stride, pad):
    from geomx_b200.ops import functional as OF
    torch.manual_seed(4)
    x = torch.randn(8, cin, hw, hw, device=dev()); w = torch.randn(cout, cin, k, k, device=dev()) * 0.1; b = torch.randn(cout, device=dev())
    f = lambda a, c, d: OF.conv2d(a, c, d, (stride, stride), (pad, pad), act="relu")
    torch.manual_seed(5); y, gr, g = _grads(f, x, w, b)
    # reference: the PyTorch definition in fp64 with the same output gradient (cuDNN's fp32 weight-gradient algorithms are only good to
    # ~1e-3 relative for some of these shapes)
    ins = [t.double().requires_grad_(True) for t in (x, w, b)]
    y2 = f(*ins); y2.backward(g.double()); gr2 = [t.grad for t in ins]
    assert rel_err(y, y2) < 2e-6
    for a, c in zip(gr, gr2):
        assert rel_err(a, c) < 1e-4      # fp32-accurate products; a ReLU mask can still flip on an activation that is zero to rounding


@pytest.mark.parametrize("C,hw,k,stride,pad", [(8, 14, 3, 1, 1), (6, 9, 3, 2, 1), (4, 12, 5, 1, 0)])
def test_depthwise_conv_fn(nat, C, hw, k, stride, pad):
    """groups == channels convolution (csrc/kernels/depthwise_conv.cu) forward + all three gradients vs torch."""
    from geomx_b200.ops import functional as OF
    torch.manual_seed(8)
    x = torch.randn(5, C, hw, hw, device=dev()); w = torch.randn(C, 1, k, k, device=dev()) * 0.3; b = torch.randn(C, device=dev())
    f = lambda a, c, d: OF.conv2d(a, c, d, (stride, stride), (pad, pad), groups=C, act="relu")
    torch.manual_seed(9); y, gr, _ = _grads(f, x, w, b)
    OF.use_native(False)
    torch.manual_seed(9); y2, gr2, _ = _grads(f, x, w, b)
    OF.use_native(True)
    assert rel_err(y, y2) < 1e-5
    for a, c in zip(gr, gr2):
        assert rel_err(a, c) < 1e-4


def test_hybridize_static_alloc_is_graph_capture(nat):
    """hybridize(static_alloc=True) = CachedOp: forward and backward of the block replay as CUDA graphs; training matches eager execution."""
    import time
    import numpy as np

    def build(seed, static):
        mx.random.seed(seed); torch.manual_seed(seed)
        net = mx.gluon.nn.HybridSequential()
        net.add(mx.gluon.nn.Conv2D(8, 3, activation="relu"), mx.gluon.nn.MaxPool2D(2, 2), mx.gluon.nn.Dense(32, activation="relu"), mx.gluon.nn.Dense(10))
        net.initialize(mx.init.Xavier(), ctx=mx.gpu(0))
        net(mx.nd.zeros((16, 1, 12, 12), ctx=mx.gpu(0)))
        if static:
            net.hybridize(static_alloc=True, static_shape=True)
        return net

    rng = np.random.RandomState(0)
    X = mx.nd.array(rng.rand(16, 1, 12, 12).astype(np.float32), ctx=mx.gpu(0)); y = mx.nd.array(rng.randint(0, 10, (16,)).astype(np.float32), ctx=mx.gpu(0))
    losses, times = {}, {}
    for static in (False, True):
        net = build(5, static)
        loss_fn = mx.gluon.loss.SoftmaxCrossEntropyLoss()
        tr = mx.gluon.Trainer(net.collect_params(), "sgd", {"learning_rate": 0.1}, kvstore=None)
        ls = []
        for it in range(25):
            if it == 5:
                torch.cuda.synchronize(); t0 = time.perf_counter()
            with mx.autograd.record():
                l = loss_fn(net(X), y)
            l.backward()
            tr.step(16)
            ls.append(float(l.mean().asscalar()))
        torch.cuda.synchronize(); times[static] = (time.perf_counter() - t0) / 20
        losses[static] = ls
        if static:
            assert any(op.ok for op in net._cached_ops.values()), "the block was not captured"
    print("hybridize(static_alloc): eager %.3f ms/step, graphed %.3f ms/step" % (times[False] * 1e3, times[True] * 1e3))
    assert losses[True][-1] < losses[True][0]
    assert np.allclose(losses[False], losses[True], rtol=2e-3, atol=2e-4), (losses[False][-3:], losses[True][-3:])


def test_pool_relu_softmax_bn(nat):
    from geomx_b200.ops import functional as OF
    torch.manual_seed(6)
    x = torch.randn(4, 8, 12, 12, device=dev())
    for f in (lambda a: OF.max_pool2d(a, (2, 2), (2, 2)), lambda a: OF.activation(a, "relu")):
        torch.manual_seed(7); y, gr, _ = _grads(f, x)
        OF.use_native(False); torch.manual_seed(7); y2, gr2, _ = _grads(f, x); OF.use_native(True)
        assert torch.allclose(y, y2) and torch.allclose(gr[0], gr2[0])
    logits = torch.randn(32, 10, device=dev()); lab = torch.randint(0, 10, (32,), device=dev()).float()
    torch.manual_seed(8); y, gr, _ = _grads(lambda a: OF.softmax_cross_entropy(a, lab), logits)
    OF.use_native(False); torch.manual_seed(8); y2, gr2, _ = _grads(lambda a: OF.softmax_cross_entropy(a, lab), logits); OF.use_native(True)
    assert rel_err(y, y2) < 1e-5 and rel_err(gr[0], gr2[0]) < 1e-5
    gamma = torch.rand(8, device=dev()) + 0.5; beta = torch.randn(8, device=dev())
    rm, rv = torch.zeros(8, device=dev()), torch.ones(8, device=dev())
    rm2, rv2 = rm.clone(), rv.clone()
    torch.manual_seed(9); y, gr, _ = _grads(lambda a, c, d: OF.batch_norm(a, c, d, rm, rv, True), x, gamma, beta)
    OF.use_native(False); torch.manual_seed(9); y2, gr2, _ = _grads(lambda a, c, d: OF.batch_norm(a, c, d, rm2, rv2, True), x, gamma, beta); OF.use_native(True)
    assert rel_err(y, y2) < 1e-4 and rel_err(rm, rm2) < 1e-4
    for a, c in zip(gr, gr2):
        assert rel_err(a, c) < 1e-3


def test_batchnorm_split_form_matches_fp64(nat):
    """Feature-map sized BatchNorm (statistics kernel on a (channel, slice) grid + streaming apply kernel) against an fp64 reference:
    forward, running statistics (population variance), input / scale / shift gradients, inference mode; vector and scalar tails."""
    from geomx_b200.ops import functional as OF
    torch.manual_seed(31)
    for shape in ((16, 24, 28, 28), (9, 5, 23, 23)):
        x = (torch.randn(*shape, device=dev()) * 1.7 + 0.6).requires_grad_(True)
        C = shape[1]
        gamma = (torch.rand(C, device=dev()) + 0.5).requires_grad_(True); beta = torch.randn(C, device=dev()).requires_grad_(True)
        rm, rv = torch.zeros(C, device=dev()), torch.ones(C, device=dev())
        wgt = torch.randn(*shape, device=dev())
        for rep in range(2):                      # twice: the accumulators must re-arm themselves
            for t in (x, gamma, beta):
                t.grad = None
            y = OF.batch_norm(x, gamma, beta, rm, rv, True, momentum=0.9, eps=1e-5)
            (y * wgt).sum().backward()
        xd = x.detach().double().requires_grad_(True); gd = gamma.detach().double().requires_grad_(True); bd = beta.detach().double().requires_grad_(True)
        mean = xd.mean((0, 2, 3), keepdim=True); var = ((xd - mean) ** 2).mean((0, 2, 3), keepdim=True)
        yd = (xd - mean) / torch.sqrt(var + 1e-5) * gd.view(1, C, 1, 1) + bd.view(1, C, 1, 1)
        (yd * wgt.double()).sum().backward()
        assert rel_err(y, yd) < 1e-5
        assert rel_err(x.grad, xd.grad) < 1e-4 and rel_err(gamma.grad, gd.grad) < 1e-5 and rel_err(beta.grad, bd.grad) < 1e-5
        m1, v1 = mean.flatten().float(), var.flatten().float()
        assert torch.allclose(rm, 0.19 * m1, atol=1e-5) and torch.allclose(rv, 0.81 + 0.19 * v1, atol=1e-4)     # two updates with momentum 0.9
        ye = OF.batch_norm(x.detach(), gamma.detach(), beta.detach(), rm, rv, False, eps=1e-5)
        ref = (x.detach() - rm.view(1, C, 1, 1)) / torch.sqrt(rv.view(1, C, 1, 1) + 1e-5) * gamma.detach().view(1, C, 1, 1) + beta.detach().view(1, C, 1, 1)
        assert rel_err(ye, ref) < 1e-5


# ---------------------------------------------------------------------------------------------------------------- optimizers
def test_adam_kernel_matches_python(nat):
    torch.manual_seed(10)
    w = torch.randn(5000, device=dev()); g = torch.randn(5000, device=dev())
    o = mx.optimizer.Adam(learning_rate=0.01, wd=0.001)
    upd = mx.optimizer.get_updater(o)
    wn = mx.nd.array(w.clone()); wn._data = w.clone()
    ref = w.clone().cpu(); m = torch.zeros(5000); v = torch.zeros(5000)
    for t in range(1, 4):
        upd(0, mx.nd.NDArray(g), wn)      # native CUDA path inside Adam.update
        gg = g.cpu() + 0.001 * ref
        m = 0.9 * m + 0.1 * gg; v = 0.999 * v + 0.001 * gg * gg
        lr = 0.01 * math.sqrt(1 - 0.999 ** t) / (1 - 0.9 ** t)
        ref = ref - lr * m / (v.sqrt() + 1e-8)
    assert rel_err(wn._t.cpu(), ref) < 1e-5


def test_trainer_multi_tensor(nat):
    import numpy as np
    torch.manual_seed(11); np.random.seed(11)
    net = mx.models.build_cnn(); net.initialize(init=mx.init.Xavier(), ctx=mx.gpu(0))
    x = mx.nd.array(torch.rand(32, 1, 28, 28), ctx=mx.gpu(0)); y = mx.nd.array(torch.randint(0, 10, (32,)).float(), ctx=mx.gpu(0))
    loss = mx.gluon.loss.SoftmaxCrossEntropyLoss()
    tr = mx.gluon.Trainer(net.collect_params(), "adam", {"learning_rate": 0.01}, kvstore=None)
    vals = []
    for _ in range(40):
        with mx.autograd.record():
            l = loss(net(x), y)
        l.backward(); tr.step(32)
        vals.append(float(l.mean().asscalar()))
    assert vals[-1] < vals[0] * 0.7, vals      # memorising 32 random labels: the loss must fall clearly (the pace depends on the init draw)


# ---------------------------------------------------------------------------------------------------------------- flagship step
def test_fused_step_matches_torch(nat, engine):
    """The fused step's gradients against torch's fp64 autograd of the demo CNN (``step_reference``), then one Adam step."""
    torch.manual_seed(15)
    eng = engine(32, mx.optimizer.Adam(learning_rate=0.01), use_graph=False, fused_zero_grad=False)
    X = torch.rand(32, 1, 28, 28, device=dev()); y = torch.randint(0, 10, (32,), device=dev()).float()
    P0 = [p.clone() for p in eng.P]
    eng.x.copy_(X); eng.label.copy_(y)
    # run everything except the optimizer: call _body with lr = 0 so weights stay put, then inspect the gradient arena
    eng.fabric.set_optimizer(dict(mx.optimizer.SGD(learning_rate=0.0).spec()))
    eng._body(); torch.cuda.synchronize()
    loss_ref, _, grads_ref, _ = step_reference(P0, X, y, eng.idx1, eng.idx2)
    assert rel_err(eng.loss, loss_ref) < 1e-5
    errs = [rel_err(g, gr) for g, gr in zip(eng.G, grads_ref)]
    print("fused-step gradient rel errors vs fp64:", ["%.2e" % e for e in errs])
    # fp32-accurate everywhere (3xTF32 tensor-core products, fp32 FMA elsewhere)
    assert max(errs) < 1e-4, errs
    # now one real Adam step on the same batch: w' = w - lr*m̂/(sqrt(v̂)+eps) with g/num_samples pushed; the expectation uses the gradient arena
    # produced by the first pass (identical inputs), so it checks scale + optimizer + broadcast exactly
    G_own = [g.clone() for g in eng.G]
    eng.fabric.set_optimizer(mx.optimizer.Adam(learning_rate=0.01).spec())
    eng.fabric.set_opt_step(0)          # optimizer step counter t restarts for the Adam run
    eng._body(); torch.cuda.synchronize()
    for i, (p, p0, g) in enumerate(zip(eng.P, P0, G_own)):
        gsc = g / 32.0
        expect = p0 - 0.01 * gsc / (gsc.abs() + 1e-8 / math.sqrt(0.001))      # first Adam step: m̂/(sqrt(v̂)+eps) = g/(|g| + eps/sqrt(1-b2))
        assert torch.allclose(p, expect, atol=2e-5), "param %d: %g" % (i, float((p - expect).abs().max()))


def test_fused_step_graph_trains(nat):
    from geomx_b200.parallel import Topology
    torch.manual_seed(16)
    eng = mx.models.HipsCNNTrainStep(batch_size=32, topo=Topology(1, 0, 1, 1), use_graph=True)
    X = torch.rand(32, 1, 28, 28).pin_memory(); y = torch.randint(0, 10, (32,)).float().pin_memory()
    l0 = eng.step(X, y)
    for _ in range(40):
        l = eng.step(X, y)
    assert l < 0.5 * l0, (l0, l)


def test_host_pipeline_direct_inputs_match_staged(nat, monkeypatch):
    """step(X_pinned, y_pinned): alternating between two graphs captured on the two H2D target buffers gives the same training as the
    single graph fed through a staging copy.  (Small learning rate: conv0's weight gradient is accumulated with atomics, so two runs differ
    in the last bits, and a large step size amplifies that chaotically within a few iterations.)"""
    from geomx_b200.parallel import Topology
    g = torch.Generator().manual_seed(5)
    Xs = [torch.rand(32, 1, 28, 28, generator=g).pin_memory() for _ in range(7)]
    ys = [torch.randint(0, 10, (32,), generator=g).float().pin_memory() for _ in range(7)]
    out = {}
    for direct in ("1", "0"):
        monkeypatch.setenv("GEOMX_E2E_DIRECT_INPUT", direct)
        torch.manual_seed(23)
        eng = mx.models.HipsCNNTrainStep(batch_size=32, optimizer=mx.optimizer.SGD(learning_rate=0.002), topo=Topology(1, 0, 1, 1), use_graph=True)
        out[direct] = ([eng.step(X, y) for X, y in zip(Xs, ys)], eng.fabric.param.tensor.clone())
        assert (eng._graph_alt is not None) == (direct == "1")
    assert all(abs(a - b) < 1e-4 * max(1.0, abs(a)) for a, b in zip(out["1"][0], out["0"][0])), (out["1"][0], out["0"][0])
    assert torch.allclose(out["1"][1], out["0"][1], atol=1e-4)      # a batch read from the wrong buffer would show up at the 1e-2 level


@pytest.mark.parametrize("use_graph", [True, False])
def test_lookahead_step_is_the_same_training(nat, use_graph):
    """The look-ahead cut of the step (head of batch k .. forward convolutions of batch k+1 in one launch) is the same arithmetic in the same
    order as the classic cut: identical loss sequence (reported one call late) and identical weights after flush()."""
    from geomx_b200.parallel import Topology
    g = torch.Generator().manual_seed(21)
    Xs = [torch.rand(32, 1, 28, 28, generator=g).pin_memory() for _ in range(6)]
    ys = [torch.randint(0, 10, (32,), generator=g).float().pin_memory() for _ in range(6)]
    runs = {}
    for look in (False, True):
        torch.manual_seed(17)
        eng = mx.models.HipsCNNTrainStep(batch_size=32, optimizer=mx.optimizer.SGD(learning_rate=0.05), topo=Topology(1, 0, 1, 1),
                                         use_graph=use_graph, lookahead=look)
        losses = [eng.step(X, y) for X, y in zip(Xs, ys)]
        if look:
            assert math.isnan(losses[0])
            losses = losses[1:] + [eng.flush()]
            assert eng.flush() is None
        torch.cuda.synchronize()
        runs[look] = (losses, eng.fabric.param.tensor.clone())
    la, lb = runs[False][0], runs[True][0]
    assert all(abs(a - b) < 1e-5 * max(1.0, abs(a)) for a, b in zip(la, lb)), (la, lb)
    assert torch.allclose(runs[False][1], runs[True][1], atol=1e-5), float((runs[False][1] - runs[True][1]).abs().max())


def test_direct_conv_kernels_exact(nat):
    """The CUDA-core (fp32 FMA) kernels must match torch to fp32 rounding: fused conv+ReLU+pool fwd, its wgrad, im2col/col2im."""
    import torch.nn.functional as F
    torch.manual_seed(17)
    N, Cin, H, W, Co, K = 8, 1, 28, 28, 16, 5
    x = torch.randn(N, Cin, H, W, device=dev()); w = (torch.randn(Co, Cin, K, K, device=dev()) * 0.2).requires_grad_(True)
    b = torch.randn(Co, device=dev()).requires_grad_(True)
    z = F.conv2d(x, w, b)
    ref = F.max_pool2d(torch.relu(z), 2)
    y = torch.empty_like(ref); idx = torch.empty(ref.shape, dtype=torch.uint8, device=dev())
    nat.conv_relu_pool_fwd(x, w.detach(), b.detach(), y, idx)
    assert torch.allclose(y, ref, atol=1e-4)
    g = torch.randn_like(ref)
    # reference gradient in fp64, routed through the pooling / ReLU of the fp32 forward (cuDNN's fp32 weight-gradient algorithms are only
    # good to ~1e-3 relative for this shape on some GPUs)
    dz, = torch.autograd.grad(ref, z, g)
    ref_dw = torch.nn.grad.conv2d_weight(x.double(), w.shape, dz.double()); ref_db = dz.double().sum((0, 2, 3))
    dw = torch.zeros_like(w); db = torch.zeros_like(b)
    nat.conv_relu_pool_wgrad(x, g, y, idx, dw, db, tuple(w.shape))
    assert rel_err(dw, ref_dw) < 1e-4 and rel_err(db, ref_db) < 1e-4
    # im2col / col2im are adjoint: <im2col(x), c> == <x, col2im(c)>
    x2 = torch.randn(4, 16, 12, 12, device=dev())
    col = nat.im2col(x2, 5, 5)
    ref_col = F.unfold(x2, 5).transpose(1, 2).reshape(-1, 400)
    assert torch.allclose(col[:, :400], ref_col)
    c = torch.randn_like(col)
    back = nat.col2im(c, tuple(x2.shape), 5, 5)
    ref_back = F.fold(c[:, :400].reshape(4, 64, 400).transpose(1, 2), (12, 12), 5)
    assert torch.allclose(back, ref_back, atol=1e-4)


@pytest.mark.gpu
def test_unique_gather_scatter_rows():
    """Row-sparse support kernels (sparse_ops.cu: CUB sort+unique, row gather / scatter-add) against torch."""
    from geomx_b200.ops import _native_api as n
    torch.manual_seed(0)
    ids = torch.randint(0, 500, (4000,), device="cuda", dtype=torch.int64)
    u = n.unique_i64(ids)
    assert torch.equal(u, torch.unique(ids, sorted=True))
    src = torch.randn(500, 24, device="cuda")
    g = n.gather_rows(src, u)
    assert torch.equal(g, src[u])
    src3 = torch.randn(500, 5, device="cuda")                 # row length not a multiple of 4: scalar path
    assert torch.equal(n.gather_rows(src3, u), src3[u])
    dst = torch.zeros(500, 24, device="cuda")
    rows = torch.randn(ids.numel(), 24, device="cuda")
    n.scatter_rows(dst, ids, rows, add=True)
    ref = torch.zeros(500, 24, device="cuda").index_add_(0, ids, rows)
    assert torch.allclose(dst, ref, atol=1e-4)
    # through the public API: dense -> row_sparse -> kv.row_sparse_pull on the GPU
    import geomx_b200 as mx
    w = mx.nd.array(src.cpu().numpy(), ctx=mx.gpu(0))
    kv = mx.kv.create("device")
    kv.init(7, w)
    out = mx.nd.sparse.zeros("row_sparse", (500, 24), ctx=mx.gpu(0))
    kv.row_sparse_pull(7, out=out, row_ids=mx.nd.array(ids.cpu().numpy(), ctx=mx.gpu(0), dtype="int64"))
    assert torch.equal(out.indices._t, u) and torch.equal(out.data._t, src[u])


@pytest.mark.gpu
def test_gemm_with_fused_maxpool_epilogue():
    """gx_gemm_tf32_pool: conv-as-GEMM + bias + ReLU + 2x2 max-pool in the wgmma GEMM's epilogue == GEMM (NCHW store) followed by the pool kernel,
    values and arg-max positions (ties resolved to the first maximum), and close to the fp32 PyTorch reference."""
    from geomx_b200.ops import _native_api as n
    torch.manual_seed(3)
    for (B, C, OH, OW, K) in ((32, 32, 8, 8, 400), (4, 16, 4, 16, 72), (2, 48, 16, 8, 36)):
        A = torch.randn(B * OH * OW, K, device="cuda")
        Wt = torch.randn(C, K, device="cuda") * 0.1
        bias = torch.randn(C, device="cuda")
        z = torch.empty(B, C, OH, OW, device="cuda")
        n.gemm(A, Wt, z, bias=bias, relu=True, store_nchw_hw=OH * OW)
        a_ref = torch.empty(B, C, OH // 2, OW // 2, device="cuda"); i_ref = torch.empty(B, C, OH // 2, OW // 2, dtype=torch.uint8, device="cuda")
        n.maxpool2x2_fwd(z, a_ref, i_ref)
        a = torch.full_like(a_ref, -7.0); idx = torch.full_like(i_ref, 9)
        assert n.gemm_pool(A, Wt, a, idx, OH, OW, bias=bias, relu=True)
        torch.cuda.synchronize()
        assert torch.equal(a, a_ref) and torch.equal(idx, i_ref), (B, C, OH, OW)
        ref = torch.nn.functional.max_pool2d(torch.relu((A @ Wt.t() + bias).view(B, OH, OW, C).permute(0, 3, 1, 2)), 2)
        assert rel_err(a, ref) < 2e-3
    # geometry the in-warp pooling cannot express -> clean refusal (the caller falls back)
    A = torch.randn(2 * 6 * 6, 16, device="cuda"); Wt = torch.randn(16, 16, device="cuda")
    assert not n.gemm_pool(A, Wt, torch.empty(2, 16, 3, 3, device="cuda"), torch.empty(2, 16, 3, 3, dtype=torch.uint8, device="cuda"), 6, 6)


@pytest.mark.gpu
def test_rtc_launch():
    """mx.rtc end to end: NVRTC cubin -> driver module -> launch on the current stream."""
    import geomx_b200 as mx
    mod = mx.rtc.CudaModule('extern "C" __global__ void axpy(const float* x, float* y, float a, int n) { int i = blockIdx.x * blockDim.x + threadIdx.x; if (i < n) y[i] += a * x[i]; }')
    k = mod.get_kernel("axpy", "const float *x, float *y, float a, int n")
    x = mx.nd.array(torch.arange(1000, dtype=torch.float32), ctx=mx.gpu(0)); y = mx.nd.ones((1000,), ctx=mx.gpu(0))
    k.launch([x, y, 2.0, 1000], mx.gpu(0), (4, 1, 1), (256, 1, 1))
    torch.cuda.synchronize()
    assert torch.equal(y._t.cpu(), 1 + 2 * torch.arange(1000, dtype=torch.float32))
