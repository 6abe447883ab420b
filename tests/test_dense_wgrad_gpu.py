"""The dense chain's weight gradients are a launch of their own (dense_wgrad_kernel in csrc/kernels/mlp_chain.cu), on a parallel branch of
the step after the cluster kernel that computes the data path.  These tests check the kernel alone against fp64 with every output pre-filled
with NaN, and that in a graph-captured step the dense keys' exchange applies the gradients this kernel writes: it runs on another stream
than the cluster kernel, so an exchange ordered only behind the cluster kernel would read gradients that do not exist yet."""
import pytest
import torch

import geomx_b200 as mx
from _cnn_ref import D0, D1, D2, engine, nan, nat, rel_err  # noqa: F401  (nat, engine: fixtures)

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("B", [1, 7, 31, 32])
def test_dense_wgrad_matches_fp64(nat, B):
    C = 10
    g = torch.Generator().manual_seed(300 + B)
    r = lambda *s: torch.randn(*s, generator=g).cuda()
    x, a3, a4 = r(B, D0).relu(), r(B, D1).relu(), r(B, D2).relu()
    dz3, dz4 = r(B, D1) * (a3 > 0), r(B, D2) * (a4 > 0)
    dl = torch.zeros(B, 16, device="cuda")
    dl[:, :C] = r(B, C)
    outs = [nan(D1, D0), nan(D1), nan(D2, D1), nan(D2), nan(C, D2), nan(C)]
    nat.dense_wgrad(x, a3, a4, dz4, dz3, dl, *outs)
    torch.cuda.synchronize()
    d = lambda t: t.double()
    ref = [d(dz3).T @ d(x), d(dz3).sum(0), d(dz4).T @ d(a3), d(dz4).sum(0), d(dl[:, :C]).T @ d(a4), d(dl[:, :C]).sum(0)]
    for name, got, want in zip(("dw0", "db0", "dw1", "db1", "dw2", "db2"), outs, ref):
        assert not torch.isnan(got).any(), (B, name, "element never written")
        assert rel_err(got, want) < 1e-6, (B, name, rel_err(got, want))


@pytest.mark.parametrize("B", [32, 20])
def test_graph_step_applies_the_dense_weight_gradients(nat, engine, B):
    """One rank, SGD at lr = 1 without momentum or weight decay: the dense parameters after one replay of the captured step must be exactly
    those an eager step gives from the same parameters and batch, and must have moved by the gradients that eager step left in the arena."""
    g = torch.Generator().manual_seed(400 + B)
    X, y = torch.rand(B, 1, 28, 28, generator=g).cuda(), torch.randint(0, 10, (B,), generator=g).float().cuda()
    eng = engine(B, mx.optimizer.SGD(learning_rate=1.0, momentum=0.0, wd=0.0), use_graph=True, fused_zero_grad=False)
    names = [n for n, _, _ in eng._steps()]
    assert eng.fused_mlp and eng.overlap and any(n.startswith("dense weight gradients") for n in names), names
    P0 = [p.clone() for p in eng.P]

    def start():
        for p, v in zip(eng.P, P0):
            p.copy_(v)
        eng.fabric.load_master_from_param()
        eng.x.copy_(X); eng.label.copy_(y)
        torch.cuda.synchronize()

    start()
    eng._body(); torch.cuda.synchronize()
    grads = [t.clone() for t in eng.G]
    eager = [p.clone() for p in eng.P]
    eng.capture()
    start()
    eng.graph.replay(); torch.cuda.synchronize()
    for i in range(4, 10):
        assert torch.equal(eng.P[i], eager[i]), "dense parameter %d differs between the captured and the eager step" % i
        moved = P0[i] - eng.P[i]
        assert rel_err(moved, grads[i] / B) < 1e-4, (i, rel_err(moved, grads[i] / B))   # (rounding of P0 - update)
