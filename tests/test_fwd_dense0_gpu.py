"""At even batches <= 32 the first dense layer runs in the forward convolution kernel (cnn_fwd_dense0_kernel, csrc/kernels/cnn_direct.cu:
clusters of two images whose 8 CTAs exchange a2 and compute a3) and the dense-chain cluster kernel starts from a3 (dense_tail_kernel,
csrc/kernels/mlp_chain.cu).  These tests check both kernels alone, with every output pre-filled with NaN (a slice never written, or read
before it landed, shows up): the convolutions against cnn_fwd bit for bit, a3 and the tail's outputs against fp64, the batch sizes the forward
kernel refuses, launch-to-launch determinism at both cluster sizes, and that the captured step runs the new pair."""
import gc
import os
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as F

import geomx_b200 as mx
from geomx_b200.models.cnn import STEP_SWITCHES

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
D0, D1, D2 = 512, 256, 128
SWITCHES = STEP_SWITCHES + ("GEOMX_MLP_CLUSTER",)


@pytest.fixture(scope="module")
def nat():
    from geomx_b200.ops import native
    native.require()
    return native


def rel_err(a, b):
    return float((a.double() - b.double()).norm() / (b.double().norm() + 1e-30))


def nan(*s, dtype=torch.float32):
    if dtype == torch.uint8:
        return torch.full(s, 255, dtype=dtype, device="cuda")
    return torch.full(s, float("nan"), dtype=dtype, device="cuda")


# ---------------------------------------------------------------------------------------------------------------- forward kernel
def _fwd_inputs(B, seed, bd_value=None):
    g = torch.Generator().manual_seed(seed)
    r = lambda *s, scale=1.0: (torch.randn(*s, generator=g) * scale).cuda()
    x = torch.rand(B, 1, 28, 28, generator=g).cuda()
    w = [r(16, 1, 5, 5, scale=0.3), r(16, scale=0.1), r(32, 16, 5, 5, scale=0.08), r(32, scale=0.1)]
    wd, bd = r(D1, D0, scale=0.05), r(D1, scale=0.1)
    if bd_value is not None:
        bd.fill_(bd_value)
    return x, w, wd, bd


def _fwd_outputs(B):
    return [nan(B, 16, 12, 12), nan(B, 16, 12, 12, dtype=torch.uint8), nan(B, 32, 4, 4), nan(B, 32, 4, 4, dtype=torch.uint8)]


@pytest.mark.parametrize("B", [2, 20, 32])
def test_fwd_dense0_matches_cnn_fwd_and_fp64(nat, B):
    x, w, wd, bd = _fwd_inputs(B, 500 + B)
    ref = _fwd_outputs(B)
    nat.cnn_fwd(x, *w, *ref)
    got = _fwd_outputs(B)
    a3 = nan(B, D1)
    assert nat.cnn_fwd_dense0(x, *w, wd, bd, *got, a3)
    torch.cuda.synchronize()
    for name, a, b in zip(("a1", "idx1", "a2", "idx2"), got, ref):
        assert torch.equal(a, b), (B, name, "differs from cnn_fwd")
    assert not torch.isnan(a3).any(), (B, "a3 element never written")
    want = torch.relu(got[2].double().view(B, D0) @ wd.double().T + bd.double())
    err = rel_err(a3, want)
    assert err < 1e-6, (B, err)
    # launch to launch: the same bits (fixed shuffle order of the 8 partial sums)
    again = nan(B, D1)
    assert nat.cnn_fwd_dense0(x, *w, wd, bd, *_fwd_outputs(B), again)
    torch.cuda.synchronize()
    assert torch.equal(a3, again), B


def test_fwd_dense0_relu_zeroes_negative_rows(nat):
    B = 20
    x, w, wd, bd = _fwd_inputs(B, 77, bd_value=-5.0)
    wd.mul_(0.01)                                           # |a2 . w| stays far below 5
    a3 = nan(B, D1)
    assert nat.cnn_fwd_dense0(x, *w, wd, bd, *_fwd_outputs(B), a3)
    torch.cuda.synchronize()
    assert torch.equal(a3, torch.zeros_like(a3))


@pytest.mark.parametrize("B", [1, 3, 31, 34, 64])
def test_fwd_dense0_refuses_odd_or_large_batches(nat, B):
    x, w, wd, bd = _fwd_inputs(B, 5)
    outs = _fwd_outputs(B)
    a3 = nan(B, D1)
    before = nat.launch_count
    assert nat.cnn_fwd_dense0(x, *w, wd, bd, *outs, a3) is False
    torch.cuda.synchronize()
    assert nat.launch_count == before and torch.isnan(a3).all() and torch.isnan(outs[0]).all()


# ---------------------------------------------------------------------------------------------------------------- the tail from a3
def _tail_inputs(B, C, seed):
    g = torch.Generator().manual_seed(seed)
    r = lambda *s, scale=1.0: (torch.randn(*s, generator=g) * scale).cuda()
    a3 = r(B, D1).relu()                                  # a3 is a ReLU output: non-negative with many zeros
    w = [r(D1, D0, scale=0.05), r(D2, D1, scale=0.08), r(D2, scale=0.1), r(C, D2, scale=0.1), r(C, scale=0.1)]   # w0, w1, b1, w2, b2
    y = torch.randint(0, C, (B,), generator=g).cuda()
    return a3, w, y


def _tail_reference(a3, w, y):
    w0, w1, b1, w2, b2 = [t.double() for t in w]
    a = a3.double().requires_grad_(True)
    z4 = F.linear(a, w1, b1); z4.retain_grad()
    h = torch.relu(z4)
    lg = F.linear(h, w2, b2); lg.retain_grad()
    loss = F.cross_entropy(lg, y, reduction="none")
    loss.sum().backward()
    dz3 = a.grad * (a3.double() > 0)
    return {"loss": loss.detach(), "logits": lg.detach(), "dx": dz3 @ w0, "a4": h.detach(), "dz4": z4.grad, "dz3": dz3, "dl": lg.grad}


def _tail_run(nat, a3, w, y):
    B, C = a3.shape[0], w[3].shape[0]
    out = {"loss": nan(B), "logits": nan(B, C), "dx": nan(B, D0), "a4": nan(B, D2), "dz4": nan(B, D2), "dz3": nan(B, D1), "dl": nan(B, 16)}
    assert nat.dense_tail(a3, *w, y.float(), out["loss"], out["logits"], out["dx"], out["a4"], out["dz4"], out["dz3"], out["dl"])
    torch.cuda.synchronize()
    return out


def check_tail_against_fp64(nat, B, C, seed):
    a3, w, y = _tail_inputs(B, C, seed)
    got = _tail_run(nat, a3, w, y)
    assert torch.equal(got["dl"][:, C:], torch.zeros_like(got["dl"][:, C:])), (B, C, "dlogits beyond the classes")
    got["dl"] = got["dl"][:, :C]
    for name, ref in _tail_reference(a3, w, y).items():
        g = got[name]
        assert not torch.isnan(g).any(), (B, C, name, "element never written")
        err = rel_err(g, ref)
        assert err < 1e-5, (B, C, name, err)


def check_tail_repeatable(nat, B, C, seed, launches=3):
    a3, w, y = _tail_inputs(B, C, seed)
    first = _tail_run(nat, a3, w, y)
    for _ in range(launches - 1):
        for name, t in _tail_run(nat, a3, w, y).items():
            assert torch.equal(first[name], t), (B, C, name, "differs between launches on the same inputs")


@pytest.mark.parametrize("B", [1, 20, 32])
@pytest.mark.parametrize("C", [10, 16])
def test_dense_tail_matches_fp64(nat, B, C):
    check_tail_against_fp64(nat, B, C, seed=600 + B + C)


def test_dense_tail_three_launches_bit_identical(nat):
    check_tail_repeatable(nat, 32, 10, seed=11)


_CLUSTER8 = """
import sys
sys.path.insert(0, {root!r}); sys.path.insert(0, {tests!r})
import torch
from geomx_b200.ops import native
import test_fwd_dense0_gpu as t
native.require()
with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
    for B in (1, 20, 32):
        t.check_tail_against_fp64(native, B, 10, seed=700 + B)
    t.check_tail_repeatable(native, 32, 10, seed=12)
names = {{e.key for e in prof.key_averages() if "dense_tail_kernel" in e.key}}
assert names and all("128, 8>" in n for n in names), names
print("cluster-8 ok", sorted(names))
"""


def test_dense_tail_cluster8_matches_fp64():
    """GEOMX_MLP_CLUSTER=8 (the portable cluster size); the choice is cached per process, hence a fresh interpreter."""
    env = dict(os.environ, GEOMX_MLP_CLUSTER="8")
    code = _CLUSTER8.format(root=ROOT, tests=os.path.join(ROOT, "tests"))
    r = subprocess.run([sys.executable, "-c", code], env=env, cwd=ROOT, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True,
                       timeout=600)
    assert r.returncode == 0 and "cluster-8 ok" in r.stdout, r.stdout[-4000:]


# ---------------------------------------------------------------------------------------------------------------- in the step
def test_captured_step_runs_the_new_pair(nat, monkeypatch):
    from geomx_b200.parallel import Topology
    for k in SWITCHES:
        monkeypatch.delenv(k, raising=False)
    B = 32
    g = torch.Generator().manual_seed(900)
    X, y = torch.rand(B, 1, 28, 28, generator=g), torch.randint(0, 10, (B,), generator=g).float()
    eng = mx.models.HipsCNNTrainStep(batch_size=B, optimizer=mx.optimizer.Adam(learning_rate=0.01), topo=Topology(1, 0, 1, 1), use_graph=True)
    try:
        names = [n for n, _, _ in eng._steps()]
        assert "conv0+conv1 fwd (direct, relu+pool fused)" in names and "mlp chain fwd+bwd (cluster)" in names, names
        eng.step(X.pin_memory(), y.pin_memory())
        assert eng.kernels_per_step == 6, eng.kernels_per_step
        torch.cuda.synchronize()
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            eng.run_device()
            torch.cuda.synchronize()
        kernels = {e.key for e in prof.key_averages()}
        assert any("cnn_fwd_dense0_kernel" in k for k in kernels), kernels
        assert any("dense_tail_kernel" in k for k in kernels), kernels
        assert not any("mlp_chain_kernel" in k or "cnn_fwd_kernel" in k for k in kernels), kernels
    finally:
        del eng
        gc.collect()
        torch.cuda.empty_cache()
