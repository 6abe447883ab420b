"""At even batches <= 32 the first dense layer runs in the forward convolution kernel (cnn_fwd_dense0_kernel, csrc/kernels/cnn_direct.cu:
clusters of two images whose 8 CTAs exchange a2 and compute a3) and the dense-chain cluster kernel starts from a3 (dense_tail_kernel,
csrc/kernels/mlp_chain.cu).  These tests check both kernels alone, with every output pre-filled with NaN (a slice never written, or read
before it landed, shows up): the convolutions against cnn_fwd bit for bit, a3 and the tail's outputs against fp64, the batch sizes the forward
kernel refuses, launch-to-launch determinism at both cluster sizes, and that the captured step runs the new pair."""
import pytest
import torch

import geomx_b200 as mx
from _cnn_ref import (D0, D1, check_dense_tail, check_dense_tail_repeatable, engine, nan, nat, rel_err,  # noqa: F401  (nat, engine: fixtures)
                      run_in_fresh_interpreter)

pytestmark = pytest.mark.gpu


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
@pytest.mark.parametrize("B", [1, 20, 32])
@pytest.mark.parametrize("C", [10, 16])
def test_dense_tail_matches_fp64(nat, B, C):
    check_dense_tail(nat, B, C, seed=600 + B + C)


def test_dense_tail_three_launches_bit_identical(nat):
    check_dense_tail_repeatable(nat, 32, 10, seed=11)


def test_dense_tail_cluster8_matches_fp64():
    """GEOMX_MLP_CLUSTER=8 (the portable cluster size); the choice is cached per process, hence a fresh interpreter."""
    run_in_fresh_interpreter({"GEOMX_MLP_CLUSTER": "8"}, """
for B in (1, 20, 32):
    ref.check_dense_tail(native, B, 10, seed=700 + B)
ref.check_dense_tail_repeatable(native, 32, 10, seed=12)
""", "dense_tail_kernel", "128, 8>")


# ---------------------------------------------------------------------------------------------------------------- in the step
def test_captured_step_runs_the_new_pair(nat, engine):
    B = 32
    g = torch.Generator().manual_seed(900)
    X, y = torch.rand(B, 1, 28, 28, generator=g), torch.randint(0, 10, (B,), generator=g).float()
    eng = engine(B, mx.optimizer.Adam(learning_rate=0.01), use_graph=True)
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
