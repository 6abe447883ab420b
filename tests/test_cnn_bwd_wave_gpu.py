"""The convolution backward grid (cnn_bwd_all, csrc/kernels/cnn_direct.cu) as one resident wave: its conv1 weight gradient is split over
clusters of two CTAs, each staging half the batch, so that the grid's shared memory is the data-gradient body's and every CTA is resident
(and staged) while the dense-chain cluster that precedes it still runs.  Checks the launch geometry with occupancy queries, the split
weight gradient against fp64, its determinism, and that the per-CTA debug stamps stay inside their 1024-slot buffer."""
import ctypes

import pytest
import torch

from _cnn_ref import dev, nan, nat, rel_err, route  # noqa: F401  (nat: fixture)

pytestmark = pytest.mark.gpu

TAIL_SMS = 16        # the dense-chain cluster (dense_tail_kernel) that runs while the backward grid becomes resident: one CTA per SM


def forward(nat, B, seed):
    """a1, idx1, a2, idx2 of the kernels' own forward pass, and a da2, for B images (biases > 0: most pooled conv1 outputs are live)."""
    g = torch.Generator().manual_seed(seed)
    x = torch.rand(B, 1, 28, 28, generator=g).to(dev())
    w0 = (torch.randn(16, 1, 5, 5, generator=g) * 0.3).to(dev())
    b0 = (torch.rand(16, generator=g) * 0.1).to(dev())
    w1 = (torch.randn(32, 16, 5, 5, generator=g) * 0.1).to(dev())
    b1 = (torch.rand(32, generator=g) * 0.05 - 0.01).to(dev())
    da2 = torch.randn(B, 32, 4, 4, generator=g).to(dev())
    a1 = torch.empty(B, 16, 12, 12, device=dev()); idx1 = torch.empty(B, 16, 12, 12, dtype=torch.uint8, device=dev())
    a2 = torch.empty(B, 32, 4, 4, device=dev()); idx2 = torch.empty(B, 32, 4, 4, dtype=torch.uint8, device=dev())
    nat.cnn_fwd(x, w0, b0, w1, b1, a1, idx1, a2, idx2)
    torch.cuda.synchronize()
    return x, w1, a1, idx1, a2, idx2, da2


def wgrad1_ref(a1, a2, idx2, da2):
    """fp64 dW1 / db1 from the kernels' a1 and routing: the pooled gradient goes to the window's arg-max where a2 > 0."""
    dz = route(torch.where(a2 > 0, da2, torch.zeros_like(da2)).double(), idx2)
    return torch.nn.grad.conv2d_weight(a1.double(), (32, 16, 5, 5), dz), dz.sum((0, 2, 3))


def test_grid_is_one_wave_beside_the_dense_chain(nat):
    geo = nat.cnn_bwd_all_geometry(32)
    assert geo is not None, geo
    # both bodies within the data-gradient body's shared memory: the weight-gradient CTAs stage half the batch each
    assert geo["wgrad_smem"] <= geo["dgrad_smem"] and geo["smem"] == geo["dgrad_smem"], geo
    assert geo["grid"] == 256 + 4 * 32, geo
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    assert geo["ctas_per_sm"] >= 5, geo
    # every CTA resident at once even if the dense-chain cluster's SMs held none of them (they hold one each)
    assert 2 * geo["clusters"] - TAIL_SMS * geo["ctas_per_sm"] >= geo["grid"], (geo, sms)
    assert geo["regs"] <= 40, geo
    assert nat.cnn_bwd_all_geometry(3) is None and nat.cnn_bwd_all_geometry(66) is None


@pytest.mark.parametrize("B", [2, 32, 64])
def test_split_wgrad1_matches_fp64(nat, B):
    x, w1, a1, idx1, a2, idx2, da2 = forward(nat, B, 100 + B)
    ref_w, ref_b = wgrad1_ref(a1, a2, idx2, da2)
    assert float(ref_w.abs().max()) > 0
    dw1, db1 = nan(32, 16, 5, 5), nan(32)
    assert nat.cnn_wgrad1(a1, a2, idx2, da2, dw1, db1)
    torch.cuda.synchronize()
    assert rel_err(dw1, ref_w) < 1e-5 and rel_err(db1, ref_b) < 1e-5, (rel_err(dw1, ref_w), rel_err(db1, ref_b))
    dw0, db0 = torch.zeros(16, 1, 5, 5, device=dev()), torch.zeros(16, device=dev())
    dw1b, db1b = nan(32, 16, 5, 5), nan(32)
    nat.cnn_bwd_all(x, w1, a1, idx1, a2, idx2, da2, dw0, db0, dw1b, db1b)
    torch.cuda.synchronize()
    assert rel_err(dw1b, ref_w) < 1e-5 and rel_err(db1b, ref_b) < 1e-5, (rel_err(dw1b, ref_w), rel_err(db1b, ref_b))
    # the separate launch and the one-grid launch run the same body: the same bits
    assert torch.equal(dw1, dw1b) and torch.equal(db1, db1b)


def test_split_wgrad1_is_bitwise_repeatable(nat):
    x, w1, a1, idx1, a2, idx2, da2 = forward(nat, 32, 7)
    outs = []
    for _ in range(3):
        dw0, db0 = torch.zeros(16, 1, 5, 5, device=dev()), torch.zeros(16, device=dev())
        dw1, db1 = nan(32, 16, 5, 5), nan(32)
        nat.cnn_bwd_all(x, w1, a1, idx1, a2, idx2, da2, dw0, db0, dw1, db1)
        torch.cuda.synchronize()
        outs.append((dw1, db1))
    for dw1, db1 in outs[1:]:
        assert torch.equal(dw1, outs[0][0]) and torch.equal(db1, outs[0][1])


@pytest.mark.parametrize("B", [32, 64])
def test_cta_stamps_stay_in_the_debug_buffer(nat, B):
    geo = nat.cnn_bwd_all_geometry(B)
    assert 64 + 3 * geo["stamped_ctas"] <= 1024, geo
    x, w1, a1, idx1, a2, idx2, da2 = forward(nat, B, 3)
    buf = torch.full((1024 + 256,), -1, dtype=torch.int64, device=dev())
    lib = nat.require()
    lib.gx_cnn_set_debug(ctypes.c_void_p(buf.data_ptr()))
    try:
        dw0, db0 = torch.zeros(16, 1, 5, 5, device=dev()), torch.zeros(16, device=dev())
        dw1, db1 = torch.empty(32, 16, 5, 5, device=dev()), torch.empty(32, device=dev())
        nat.cnn_bwd_all(x, w1, a1, idx1, a2, idx2, da2, dw0, db0, dw1, db1)
        torch.cuda.synchronize()
    finally:
        lib.gx_cnn_set_debug(ctypes.c_void_p(0))
    assert bool((buf[1024:] == -1).all()), "stamps written past slot 1023"
    n = geo["stamped_ctas"]
    stamps = buf[64:64 + 3 * n].view(n, 3)
    assert bool((stamps[:, 1] >= stamps[:, 0]).all()) and bool((stamps[:, 0] > 0).all())
