"""da2 = dz3 W0 from dense_tail_kernel's from-dz3 mode (csrc/kernels/mlp_chain.cu, dense_dx_rows), which runs over one cluster per four
batch rows: 1, 1, 2 and 8 clusters at the batch sizes below.  Against fp64 with a ReLU-sparse dz3, and bit for bit over three launches."""
import pytest
import torch

from _cnn_ref import D0, D1, D2, dense_chain_ref, nan, nat, rel_err  # noqa: F401  (nat: fixture)

pytestmark = pytest.mark.gpu

C = 10
BATCHES = [1, 2, 8, 32]


def da2_from_dz3(nat, dz3, w0):
    """from-dz3 mode: every operand but dz3 and w0 is NaN, so that a read of one shows up in dx"""
    B = dz3.shape[0]
    dx = nan(B, D0)
    assert nat.dense_tail(nan(B, D1), w0, nan(D2, D1), nan(D2), nan(C, D2), nan(C), nan(B), nan(B), nan(B, C), dx, nan(B, D2), nan(B, D2),
                          dz3, nan(B, 16), from_dz3=True)
    torch.cuda.synchronize()
    return dx


@pytest.mark.parametrize("B", BATCHES)
def test_da2_matches_fp64_and_repeats_bitwise(nat, B):
    g = torch.Generator().manual_seed(1200 + B)
    dz3 = torch.relu(torch.randn(B, D1, generator=g)).cuda()          # ReLU-sparse, like the head's dz3
    w0 = (torch.randn(D1, D0, generator=g) * 0.05).cuda()
    outs = [da2_from_dz3(nat, dz3, w0) for _ in range(3)]
    assert not torch.isnan(outs[0]).any(), B
    assert rel_err(outs[0], dense_chain_ref([w0] + [None] * 5, dz3=dz3)["dx"]) < 1e-6, B
    for dx in outs[1:]:
        assert torch.equal(dx, outs[0]), (B, "da2 differs between launches")
