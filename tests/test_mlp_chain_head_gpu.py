"""The classifier head of the dense-chain cluster kernel (csrc/kernels/mlp_chain.cu) computes the 32 x C logits as 4x4 register tiles, runs
softmax-CE on the four lanes that hold a row, and every CTA then computes the whole dz4 itself instead of receiving it.  These tests cover
what that layout has to get right: class counts that are not a multiple of four (C = 1, 3, 13) with the last class as a label, batches that
fill the last 4-row tile only partly (B = 7, 31: the padded rows must add nothing to any output), logit margins up to 60, and
bit-identical outputs from launch to launch at both cluster sizes.  Outputs are pre-filled with NaN and checked against fp64 autograd."""
import pytest

from _cnn_ref import check_mlp_chain, check_mlp_chain_repeatable, nat, run_in_fresh_interpreter  # noqa: F401  (nat: fixture)

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("margin", [0, 60])
@pytest.mark.parametrize("C", [1, 3, 13])
@pytest.mark.parametrize("B", [7, 31])
def test_mlp_chain_head_matches_fp64(nat, B, C, margin):
    check_mlp_chain(nat, B, C, seed=300 + 3 * B + C, margin=margin)


@pytest.mark.parametrize("B,C", [(31, 13), (7, 3)])
def test_mlp_chain_head_three_launches_bit_identical(nat, B, C):
    check_mlp_chain_repeatable(nat, B, C, seed=400 + B, margin=60)


def test_mlp_chain_head_cluster8():
    """GEOMX_MLP_CLUSTER=8 (the portable cluster size); the choice is cached per process, hence a fresh interpreter."""
    run_in_fresh_interpreter({"GEOMX_MLP_CLUSTER": "8"}, """
for B in (7, 31):
    for C in (1, 3, 13):
        ref.check_mlp_chain(native, B, C, seed=500 + B + C, margin=60)
ref.check_mlp_chain_repeatable(native, 31, 13, seed=9, margin=60)
""", "mlp_chain_kernel", "128, 8>")
