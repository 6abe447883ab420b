"""The dense-chain cluster kernel (csrc/kernels/mlp_chain.cu) hands every layer's output to the other CTAs of its cluster with st.async and
per-buffer transaction barriers instead of cluster-wide barriers.  These tests check what that hand-off must preserve: every output against
fp64 autograd at the batch sizes it covers, at both cluster sizes, with every output buffer pre-filled with NaN (a slice that is never
written, or read before it has landed, shows up), and bit-identical results from launch to launch (every sum has a fixed order)."""
import pytest

from _cnn_ref import check_mlp_chain, check_mlp_chain_repeatable, nat, run_in_fresh_interpreter  # noqa: F401  (nat: fixture)

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("B", [1, 20, 32])
@pytest.mark.parametrize("C", [10, 16])
def test_mlp_chain_cluster16_matches_fp64(nat, B, C):
    check_mlp_chain(nat, B, C, seed=100 + B + C)


@pytest.mark.parametrize("B", [1, 32])
def test_mlp_chain_three_launches_bit_identical(nat, B):
    check_mlp_chain_repeatable(nat, B, 10, seed=7 + B)


def test_mlp_chain_cluster8_matches_fp64():
    """GEOMX_MLP_CLUSTER=8 (the portable cluster size); the choice is cached per process, hence a fresh interpreter."""
    run_in_fresh_interpreter({"GEOMX_MLP_CLUSTER": "8"}, """
for B in (1, 20, 32):
    ref.check_mlp_chain(native, B, 10, seed=200 + B)
ref.check_mlp_chain_repeatable(native, 32, 10, seed=9)
""", "mlp_chain_kernel", "128, 8>")
