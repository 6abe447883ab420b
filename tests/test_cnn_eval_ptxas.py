"""cnn_eval_kernel (csrc/kernels/cnn_direct.cu) has no co-residency budget to meet, but a spill to local memory would put every image's
dense1 / classifier operands through L1 / L2.  ptxas reports spills at the build's own flags; no GPU needed."""
from test_fwd_dense0_ptxas import _ptxas


def test_cnn_eval_kernel_does_not_spill(tmp_path):
    found = {k: v for k, v in _ptxas(tmp_path, "cnn_direct").items() if "cnn_eval_kernel" in k}
    assert len(found) == 1, found
    for name, (regs, spills) in found.items():
        assert spills and not any(spills), (name, regs, spills)
