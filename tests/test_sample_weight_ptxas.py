"""Short and sample-weighted batches run the weighted instances of the kernels that produce the dlogits (cnn_fwd_dense0_weighted_kernel,
mlp_chain_weighted_kernel, dense_tail_weighted_kernel, head_fwd_bwd_weighted_kernel).  They replace their unweighted twins in the same step,
so they must meet the same budgets: the forward kernel's instance <= 64 registers (it shares an SM with a dense_tail CTA), the cluster
kernels' <= 96, and no spills.  ptxas reports what each instance uses at the build's own flags; no GPU needed."""
import pytest

from test_fwd_dense0_ptxas import _ptxas


@pytest.mark.parametrize("src,kernel,count,regs", [
    ("cnn_direct", "cnn_fwd_dense0_weighted_kernel", 1, 64),
    ("mlp_chain", "mlp_chain_weighted_kernel", 2, 96),          # the 16-CTA and the 8-CTA cluster instances
    ("mlp_chain", "dense_tail_weighted_kernel", 2, 96),
    ("loss_head", "head_fwd_bwd_weighted_kernel", 1, 64),       # 1024 threads per CTA: at most 64 registers each
])
def test_weighted_instances_within_budget(tmp_path, src, kernel, count, regs):
    found = {k: v for k, v in _ptxas(tmp_path, src).items() if kernel in k}
    assert len(found) == count, found
    for name, (r, spills) in found.items():
        assert r <= regs, (name, r)
        assert spills and not any(spills), (name, spills)
