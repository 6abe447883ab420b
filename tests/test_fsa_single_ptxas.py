"""The one-rank exchange (hips_fsa_step_single_kernel, csrc/kernels/hips_fabric.cu) stages its tile before its grid dependency resolves, so
its CTAs must find room on SMs that still run the grid producing the gradients: beside two or three CTAs of the convolution backward wave
(288 threads, <= 40 registers, 41,344 bytes of shared memory each) and the dense weight-gradient CTAs.  At 256 threads and <= 64 registers a
CTA takes 16,384 registers, so two of them fit beside two backward CTAs (2 x 11,520 + 2 x 16,384 <= 65,536) and one beside three.  ptxas
reports what each instance (constant / scheduled lr, with / without the later optimizer kinds) uses; no GPU needed."""
from test_fwd_dense0_ptxas import _ptxas


def test_single_rank_exchange_within_budget(tmp_path):
    found = _ptxas(tmp_path, "hips_fabric")
    inst = {k: v for k, v in found.items() if "hips_fsa_step_single_kernel" in k}
    assert len(inst) == 4, inst
    for name, (regs, spills) in inst.items():
        assert regs <= 64, (name, regs)
        assert spills and not any(spills), (name, spills)
