"""Register and spill budgets of the sm_90a kernels, from ptxas at the build's own flags; no GPU needed.  Each source is compiled once;
each row of BUDGETS is one test."""
import os
import re
import shutil
import subprocess

import pytest

from geomx_b200 import build
from geomx_b200.ops import _native_api as api

# (source, kernel-name substring ("" = every entry function), instances (None = any number), register ceiling (None = none), spills allowed)
BUDGETS = [
    # the forward kernel's CTAs share an SM with the dense_tail CTAs that stage their weights beside them: 256 x 64 + 512 x 96 = 65,536
    # registers (the shared-memory side is a static_assert in mlp_chain.cu)
    ("cnn_direct", "cnn_fwd_dense0_kernel", 1, 64, False),
    ("mlp_chain", "dense_tail_kernel", 2, 96, False),                  # the 16-CTA and the 8-CTA cluster instances; the same sum
    # the dense-chain cluster kernel fits on an SM beside a cnn_fwd CTA (256 threads at 64 registers): 512 x 96 + 256 x 64 = 65,536
    ("mlp_chain", "mlp_chain_kernel", 2, 96, False),
    # the weighted instances (short and sample-weighted batches) replace their unweighted twins in the same step: the same budgets
    ("cnn_direct", "cnn_fwd_dense0_weighted_kernel", 1, 64, False),
    ("mlp_chain", "mlp_chain_weighted_kernel", 2, 96, False),
    ("mlp_chain", "dense_tail_weighted_kernel", 2, 96, False),
    ("loss_head", "head_fwd_bwd_weighted_kernel", 1, 64, False),       # 1024 threads per CTA: at most 64 registers each
    # no co-residency budget, but a spill would put every image's dense1 / classifier operands through L1 / L2
    ("cnn_direct", "cnn_eval_kernel", 1, None, False),
    # the one-rank exchange stages its tile before its grid dependency resolves, beside two or three CTAs of the convolution backward wave
    # (288 threads, <= 40 registers): at 256 threads and <= 64 registers, 2 x 11,520 + 2 x 16,384 <= 65,536.  Constant / scheduled lr,
    # with / without the later optimizer kinds
    ("hips_fabric", "hips_fsa_step_single_kernel", 4, 64, False),
    # constant / scheduled lr, with / without the kinds after DCASGD; __launch_bounds__(256, 2)
    ("hips_fabric", "hips_fsa_ll_kernel", 4, 128, True),
    ("hips_fabric", "hips_fsa_direct_kernel", 4, 128, True),
    # two 288-thread CTAs per SM, which the kernel's ticket wait needs
    ("cnn_direct", "cnn_bwd_exchange_kernel", 4, 112, True),
    # one instance per optimizer kind: arena x {constant, scheduled lr}, multi-tensor, single-tensor
    ("optim", "arena_opt_kernel", 2 * len(api.OPT_KINDS), None, True),
    ("optim", "multi_tensor_opt_kernel", len(api.OPT_KINDS), None, True),
    ("optim", "single_opt_kernel", len(api.OPT_KINDS), None, True),
    # every update kernel has a constant-lr and a scheduled instance (step_lr<SCHED>): none of them, nor anything else in these files, spills
    ("optim", "", None, None, False),
    ("hips_fabric", "", None, None, False),
    ("cnn_direct", "", None, None, False),
    # the gradient-compression kernels (bsc_kernel<0> at 1024 threads: at most 64 registers, enforced by its __launch_bounds__)
    ("compress", "", None, None, False),
]


@pytest.fixture(scope="module")
def ptxas(tmp_path_factory):
    """source name -> {entry function: (registers, [spill store bytes, spill load bytes])}, compiling each source once."""
    if not (os.path.exists(build.NVCC) or shutil.which(build.NVCC)):
        pytest.skip("nvcc not available")
    out, cache = tmp_path_factory.mktemp("ptxas"), {}

    def get(name):
        if name not in cache:
            src = os.path.join(build.CSRC, "kernels", name + ".cu")
            r = subprocess.run([build.NVCC] + build.NVCC_FLAGS + ["-Xptxas", "-v", "-c", src, "-o", str(out / (name + ".o"))],
                               stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
            assert r.returncode == 0, r.stdout[-4000:]
            # per entry function: "Compiling entry function '<name>'", "... N bytes spill stores, M bytes spill loads", "Used R registers"
            found = {}
            for block in r.stdout.split("Compiling entry function ")[1:]:
                spills = [int(v) for v in re.findall(r"(\d+) bytes spill (?:stores|loads)", block)]
                found[block.split("'")[1]] = (int(re.search(r"Used (\d+) registers", block).group(1)), spills)
            cache[name] = found
        return cache[name]

    return get


@pytest.mark.parametrize("src,kernel,count,max_regs,spills_ok", BUDGETS, ids=["%s-%s" % (s, k or "all") for s, k, *_ in BUDGETS])
def test_kernel_budget(ptxas, src, kernel, count, max_regs, spills_ok):
    found = {k: v for k, v in ptxas(src).items() if kernel in k}
    assert found if count is None else len(found) == count, (src, kernel, count, sorted(found))
    for name, (regs, spills) in found.items():
        if max_regs is not None:
            assert regs <= max_regs, (name, regs, max_regs)
        if not spills_ok:
            assert spills and not any(spills), (name, regs, spills)
