"""At even batches <= 32 the step runs cnn_fwd_dense0_kernel (csrc/kernels/cnn_direct.cu) and then dense_tail_kernel
(csrc/kernels/mlp_chain.cu), whose CTAs stage their weights on the SMs beside the forward CTAs while those still run.  That needs both in one
SM's register file: 256 x 64 + 512 x 96 = 65,536 registers.  ptxas reports what each kernel uses; this checks it at the build's own flags,
with no GPU needed (the shared-memory side is a static_assert in mlp_chain.cu)."""
import os
import re
import shutil
import subprocess

import pytest

from geomx_b200 import build


def _ptxas(tmp_path, name):
    if not (os.path.exists(build.NVCC) or shutil.which(build.NVCC)):
        pytest.skip("nvcc not available")
    src = os.path.join(build.CSRC, "kernels", name + ".cu")
    r = subprocess.run([build.NVCC] + build.NVCC_FLAGS + ["-Xptxas", "-v", "-c", src, "-o", str(tmp_path / (name + ".o"))],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout[-4000:]
    found = {}
    for block in r.stdout.split("Compiling entry function ")[1:]:
        spills = [int(v) for v in re.findall(r"(\d+) bytes spill (?:stores|loads)", block)]
        regs = int(re.search(r"Used (\d+) registers", block).group(1))
        found[block.split("'")[1]] = (regs, spills)
    return found


def test_fwd_dense0_within_64_registers(tmp_path):
    found = {k: v for k, v in _ptxas(tmp_path, "cnn_direct").items() if "cnn_fwd_dense0_kernel" in k}
    assert len(found) == 1, found
    for name, (regs, spills) in found.items():
        assert regs <= 64, (name, regs)
        assert spills and not any(spills), (name, spills)


def test_dense_tail_within_96_registers(tmp_path):
    found = {k: v for k, v in _ptxas(tmp_path, "mlp_chain").items() if "dense_tail_kernel" in k}
    assert len(found) == 2, found               # the 16-CTA and the 8-CTA cluster instances
    for name, (regs, spills) in found.items():
        assert regs <= 96, (name, regs)
        assert spills and not any(spills), (name, spills)
