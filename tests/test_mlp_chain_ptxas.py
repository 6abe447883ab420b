"""The dense-chain cluster kernel (csrc/kernels/mlp_chain.cu) has to fit on an SM beside a cnn_fwd CTA (256 threads allocated 64 registers
each), so that the convolution forward pass of the next step can overlap it: 512 x 96 + 256 x 64 = 65,536 registers.  ptxas reports what
each instance of the kernel uses; this checks both cluster sizes at the build's own flags, with no GPU needed."""
import os
import re
import shutil
import subprocess

import pytest

from geomx_b200 import build

SRC = os.path.join(build.CSRC, "kernels", "mlp_chain.cu")


def test_mlp_chain_fits_beside_cnn_fwd(tmp_path):
    if not (os.path.exists(build.NVCC) or shutil.which(build.NVCC)):
        pytest.skip("nvcc not available")
    r = subprocess.run([build.NVCC] + build.NVCC_FLAGS + ["-Xptxas", "-v", "-c", SRC, "-o", str(tmp_path / "mlp_chain.o")],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout[-4000:]
    # ptxas prints, per entry function: "Compiling entry function '<name>'", "... N bytes spill stores, M bytes spill loads", "Used R registers"
    found = {}
    for block in r.stdout.split("Compiling entry function ")[1:]:
        name = block.split("'")[1]
        if "mlp_chain_kernel" not in name:
            continue
        spills = [int(v) for v in re.findall(r"(\d+) bytes spill (?:stores|loads)", block)]
        regs = int(re.search(r"Used (\d+) registers", block).group(1))
        found[name] = (regs, spills)
    assert len(found) == 2, found               # the 16-CTA and the 8-CTA cluster instances
    for name, (regs, spills) in found.items():
        assert regs <= 96, (name, regs)
        assert spills and not any(spills), (name, spills)
