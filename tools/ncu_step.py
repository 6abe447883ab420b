"""Driver for `ncu --set full`: a few EAGER flagship steps (one launch per kernel, no CUDA graph) so that every kernel of the step can be
captured on its own.  Launch order per step: cnn_fwd, mlp_chain, dense_wgrad, dense-key channel, cnn_bwd_all, conv-key channel
(6 launches; with GEOMX_FUSED_EXCHANGE=1: 5).  Then one BatchNorm forward/backward and the large GEMM in both precisions.

  ncu --set full --clock-control none --import-source on --launch-skip 15 --launch-count 9 -o gpurun_out/r2_step python tools/ncu_step.py
"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import geomx_b200 as mx  # noqa: E402
from geomx_b200.ops import native  # noqa: E402
from geomx_b200.parallel import Topology  # noqa: E402

native.set_gemm_precision("3xtf32")
torch.manual_seed(0)
eng = mx.models.HipsCNNTrainStep(batch_size=32, optimizer=mx.optimizer.Adam(learning_rate=0.01), topo=Topology(1, 0, 1, 0), use_graph=False,
                                 loopback=os.environ.get("NCU_LOOPBACK", "1") == "1")
eng.x.copy_(torch.rand(32, 1, 28, 28)); eng.label.copy_(torch.randint(0, 10, (32,)).float())
flush = torch.empty(64 * 1024 * 1024, device="cuda")
for it in range(4):                       # steps 0-2: warm-up (15 launches), step 3: captured
    flush.fill_(float(it))                # torch kernels are not counted by the -k filter of the command line below
    eng._body()
    torch.cuda.synchronize()
# BatchNorm (generic Gluon path) and the large GEMM
x = torch.randn(64, 128, 28, 28, device="cuda", requires_grad=True)
g = torch.ones(128, device="cuda", requires_grad=True); b = torch.zeros(128, device="cuda", requires_grad=True)
rm, rv = torch.zeros(128, device="cuda"), torch.ones(128, device="cuda")
from geomx_b200.ops import functional as OF  # noqa: E402
y = OF.batch_norm(x, g, b, rm, rv, True)
y.sum().backward()
A = torch.randn(8192, 4096, device="cuda"); B = torch.randn(4096, 4096, device="cuda"); D = torch.empty(8192, 4096, device="cuda")
native.set_gemm_precision("tf32"); native.gemm(A, B, D)
native.set_gemm_precision("3xtf32"); native.gemm(A, B, D)
torch.cuda.synchronize()
print("ok", float(eng.loss.mean()), float(D[0, 0]))
