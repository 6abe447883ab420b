"""Per-kernel cost of the flagship step (1 GPU): every launch of HipsCNNTrainStep is captured alone, REP times back to back, in a CUDA graph
(PDL edges, L2 warm) and timed with CUDA events -> steady-state us per launch; plus in-kernel %globaltimer phase stamps of the fused MLP
cluster kernel, of the dense weight-gradient kernel behind it and of the conv1 wgmma GEMM.  Usage: python tools/kernel_times.py [--fast]"""
import ctypes
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import geomx_b200 as mx  # noqa: E402
from geomx_b200.ops import native  # noqa: E402
from geomx_b200.parallel import Topology  # noqa: E402

native.set_gemm_precision("tf32" if "--fast" in sys.argv else "3xtf32")
eng = mx.models.HipsCNNTrainStep(batch_size=32, topo=Topology(1, 0, 1, 0), use_graph=False)
eng.x.copy_(torch.rand(32, 1, 28, 28)); eng.label.copy_(torch.randint(0, 10, (32,)).float())
for _ in range(3):
    eng._body()
torch.cuda.synchronize()
REP = 20
print("# precision=%s fused_mlp=%s overlap=%s  (us per launch, %d back-to-back launches in one graph)" % (native.gemm_precision(), eng.fused_mlp, eng.overlap, REP))
total = 0.0
for name, where, fn in eng._steps():
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        fn(); fn()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(REP):
            fn()
    ts = []
    for _ in range(20):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); g.replay(); b.record(); torch.cuda.synchronize()
        ts.append(a.elapsed_time(b) * 1e3 / REP)
    ts.sort()
    total += ts[len(ts) // 2]
    print("%-52s %-5s %8.2f" % (name, where, ts[len(ts) // 2]))
print("%-52s %-5s %8.2f" % ("sum", "", total))
eng._body(); torch.cuda.synchronize()
lib = native.require()
if eng.fused_mlp:
    dbg = torch.zeros(32, dtype=torch.int64, device="cuda")
    lib.gx_mlp_chain_set_debug(ctypes.c_void_p(dbg.data_ptr()))
    for rep in range(3):
        eng._body(); torch.cuda.synchronize()
        st = dbg.cpu().tolist()
        # (the cluster kernel that starts from a3, dense_tail_kernel, leaves slots 4 and 10..13 at 0)
        print("mlp chain phases (us since kernel start): 0 start|1 prologue issued|2 pdl wait done|3 inputs landed+sync|4 a3 landed|5 a4 landed|"
              "6 dz4 computed|7 dz3 pushed|8 dz3 landed|9 end (da2 stored):",
              ["%.2f" % ((v - st[0]) / 1e3) for v in st[:10]], "| P1: 10 products done|11 partials synced|12 W0 prefetch issued|13 a3 pushed:",
              ["%.2f" % ((v - st[0]) / 1e3) for v in st[10:14]], "| P5: 14 da2 products done:", "%.2f" % ((st[14] - st[0]) / 1e3),
              "| dense_wgrad: 16 start|17 dependency resolved|18 last CTA done:", ["%.2f" % ((v - st[0]) / 1e3) for v in st[16:19]])
    lib.gx_mlp_chain_set_debug(ctypes.c_void_p(0))
if eng.direct_conv:
    dbg = torch.zeros(1024, dtype=torch.int64, device="cuda")
    lib.gx_cnn_set_debug(ctypes.c_void_p(dbg.data_ptr()))
    for rep in range(2):
        eng._body(); torch.cuda.synchronize()
        st = dbg.cpu().tolist()
        r = lambda a, b: ["%.2f" % ((v - st[a]) / 1e3) for v in st[a:b]]
        print("cnn_fwd  (us): 0 start|1 operands staged|2 conv0 done|3 conv1 partials|4 end|5 a2 landed|6 a3 stored (5, 6: with dense0):", r(0, 7))
        print("cnn_bwd  (us): 8 start|9 staged|10 dz2 scattered|11 dgrad partials|12 da1 routed|13 end:", r(8, 14))
        print("cnn_wgrad1 (us): 16 start|17 staged|18 end:", r(16, 19))
    lib.gx_cnn_set_debug(ctypes.c_void_p(0))
dbg = torch.zeros(16, dtype=torch.int64, device="cuda")
lib.gx_gemm_set_debug(ctypes.c_void_p(dbg.data_ptr()))
gemm_steps = [(s[0], s[2]) for s in eng._steps() if "gemm" in s[0]]
for label, fn in gemm_steps:
    for rep in range(2):
        fn(); torch.cuda.synchronize()
    st = dbg.cpu().tolist()
    print("%s phases (us): 0 start|1 prologue|2 pdl wait|3 first stage ready|4 last MMA issued|5 accumulator visible|6 epilogue done:" % label,
          ["%.2f" % ((v - st[0]) / 1e3) for v in st[:7]])
lib.gx_gemm_set_debug(ctypes.c_void_p(0))
