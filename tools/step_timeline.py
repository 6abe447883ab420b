"""In-graph timeline of the flagship step on every rank (run under torchrun, or plain python for 1 GPU).

Every kernel of the step writes %globaltimer stamps (debug buffers of cnn_direct.cu / mlp_chain.cu, phase stamps of the exchange channels); the
graph is captured with stamping on and replayed like bench.py does (L2 flushed, ranks re-aligned before each step).  Prints, per rank, the
median start / end of each kernel relative to the start of the first one — where the step's microseconds go at N GPUs.

  python -m torch.distributed.run --nproc-per-node 2 --master-addr 127.0.0.1 tools/step_timeline.py [--lookahead]
"""
import ctypes
import os
import statistics
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import geomx_b200 as mx  # noqa: E402
from geomx_b200.ops import native  # noqa: E402
from geomx_b200.parallel import Topology  # noqa: E402

# in-kernel %globaltimer stamps of the direct-convolution kernels (gx_cnn_set_debug slots, written by the first CTA of each body).  The
# forward kernel that also computes dense0 (even batches <= 32) stamps 5 a2 landed | 6 a3 stored before its end (4).
# The data-gradient body splits its staging: 25 W1 issued | 26 x, a1, idx1 issued | 27 list ballots done | 9 staging landed; 28 is the end
# of its db0 thread (shown relative to 13, the end of thread 0's conv0 weight gradient).
CNN_PHASES = {"cnn_fwd": (0, 1, 2, 3, 4), "cnn_bwd": (8, 25, 26, 27, 9, 10, 11, 12, 13, 28), "cnn_wgrad1": (16, 17, 18)}
CNN_PHASE_LABELS = {"cnn_fwd": ("staging", "conv0", "conv1", "epilogue"),
                    "cnn_bwd": ("W1 issued", "x/a1/idx1", "ballots", "landed", "pdl-wait+dz2", "dgrad", "routing", "wgrad0", "db0 thread end"),
                    "cnn_wgrad1": ("staging+pdl-wait", "wgrad1")}
FWD_DENSE0_PHASES, FWD_DENSE0_LABELS = (0, 1, 2, 3, 5, 6), ("staging", "conv0", "conv1", "a2 landed", "dense0 -> a3 stored")
# with its training head (the classic step) it goes on: 7 a3 landed | 14 a4 landed | 15 dz3 stored
FWD_HEAD_PHASES = FWD_DENSE0_PHASES + (7, 14, 15)
FWD_HEAD_LABELS = FWD_DENSE0_LABELS + ("a3 landed", "dense1 -> a4 landed", "head -> dz4 -> dz3 stored")
# the same for the dense-chain cluster kernel (gx_mlp_chain_set_debug slots of cluster CTA 0): 0 start | 3 inputs landed | 4 a3 landed |
# 5 a4 landed | 6 dz4 computed | 7 dz3 pushed | 8 dz3 landed | 9 end (da2 stored); and of the dense weight-gradient kernel: 16 start of its
# CTA 0 | 17 its grid dependency resolved | 18 end of its last CTA.  The kernel that starts from a3 (dense_tail_kernel) has no slot 4.
MLP_PHASES = (0, 3, 4, 5, 6, 7, 8, 9)
MLP_PHASE_LABELS = ("staging+pdl-wait", "dense0 -> a3", "dense1 -> a4", "head -> dz4", "dz3 pushed", "dz3 landed", "da2")
TAIL_PHASES = (0, 3, 5, 6, 7, 8, 9)
TAIL_PHASE_LABELS = ("staging+pdl-wait", "a3 staged -> a4", "head -> dz4", "dz3 pushed", "dz3 landed", "da2")
# ... and from dz3 (after the forward kernel's training head): 0 start | 1 W0 issued | 2 grid dependency resolved | 3 dz3 staged | 14 product done |
# 9 end (da2 stored)
TAIL_DZ3_PHASES, TAIL_DZ3_LABELS = (0, 1, 2, 3, 14, 9), ("W0 issued", "pdl-wait", "dz3 staged", "da2 product", "da2 stored")


def main():
    world, rank, local = int(os.environ.get("WORLD_SIZE", 1)), int(os.environ.get("RANK", 0)), int(os.environ.get("LOCAL_RANK", 0))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if world > 1:
        dist.init_process_group("nccl", device_id=dev)
    parties = 2 if world >= 2 and world % 2 == 0 else 1
    topo = Topology(world, rank, parties, 0)
    native.set_gemm_precision("3xtf32")
    lib = native.require()
    cdbg = torch.zeros(1024, dtype=torch.int64, device=dev)
    mdbg = torch.zeros(32, dtype=torch.int64, device=dev)
    lib.gx_cnn_set_debug(ctypes.c_void_p(cdbg.data_ptr()))
    lib.gx_mlp_chain_set_debug(ctypes.c_void_p(mdbg.data_ptr()))
    torch.manual_seed(1)
    eng = mx.models.HipsCNNTrainStep(batch_size=32, optimizer=mx.optimizer.Adam(learning_rate=0.01), topo=topo, device=dev, use_graph=True,
                                     lookahead="--lookahead" in sys.argv)
    X = torch.rand(32, 1, 28, 28).pin_memory(); y = torch.randint(0, 10, (32,)).float().pin_memory()
    for _ in range(5):
        eng.step(X, y)
    fab = eng.fabric
    chans = list(fab.channels) or ["fsa"]
    tail, head = getattr(eng, "_fwd_dense0", False), getattr(eng, "_fwd_head", False)
    cnn_phases, cnn_labels = dict(CNN_PHASES), dict(CNN_PHASE_LABELS)
    if tail:
        cnn_phases["cnn_fwd"], cnn_labels["cnn_fwd"] = (FWD_HEAD_PHASES, FWD_HEAD_LABELS) if head else (FWD_DENSE0_PHASES, FWD_DENSE0_LABELS)
    mlp_phases, mlp_labels = ((TAIL_DZ3_PHASES, TAIL_DZ3_LABELS) if head else (TAIL_PHASES, TAIL_PHASE_LABELS)) if tail else (MLP_PHASES, MLP_PHASE_LABELS)
    for c in chans:
        fab.state[c][3] = 1
    # cnn_bwd_all: weight-gradient CTAs [0, 256) (pairs that split the batch), data-gradient CTAs [256, grid); its last `stamped_ctas` CTAs
    # record (start, end, SM)
    geo = native.cnn_bwd_all_geometry(32)
    first = geo["grid"] - geo["stamped_ctas"]
    flush = torch.empty(64 * 1024 * 1024, device=dev)
    rows = []
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    for it in range(24):
        flush.fill_(float(it))
        if world > 1:
            fab.barrier()
        ev[0].record(); eng.run_device(); ev[1].record()
        torch.cuda.synchronize()
        c, m = cdbg.tolist(), mdbg.tolist()
        st = {k: fab.state[k][8:8 + 12].view(torch.int64).tolist() for k in chans}
        row = {"cnn_fwd": (c[0], c[4]), "mlp_chain": (m[0], m[9]), "cnn_bwd": (c[8], c[13]), "cnn_wgrad1": (c[16], c[18])}
        if m[16] > 0:
            row["dense_wgrad"] = (m[17], m[18])         # from its grid dependency (the cluster kernel's end) to its last CTA
        for k in chans:
            if st[k][0] > 0:
                row["chan:" + k] = (st[k][0], st[k][5])
        if getattr(eng, "fused_exchange", False):       # exchange tail of the backward launch: 20 ticket | 21 grid done | 22 sent | 23 received | 24 end
            row["bwd tail"] = (c[20], c[24])
            row["_tail"] = [(v - c[20]) / 1e3 for v in c[20:25]]
        if not getattr(eng, "fused_exchange", False):
            # (start, end, SM) of the backward grid's CTAs [first, grid), keyed by CTA index
            row["_cta"] = {first + k: (c[64 + 3 * k], c[65 + 3 * k], c[66 + 3 * k]) for k in range(geo["stamped_ctas"])}
        row["_ms"] = ev[0].elapsed_time(ev[1])
        row["_cnn_ph"] = {name: [(c[s1] - c[s0]) / 1e3 for s0, s1 in zip(slots, slots[1:])] for name, slots in cnn_phases.items()}
        row["_mlp_ph"] = [(m[s1] - m[s0]) / 1e3 for s0, s1 in zip(mlp_phases, mlp_phases[1:])]
        if "chan:dense" in row and "chan:conv" in row:
            # the dense branch (weight gradients + dense channel) must end before the conv-key exchange does, or it is exposed
            row["_dense_vs_conv"] = (row["chan:dense"][1] - row["chan:conv"][1]) / 1e3
        row["_ph"] = {k: [(v - st[k][0]) / 1e3 for v in st[k][:6]] for k in chans if st[k][0] > 0}
        rows.append(row)
    rows = rows[4:]
    names = [k for k in rows[0] if not k.startswith("_")]
    lines = ["rank %d  step %.2f us (event-timed median)" % (rank, 1e3 * statistics.median(r["_ms"] for r in rows))]
    for k in sorted(names, key=lambda k: statistics.median(r[k][0] - min(v[0] for kk, v in r.items() if not kk.startswith("_") and v[0] > 0) for r in rows)):
        rel0 = [(r[k][0] - min(v[0] for kk, v in r.items() if not kk.startswith("_") and v[0] > 0)) / 1e3 for r in rows]
        rel1 = [(r[k][1] - min(v[0] for kk, v in r.items() if not kk.startswith("_") and v[0] > 0)) / 1e3 for r in rows]
        lines.append("  %-12s start %7.2f  end %7.2f  (dur %6.2f us)" % (k, statistics.median(rel0), statistics.median(rel1),
                                                                        statistics.median(b - a for a, b in zip(rel0, rel1))))
    if "_cta" in rows[0]:
        # how the convolution-backward grid packs onto the SMs (last sampled step; the stamped CTAs only)
        r = rows[-1]
        base = min(v[0] for kk, v in r.items() if not kk.startswith("_") and v[0] > 0)
        for name, lo, hi in (("wgrad CTAs (%d..255)" % first, first, 256), ("bwd CTAs  (256..%d)" % (geo["grid"] - 1), 256, geo["grid"])):
            cs = [r["_cta"][i] for i in range(max(lo, first), hi)]
            st = sorted((a - base) / 1e3 for a, b, sm_ in cs); en = sorted((b - base) / 1e3 for a, b, sm_ in cs)
            du = sorted((b - a) / 1e3 for a, b, sm_ in cs)
            m = len(cs) // 2
            lines.append("  %-22s start min/med/max %.2f %.2f %.2f | end %.2f %.2f %.2f | duration %.2f %.2f %.2f" % (
                name, st[0], st[m], st[-1], en[0], en[m], en[-1], du[0], du[m], du[-1]))
        sms = {}
        for i, (a, b, sm_) in r["_cta"].items():
            sms.setdefault(sm_, []).append(i)
        shared = sorted(len(v) for v in sms.values())
        lines.append("  SMs used %d; CTAs per SM: %s" % (len(sms), {k: shared.count(k) for k in sorted(set(shared))}))
        mix = {}
        for v in sms.values():
            k = "%d wgrad + %d bwd" % (sum(1 for i in v if i < 256), sum(1 for i in v if i >= 256))
            mix[k] = mix.get(k, 0) + 1
        lines.append("  SM sharing: %s" % dict(sorted(mix.items())))
        # the part of the step after da2: CTAs that could only start once the dense-chain cluster had ended, and where the segment ends
        late = [sum(1 for a, b, sm_ in q["_cta"].values() if a > q["mlp_chain"][1]) for q in rows]
        to_bwd = [(max(max(b for a, b, sm_ in q["_cta"].values()), q["cnn_wgrad1"][1], q["cnn_bwd"][1]) - q["mlp_chain"][1]) / 1e3 for q in rows]
        line = "  after da2 stored: CTAs starting later %s (median %d); to the end of cnn_bwd_all %.2f us" % (
            max(late), statistics.median(late), statistics.median(to_bwd))
        if "chan:conv" in rows[0]:
            line += ", to the end of the conv-key exchange %.2f us" % statistics.median((q["chan:conv"][1] - q["mlp_chain"][1]) / 1e3 for q in rows)
        lines.append(line)
    for name, labels in cnn_labels.items():
        lines.append("  %s phases of CTA 0 (us): %s" % (name, "  ".join("%s %.2f" % (lab, statistics.median(r["_cnn_ph"][name][i] for r in rows))
                                                                      for i, lab in enumerate(labels))))
    lines.append("  %s phases of CTA 0 (us): %s" % ("dense_tail" if tail else "mlp_chain", "  ".join(
        "%s %.2f" % (lab, statistics.median(r["_mlp_ph"][i] for r in rows)) for i, lab in enumerate(mlp_labels))))
    if "_dense_vs_conv" in rows[0]:
        d = statistics.median(r["_dense_vs_conv"] for r in rows)
        lines.append("  dense branch (weight gradients + dense channel) ends %.2f us %s the end of the conv-key exchange" % (abs(d), "after" if d > 0 else "before"))
    if "_tail" in rows[0]:
        lines.append("  bwd tail (us since first tail ticket): ticket|grid done|sent|received|end %s" % ["%.2f" % statistics.median(r["_tail"][i] for r in rows) for i in range(5)])
    for k in rows[0]["_ph"]:
        lines.append("  chan:%s phases since its start (us): %s" % (k, ["%.2f" % statistics.median(r["_ph"][k][i] for r in rows) for i in range(6)]))
    for r in range(world):
        if r == rank:
            print("\n".join(lines), flush=True)
        if world > 1:
            dist.barrier()
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
