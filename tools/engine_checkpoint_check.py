"""Resume the training engine on another number of ranks (torchrun --nproc-per-node 2): ``2to1`` — both ranks train a two-rank engine and
save, rank 0 resumes on one rank; ``1to2`` — rank 0 trains a one-rank engine and saves, both ranks resume on two.  The resumed engine's
first update must be the fp64 reference's (tests/_optim_ref.py) from the saved state and the gradient sums that the resuming ranks pushed,
read from their gradient arenas (each checked against its own batch's fp32 autograd sums, so that an arena the exchange had reduced in
place would be caught).  ``lookahead`` — two look-ahead ranks
save with a primed batch each and two resume: every rank must prime its own batch again.  Prints ``CKPT_CHECK PASS``."""
import os
import sys

import torch
import torch.distributed as dist
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import geomx_b200 as mx  # noqa: E402
from geomx_b200.models.cnn import CNN_PARAM_NAMES  # noqa: E402
from geomx_b200.parallel import Topology  # noqa: E402

import _optim_ref as R  # noqa: E402

B = 32


def engine(world, rank, lookahead=False):
    topo = Topology(world, rank, 2 if world > 1 else 1, 0) if world > 1 else Topology(1, 0, 1, 1)
    return mx.models.HipsCNNTrainStep(batch_size=B, optimizer=mx.optimizer.Adam(learning_rate=0.01, wd=0.01), topo=topo, use_graph=False,
                                      fused_zero_grad=False, lookahead=lookahead)


def grad_sums(P, X, y):
    """The gradient sums over the batch (what a rank pushes) of the demo CNN at weights ``P``, fp32 autograd."""
    ps = [p.detach().clone().requires_grad_(True) for p in P]
    h = F.max_pool2d(torch.relu(F.conv2d(X, ps[0], ps[1])), 2)
    h = F.max_pool2d(torch.relu(F.conv2d(h, ps[2], ps[3])), 2).flatten(1)
    h = torch.relu(F.linear(h, ps[4], ps[5]))
    h = torch.relu(F.linear(h, ps[6], ps[7]))
    F.cross_entropy(F.linear(h, ps[8], ps[9]), y.long(), reduction="sum").backward()
    return [p.grad.detach() for p in ps]


def lookahead_check(rank, path):
    """Two look-ahead ranks, each with its own batches: after the resume each rank's primed batch is its own last one."""
    a = engine(2, rank, lookahead=True)
    for k in range(3):
        last = batch(100 * k + rank)
        a.step(*last)
    a.save_states(path)
    del a
    b = engine(2, rank, lookahead=True)
    b.load_states(path)
    ok = b._primed and torch.equal(b.x_cur, last[0]) and torch.equal(b.label_cur, last[1])
    print("[ckpt lookahead] rank %d primes its own batch again: %s" % (rank, ok), flush=True)
    loss = b.step(*batch(1000 + rank))
    return ok and loss == loss


def batch(seed):
    g = torch.Generator().manual_seed(seed)
    return torch.rand(B, 1, 28, 28, generator=g).cuda(), torch.randint(0, 10, (B,), generator=g).float().cuda()


def main():
    direction, path = sys.argv[1], sys.argv[2]
    rank = int(os.environ["RANK"])
    torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", rank)))
    dist.init_process_group("nccl")
    if direction == "lookahead":
        ok = lookahead_check(rank, path)
        flag = torch.tensor([int(ok)], device="cuda")
        dist.all_reduce(flag, op=dist.ReduceOp.MIN)
        if rank == 0:
            print("CKPT_CHECK %s" % ("PASS" if int(flag) else "FAIL"), flush=True)
        dist.destroy_process_group()
        sys.exit(0 if int(flag) else 1)
    save_world, load_world = (2, 1) if direction == "2to1" else (1, 2)
    if rank < save_world:
        a = engine(save_world, rank)
        for k in range(4):
            a.step(*batch(100 * k + rank))
        a.save_states(path)
        del a
    dist.barrier()
    ok = True
    if rank < load_world:
        b = engine(load_world, rank)
        b.load_states(path)
        torch.backends.cudnn.allow_tf32 = False
        torch.backends.cuda.matmul.allow_tf32 = False
        X, y = batch(1000 + rank)
        grads = grad_sums(b.P, X, y)          # from the loaded weights, before the step changes them
        b.step(X, y)
        torch.cuda.synchronize()
        # the step's own gradient sums stay in the arena (fused_zero_grad=False): they must be this rank's, not an aggregate
        e_own = max(float((g - G).norm() / (g.norm() + 1e-30)) for g, G in zip(grads, b.G))
        print("[ckpt %s] rank %d: arena gradient vs fp32 autograd %.1e" % (direction, rank, e_own), flush=True)
        ok = e_own < 1e-4
        grads = [G.detach().clone() for G in b.G]
        if load_world > 1:
            for g in grads:
                dist.all_reduce(g)                     # the pushed sums of every rank: what the server tier aggregates
        master = b.fabric.export_state()["w"]          # full master weights, whoever owns each tile
        if rank == 0:
            saved = {k: v.asnumpy() for k, v in mx.nd.load(path).items()}
            h = R.hyper(b.fabric.opt_spec)
            M, M0, ref = [], [], []
            for i, n in enumerate(CNN_PARAM_NAMES):
                sl = b.layout.slots[i]
                w = torch.from_numpy(saved["master:" + n]).double()
                s0, s1 = torch.from_numpy(saved["s0:" + n]).double(), torch.from_numpy(saved["s1:" + n]).double()
                R.update(h, w, grads[i].cpu().double() / B, s0, s1, int(saved["step:" + n].max()) + 1)
                ref.append(w)
                M0.append(torch.from_numpy(saved["master:" + n]))
                M.append(torch.from_numpy(master[sl.offset:sl.offset + sl.numel]).reshape(w.shape))
            e = R.displacement_err(M, M0, ref, stores=1)
            print("[ckpt %s] first update after the load: %.2e (tolerance %.0e)" % (direction, e, R.DISP_TOL), flush=True)
            ok = ok and e < R.DISP_TOL and not b.fabric.check_protocol_errors()
        del b
    flag = torch.tensor([int(ok)], device="cuda")
    dist.all_reduce(flag, op=dist.ReduceOp.MIN)
    dist.barrier()
    if rank == 0:
        print("CKPT_CHECK %s" % ("PASS" if int(flag) else "FAIL"), flush=True)
    dist.destroy_process_group()
    sys.exit(0 if int(flag) else 1)


if __name__ == "__main__":
    main()
