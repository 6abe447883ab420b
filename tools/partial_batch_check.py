"""Two ranks pass batches of different sizes in the same step (torchrun --nproc-per-node 2): rank 0 a short, sample-weighted batch of
N0 rows, rank 1 a full one.  The exchange is unchanged, so the update must be the fp64 reference's on the sum of both ranks' contributions,
``sum_r sum_i c_ri grad_ri / B`` with ``c_ri = w_ri * B / n_r``.  SGD without momentum: the update is ``-lr`` times that sum.
Prints ``PARTIAL_BATCH_CHECK PASS``."""
import os
import sys

import torch
import torch.distributed as dist
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import geomx_b200 as mx  # noqa: E402
from geomx_b200.parallel import Topology  # noqa: E402

B, N0, LR = 32, 11, 0.1


def weighted_grad_sums(P, X, y, c):
    """fp64 autograd of sum_i c_i loss_i of the demo CNN at weights ``P``."""
    ps = [p.detach().double().requires_grad_(True) for p in P]
    h = F.max_pool2d(torch.relu(F.conv2d(X.double(), ps[0], ps[1])), 2)
    h = F.max_pool2d(torch.relu(F.conv2d(h, ps[2], ps[3])), 2).flatten(1)
    h = torch.relu(F.linear(h, ps[4], ps[5]))
    h = torch.relu(F.linear(h, ps[6], ps[7]))
    (F.cross_entropy(F.linear(h, ps[8], ps[9]), y.long(), reduction="none") * c).sum().backward()
    return [p.grad.detach() for p in ps]


def main():
    rank = int(os.environ["RANK"])
    torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", rank)))
    dist.init_process_group("nccl")
    eng = mx.models.HipsCNNTrainStep(batch_size=B, optimizer=mx.optimizer.SGD(learning_rate=LR), topo=Topology(2, rank, 2, 0),
                                     use_graph=False, fused_zero_grad=False)
    g = torch.Generator().manual_seed(7 + rank)
    n = N0 if rank == 0 else B
    X, y = torch.rand(n, 1, 28, 28, generator=g), torch.randint(0, 10, (n,), generator=g).float()
    w = torch.rand(n, generator=g) + 0.5 if rank == 0 else None
    P0 = [p.detach().clone() for p in eng.P]
    c = torch.zeros(B, dtype=torch.float64, device="cuda")
    c[:n] = (w.double().cuda() if w is not None else 1.0) * B / n
    Xp = torch.zeros(B, 1, 28, 28, device="cuda"); Xp[:n] = X.cuda()
    yp = torch.zeros(B, device="cuda"); yp[:n] = y.cuda()
    ref = weighted_grad_sums(P0, Xp, yp, c)
    for t in ref:
        dist.all_reduce(t)
    eng.step(X, y, w)
    torch.cuda.synchronize()
    errs = []
    for p, p0, gr in zip(eng.P, P0, ref):
        want = -LR * gr / B
        errs.append(float(((p.double() - p0.double()) - want).norm() / (want.norm() + 1e-300)))
    e = max(errs)
    print("[partial batch] rank %d (n = %d): worst displacement error %.2e" % (rank, n, e), flush=True)
    ok = e < 1e-4 and not eng.fabric.check_protocol_errors()
    flag = torch.tensor([int(ok)], device="cuda")
    dist.all_reduce(flag, op=dist.ReduceOp.MIN)
    dist.barrier()
    if rank == 0:
        print("PARTIAL_BATCH_CHECK %s" % ("PASS" if int(flag) else "FAIL"), flush=True)
    del eng
    dist.destroy_process_group()
    sys.exit(0 if int(flag) else 1)


if __name__ == "__main__":
    main()
