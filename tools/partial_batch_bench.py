"""Cost of short and sample-weighted batches in the training step: one engine (the demo CNN's graph-captured ``HipsCNNTrainStep``, Adam,
one GPU) fed through the public ``step_async`` from pinned host batches, timed end to end for three kinds of step that alternate in rounds:

  full       B rows, no weights: the step as it ran before weights existed
  weighted   B rows with ``sample_weight``: the weighted graphs, plus the coefficient vector built on the host and copied with the batch
  short      B / 2 rows: the same weighted graphs, padding rows cleared on the copy stream

Each round runs ``--steps`` steps of one kind and reads the loss of the last one (a host clock around work that ends in a device
synchronise), after ``--warmup`` untimed steps of that kind.  Prints the card, its power limit and one JSON line: the median, 10th and 90th
percentile of each kind's ms per step over the rounds.

    python tools/partial_batch_bench.py --steps 200 --rounds 5
"""
import argparse
import json
import os
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools.lr_schedule_bench import card  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200, help="timed steps per kind and round")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--batch-size", type=int, default=32)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("partial_batch_bench needs a CUDA device")
    import geomx_b200 as mx
    from geomx_b200.parallel import Topology

    B = args.batch_size
    torch.cuda.set_device(0)
    g = torch.Generator().manual_seed(1234)
    eng = mx.models.HipsCNNTrainStep(batch_size=B, optimizer=mx.optimizer.Adam(learning_rate=0.001), topo=Topology(1, 0, 1, 1))
    X = [torch.rand(B, 1, 28, 28, generator=g).pin_memory() for _ in range(2)]
    y = [torch.randint(0, 10, (B,), generator=g).float().pin_memory() for _ in range(2)]
    w = [(torch.rand(B, generator=g) + 0.5).pin_memory() for _ in range(2)]
    kinds = {
        "full": lambda i: eng.step_async(X[i % 2], y[i % 2]),
        "weighted": lambda i: eng.step_async(X[i % 2], y[i % 2], w[i % 2]),
        "short": lambda i: eng.step_async(X[i % 2][:B // 2], y[i % 2][:B // 2]),
    }
    times = {k: [] for k in kinds}
    for _ in range(args.rounds):
        for name, fn in kinds.items():
            for i in range(args.warmup):
                h = fn(i)
            h.item()
            t0 = time.perf_counter()
            for i in range(args.steps):
                h = fn(i)
            h.item()
            torch.cuda.synchronize()
            times[name].append((time.perf_counter() - t0) * 1e3 / args.steps)
    name, power = card()
    print("card: %s, power limit %s" % (name, power))

    def pct(v, q):
        v = sorted(v)
        return v[min(len(v) - 1, int(round(q * (len(v) - 1))))]
    print(json.dumps({"batch_size": B, "steps": args.steps, "rounds": args.rounds, "card": name, "power_limit": power,
                      "ms_per_step": {k: {"median": pct(v, 0.5), "p10": pct(v, 0.1), "p90": pct(v, 0.9)} for k, v in times.items()},
                      "kernels_per_step": eng.kernels_per_step}))


if __name__ == "__main__":
    main()
