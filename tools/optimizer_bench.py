"""Cost of the optimizer in the training step: the demo CNN's graph-captured step (``HipsCNNTrainStep``, one GPU) timed with Adam and with
each of the other optimizers the update kernels run (NAG, Signum, RMSProp, AdaGrad, AdaDelta, Ftrl).  The update runs inside the exchange
kernels, which pick the rule at run time, so the difference to Adam is that rule's arithmetic plus whatever the weights it produces change in
the data-dependent parts of the step (the direct convolutions skip all-zero work).

Same method as ``tools/lr_schedule_bench.py``: a device-resident batch of B = 32, one CUDA-event pair per step, a 256 MiB buffer written
between timed steps to flush the L2, the engines in one process alternating in rounds.  Prints the card, its power limit and one JSON line:
the median and the 10th / 90th percentiles of each engine's step time in milliseconds.

    python tools/optimizer_bench.py --steps 200 --rounds 3
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from lr_schedule_bench import card  # noqa: E402


def optimizers(mx):
    O = mx.optimizer
    return {
        "adam": O.Adam(learning_rate=0.01),
        "nag": O.NAG(learning_rate=0.01, momentum=0.9),
        "signum": O.Signum(learning_rate=0.001, momentum=0.9),
        "rmsprop": O.RMSProp(learning_rate=0.001),
        "adagrad": O.AdaGrad(learning_rate=0.01),
        "adadelta": O.AdaDelta(),
        "ftrl": O.Ftrl(learning_rate=0.01, lamda1=1e-5, beta=1e-6),
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200, help="timed steps per engine and round")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--batch-size", type=int, default=32)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("optimizer_bench needs a CUDA device")
    import geomx_b200 as mx
    from geomx_b200.parallel import Topology

    B = args.batch_size
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    torch.manual_seed(1234)
    g = torch.Generator().manual_seed(100)
    X = torch.rand(B, 1, 28, 28, generator=g).pin_memory()
    y = torch.randint(0, 10, (B,), generator=g).float().pin_memory()
    engines = {k: mx.models.HipsCNNTrainStep(batch_size=B, optimizer=o, topo=Topology(1, 0, 1, 1), device=dev)
               for k, o in optimizers(mx).items()}
    for eng in engines.values():
        for _ in range(args.warmup):
            eng.step(X, y)                # also captures the graph
        eng.x.copy_(X.to(dev)); eng.label.copy_(y.to(dev))
    torch.cuda.synchronize()
    flush = torch.empty(256 * 1024 * 1024 // 4, dtype=torch.float32, device=dev)
    times = {k: [] for k in engines}
    for r in range(args.rounds):
        for name in (list(engines) if r % 2 == 0 else list(engines)[::-1]):
            eng = engines[name]
            ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(args.steps)]
            for i, (s, e) in enumerate(ev):
                flush.fill_(float(i))
                s.record()
                eng.run_device()
                e.record()
            torch.cuda.synchronize()
            times[name] += [s.elapsed_time(e) for s, e in ev]
    name, power = card()
    print("card: %s, power limit %s" % (name, power))
    out = {"card": name, "power_limit": power, "batch": B, "steps_per_engine": args.rounds * args.steps, "l2": "256 MiB flush between steps"}
    for k, ts in times.items():
        ts = sorted(ts)
        q = lambda p: ts[min(len(ts) - 1, int(p * len(ts)))]
        out[k] = {"median_ms": q(0.5), "p10_ms": q(0.1), "p90_ms": q(0.9), "kernels_per_step": engines[k].kernels_per_step,
                  "over_adam": q(0.5) / sorted(times["adam"])[len(times["adam"]) // 2]}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
