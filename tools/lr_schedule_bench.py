"""Cost of a learning-rate schedule in the training step: the demo CNN's graph-captured step (``HipsCNNTrainStep``, Adam, one GPU) timed
with a constant lr and with ``CosineScheduler`` plus a linear warm-up, which the update kernels evaluate from the device step count.
A third engine runs the same schedule with base, warm-up and final lr all equal: it pays for evaluating the schedule but trains exactly like
the constant engine.  The real cosine run changes the weights, and the step's time depends on them (the direct convolutions skip all-zero
work), so ``cosine_flat`` against ``constant`` is the cost of the schedule itself.

Same method as ``bench.py``: a device-resident batch of B = 32, one CUDA-event pair per step, a 256 MiB buffer written between timed steps to
flush the L2.  The two engines run in one process and alternate in rounds, so that both see the same clocks and neighbours.  Prints the
card, its power limit and one JSON line: the median and the 10th / 90th percentiles of each engine's step time in milliseconds.

    python tools/lr_schedule_bench.py --steps 200 --rounds 5
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    """Name and power limit of GPU 0 (nvidia-smi query; 'unknown' where it cannot be read)."""
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip()
        name, power = [s.strip() for s in out.split(",")]
        return name, power
    except Exception:
        return torch.cuda.get_device_name(0), "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200, help="timed steps per engine and round")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--batch-size", type=int, default=32)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("lr_schedule_bench needs a CUDA device")
    import geomx_b200 as mx
    from geomx_b200.parallel import Topology

    B = args.batch_size
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    torch.manual_seed(1234)
    g = torch.Generator().manual_seed(100)
    X = torch.rand(B, 1, 28, 28, generator=g).pin_memory()
    y = torch.randint(0, 10, (B,), generator=g).float().pin_memory()
    total = args.warmup + args.rounds * args.steps + 10
    opts = {
        "constant": mx.optimizer.Adam(learning_rate=0.01),
        "cosine": mx.optimizer.Adam(learning_rate=0.01, lr_scheduler=mx.lr_scheduler.CosineScheduler(
            max_update=2 * total, warmup_steps=total // 4, warmup_begin_lr=0.001, final_lr=1e-4)),
        # the same two branches of the device schedule (linear warm-up, then cosine) with base = begin = final lr: the rate is the constant
        # one, so the weights, and with them the data-dependent parts of the step, follow the constant run exactly
        "cosine_flat": mx.optimizer.Adam(learning_rate=0.01, lr_scheduler=mx.lr_scheduler.CosineScheduler(
            max_update=2 * total, warmup_steps=total // 4, warmup_begin_lr=0.01, final_lr=0.01)),
    }
    engines = {k: mx.models.HipsCNNTrainStep(batch_size=B, optimizer=o, topo=Topology(1, 0, 1, 1), device=dev) for k, o in opts.items()}
    for eng in engines.values():
        for _ in range(args.warmup):
            eng.step(X, y)                # also captures the graph
        eng.x.copy_(X.to(dev)); eng.label.copy_(y.to(dev))
    torch.cuda.synchronize()
    flush = torch.empty(256 * 1024 * 1024 // 4, dtype=torch.float32, device=dev)
    times = {k: [] for k in engines}
    kernels = {k: e.kernels_per_step for k, e in engines.items()}
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
        out[k] = {"median_ms": q(0.5), "p10_ms": q(0.1), "p90_ms": q(0.9), "kernels_per_step": kernels[k],
                  "learning_rate_next": engines[k].learning_rate}
    out["cosine_over_constant"] = out["cosine"]["median_ms"] / out["constant"]["median_ms"]
    out["cosine_flat_over_constant"] = out["cosine_flat"]["median_ms"] / out["constant"]["median_ms"]
    print(json.dumps(out))


if __name__ == "__main__":
    main()
