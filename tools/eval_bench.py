"""Time the scoring of a 10 000-image test set with the training engine's one-launch evaluation against the generic Gluon path.

    python tools/eval_bench.py [--n 10000] [--reps 20] [--warmup 3]

On a seeded image set (uniform noise in [0, 1), seeded labels) and the demo CNN re-homed onto a ``HipsCNNTrainStep`` (one rank):
  evaluate_N       ``eng.evaluate(X, y)`` of all N images: one cnn_eval_kernel launch, the fp64 / integer totals and their read-back
  evaluate_32      ``eng.evaluate`` of one batch of 32
  gluon_batches_32 what ``examples/common.py::accuracy`` does, over the whole set: ``net(X).argmax`` per batch of 32 plus one
                   ``asscalar()`` read-back of the hit count per batch
  gluon_N          ``net(X)`` of all N images at once (logits only, no argmax); where the generic path refuses a batch that large, the
                   error is reported instead and ``gluon_chunks_1000`` times ``net(X)`` over chunks of 1000 images
Inputs are CUDA tensors / NDArrays, so no host-to-device copy is timed.  Each figure is the mean over ``--reps`` calls between CUDA events,
after ``--warmup`` untimed calls.  Prints one JSON line, with the GPU's name and power limit read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402


def gpu_info():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                       text=True)
    line = r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else ""
    name, _, power = line.partition(",")
    return name.strip() or torch.cuda.get_device_name(0), power.strip() or "unknown"


def timed(fn, reps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / reps


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--n", type=int, default=10000, help="test-set size")
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("eval_bench: no CUDA device")
    import geomx_b200 as mx
    from geomx_b200.ops import native
    from geomx_b200.parallel import Topology
    native.require()
    torch.cuda.set_device(0)
    torch.manual_seed(0)
    net = mx.models.build_cnn()
    net.initialize(init=mx.init.Xavier(), ctx=mx.gpu(0))
    net(mx.nd.array(torch.zeros(1, 1, 28, 28), ctx=mx.gpu(0)))          # deferred shapes -> parameters, then re-homed onto the engine
    eng = mx.models.HipsCNNTrainStep(net=net, batch_size=32, optimizer=mx.optimizer.Adam(learning_rate=0.01), topo=Topology(1, 0, 1, 1))
    g = torch.Generator().manual_seed(1)
    N = args.n
    X = torch.rand(N, 1, 28, 28, generator=g).cuda()
    y = torch.randint(0, 10, (N,), generator=g).float().cuda()
    Xnd, ynd = mx.nd.array(X, ctx=mx.gpu(0)), mx.nd.array(y, ctx=mx.gpu(0))
    batches = [(Xnd[i:i + 32], ynd[i:i + 32]) for i in range(0, N - N % 32, 32)]

    def gluon_batches():
        hit = 0.0
        for xb, yb in batches:
            hit += float((net(xb).argmax(axis=1) == yb).sum().asscalar())
        return hit / (32 * len(batches))

    res = {"evaluate_N_ms": timed(lambda: eng.evaluate(X, y), args.reps, args.warmup),
           "evaluate_32_ms": timed(lambda: eng.evaluate(X[:32], y[:32]), args.reps, args.warmup),
           "gluon_batches_32_ms": timed(gluon_batches, max(1, args.reps // 4), 1)}
    try:
        res["gluon_N_ms"] = timed(lambda: net(Xnd), args.reps, args.warmup)
    except RuntimeError as e:
        res["gluon_N_ms"], res["gluon_N_error"] = None, str(e)
        res["gluon_chunks_1000_ms"] = timed(lambda: [net(Xnd[i:i + 1000]) for i in range(0, N, 1000)], args.reps, args.warmup)
    # the two paths score the same weights: their accuracies over the batched part of the set agree up to arg-max ties
    n_b = 32 * len(batches)
    launches = native.launch_count
    acc_engine = eng.evaluate(X[:n_b], y[:n_b])[1]
    launches = native.launch_count - launches
    acc_gluon = gluon_batches()
    name, power = gpu_info()
    out = {"metric": "cnn_eval", "n": N, "gpu": name, "power_limit": power, "reps": args.reps, "warmup": args.warmup,
           **{k: round(v, 4) if isinstance(v, float) else v for k, v in res.items()},
           "speedup_vs_gluon_batches": round(res["gluon_batches_32_ms"] / res["evaluate_N_ms"], 1),
           "speedup_vs_gluon_N": round((res["gluon_N_ms"] or res["gluon_chunks_1000_ms"]) / res["evaluate_N_ms"], 1),
           "accuracy_engine": acc_engine, "accuracy_gluon": acc_gluon, "native_launches_per_evaluate": launches}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
