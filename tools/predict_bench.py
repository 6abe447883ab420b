"""Time the C predict API serving a checkpoint on the GPU (dev_type 2) and on the host (dev_type 1).

    python tools/predict_bench.py [--min-time 1.0] [--models cnn,resnet18_v1] [--batches 1,32]

Models: the demo CNN (``models.build_cnn``, 1x28x28 inputs) and the model zoo's ``resnet18_v1`` (1000 classes, 3x224x224 inputs), Xavier
weights, exported to a temporary directory and served through ctypes on ``libgeomx_capi.so``.  Two more use operators outside the planned
predictor's set, so the host serves them on its general executor: ``encdec``, an encoder-decoder on 3x64x64 inputs (Convolution /
BatchNorm / Pooling, then UpSampling, Deconvolution with ``adj``, Concat, reflect Pad and InstanceNorm), and ``transformer``, a
token-mixing block on (16, 64) sequences (FullyConnected with ``flatten=False``, LayerNorm, SwapAxis, softmax, mean, broadcast ops,
slice_axis).  Both are written as nnvm symbol JSON with seeded random parameters and saved as a checkpoint.  Each figure is the mean wall time of
``GXPredForward`` followed by ``GXPredGetOutput`` (which ends in a stream synchronise on the device), measured with a host clock over at
least ``--min-time`` seconds and 3 calls, after one untimed call of every shape (the device handle's first call records its CUDA graph).
The input is set once before timing.  Prints one JSON line, with the GPU's name and power limit read in the same run.
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import tempfile
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402


def gpu_info():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                       text=True)
    line = r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else ""
    name, _, power = line.partition(",")
    return name.strip() or "unknown", power.strip() or "unknown"


def symbol_json(ops, heads):
    """nnvm-dialect symbol JSON: `ops` = [(op, name, attrs, inputs)], an input "n:j" is output j of node n; names no op defines are variables."""
    nodes, idx = [], {}

    def ref(i):
        name, _, j = i.partition(":")
        return [idx[name], int(j or 0), 0]
    for op, name, attrs, ins in ops:
        for i in ins:
            if i.partition(":")[0] not in idx:
                idx[i] = len(nodes)
                nodes.append({"op": "null", "name": i, "inputs": []})
        idx[name] = len(nodes)
        nodes.append({"op": op, "name": name, "attrs": {k: str(v) for k, v in attrs.items()}, "inputs": [ref(i) for i in ins]})
    return json.dumps({"nodes": nodes, "arg_nodes": [i for i, n in enumerate(nodes) if n["op"] == "null"], "heads": [ref(h) for h in heads]})


def encdec_model():
    """(ops, parameter shapes, per-sample input shape) of the encoder-decoder."""
    conv = lambda k, f, p: {"kernel": (k, k), "num_filter": f, "pad": (p, p)}
    bn = {"fix_gamma": False, "eps": 1e-3}
    pool = {"kernel": (2, 2), "stride": (2, 2), "pool_type": "max"}
    ops = [("Convolution", "c1", conv(3, 16, 1), ["data", "c1_weight", "c1_bias"]), ("BatchNorm", "bn1", bn, ["c1", "bn1_gamma", "bn1_beta", "bn1_mean", "bn1_var"]),
           ("relu", "r1", {}, ["bn1"]), ("Pooling", "p1", pool, ["r1"]),
           ("Convolution", "c2", conv(3, 32, 1), ["p1", "c2_weight", "c2_bias"]), ("BatchNorm", "bn2", bn, ["c2", "bn2_gamma", "bn2_beta", "bn2_mean", "bn2_var"]),
           ("relu", "r2", {}, ["bn2"]), ("Pooling", "p2", pool, ["r2"]),
           ("UpSampling", "up", {"scale": 2, "sample_type": "nearest", "num_args": 1}, ["p2"]),
           ("Deconvolution", "dc", {"kernel": (3, 3), "stride": (2, 2), "pad": (1, 1), "adj": (1, 1), "num_filter": 16, "no_bias": False},
            ["p2", "dc_weight", "dc_bias"]),
           ("Concat", "cat", {"dim": 1, "num_args": 3}, ["up", "dc", "p1"]),
           ("Pad", "pad", {"mode": "reflect", "pad_width": (0, 0, 0, 0, 1, 1, 1, 1)}, ["cat"]),
           ("Convolution", "c3", conv(3, 16, 0), ["pad", "c3_weight", "c3_bias"]), ("InstanceNorm", "in3", {"eps": 1e-3}, ["c3", "in3_gamma", "in3_beta"]),
           ("relu", "r3", {}, ["in3"]), ("Convolution", "c4", conv(1, 2, 0), ["r3", "c4_weight", "c4_bias"])]
    shapes = {"c1_weight": (16, 3, 3, 3), "c1_bias": (16,), "c2_weight": (32, 16, 3, 3), "c2_bias": (32,), "dc_weight": (32, 16, 3, 3), "dc_bias": (16,),
              "c3_weight": (16, 64, 3, 3), "c3_bias": (16,), "in3_gamma": (16,), "in3_beta": (16,), "c4_weight": (2, 16, 1, 1), "c4_bias": (2,)}
    for b, c in (("bn1", 16), ("bn2", 32)):
        shapes.update({b + "_gamma": (c,), b + "_beta": (c,), b + "_mean": (c,), b + "_var": (c,)})
    return ops, shapes, (3, 64, 64)


def transformer_model(T=16, D=64):
    """(ops, parameter shapes, per-sample input shape) of the token-mixing block on (T, D) sequences."""
    fc = lambda h: {"num_hidden": h, "flatten": False}
    ops = [("LayerNorm", "ln1", {"axis": -1}, ["data", "ln1_gamma", "ln1_beta"]), ("SwapAxis", "sw1", {"dim1": 1, "dim2": 2}, ["ln1"]),
           ("FullyConnected", "tok", fc(T), ["sw1", "tok_weight", "tok_bias"]), ("SwapAxis", "sw2", {"dim1": 1, "dim2": 2}, ["tok"]),
           ("softmax", "att", {"axis": 1}, ["sw2"]), ("broadcast_mul", "mix", {}, ["att", "ln1"]), ("elemwise_add", "res1", {}, ["data", "mix"]),
           ("LayerNorm", "ln2", {"axis": -1}, ["res1", "ln2_gamma", "ln2_beta"]), ("FullyConnected", "f1", fc(4 * D), ["ln2", "f1_weight", "f1_bias"]),
           ("relu", "a1", {}, ["f1"]), ("FullyConnected", "f2", fc(D), ["a1", "f2_weight", "f2_bias"]), ("elemwise_add", "res2", {}, ["res1", "f2"]),
           ("mean", "mu", {"axis": (1,), "keepdims": True}, ["res2"]), ("broadcast_sub", "cen", {}, ["res2", "mu"]),
           ("slice_axis", "first", {"axis": 1, "begin": 0, "end": 1}, ["cen"]), ("FullyConnected", "head", {"num_hidden": 10}, ["first", "head_weight", "head_bias"]),
           ("softmax", "prob", {"axis": -1}, ["head"])]
    shapes = {"ln1_gamma": (D,), "ln1_beta": (D,), "tok_weight": (T, T), "tok_bias": (T,), "ln2_gamma": (D,), "ln2_beta": (D,), "f1_weight": (4 * D, D),
              "f1_bias": (4 * D,), "f2_weight": (D, 4 * D), "f2_bias": (D,), "head_weight": (10, D), "head_bias": (10,)}
    return ops, shapes, (T, D)


SYMBOL_MODELS = {"encdec": encdec_model, "transformer": transformer_model}


def symbol_params(shapes, seed=0):
    """Seeded parameters: weights scaled by 1/sqrt(fan-in), positive variances and scales."""
    rng = np.random.RandomState(seed)
    out = {}
    for k, s in sorted(shapes.items()):
        if k.endswith(("_var", "_gamma")):
            out[k] = (rng.rand(*s) + 0.5).astype(np.float32)
        elif k.endswith("_weight"):
            out[k] = (rng.randn(*s) / np.sqrt(np.prod(s[1:]))).astype(np.float32)
        else:
            out[k] = (rng.randn(*s) * 0.1).astype(np.float32)
    return out


def export(model, tmp):
    import geomx_b200 as mx
    if model in SYMBOL_MODELS:
        ops, shapes, shape = SYMBOL_MODELS[model]()
        prefix = os.path.join(tmp, model)
        with open(prefix + "-symbol.json", "w") as f:
            f.write(symbol_json(ops, [ops[-1][1]]))
        mx.nd.save(prefix + "-0000.params", {"arg:" + k: mx.nd.array(v) for k, v in symbol_params(shapes).items()})
        return open(prefix + "-symbol.json").read(), open(prefix + "-0000.params", "rb").read(), shape
    from geomx_b200.gluon import nn
    from geomx_b200.gluon.model_zoo import vision
    if model == "cnn":
        net = nn.HybridSequential()                   # models.build_cnn's layers in a container that exports
        for layer in mx.models.build_cnn()._children.values():
            net.add(layer)
        shape = (1, 28, 28)
    else:
        net = vision.get_model(model, classes=1000)
        shape = (3, 224, 224)
    net.initialize(mx.init.Xavier())
    with mx.autograd.predict_mode():
        net(mx.nd.array(np.zeros((1,) + shape, np.float32)))
    prefix = os.path.join(tmp, model)
    net.export(prefix)
    return open(prefix + "-symbol.json").read(), open(prefix + "-0000.params", "rb").read(), shape


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--min-time", type=float, default=1.0)
    ap.add_argument("--models", default="cnn,resnet18_v1")
    ap.add_argument("--batches", default="1,32")
    a = ap.parse_args()
    lib = ctypes.CDLL(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "geomx_b200", "lib", "libgeomx_capi.so"))
    lib.GXRTGetLastError.restype = ctypes.c_char_p

    def ck(rc):
        if rc != 0:
            raise RuntimeError(lib.GXRTGetLastError().decode(errors="replace"))

    name, power = gpu_info()
    result = {"bench": "predict_capi", "gpu": name, "power_limit": power, "ms": {}}
    rng = np.random.RandomState(0)
    with tempfile.TemporaryDirectory() as tmp:
        for model in a.models.split(","):
            text, blob, shape = export(model, tmp)
            for batch in [int(b) for b in a.batches.split(",")]:
                dims = (batch,) + shape
                x = rng.rand(*dims).astype(np.float32)
                for dev_type, dev_name in ((2, "gpu"), (1, "host")):
                    h = ctypes.c_void_p()
                    ck(lib.GXPredCreate(text.encode(), blob, len(blob), dev_type, 0, 1, (ctypes.c_char_p * 1)(b"data"), (ctypes.c_uint32 * 2)(0, len(dims)),
                                        (ctypes.c_uint32 * len(dims))(*dims), ctypes.byref(h)))
                    pd, nd = ctypes.POINTER(ctypes.c_uint32)(), ctypes.c_uint32()
                    ck(lib.GXPredGetOutputShape(h, 0, ctypes.byref(pd), ctypes.byref(nd)))
                    out = np.empty([pd[i] for i in range(nd.value)], np.float32)
                    fp = ctypes.POINTER(ctypes.c_float)
                    ck(lib.GXPredSetInput(h, b"data", x.ctypes.data_as(fp), x.size))

                    def call():
                        ck(lib.GXPredForward(h))
                        ck(lib.GXPredGetOutput(h, 0, out.ctypes.data_as(fp), out.size))
                    call()                                  # warm-up of this shape
                    n, t0 = 0, time.perf_counter()
                    while n < 3 or time.perf_counter() - t0 < a.min_time:
                        call(); n += 1
                    ms = (time.perf_counter() - t0) / n * 1e3
                    result["ms"]["%s_b%d_%s" % (model, batch, dev_name)] = round(ms, 4)
                    ck(lib.GXPredFree(h))
    print(json.dumps(result))


if __name__ == "__main__":
    main()
