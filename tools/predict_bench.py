"""Time the C predict API serving a checkpoint on the GPU (dev_type 2) and on the host (dev_type 1).

    python tools/predict_bench.py [--min-time 1.0] [--models cnn,resnet18_v1] [--batches 1,32]

Models: the demo CNN (``models.build_cnn``, 1x28x28 inputs) and the model zoo's ``resnet18_v1`` (1000 classes, 3x224x224 inputs), Xavier
weights, exported to a temporary directory and served through ctypes on ``libgeomx_capi.so``.  Each figure is the mean wall time of
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


def export(model, tmp):
    import geomx_b200 as mx
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
                    ck(lib.GXPredCreate(text.encode(), blob, len(blob), dev_type, 0, 1, (ctypes.c_char_p * 1)(b"data"), (ctypes.c_uint32 * 2)(0, 4),
                                        (ctypes.c_uint32 * 4)(*dims), ctypes.byref(h)))
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
