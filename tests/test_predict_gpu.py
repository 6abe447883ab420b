"""The C predict API on the GPU (GXPredCreate* with dev_type 2: csrc/runtime/predict_device.h, kernels/predict_dev.cu), through ctypes on
libgeomx_capi.so: every planned operator against the host predictor (dev_type 1, the same bytes) and an fp64 reference, whole graphs
(the model zoo's families at small and full resolution, with attribute mutations the device output must miss), the CUDA-graph replay,
operator-at-a-time forward, partial outputs, reshape, threads, refusals and memory."""
import ctypes
import json
import os
import re
import shutil
import subprocess
import sys
import threading

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIBDIR = os.path.join(ROOT, "geomx_b200", "lib")
CAPI = os.path.join(LIBDIR, "libgeomx_capi.so")
u32, vp, cp = ctypes.c_uint32, ctypes.c_void_p, ctypes.c_char_p
_lib = None


def lib():
    global _lib
    if _lib is None:
        _lib = ctypes.CDLL(CAPI)
        _lib.GXRTGetLastError.restype = cp
    return _lib


def err():
    return lib().GXRTGetLastError().decode(errors="replace")


def ck(rc):
    assert rc == 0, err()


def save_params(params):
    """`.params` bytes of {name: array}, written by the Python front end's NDArray-list writer."""
    import tempfile
    import geomx_b200 as mx
    with tempfile.TemporaryDirectory() as d:
        f = os.path.join(d, "p.params")
        mx.nd.save(f, {"arg:" + k: mx.nd.array(np.ascontiguousarray(v, dtype=np.float32)) for k, v in params.items()})
        return open(f, "rb").read()


class Pred:
    def __init__(self, text, blob, shapes, dev_type, dev_id=0, output_keys=None, handle=None):
        if handle is not None:
            self.h = handle
            return
        keys = (cp * len(shapes))(*[k.encode() for k in shapes])
        indptr, data = [0], []
        for s in shapes.values():
            data += list(s); indptr.append(len(data))
        self.h = vp()
        args = (text.encode(), blob, len(blob), dev_type, dev_id, len(shapes), keys, (u32 * len(indptr))(*indptr), (u32 * max(len(data), 1))(*data))
        if output_keys:
            ck(lib().GXPredCreatePartialOut(*args, len(output_keys), (cp * len(output_keys))(*[k.encode() for k in output_keys]), ctypes.byref(self.h)))
        else:
            ck(lib().GXPredCreate(*args, ctypes.byref(self.h)))

    def set(self, **inputs):
        for k, v in inputs.items():
            v = np.ascontiguousarray(v, dtype=np.float32)
            ck(lib().GXPredSetInput(self.h, k.encode(), v.ctypes.data_as(ctypes.POINTER(ctypes.c_float)), v.size))

    def forward(self, **inputs):
        self.set(**inputs)
        ck(lib().GXPredForward(self.h))
        return self

    def num_outputs(self):
        n = u32(); ck(lib().GXPredGetNumOutputs(self.h, ctypes.byref(n))); return n.value

    def out(self, i=0):
        pdata, ndim = ctypes.POINTER(u32)(), u32()
        ck(lib().GXPredGetOutputShape(self.h, i, ctypes.byref(pdata), ctypes.byref(ndim)))
        shape = tuple(pdata[j] for j in range(ndim.value))
        o = np.empty(shape, np.float32)
        ck(lib().GXPredGetOutput(self.h, i, o.ctypes.data_as(ctypes.POINTER(ctypes.c_float)), o.size))
        return o

    def engine(self):
        e = ctypes.c_int(); ck(lib().GXPredGetEngine(self.h, ctypes.byref(e))); return e.value

    def plan(self):
        a, n = ctypes.c_uint64(), u32(); ck(lib().GXPredGetPlan(self.h, ctypes.byref(a), ctypes.byref(n))); return a.value, n.value

    def free(self):
        ck(lib().GXPredFree(self.h))


def graph(ops, heads=None):
    """nnvm-dialect JSON: `ops` = [(op, name, attrs, [input names])]; names that no op defines become variables."""
    nodes, idx = [], {}
    for op, name, attrs, ins in ops:
        for i in ins:
            if i not in idx:
                idx[i] = len(nodes); nodes.append({"op": "null", "name": i, "inputs": []})
        idx[name] = len(nodes)
        nodes.append({"op": op, "name": name, "attrs": {k: str(v) for k, v in attrs.items()}, "inputs": [[idx[i], 0, 0] for i in ins]})
    heads = heads or [ops[-1][1]]
    return json.dumps({"nodes": nodes, "arg_nodes": [i for i, n in enumerate(nodes) if n["op"] == "null"], "heads": [[idx[h], 0, 0] for h in heads]})


# ------------------------------------------------------------------------------------------------ fp64 references
def pool_ref(x, k, s, p, kind, full=False, count_pad=True, glob=False):
    """The host predictor's pooling in fp64: windows clipped to the padded plane, then to the input; an empty max window gives 0."""
    N, C, H, W = x.shape
    if glob:
        k, s, p = (H, W), (1, 1), (0, 0)
    def out(n, kk, ss, pp):
        span = n + 2 * pp - kk
        return ((span + ss - 1) // ss if full else span // ss) + 1
    OH, OW = out(H, k[0], s[0], p[0]), out(W, k[1], s[1], p[1])
    y = np.zeros((N, C, OH, OW))
    for oh in range(OH):
        for ow in range(OW):
            h0, w0 = oh * s[0] - p[0], ow * s[1] - p[1]
            h1, w1 = min(h0 + k[0], H + p[0]), min(w0 + k[1], W + p[1])
            hs, ws, he, we = max(h0, 0), max(w0, 0), min(h1, H), min(w1, W)
            win = x[:, :, hs:he, ws:we].astype(np.float64)
            if kind == "max":
                y[:, :, oh, ow] = win.max((2, 3)) if he > hs and we > ws else 0
            else:
                v = win.sum((2, 3))
                if kind == "avg":
                    v = v / max((h1 - h0) * (w1 - w0) if count_pad else (he - hs) * (we - ws), 1)
                y[:, :, oh, ow] = v
    return y


def softmax_ref(x, axis):
    x = x.astype(np.float64)
    e = np.exp(x - x.max(axis, keepdims=True))
    return e / e.sum(axis, keepdims=True)


def embedding_rows(idx, rows):
    """float -> int64 as the host's static_cast does on x86-64 (truncation; NaN / out of range -> INT64_MIN), clamped to the table."""
    out = []
    for v in idx.ravel():
        r = int(v) if np.isfinite(v) and -2.0 ** 63 <= v < 2.0 ** 63 else -(2 ** 63)
        out.append(min(max(r, 0), rows - 1))
    return np.array(out).reshape(idx.shape)


def ref_eval(text, params, inputs, shapes=None):
    """fp64 evaluation (torch, CPU) of the operators that the demo graphs and every network of the model zoo use, in both JSON dialects.
    A value is dropped after its last consumer, so full-resolution networks fit; `shapes`, if given, receives every node's output shape."""
    import torch
    import torch.nn.functional as F
    d = json.loads(text)
    nnvm = "arg_nodes" in d or "format" not in d
    val = []
    T = lambda a: torch.tensor(np.asarray(a, dtype=np.float64))
    src = lambda n: [e[0] if isinstance(e, list) else e for e in n.get("inputs", []) + n.get("aux", [])]
    h = d["heads"][0]
    h = h[0] if isinstance(h, list) else h
    last = {j: i for i, n in enumerate(d["nodes"]) for j in src(n)}
    for i, n in enumerate(d["nodes"]):
        op, a = n["op"], n.get("attrs", {})
        ins = [val[j] for j in src(n)]
        for j in src(n):
            if last[j] == i and j != h:
                val[j] = None
        if op == "_nd":
            op, a = a["fn"].split(".")[-1], a.get("kwargs", {})
        tup = lambda k, dv: tuple(json.loads(str(a[k]).replace("(", "[").replace(")", "]"))) if a.get(k) not in (None, "None") else dv
        if op == "null":
            v = inputs.get(n["name"], params.get(n["name"]))
            val.append(None if v is None else T(v))
        elif op == "Convolution":
            nb = str(a.get("no_bias", False)) in ("True", "true", "1")
            val.append(F.conv2d(ins[0], ins[1], None if nb else ins[2], tup("stride", (1, 1)), tup("pad", (0, 0)), tup("dilate", (1, 1)), int(a.get("num_group", 1))))
        elif op == "BatchNorm":
            x, g, b, m, v = ins
            if str(a.get("fix_gamma", nnvm)) in ("True", "true", "1"):
                g = torch.ones_like(g)
            sh = (1, -1) + (1,) * (x.dim() - 2)
            val.append((x - m.view(sh)) / torch.sqrt(v.view(sh) + float(a.get("eps", 1e-3))) * g.view(sh) + b.view(sh))
        elif op in ("Activation", "relu"):
            t = a.get("act_type", "relu") if op == "Activation" else "relu"
            val.append({"relu": torch.relu, "tanh": torch.tanh, "sigmoid": torch.sigmoid}[t](ins[0]))
        elif op == "Pooling":
            k = tup("kernel", None)
            s = tup("stride", None) or ((1, 1) if nnvm else k)
            val.append(T(pool_ref(ins[0].numpy(), k, s, tup("pad", (0, 0)), a.get("pool_type", "max"), a.get("pooling_convention", "valid") == "full",
                                  str(a.get("count_include_pad", True)) in ("True", "true", "1"), str(a.get("global_pool", False)) in ("True", "true", "1"))))
        elif op in ("Concat", "concat"):
            val.append(torch.cat(ins, int(a.get("dim", 1))))
        elif op == "clip":
            val.append(ins[0].clamp(float(a["a_min"]), float(a["a_max"])))
        elif op in ("_plus", "elemwise_add", "broadcast_add"):
            val.append(ins[0] + ins[1])
        elif op == "_mul_scalar":
            val.append(ins[0] * float(a["scalar"]))
        elif op in ("Flatten", "flatten"):
            val.append(ins[0].reshape(ins[0].shape[0], -1))
        elif op == "Dropout":
            val.append(ins[0])
        elif op == "FullyConnected":
            nb = str(a.get("no_bias", False)) in ("True", "true", "1")
            y = ins[0].reshape(ins[0].shape[0], -1) @ ins[1].T
            val.append(y if nb else y + ins[2])
        elif op == "SoftmaxOutput":
            val.append(torch.softmax(ins[0], 1))
        else:
            raise NotImplementedError(op)
        if shapes is not None and val[-1] is not None:
            shapes[n["name"]] = tuple(val[-1].shape)
    return val[h].numpy()


def close(got, ref, rel):
    scale = float(np.abs(ref).max()) or 1.0
    err_ = float(np.abs(got.astype(np.float64) - ref).max())
    assert err_ <= rel * scale, (err_, scale, err_ / scale)


# ------------------------------------------------------------------------------------------------ per-operator cases
def _cases():
    rng = np.random.RandomState(0)
    r = lambda *s: rng.randn(*s).astype(np.float32)
    C = {}

    def conv(name, xs, F, k, stride=(1, 1), pad=(0, 0), dil=(1, 1), groups=1, bias=True):
        import torch
        w = r(F, xs[1] // groups, *k) * 0.3
        b = r(F)
        x = r(*xs)
        attrs = {"kernel": k, "num_filter": F, "stride": stride, "pad": pad, "dilate": dil, "num_group": groups, "no_bias": not bias}
        params = {"w": w, "b": b} if bias else {"w": w}
        ref = torch.nn.functional.conv2d(torch.tensor(x, dtype=torch.float64), torch.tensor(w, dtype=torch.float64),
                                         torch.tensor(b, dtype=torch.float64) if bias else None, stride, pad, dil, groups).numpy()
        C[name] = (graph([("Convolution", "y", attrs, ["data", "w"] + (["b"] if bias else []))]), params, {"data": x}, ref)

    conv("conv_groups_dilate_pad", (3, 4, 11, 13), 6, (3, 3), stride=(2, 1), pad=(1, 2), dil=(2, 1), groups=2)      # K = 18: padded weight rows
    conv("conv_tma", (5, 4, 16, 16), 32, (3, 3), pad=(1, 1))                                                            # K = 36: whole-batch product
    conv("conv_7x7_stride2_nobias", (2, 3, 30, 30), 16, (7, 7), stride=(2, 2), pad=(3, 3), bias=False)
    conv("conv_depthwise", (2, 8, 9, 9), 8, (3, 3), pad=(1, 1), groups=8)
    conv("conv_1x1_aligned", (3, 8, 8, 8), 16, (1, 1))                                                                 # MN-major input planes
    conv("conv_1x1_odd_plane", (2, 6, 7, 9), 10, (1, 1), groups=2)                                                     # P = 63: CUDA-core product
    # 64 x 64 planes x 576 columns = 2.4M floats of column matrix per image: the 16M-float workspace holds 7 images, so the batch of 8 runs
    # as two im2col + product rounds, the second writing image 7
    assert (16 << 20) // (64 * 64 * 576) == 7
    conv("conv_two_chunks", (8, 64, 64, 64), 64, (3, 3), pad=(1, 1))

    for name, xs, h, flat, bias in [("fc_aligned", (6, 64), 10, True, True), ("fc_odd_k", (7, 3, 5), 9, True, True),
                                    ("fc_no_flatten_no_bias", (2, 3, 8), 5, False, False)]:
        x = r(*xs); K = int(np.prod(xs[1:])) if flat else xs[-1]
        w = r(h, K) * 0.3; b = r(h)
        ref = (x.reshape(xs[0], -1) if flat else x).astype(np.float64) @ w.T.astype(np.float64) + (b if bias else 0)
        params = {"w": w, "b": b} if bias else {"w": w}
        C[name] = (graph([("FullyConnected", "y", {"num_hidden": h, "flatten": flat, "no_bias": not bias}, ["data", "w"] + (["b"] if bias else []))]),
                   params, {"data": x}, ref)

    for name, xs, a, k, s, p in [("pool_max_pad", (2, 3, 9, 10), {"pool_type": "max"}, (3, 3), (2, 2), (1, 1)),
                                 ("pool_max_full", (2, 3, 10, 11), {"pool_type": "max", "pooling_convention": "full"}, (3, 3), (2, 2), (0, 0)),
                                 ("pool_avg_count_pad", (2, 3, 9, 10), {"pool_type": "avg", "count_include_pad": True}, (3, 3), (2, 2), (1, 1)),
                                 ("pool_avg_no_count_pad_full", (2, 3, 9, 10), {"pool_type": "avg", "count_include_pad": False, "pooling_convention": "full"},
                                  (3, 2), (2, 3), (1, 1)),
                                 ("pool_sum", (1, 4, 8, 8), {"pool_type": "sum"}, (2, 3), (2, 1), (0, 1)),
                                 ("pool_global_avg", (2, 5, 7, 6), {"pool_type": "avg", "global_pool": True}, (1, 1), (1, 1), (0, 0)),
                                 ("pool_global_max", (2, 5, 7, 6), {"pool_type": "max", "global_pool": True}, (1, 1), (1, 1), (0, 0))]:
        x = r(*xs)
        attrs = dict(a, kernel=k, stride=s, pad=p)
        ref = pool_ref(x, k, s, p, a["pool_type"], a.get("pooling_convention") == "full", a.get("count_include_pad", True), a.get("global_pool", False))
        C[name] = (graph([("Pooling", "y", attrs, ["data"])]), {}, {"data": x}, ref)

    x = r(4, 6, 5); xd = x.astype(np.float64)
    unary = {"relu": np.maximum(xd, 0), "sigmoid": 1 / (1 + np.exp(-xd)), "tanh": np.tanh(xd), "exp": np.exp(xd), "abs": np.abs(xd), "negative": -xd,
             "square": xd * xd, "softsign": xd / (1 + np.abs(xd)), "softrelu": np.where(xd > 20, xd, np.log1p(np.exp(xd)))}
    for k, ref in unary.items():
        C["unary_" + k] = (graph([(k, "y", {}, ["data"])]), {}, {"data": x}, ref)
    xp = np.abs(x) + 0.1
    C["unary_log"] = (graph([("log", "y", {}, ["data"])]), {}, {"data": xp}, np.log(xp.astype(np.float64)))
    C["unary_sqrt"] = (graph([("sqrt", "y", {}, ["data"])]), {}, {"data": xp}, np.sqrt(xp.astype(np.float64)))
    for t in ("relu", "sigmoid", "tanh", "softrelu", "softsign"):
        C["activation_" + t] = (graph([("Activation", "y", {"act_type": t}, ["data"])]), {}, {"data": x}, unary[t])
    C["leaky"] = (graph([("LeakyReLU", "y", {"act_type": "leaky", "slope": 0.1}, ["data"])]), {}, {"data": x}, np.where(xd > 0, xd, 0.1 * xd))
    C["elu"] = (graph([("LeakyReLU", "y", {"act_type": "elu", "slope": 0.7}, ["data"])]), {}, {"data": x}, np.where(xd > 0, xd, 0.7 * (np.exp(xd) - 1)))
    C["clip"] = (graph([("clip", "y", {"a_min": -0.5, "a_max": 0.8}, ["data"])]), {}, {"data": x}, np.clip(xd, -0.5, 0.8))
    C["logistic_output"] = (graph([("LogisticRegressionOutput", "y", {}, ["data", "label"])]), {}, {"data": x}, unary["sigmoid"])
    for op, f in [("_plus_scalar", lambda v: v + 1.5), ("_minus_scalar", lambda v: v - 1.5), ("_mul_scalar", lambda v: v * 1.5),
                  ("_div_scalar", lambda v: v / 1.5), ("_rminus_scalar", lambda v: 1.5 - v), ("_rdiv_scalar", lambda v: 1.5 / v)]:
        C["scalar" + op] = (graph([(op, "y", {"scalar": 1.5}, ["data"])]), {}, {"data": xp}, f(xp.astype(np.float64)))

    for name, xs, axis, fix in [("batchnorm_nchw", (3, 5, 4, 6), 1, False), ("batchnorm_fix_gamma_last_axis", (4, 7), -1, True)]:
        x = r(*xs); c = xs[axis]
        g, b, m, v = r(c), r(c), r(c), np.abs(r(c)) + 0.5
        sh = [1] * len(xs); sh[axis] = c
        gg = np.ones(c) if fix else g.astype(np.float64)
        ref = (x - m.reshape(sh)) / np.sqrt(v.reshape(sh).astype(np.float64) + 1e-4) * gg.reshape(sh) + b.reshape(sh)
        C[name] = (graph([("BatchNorm", "y", {"axis": axis, "eps": 1e-4, "fix_gamma": fix}, ["data", "g", "b", "m", "v"])]),
                   {"g": g, "b": b, "m": m, "v": v}, {"data": x}, ref)

    a, b, c = r(2, 3, 4, 5), r(2, 1, 4, 5), r(2, 2, 4, 5)
    C["concat_dim1"] = (graph([("Concat", "y", {"dim": 1, "num_args": 3}, ["a", "b", "c"])]), {}, {"a": a, "b": b, "c": c}, np.concatenate([a, b, c], 1))
    C["concat_dim0"] = (graph([("Concat", "y", {"dim": 0, "num_args": 2}, ["a", "c"])]), {}, {"a": a[:, :2], "c": c}, np.concatenate([a[:, :2], c], 0))

    x4 = r(2, 7, 3, 4) * 3
    C["softmax_last"] = (graph([("softmax", "y", {"axis": -1}, ["data"])]), {}, {"data": x4}, softmax_ref(x4, -1))
    C["log_softmax_axis1"] = (graph([("log_softmax", "y", {"axis": 1}, ["data"])]), {}, {"data": x4}, np.log(softmax_ref(x4, 1)))
    x2 = r(5, 1000) * 4
    C["softmax_output_wide"] = (graph([("SoftmaxOutput", "y", {}, ["data", "label"])]), {}, {"data": x2}, softmax_ref(x2, 1))
    C["softmax_output_preserve_shape"] = (graph([("SoftmaxOutput", "y", {"preserve_shape": True}, ["data", "label"])]), {}, {"data": x4}, softmax_ref(x4, -1))
    C["softmax_activation_channel"] = (graph([("SoftmaxActivation", "y", {"mode": "channel"}, ["data"])]), {}, {"data": x4}, softmax_ref(x4, 1))
    C["softmax_activation_instance"] = (graph([("SoftmaxActivation", "y", {}, ["data"])]), {}, {"data": x4},
                                        softmax_ref(x4.reshape(2, -1), 1).reshape(x4.shape))

    idx = np.array([[0, 3, 9, 10], [-1, -7.5, 2.9, 100], [1e30, -1e30, np.nan, 5.5]], np.float32)
    w = r(10, 6)
    C["embedding_out_of_range"] = (graph([("Embedding", "y", {"input_dim": 10, "output_dim": 6}, ["data", "w"])]), {"w": w}, {"data": idx},
                                   w[embedding_rows(idx, 10)].astype(np.float64))

    C["transpose_axes"] = (graph([("transpose", "y", {"axes": (0, 2, 3, 1)}, ["data"])]), {}, {"data": x4}, x4.transpose(0, 2, 3, 1))
    C["transpose_default"] = (graph([("transpose", "y", {}, ["data"])]), {}, {"data": x4[:, :, :2]}, x4[:, :, :2].transpose())

    ins = {"x%d" % i: r(3, 4, 5) for i in range(11)}                                  # more inputs than one launch sums
    C["add_n_11"] = (graph([("add_n", "y", {"num_args": 11}, list(ins))]), {}, ins, sum(v.astype(np.float64) for v in ins.values()))

    p, q = r(2, 1, 4), r(3, 1)
    qa = np.abs(q) + 0.5
    for op, f, qq in [("broadcast_add", np.add, q), ("broadcast_sub", np.subtract, q), ("broadcast_mul", np.multiply, q), ("broadcast_div", np.divide, qa),
                      ("broadcast_maximum", np.maximum, q), ("broadcast_minimum", np.minimum, q)]:
        C[op] = (graph([(op, "y", {}, ["p", "q"])]), {}, {"p": p, "q": qq}, f(p.astype(np.float64), qq.astype(np.float64)))
    s1, s2 = r(3, 4), r(3, 4)
    C["elemwise_sub_same_shape"] = (graph([("elemwise_sub", "y", {}, ["p", "q"])]), {}, {"p": s1, "q": s2}, s1.astype(np.float64) - s2)

    v = r(2, 3, 4)
    C["views_reshape_flatten_expand"] = (graph([("Reshape", "r", {"shape": (0, -1)}, ["data"]), ("expand_dims", "e", {"axis": 1}, ["r"]),
                                                ("Flatten", "f", {}, ["e"]), ("Dropout", "d", {"p": 0.5}, ["f"]), ("_mul_scalar", "y", {"scalar": 2.0}, ["d"])]),
                                         {}, {"data": v}, v.reshape(2, -1).astype(np.float64) * 2)
    return C


CASES = _cases()


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(CASES))
def test_operator_matches_host_and_fp64(name):
    text, params, inputs, ref = CASES[name]
    blob = save_params(params) if params else b""
    shapes = {k: v.shape for k, v in inputs.items()}
    dev = Pred(text, blob, shapes, 2)
    host = Pred(text, blob, shapes, 1)
    try:
        assert dev.engine() == 3 and host.engine() == 1
        got, want = dev.forward(**inputs).out(), host.forward(**inputs).out()
        assert got.shape == want.shape == ref.shape
        close(got, ref, 2e-5)
        close(got, want.astype(np.float64), 2e-5)
        close(want, ref, 2e-5)
    finally:
        dev.free(); host.free()


def _mixed(tmp_path):
    import geomx_b200 as mx
    from test_predict_api import _net, _params
    net, shapes = _net(), {"data": (4, 3, 14, 14)}
    args, aux, save = _params(net, shapes)
    params = {k.split(":", 1)[1]: v.asnumpy() for k, v in save.items()}
    f = str(tmp_path / "net.params")
    mx.nd.save(f, save)
    return net.tojson(), open(f, "rb").read(), params, args["data"].asnumpy()


def zoo_net(name, batch, size, seed=0):
    """Model-zoo network `name` with Xavier weights, random BatchNorm scales and shifts, and a seeded (batch, 3, size, size) input.
    Each BatchNorm's running statistics are those of its input on a calibration batch of 8 other images, so every layer sees activations
    of order one and the output depends on all of them: with arbitrary statistics a deep network's output hardly depends on its input
    (MobileNetV2's by 1e-11), and neither would a wrong layer show."""
    import geomx_b200 as mx
    from geomx_b200.gluon import nn
    from geomx_b200.gluon.model_zoo import vision
    rng = np.random.RandomState(seed)
    mx.random.seed(seed)
    net = vision.get_model(name, classes=7)
    net.initialize(mx.init.Xavier())
    x = rng.randn(batch, 3, size, size).astype(np.float32)
    with mx.autograd.predict_mode():
        net(mx.nd.array(x))
    for pname, p in net.collect_params().items():
        if pname.endswith(("gamma", "beta")):
            v = rng.rand(*p.shape).astype(np.float32)
            p.set_data(mx.nd.array(v + 0.5 if pname.endswith("gamma") else v - 0.5))
    bns = []
    net.apply(lambda b: bns.append(b) if isinstance(b, nn.BatchNorm) else None)
    for b in bns:
        b._momentum = 0.0                                          # the training forward stores the batch's statistics
    with mx.autograd.train_mode():
        net(mx.nd.array(rng.randn(8, 3, size, size).astype(np.float32)))
    for b in bns:
        b._momentum = 0.9
    return net, x


def fp32_tol(net, x, ref):
    """Tolerances (host, device), relative to max|fp64|, for an fp32 evaluation of a zoo network: 1e-4, or four times the error of the imperative fp32
    forward where the network's conditioning makes that larger (with calibrated statistics the 100-layer ResNets and Inception v3 reach
    1e-4 - 2.4e-4 in torch's own fp32 forward).  The device's products run at 3xTF32, whose split operands keep about 21 of fp32's 24
    bits, so its bound is eight times that (measured on an H100: 6 to 10 times the imperative error where that exceeds 2.5e-5)."""
    import geomx_b200 as mx
    with mx.autograd.predict_mode():
        e = rel_err(net(mx.nd.array(x)).asnumpy(), ref)
    return max(1e-4, 4 * e), max(1e-4, 32 * e)


def export_net(net, prefix, nnvm=False):
    """`net.export` in one dialect: (symbol JSON, .params bytes, {parameter name: array})."""
    import geomx_b200 as mx
    net.export(prefix, nnvm=nnvm)
    text = open(prefix + "-symbol.json").read()
    blob = open(prefix + "-0000.params", "rb").read()
    params = {k.split(":", 1)[1]: v.asnumpy() for k, v in mx.nd.load(prefix + "-0000.params").items()}
    return text, blob, params


def _resnet(tmp_path, batch=2, size=32):
    net, x = zoo_net("resnet18_v1", batch, size)
    return export_net(net, str(tmp_path / "rn")) + (x,)


def rel_err(got, ref):
    return float(np.abs(got.astype(np.float64) - ref).max()) / (float(np.abs(ref).max()) or 1.0)


def mutate(text, op, change):
    """`text` with `change(node, attributes)` applied to every node of operator `op`; an `_nd` node's attributes are its keyword arguments."""
    d = json.loads(text)
    for n in d["nodes"]:
        a = n.get("attrs", {})
        if n["op"] == "_nd" and a["fn"].split(".")[-1] == op:
            change(n, a["kwargs"])
        elif n["op"] == op:
            change(n, a)
    return json.dumps(d)


# the smallest input each model-zoo family accepts (32 where not listed); at 37 and 33 every ceil-mode pooling of SqueezeNet 1.0 and 1.1
# gives a larger plane than valid pooling would, and a valid pooling would still leave a plane
ZOO_SIZE = {"alexnet": 63, "inceptionv3": 75, "squeezenet1.0": 37, "squeezenet1.1": 33, "lenet": 28}
# one network per family, Inception v3 at its native 299
ZOO_SMALL = {n: 299 if n == "inceptionv3" else ZOO_SIZE.get(n, 32) for n in ("alexnet", "vgg11_bn", "resnet18_v2", "resnet50_v1", "resnet50_v2",
                                                                            "densenet121", "squeezenet1.0", "squeezenet1.1", "mobilenet1.0",
                                                                            "mobilenetv2_1.0", "inceptionv3")}
# plausible wrong results that the device output must not match: fp64 of the same graph with one attribute changed
ZOO_MUTATIONS = {
    "squeezenet1.0": ("pooling convention full -> valid", "Pooling",
                      lambda n, a: a.__setitem__("pooling_convention", "valid") if a.get("pooling_convention") == "full" else None),
    "inceptionv3": ("count_include_pad flipped", "Pooling",
                    lambda n, a: a.__setitem__("count_include_pad", str(a.get("count_include_pad", True)) not in ("True", "true", "1"))
                    if a.get("pool_type") == "avg" else None),
    "mobilenetv2_1.0": ("clip upper bound removed", "clip", lambda n, a: a.__setitem__("a_max", 1e30)),
    "densenet121": ("concat operands swapped", "concat", lambda n, a: n["inputs"].reverse()),
}


@pytest.mark.gpu
@pytest.mark.parametrize("model", ["mixed", "resnet18_v1"] + ["%s-b%d" % (n, b) for n in ZOO_SMALL for b in (1, 3)])
def test_whole_graph_matches_host_and_fp64(tmp_path, model):
    net = None
    if model == "mixed":
        text, blob, params, x = _mixed(tmp_path)
    else:
        name, batch = model.rsplit("-b", 1) if "-b" in model else (model, 2)
        net, x = zoo_net(name, int(batch), ZOO_SMALL.get(name, 32))
        text, blob, params = export_net(net, str(tmp_path / "zoo"))
    ref = ref_eval(text, params, {"data": x})
    if net is not None:
        tol, dtol = fp32_tol(net, x, ref)
    else:
        tol = dtol = 1e-4
    dev, host = Pred(text, blob, {"data": x.shape}, 2), Pred(text, blob, {"data": x.shape}, 1)
    got, want = dev.forward(data=x).out(), host.forward(data=x).out()
    print("%s %s: device %.2e (tolerance %.1e), host %.2e (tolerance %.1e) of max|fp64|" % (model, x.shape, rel_err(got, ref), dtol, rel_err(want, ref), tol))
    close(got, ref, dtol); close(got, want.astype(np.float64), dtol); close(want, ref, tol)
    assert dev.plan() == host.plan()                               # the same plan, the same arena
    dev.free(); host.free()
    what, op, change = ZOO_MUTATIONS.get(model.rsplit("-b", 1)[0], (None, None, None))
    if what:
        e = rel_err(got, ref_eval(mutate(text, op, change), params, {"data": x}))
        print("%s, %s: device %.2e of max|mutant|" % (model, what, e))
        assert e > dtol


def _two_round_convs(text, shapes, batch):
    """Names of the convolutions that run in more than one im2col round: the handle's workspace is the largest that any of its
    convolutions asks gx_pred_conv_workspace for, and a layer takes as many images per round as fit in it."""
    k = ctypes.CDLL(os.path.join(LIBDIR, "libgeomx_kernels.so"))
    k.gx_pred_conv_workspace.restype = ctypes.c_longlong
    d = json.loads(text)
    convs = []
    for n in d["nodes"]:
        if n["op"] == "Convolution":
            a = n["attrs"]
            e = n["inputs"][0]
            (C, H, W), (F, OH, OW) = shapes[d["nodes"][e[0] if isinstance(e, list) else e]["name"]][1:], shapes[n["name"]][1:]
            g, (kh, kw) = int(a.get("num_group", 1)), tuple(a["kernel"])
            pointwise = (kh, kw) == (1, 1) and (H, W) == (OH, OW) and tuple(a.get("pad", (0, 0))) == (0, 0)
            convs.append((n["name"], C, OH, OW, kh, kw, g, pointwise))
    ws = max(k.gx_pred_conv_workspace(batch, C, OH, OW, kh, kw, g, int(pw)) for _, C, OH, OW, kh, kw, g, pw in convs)
    return {name for name, C, OH, OW, kh, kw, g, pw in convs if not pw and ws // (OH * OW * ((C // g * kh * kw + 3) // 4 * 4)) < batch}


# full-resolution networks, device against fp64 (the host predictor takes seconds per image here, so it runs only where it is cheap):
# the two-round stem and 56x56 layers of ResNet-50 at batch 10, depthwise layers with up to 1024 groups, big-K FC layers at M = 1,
# DenseNet's growing concats, SqueezeNet's ceil-mode pooling and Inception's factorised kernels
ZOO_FULL = [("resnet50_v1", 10, 224, False), ("mobilenet1.0", 2, 224, False), ("mobilenetv2_1.0", 2, 224, False), ("vgg16", 1, 224, False),
            ("alexnet", 1, 224, True), ("densenet121", 2, 224, False), ("squeezenet1.0", 2, 224, True), ("inceptionv3", 2, 299, False)]


@pytest.mark.gpu
@pytest.mark.parametrize("name,batch,size,with_host", ZOO_FULL, ids=["%s-b%d-%d" % c[:3] for c in ZOO_FULL])
def test_zoo_full_resolution_matches_fp64(tmp_path, name, batch, size, with_host):
    net, x = zoo_net(name, batch, size)
    text, blob, params = export_net(net, str(tmp_path / "zoo"))
    shapes = {}
    ref = ref_eval(text, params, {"data": x}, shapes)
    tol, dtol = fp32_tol(net, x, ref)
    if name == "resnet50_v1":
        two = _two_round_convs(text, shapes, batch)
        stem = next(n["name"] for n in json.loads(text)["nodes"] if n["op"] == "Convolution")
        assert stem in two and sum(shapes[c][2:] == (56, 56) for c in two) == 3, two     # the stem and the three 56x56 3x3 layers
    dev = Pred(text, blob, {"data": x.shape}, 2)
    got = dev.forward(data=x).out()
    dev.free()
    msg = "%s %s: device %.2e of max|fp64| (tolerance %.1e)" % (name, x.shape, rel_err(got, ref), dtol)
    if with_host:
        host = Pred(text, blob, {"data": x.shape}, 1)
        want = host.forward(data=x).out()
        host.free()
        msg += ", host %.2e" % rel_err(want, ref)
        close(got, want.astype(np.float64), dtol); close(want, ref, tol)
    print(msg)
    close(got, ref, dtol)
    text2, blob2, _ = export_net(net, str(tmp_path / "zoo_nnvm"), nnvm=True)     # the reference's dialect: the same bytes
    dev2 = Pred(text2, blob2, {"data": x.shape}, 2)
    assert dev2.forward(data=x).out().tobytes() == got.tobytes()
    dev2.free()


@pytest.mark.gpu
def test_replay_partial_forward_partial_out_reshape(tmp_path):
    text, blob, params, x = _mixed(tmp_path)
    dev, host = Pred(text, blob, {"data": x.shape}, 2), Pred(text, blob, {"data": x.shape}, 1)
    a = dev.forward(data=x).out()
    b = dev.forward().out()                                         # graph replay, same input
    assert a.tobytes() == b.tobytes()
    x2 = np.random.RandomState(9).randn(*x.shape).astype(np.float32)
    c = dev.forward(data=x2).out()
    assert not np.array_equal(a, c)
    close(c, host.forward(data=x2).out().astype(np.float64), 1e-4)
    # one operator at a time gives Forward's bytes
    dev.set(data=x)
    _, nops = dev.plan()
    step, left = 0, ctypes.c_int(1)
    while left.value:
        ck(lib().GXPredPartialForward(dev.h, step, ctypes.byref(left)))
        step += 1
        assert left.value == nops - step
    assert step == nops and dev.out().tobytes() == a.tobytes()
    # internal outputs
    q, qh = Pred(text, blob, {"data": x.shape}, 2, output_keys=["pool1", "fc_output"]), Pred(text, blob, {"data": x.shape}, 1, output_keys=["pool1", "fc_output"])
    q.forward(data=x); qh.forward(data=x)
    assert q.num_outputs() == 2 and q.engine() == 3
    for i in range(2):
        close(q.out(i), qh.out(i).astype(np.float64), 1e-4)
    # reshape: a new handle with another batch over the same device parameters
    r = vp()
    keys = (cp * 1)(b"data")
    ck(lib().GXPredReshape(1, keys, (u32 * 2)(0, 4), (u32 * 4)(2, 3, 14, 14), dev.h, ctypes.byref(r)))
    rp = Pred(None, None, None, None, handle=r)
    assert rp.engine() == 3
    close(rp.forward(data=x[:2]).out(), a[:2].astype(np.float64), 1e-5)
    for p in (dev, host, q, qh, rp):
        p.free()


@pytest.mark.gpu
def test_multithread_handles(tmp_path):
    text, blob, params, x = _mixed(tmp_path)
    shape = (2, 3, 14, 14)
    hs = (vp * 4)()
    ck(lib().GXPredCreateMultiThread(text.encode(), blob, len(blob), 2, 0, 1, (cp * 1)(b"data"), (u32 * 2)(0, 4), (u32 * 4)(*shape), 4, hs))
    preds = [Pred(None, None, None, None, handle=vp(hs[i])) for i in range(4)]
    single = Pred(text, blob, {"data": shape}, 2)
    rng = np.random.RandomState(4)
    xs = [rng.randn(*shape).astype(np.float32) for _ in preds]
    want = [single.forward(data=v).out() for v in xs]
    outs, errors = [None] * 4, []

    def work(i):
        try:
            for _ in range(5):
                outs[i] = preds[i].forward(data=xs[i]).out()
        except AssertionError as e:
            errors.append(e)
    th = [threading.Thread(target=work, args=(i,)) for i in range(4)]
    [t.start() for t in th]; [t.join() for t in th]
    assert not errors, errors
    for o, w in zip(outs, want):
        assert o.tobytes() == w.tobytes()
    for p in preds + [single]:
        p.free()


@pytest.mark.gpu
def test_two_devices_in_one_process(tmp_path):
    """One process serving the mixed net on GPUs 0 and 1: each device's handle runs its own products (the GEMM's shared-memory attribute is
    per device), and the caller's current device is left alone."""
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    text, blob, params, x = _mixed(tmp_path)
    torch.cuda.set_device(0)
    host = Pred(text, blob, {"data": x.shape}, 1)
    want = host.forward(data=x).out().astype(np.float64)
    d0 = Pred(text, blob, {"data": x.shape}, 2, dev_id=0)
    close(d0.forward(data=x).out(), want, 1e-4)                   # device 0 runs a product first ...
    d1 = Pred(text, blob, {"data": x.shape}, 2, dev_id=1)
    close(d1.forward(data=x).out(), want, 1e-4)                   # ... then device 1 its own
    close(d0.forward(data=x).out(), want, 1e-4)
    assert torch.cuda.current_device() == 0
    for p in (host, d0, d1):
        p.free()


@pytest.mark.gpu
def test_refusals(tmp_path):
    import torch
    text, blob, params, x = _mixed(tmp_path)
    h = vp()
    keys, indptr, shp = (cp * 1)(b"data"), (u32 * 2)(0, 4), (u32 * 4)(*x.shape)
    other = json.dumps({"nodes": [{"op": "null", "name": "data", "inputs": []}, {"op": "relu", "name": "r", "inputs": [[0, 0, 0]]},
                                  {"op": "Correlation", "name": "c", "inputs": [[1, 0, 0], [1, 0, 0]]}], "arg_nodes": [0], "heads": [[2, 0, 0]]})
    assert lib().GXPredCreate(other.encode(), b"", 0, 2, 0, 1, keys, indptr, shp, ctypes.byref(h)) == -1
    assert "operator Correlation" in err() and "dev_type 1" in err() and "Python Executor" in err()
    n = torch.cuda.device_count()
    assert lib().GXPredCreate(text.encode(), blob, len(blob), 2, n, 1, keys, indptr, shp, ctypes.byref(h)) == -1
    assert "out of range" in err() and "Python Executor" in err()
    assert lib().GXPredCreate(text.encode(), b"", 0, 2, 0, 1, keys, indptr, shp, ctypes.byref(h)) == -1           # parameters missing
    assert "c1_weight" in err() and "Python Executor" in err()
    p = Pred(text, blob, {"data": x.shape}, 2)
    bad = np.zeros(7, np.float32)
    assert lib().GXPredSetInput(p.h, b"data", bad.ctypes.data_as(ctypes.POINTER(ctypes.c_float)), bad.size) == -1
    assert "expects %d values, got 7" % x.size in err()
    before = torch.cuda.current_device()
    p.forward(data=x).out()
    p.free()
    assert torch.cuda.current_device() == before


@pytest.mark.gpu
def test_create_free_cycles_release_device_memory(tmp_path):
    import torch
    text, blob, params, x = _resnet(tmp_path, batch=4)
    def cycle():
        p = Pred(text, blob, {"data": x.shape}, 2)
        p.forward(data=x).out()
        p.free()
    cycle()                                                          # first use: module loading, allocator pools
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    for _ in range(20):
        cycle()
    torch.cuda.synchronize()
    assert abs(torch.cuda.mem_get_info()[0] - free0) <= 8 << 20


@pytest.mark.gpu
def test_c_example_serves_a_checkpoint(tmp_path):
    cc = shutil.which("gcc") or shutil.which("cc")
    if cc is None:
        pytest.skip("no C compiler")
    text, blob, params, x = _resnet(tmp_path)
    exe = str(tmp_path / "predict_gpu")
    subprocess.run([cc, "-O2", "-Wall", "-Werror", "-std=c99", "-I", os.path.join(ROOT, "geomx_b200", "include"), os.path.join(ROOT, "examples", "c_api", "predict_gpu.c"),
                    "-L", LIBDIR, "-lgeomx_capi", "-Wl,-rpath," + LIBDIR, "-o", exe], check=True)
    x.tofile(str(tmp_path / "x.f32"))
    r = subprocess.run([exe, str(tmp_path / "rn-symbol.json"), str(tmp_path / "rn-0000.params"), str(tmp_path / "x.f32")] + [str(d) for d in x.shape],
                       capture_output=True, text=True, timeout=300, env={k: v for k, v in os.environ.items() if not k.startswith("PYTHON")})
    assert r.returncode == 0, r.stdout + r.stderr
    assert "engine 3" in r.stderr
    got = np.array([float(v) for v in r.stdout.split()])
    host = Pred(text, blob, {"data": x.shape}, 1)
    want = host.forward(data=x).out().ravel().astype(np.float64)
    host.free()
    close(got, want, 1e-4)


# ------------------------------------------------------------------------------------------------ no GPU needed
def test_predict_dev_compiles_without_spills(tmp_path):
    from geomx_b200 import build
    if not (os.path.exists(build.NVCC) or shutil.which(build.NVCC)):
        pytest.skip("nvcc not available")
    src = os.path.join(build.CSRC, "kernels", "predict_dev.cu")
    r = subprocess.run([build.NVCC] + build.NVCC_FLAGS + ["-Xptxas", "-v", "-c", src, "-o", str(tmp_path / "p.o")], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout[-4000:]
    blocks = r.stdout.split("Compiling entry function ")[1:]
    assert len(blocks) >= 12, r.stdout[-2000:]
    for b in blocks:
        assert re.search(r" 0 bytes spill stores, 0 bytes spill loads", b), b


_NO_GPU = r"""
import ctypes, json, sys
lib = ctypes.CDLL(sys.argv[1]); lib.GXRTGetLastError.restype = ctypes.c_char_p
g = json.dumps({"nodes": [{"op": "null", "name": "data", "inputs": []}, {"op": "relu", "name": "r", "inputs": [[0, 0, 0]]}], "arg_nodes": [0], "heads": [[1, 0, 0]]})
h = ctypes.c_void_p(); keys = (ctypes.c_char_p * 1)(b"data"); ip = (ctypes.c_uint32 * 2)(0, 2); sh = (ctypes.c_uint32 * 2)(2, 3)
rc = lib.GXPredCreate(g.encode(), b"", 0, 2, 0, 1, keys, ip, sh, ctypes.byref(h))
print(rc, lib.GXRTGetLastError().decode())
assert lib.GXPredCreate(g.encode(), b"", 0, 1, 0, 1, keys, ip, sh, ctypes.byref(h)) == 0
x = (ctypes.c_float * 6)(-1, 2, -3, 4, -5, 6); y = (ctypes.c_float * 6)()
assert lib.GXPredSetInput(h, b"data", x, 6) == 0 and lib.GXPredForward(h) == 0 and lib.GXPredGetOutput(h, 0, y, 6) == 0
print(list(y))
assert "torch" not in sys.modules and "numpy" not in sys.modules
"""


def test_device_request_without_a_gpu_is_refused():
    if not os.path.exists(CAPI):
        pytest.skip("libgeomx_capi.so not built")
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    r = subprocess.run([sys.executable, "-S", "-c", _NO_GPU, CAPI], capture_output=True, text=True, timeout=120, env=env)
    assert r.returncode == 0, r.stdout + r.stderr
    first, second = r.stdout.splitlines()[:2]
    rc, msg = first.split(" ", 1)
    assert rc == "-1" and "device" in msg and "dev_type 1" in msg and "Python Executor" in msg, msg
    assert second == "[0.0, 2.0, 0.0, 4.0, 0.0, 6.0]"
