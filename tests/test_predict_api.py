"""C predict API (csrc/runtime/{predict.h,c_predict_api.cc}) through geomx_b200.predictor: the native interpreter against the Python Executor
on the same graph and parameters, both JSON dialects, partial outputs, reshape, per-thread clones, operator-at-a-time forward, NDList and
the error paths.  Reference surface: include/mxnet/c_predict_api.h."""
import ctypes
import json
import threading

import numpy as np
import pytest

import geomx_b200 as mx
from geomx_b200 import predictor
from geomx_b200.base import MXNetError

sym = mx.sym


def _net():
    data = sym.Variable("data")
    c1 = sym.Convolution(data, kernel=(3, 3), num_filter=8, pad=(1, 1), name="c1")
    b1 = sym.BatchNorm(c1, name="bn1")
    a1 = sym.Activation(b1, "relu", name="relu1")
    p1 = sym.Pooling(a1, kernel=(2, 2), pool_type="max", name="pool1")
    c2 = sym.Convolution(p1, kernel=(3, 3), num_filter=8, stride=(2, 2), num_group=2, no_bias=True, name="c2")
    c3 = sym.Convolution(p1, kernel=(1, 1), num_filter=4, name="c3")
    p3 = sym.Pooling(c3, kernel=(3, 3), pool_type="avg", stride=(2, 2), name="pool3")
    cat = sym.Concat(c2, p3, dim=1, name="cat")
    t = sym.Activation(cat, "tanh") + cat * 0.5
    fc = sym.FullyConnected(sym.Dropout(sym.Flatten(t), p=0.3), num_hidden=10, name="fc")
    return sym.SoftmaxOutput(fc, name="softmax")


def _params(net, shapes, seed=0):
    arg_shapes, _, aux_shapes = net.infer_shape(**shapes)
    rng = np.random.RandomState(seed)
    args, aux, save = {}, {}, {}
    for n, s in zip(net.list_arguments(), arg_shapes):
        args[n] = mx.nd.array(rng.randn(*s).astype(np.float32) * 0.3)
        if n not in shapes and not n.endswith("_label"):
            save["arg:" + n] = args[n]
    for n, s in zip(net.list_auxiliary_states(), aux_shapes):
        aux[n] = mx.nd.array(rng.rand(*s).astype(np.float32) + 0.5)
        save["aux:" + n] = aux[n]
    return args, aux, save


def _blob(save, tmp_path):
    f = str(tmp_path / "net.params")
    mx.nd.save(f, save)
    return open(f, "rb").read()


def _executor_out(net, args, aux):
    return net.bind(mx.cpu(), args, aux_states=aux, grad_req="null").forward(is_train=False)[0].asnumpy()


def test_native_predictor_matches_executor(tmp_path):
    net, shapes = _net(), {"data": (4, 3, 14, 14)}
    args, aux, save = _params(net, shapes)
    blob = _blob(save, tmp_path)
    ref = _executor_out(net, args, aux)
    p = predictor.Predictor(net, blob, shapes)
    x = args["data"].asnumpy()
    p.forward(data=x)
    assert p.num_outputs == 1 and p.get_output_shape(0) == (4, 10)
    np.testing.assert_allclose(p.get_output(0), ref, atol=2e-6)
    arena, nops = p.plan()
    live = 4 * sum(int(np.prod(s)) for s in net.get_internals().infer_shape(**shapes)[1])
    assert 0 < arena < live / 2, (arena, live)               # the planner reuses blocks: far less than one buffer per intermediate
    # one operator at a time gives the same answer
    p.forward(data=np.zeros_like(x))
    p._set = None
    lib = predictor._lib()
    xx = np.ascontiguousarray(x)
    assert lib.GXPredSetInput(p._h, b"data", xx.ctypes.data_as(ctypes.POINTER(ctypes.c_float)), xx.size) == 0
    step, left = 0, 1
    while left:
        left = p.partial_forward(step); step += 1
    assert step == nops
    np.testing.assert_allclose(p.get_output(0), ref, atol=2e-6)
    # reshape: other batch size, same parameters
    p.reshape({"data": (2, 3, 14, 14)})
    p.forward(data=x[:2])
    np.testing.assert_allclose(p.get_output(0), ref[:2], atol=2e-6)
    # internal outputs by name
    q = predictor.Predictor(net, blob, shapes, output_keys=["pool1", "fc_output"])
    q.forward(data=x)
    internals = net.get_internals()
    grp = sym.Group([internals["pool1_output"], internals["fc_output"]])
    ex = grp.bind(mx.cpu(), args, aux_states=aux, grad_req="null").forward(is_train=False)
    assert q.num_outputs == 2
    np.testing.assert_allclose(q.get_output(0), ex[0].asnumpy(), atol=2e-6)
    np.testing.assert_allclose(q.get_output(1), ex[1].asnumpy(), atol=1e-5)


def test_predictor_threads_share_parameters(tmp_path):
    net, shapes = _net(), {"data": (2, 3, 14, 14)}
    args, aux, save = _params(net, shapes, seed=3)
    blob = _blob(save, tmp_path)
    preds = predictor.create_multi_thread(net.tojson(), blob, shapes, 4)
    rng = np.random.RandomState(1)
    xs = [rng.randn(2, 3, 14, 14).astype(np.float32) for _ in preds]
    outs = [None] * len(preds)

    def work(i):
        for _ in range(5):
            preds[i].forward(data=xs[i])
        outs[i] = preds[i].get_output(0)
    th = [threading.Thread(target=work, args=(i,)) for i in range(len(preds))]
    [t.start() for t in th]; [t.join() for t in th]
    for i, x in enumerate(xs):
        a = dict(args); a["data"] = mx.nd.array(x)
        np.testing.assert_allclose(outs[i], _executor_out(net, a, aux), atol=2e-6)


def test_nnvm_dialect_roundtrip_and_native(tmp_path):
    net, shapes = _net(), {"data": (3, 3, 14, 14)}
    args, aux, save = _params(net, shapes, seed=5)
    blob = _blob(save, tmp_path)
    ref = _executor_out(net, args, aux)
    text = net.tojson(nnvm=True)
    d = json.loads(text)
    assert "arg_nodes" in d and all(isinstance(v, str) for n in d["nodes"] for v in n.get("attrs", {}).values())
    conv = next(n for n in d["nodes"] if n["name"] == "c2")
    assert conv["attrs"]["kernel"] == "(3, 3)" and conv["attrs"]["no_bias"] == "True" and conv["inputs"][0][1:] == [0, 0]
    back = sym.load_json(text)                              # python front end reads the reference dialect
    assert back.list_arguments() == net.list_arguments() and back.list_auxiliary_states() == net.list_auxiliary_states()
    np.testing.assert_allclose(_executor_out(back, args, aux), ref, atol=1e-6)
    p = predictor.Predictor(text, blob, shapes)             # and so does the native runtime
    p.forward(data=args["data"].asnumpy())
    np.testing.assert_allclose(p.get_output(0), ref, atol=2e-6)


def test_handwritten_reference_json_defaults(tmp_path):
    """A file as MXNet 0.x/1.x writes it: string attributes, defaults left out (Pooling stride 1, BatchNorm fix_gamma True / eps 1e-3),
    pre-1.0 "param" + "attr" keys, generic operators by registry name."""
    nodes = [
        {"op": "null", "name": "data", "inputs": []},
        {"op": "null", "name": "bn_gamma", "attr": {"__lr_mult__": "0.0"}, "inputs": []},
        {"op": "null", "name": "bn_beta", "inputs": []},
        {"op": "null", "name": "bn_moving_mean", "inputs": []},
        {"op": "null", "name": "bn_moving_var", "inputs": []},
        {"op": "BatchNorm", "name": "bn", "param": {}, "attr": {"ctx_group": "dev1"}, "inputs": [[0, 0, 0], [1, 0, 0], [2, 0, 0], [3, 0, 1], [4, 0, 1]]},
        {"op": "Pooling", "name": "pool", "param": {"kernel": "(2, 2)", "pool_type": "max"}, "inputs": [[5, 0, 0]]},
        {"op": "LeakyReLU", "name": "lrelu", "param": {"act_type": "leaky", "slope": "0.1"}, "inputs": [[6, 0, 0]]},
        {"op": "_mul_scalar", "name": "scale", "param": {"scalar": "2.0"}, "inputs": [[7, 0, 0]]},
        {"op": "elemwise_add", "name": "res", "inputs": [[8, 0, 0], [6, 0, 0]]},
        {"op": "transpose", "name": "tr", "param": {"axes": "(0, 2, 3, 1)"}, "inputs": [[9, 0, 0]]},
        {"op": "softmax", "name": "sm", "param": {"axis": "-1"}, "inputs": [[10, 0, 0]]},
    ]
    text = json.dumps({"nodes": nodes, "arg_nodes": [0, 1, 2, 3, 4], "heads": [[11, 0, 0]]})
    rng = np.random.RandomState(2)
    C = 5
    vals = {"bn_gamma": rng.rand(C) + 0.5, "bn_beta": rng.randn(C), "bn_moving_mean": rng.randn(C), "bn_moving_var": rng.rand(C) + 0.5}
    x = rng.randn(2, C, 6, 7).astype(np.float32)
    f = str(tmp_path / "hand.params")
    mx.nd.save(f, {("aux:" if "moving" in k else "arg:") + k: mx.nd.array(v.astype(np.float32)) for k, v in vals.items()})
    p = predictor.Predictor(text, open(f, "rb").read(), {"data": x.shape})
    p.forward(data=x)
    got = p.get_output(0)
    # numpy oracle with the reference's defaults
    bn = (x - vals["bn_moving_mean"][None, :, None, None]) / np.sqrt(vals["bn_moving_var"][None, :, None, None] + 1e-3) + vals["bn_beta"][None, :, None, None]
    pool = np.stack([bn[:, :, i:i + 2, :] for i in range(5)], 2).max(3)                      # stride 1
    pool = np.stack([pool[:, :, :, j:j + 2] for j in range(6)], 3).max(4)
    lre = np.where(pool > 0, pool, 0.1 * pool)
    t = (lre * 2.0 + pool).transpose(0, 2, 3, 1)
    e = np.exp(t - t.max(-1, keepdims=True)); want = e / e.sum(-1, keepdims=True)
    assert got.shape == (2, 5, 6, C)
    np.testing.assert_allclose(got, want, atol=2e-6)
    s = sym.load_json(text)                                  # the Python loader agrees
    assert s.list_auxiliary_states() == ["bn_moving_mean", "bn_moving_var"] and s.attr_dict()["bn"] == {"ctx_group": "dev1"}
    args = {"data": mx.nd.array(x), "bn_gamma": mx.nd.array(vals["bn_gamma"].astype(np.float32)), "bn_beta": mx.nd.array(vals["bn_beta"].astype(np.float32))}
    aux = {k: mx.nd.array(vals[k].astype(np.float32)) for k in ("bn_moving_mean", "bn_moving_var")}
    np.testing.assert_allclose(_executor_out(s, args, aux), want, atol=2e-6)


def test_ndlist_and_errors(tmp_path):
    f = str(tmp_path / "l.params")
    mx.nd.save(f, {"arg:w": mx.nd.array(np.arange(6, dtype=np.float32).reshape(2, 3)), "aux:h": mx.nd.array(np.ones(4, dtype=np.float16), dtype="float16")})
    d = predictor.load_ndarray_file(open(f, "rb").read())
    assert d["arg:w"].tolist() == [[0, 1, 2], [3, 4, 5]] and d["aux:h"].dtype == np.float32 and d["aux:h"].tolist() == [1, 1, 1, 1]
    with pytest.raises(MXNetError, match="NDArray list"):
        predictor.load_ndarray_file(b"\x00" * 40)
    net = sym.FullyConnected(sym.Variable("data"), num_hidden=3, name="fc")
    with pytest.raises(MXNetError, match="fc_weight"):
        predictor.Predictor(net, b"", {"data": (2, 4)})                        # parameter missing
    f2 = str(tmp_path / "w.params")
    mx.nd.save(f2, {"arg:fc_weight": mx.nd.zeros((3, 5)), "arg:fc_bias": mx.nd.zeros((3,))})
    with pytest.raises(MXNetError, match=r"fc_weight has shape \(3, 5\), expected \(3, 4\)"):
        predictor.Predictor(net, open(f2, "rb").read(), {"data": (2, 4)})
    p = predictor.Predictor(net, open(f2, "rb").read(), {"data": (2, 5)})
    with pytest.raises(MXNetError, match="expects 10 values"):
        p.forward(data=np.zeros((2, 4), np.float32))
    with pytest.raises(MXNetError, match="unknown input"):
        p.forward(other=np.zeros((2, 5), np.float32))
    with pytest.raises(MXNetError, match="not supported by the native predictor"):
        predictor.Predictor(json.dumps({"nodes": [{"op": "null", "name": "data", "inputs": []}, {"op": "Correlation", "name": "c", "inputs": [[0, 0, 0]]}],
                                        "arg_nodes": [0], "heads": [[1, 0, 0]]}), b"", {"data": (1, 2)})
    with pytest.raises(MXNetError, match="symbol JSON"):
        predictor.Predictor('{"nodes": [', b"", {"data": (1, 2)})
    with pytest.raises(MXNetError, match="earlier nodes"):
        predictor.Predictor(json.dumps({"nodes": [{"op": "relu", "name": "r", "inputs": [[0, 0, 0]]}], "arg_nodes": [], "heads": [[0, 0, 0]]}), b"", {})
    # raw ABI: device type 2 is refused with an explanation
    lib = predictor._lib()
    h = ctypes.c_void_p()
    keys = (ctypes.c_char_p * 1)(b"data"); indptr = (ctypes.c_uint32 * 2)(0, 2); shp = (ctypes.c_uint32 * 2)(2, 5)
    assert lib.GXPredCreate(net.tojson().encode(), b"", 0, 2, 0, 1, keys, indptr, shp, ctypes.byref(h)) == -1
    assert b"Python Executor" in lib.GXRTGetLastError()


def test_hybridblock_export_traces_a_graph(tmp_path):
    """HybridBlock.export of imperative nets: built-in layers through their symbolic rules, user blocks through hybrid_forward(F=mx.sym);
    the files load into SymbolBlock, Module-style checkpoints and the native predictor (gluon/block.py export :866-927)."""
    from geomx_b200 import gluon
    from geomx_b200.gluon import nn
    from geomx_b200.gluon.model_zoo import vision

    class Gate(gluon.HybridBlock):
        def __init__(self, **kw):
            super().__init__(**kw)
            with self.name_scope():
                self.fc = nn.Dense(6, flatten=True)
                self.scale = self.params.get("scale", shape=(6,), init=mx.init.Constant(0.5))

        def hybrid_forward(self, F, x, scale):
            h = F.tanh(self.fc(x))
            return F.broadcast_mul(h, F.reshape(scale, shape=(1, -1))) + h

    rng = np.random.RandomState(0)
    net = nn.HybridSequential()
    net.add(nn.Conv2D(4, 3, padding=1, activation="relu"), nn.BatchNorm(), nn.AvgPool2D(2), nn.Dropout(0.2), Gate(), nn.LeakyReLU(0.1), nn.Dense(3))
    net.initialize(mx.init.Xavier())
    x = mx.nd.array(rng.randn(3, 2, 8, 8).astype(np.float32))
    with mx.autograd.predict_mode():
        ref = net(x).asnumpy()
    prefix = str(tmp_path / "gate")
    graph = net.export(prefix, epoch=2)
    assert graph.list_arguments()[0] == "data" and len(graph.list_auxiliary_states()) == 2
    blob = open(prefix + "-0002.params", "rb").read()
    for nnvm in (False, True):
        if nnvm:
            net.export(prefix, epoch=2, nnvm=True)
        p = predictor.Predictor(open(prefix + "-symbol.json").read(), blob, {"data": x.shape})
        p.forward(data=x.asnumpy())
        np.testing.assert_allclose(p.get_output(0), ref, atol=2e-6)
        blk = gluon.SymbolBlock.imports(prefix + "-symbol.json", ["data"], prefix + "-0002.params")
        with mx.autograd.predict_mode():
            np.testing.assert_allclose(blk(x).asnumpy(), ref, atol=1e-6)
    s, arg_params, aux_params = mx.model.load_checkpoint(prefix, 2)
    assert set(arg_params) | {"data"} == set(s.list_arguments()) and set(aux_params) == set(s.list_auxiliary_states())
    # a residual network from the model zoo
    rn = vision.get_model("resnet18_v1", classes=5)
    rn.initialize()
    xi = mx.nd.array(rng.randn(2, 3, 32, 32).astype(np.float32))
    with mx.autograd.predict_mode():
        want = rn(xi).asnumpy()
    rn.export(str(tmp_path / "rn"))
    p = predictor.Predictor(open(str(tmp_path / "rn-symbol.json")).read(), open(str(tmp_path / "rn-0000.params"), "rb").read(), {"data": xi.shape})
    p.forward(data=xi.asnumpy())
    np.testing.assert_allclose(p.get_output(0), want, atol=1e-5)
    arena, nops = p.plan()
    assert arena < 1 << 20 and nops > 60

    class Opaque(gluon.HybridBlock):                       # computes on tensors directly: reported, not mis-exported
        def hybrid_forward(self, F, x):
            return mx.nd.NDArray(x._t * 2)
    with pytest.raises(MXNetError, match="no symbolic rule"):
        Opaque().export(str(tmp_path / "op"))


def _zoo_names():
    from geomx_b200.gluon.model_zoo import vision
    return sorted(vision._models)


@pytest.mark.parametrize("name", _zoo_names())
def test_model_zoo_exports_and_serves(tmp_path, name):
    """Every network of get_model's table at the smallest input its family accepts: it exports in both JSON dialects, and the host
    predictor's output matches the imperative forward and the fp64 evaluation of the exported graph, with the same bytes from both."""
    from test_predict_gpu import ZOO_SIZE, export_net, fp32_tol, ref_eval, rel_err, zoo_net
    net, x = zoo_net(name, 2, ZOO_SIZE.get(name, 32))
    with mx.autograd.predict_mode():
        want = net(mx.nd.array(x)).asnumpy()
    outs = []
    for nnvm in (False, True):
        text, blob, params = export_net(net, str(tmp_path / name), nnvm=nnvm)
        assert ("arg_nodes" in json.loads(text)) == nnvm
        p = predictor.Predictor(text, blob, {"data": x.shape})
        engine = ctypes.c_int()
        assert predictor._lib().GXPredGetEngine(p._h, ctypes.byref(engine)) == 0 and engine.value == 1     # the planned interpreter
        p.forward(data=x)
        outs.append(p.get_output(0))
        ref = ref_eval(text, params, {"data": x})
        tol = fp32_tol(net, x, ref)[0]
        assert rel_err(outs[-1], ref) <= tol, (nnvm, rel_err(outs[-1], ref))
    assert outs[0].shape == want.shape == (2, 7)
    assert rel_err(outs[0], want.astype(np.float64)) <= tol, rel_err(outs[0], want.astype(np.float64))
    assert outs[0].tobytes() == outs[1].tobytes()


def test_user_blocks_with_concurrent_branches_and_clip_export(tmp_path):
    """HybridConcurrent (an Identity branch beside a layer) and ReLU6 written as F.clip(x, 0, 6) / mx.sym.clip(x, 0, 6) export and serve."""
    from geomx_b200 import gluon
    from geomx_b200.gluon import nn
    from geomx_b200.gluon.contrib.nn import HybridConcurrent, Identity

    class ReLU6(gluon.HybridBlock):
        def hybrid_forward(self, F, x):
            return F.clip(x, 0, 6)

    net = nn.HybridSequential()
    cat = HybridConcurrent(axis=1)
    cat.add(Identity(), nn.Conv2D(3, 3, padding=1))
    net.add(nn.Conv2D(4, 1), cat, ReLU6(), nn.Dense(5))
    net.initialize(mx.init.Xavier())
    x = np.random.RandomState(0).randn(2, 2, 6, 6).astype(np.float32) * 8
    with mx.autograd.predict_mode():
        want = net(mx.nd.array(x)).asnumpy()
    for nnvm in (False, True):
        net.export(str(tmp_path / "blk"), nnvm=nnvm)
        text = open(str(tmp_path / "blk-symbol.json")).read()
        assert text.count('"concat"') == 1 and text.count('"clip"') == 1, text
        p = predictor.Predictor(text, open(str(tmp_path / "blk-0000.params"), "rb").read(), {"data": x.shape})
        p.forward(data=x)
        np.testing.assert_allclose(p.get_output(0), want, rtol=1e-5, atol=1e-5)
    # positional attributes bind to mx.nd.clip's parameter names, from mx.sym and from Symbol.clip
    data = sym.Variable("data")
    xs = np.linspace(-9, 9, 12, dtype=np.float32).reshape(3, 4)
    for s in (sym.clip(data, 0, 6), data.clip(0, 6), sym.clip(data, 0, a_max=6)):
        assert s.attrs["kwargs"] == {"a_min": 0, "a_max": 6}
        p = predictor.Predictor(s.tojson(nnvm=True), b"", {"data": xs.shape})
        p.forward(data=xs)
        np.testing.assert_array_equal(p.get_output(0), np.clip(xs, 0, 6))
    with pytest.raises(MXNetError, match="positional arguments must be Symbols"):
        sym.clip(data, 0, 6, 7)                                  # more values than clip has parameters
    with pytest.raises(MXNetError, match="positional arguments must be Symbols"):
        sym.clip(data, 0, a_min=1)                               # a_min twice
    with pytest.raises(MXNetError, match="positional arguments must be Symbols"):
        sym.concat(data, 1)                                      # concat's arrays are variadic
