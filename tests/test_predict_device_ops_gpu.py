"""The C predict API's device-only operator set (GXPredCreate* with dev_type 2 on graphs the host serves with its general executor): every
operator and attribute variant against the host general executor on the same bytes (dev_type 1, engine 2) and an fp64 reference, whole
graphs, CUDA-graph replay with new indices, operator-at-a-time forward, secondary and internal outputs, handles, refusals and memory."""
import ctypes
import os
import sys

import numpy as np
import pytest

from test_predict_gpu import Pred, ck, cp, err, lib, save_params, u32, vp

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
from predict_bench import SYMBOL_MODELS, symbol_json, symbol_params  # noqa: E402


def graph(ops, heads=None):
    return symbol_json(ops, heads or [ops[-1][1]])


def ulp_close(got, want, ulps):
    """|got - want| within `ulps` units in the last place of the fp32 host value (equal NaNs and infinities pass)."""
    g, w = got.astype(np.float32), want.astype(np.float32)
    same = (g == w) | (np.isnan(g) & np.isnan(w))
    tol = ulps * np.spacing(np.abs(w))
    ok = same | (np.abs(g.astype(np.float64) - w.astype(np.float64)) <= tol)
    assert ok.all(), (g[~ok][:5], w[~ok][:5])


def close(got, ref, rel):
    ref = np.asarray(ref, np.float64)
    scale = float(np.abs(ref).max()) or 1.0
    e = float(np.abs(got.astype(np.float64) - ref).max())
    assert e <= rel * scale, (e, scale, e / scale)


def both(text, params, inputs, output_keys=None):
    blob = save_params(params) if params else b""
    shapes = {k: v.shape for k, v in inputs.items()}
    dev = Pred(text, blob, shapes, 2, output_keys=output_keys)
    host = Pred(text, blob, shapes, 1, output_keys=output_keys)
    assert dev.engine() == 3 and host.engine() == 2
    return dev, host


def outputs(p, inputs):
    p.forward(**inputs)
    return [p.out(i) for i in range(p.num_outputs())]


# ------------------------------------------------------------------------------------------------ per-operator cases
DECONV_TWO_CHUNKS = {"x": (8, 8, 64, 64), "F": 64, "k": (3, 3)}

# name -> (ops, heads, params, inputs, fp64 references, tolerance): "exact" (bitwise equal to the host, equal to the reference), "ulp" (within
# 4 ulp of the host), "exact_ew" (elementwise, bitwise equal), "red" (1e-5 relative to fp64), "gemm" (1e-4)
def _cases():
    rng = np.random.RandomState(0)
    r = lambda *s: rng.randn(*s).astype(np.float32)
    C = {}

    def add(name, ops, inputs, refs, tol, params=None, heads=None):
        C[name] = (ops, heads, params or {}, inputs, [np.asarray(v, np.float64) for v in (refs if isinstance(refs, list) else [refs])], tol)

    def one(name, op, attrs, x, ref, tol, extra=None, params=None):
        ins = {"data": x}
        ins.update(extra or {})
        add(name, [(op, "y", attrs, list(ins) + list(params or {}))], ins, ref, tol, params)

    # ---- layout / index rules
    x = r(4, 7, 5)
    one("slice_axis_negative", "slice_axis", {"axis": 1, "begin": -5, "end": -1}, x, x[:, 2:6], "exact")
    one("slice_axis_end_none", "slice_axis", {"axis": 2, "begin": 1, "end": None}, x, x[:, :, 1:], "exact")
    one("slice_mixed_none", "slice", {"begin": (1, None, -3), "end": (None, 5, None)}, x, x[1:, :5, -3:], "exact")
    one("slice_prefix_axes", "slice", {"begin": (-3,), "end": (-1,)}, x, x[1:3], "exact")
    one("swapaxis", "SwapAxis", {"dim1": 0, "dim2": 2}, x, np.swapaxes(x, 0, 2), "exact")
    one("swapaxes_alias", "swapaxes", {"dim1": -1, "dim2": 1}, x, np.swapaxes(x, 2, 1), "exact")
    x2 = r(2, 3)
    one("tile_rank_up", "tile", {"reps": (2, 1, 3)}, x2, np.tile(x2, (2, 1, 3)), "exact")
    one("repeat", "repeat", {"repeats": 3, "axis": 1}, x, np.repeat(x, 3, 1), "exact")
    x4 = r(2, 3, 5, 6)
    pw = (0, 0, 0, 0, 1, 2, 2, 1)
    npw = [(0, 0), (0, 0), (1, 2), (2, 1)]
    one("pad_constant", "Pad", {"mode": "constant", "pad_width": pw, "constant_value": 1.5}, x4, np.pad(x4, npw, constant_values=1.5), "exact")
    one("pad_edge", "Pad", {"mode": "edge", "pad_width": pw}, x4, np.pad(x4, npw, mode="edge"), "exact")
    one("pad_reflect", "pad", {"mode": "reflect", "pad_width": pw}, x4, np.pad(x4, npw, mode="reflect"), "exact")
    one("reverse", "reverse", {"axis": (0, 2)}, x, x[::-1, :, ::-1], "exact")
    one("flip_alias", "flip", {"axis": (1,)}, x, x[:, ::-1], "exact")
    xb = r(1, 3, 1)
    one("broadcast_to", "broadcast_to", {"shape": (4, 0, 5)}, xb, np.broadcast_to(xb, (4, 3, 5)), "exact")
    one("broadcast_axis", "broadcast_axis", {"axis": (0, 2), "size": (4, 5)}, xb, np.broadcast_to(xb, (4, 3, 5)), "exact")
    one("upsampling_nearest", "UpSampling", {"scale": 3, "sample_type": "nearest", "num_args": 1}, x4, x4.repeat(3, 2).repeat(3, 3), "exact")
    xs = r(2, 6, 5)
    add("slice_channel", [("SliceChannel", "sp", {"num_outputs": 3, "axis": 1}, ["data"])], {"data": xs}, [xs[:, 0:2], xs[:, 2:4], xs[:, 4:6]], "exact",
        heads=["sp:0", "sp:1", "sp:2"])
    xq = r(2, 3, 4)
    add("split_squeeze_axis", [("split", "sp", {"num_outputs": 3, "axis": 1, "squeeze_axis": True}, ["data"])], {"data": xq},
        [xq[:, 0], xq[:, 1], xq[:, 2]], "exact", heads=["sp:0", "sp:1", "sp:2"])
    # rank 1 .. 8, odd extents
    x8 = r(3, 1, 2, 5, 1, 3, 2, 3)
    one("reverse_rank8", "reverse", {"axis": (0, 3, 7)}, x8, x8[::-1, :, :, ::-1, :, :, :, ::-1], "exact")
    x1 = r(11)
    one("slice_axis_rank1", "slice_axis", {"axis": 0, "begin": 2, "end": -3}, x1, x1[2:-3], "exact")
    x5 = r(2, 3, 1, 5, 3)
    one("tile_rank5", "tile", {"reps": (1, 2, 3, 1, 2)}, x5, np.tile(x5, (1, 2, 3, 1, 2)), "exact")
    x7 = r(3, 1, 2, 3, 1, 5, 2)
    one("pad_edge_rank7", "Pad", {"mode": "edge", "pad_width": (0, 0, 1, 0, 0, 2, 0, 0, 1, 1, 0, 0, 0, 1)}, x7,
        np.pad(x7, [(0, 0), (1, 0), (0, 2), (0, 0), (1, 1), (0, 0), (0, 1)], mode="edge"), "exact")

    # ---- data-dependent gathers (indices converted and clamped as the host does)
    idx = np.array([[0, 3, -1], [6.9, -7.5, 100]], np.float32)
    cl = lambda v, n: np.clip(np.trunc(v).astype(np.int64), 0, n - 1)
    one("take_axis1", "take", {"axis": 1}, x, np.take(x, cl(idx, 7), 1), "exact", {"indices": idx})
    one("take_default_axis", "take", {}, x, np.take(x, cl(idx, 4), 0), "exact", {"indices": idx})
    pidx = np.array([[0, 4.7, -2, 9, 1, 3, 2]] * 4, np.float32)
    one("pick_last_axis", "pick", {"axis": -1}, x, np.take_along_axis(x, cl(pidx, 5)[..., None], -1)[..., 0], "exact", {"index": pidx})
    pk = np.array([[1, 0, 6, 2, 3]] * 4, np.float32)
    one("pick_axis1_keepdims", "pick", {"axis": 1, "keepdims": True}, x, np.take_along_axis(x, cl(pk, 7)[:, None, :], 1), "exact", {"index": pk})
    oh = np.array([[0, 2.9, -1], [4, 7, 1]], np.float32)
    ohr = np.where(np.trunc(oh).astype(np.int64)[..., None] == np.arange(5), 2.0, -0.5)
    one("one_hot", "one_hot", {"depth": 5, "on_value": 2.0, "off_value": -0.5}, oh, ohr, "exact")
    cond = (rng.rand(3, 4) > 0.5).astype(np.float32) * r(3, 4)
    wx, wy = r(3, 4), r(3, 4)
    one("where", "where", {}, cond, np.where(cond != 0, wx, wy), "exact", {"on_true": wx, "on_false": wy})
    ties = np.array([[[1, 3, 3, 0], [2, 2, 1, 2], [5, 5, 5, 5]], [[-1, -4, -4, 0], [7, 0, 7, 0], [0, 0, 0, 0]]], np.float32)
    for ax in (1, 2):
        one("argmax_ties_axis%d" % ax, "argmax", {"axis": ax}, ties, ties.argmax(ax), "exact")
        one("argmin_ties_axis%d" % ax, "argmin", {"axis": ax, "keepdims": True}, ties, np.expand_dims(ties.argmin(ax), ax), "exact")

    # ---- views
    xv = r(3, 1, 4, 1)
    one("squeeze_all", "squeeze", {}, xv, xv.reshape(3, 4), "exact")
    one("squeeze_axis", "squeeze", {"axis": (3,)}, xv, xv.reshape(3, 1, 4), "exact")
    one("cast", "Cast", {"dtype": "float32"}, xv, xv, "exact")
    one("make_loss", "MakeLoss", {}, xv, xv, "exact")

    # ---- reductions
    xr = r(3, 4, 5, 6)
    d = xr.astype(np.float64)
    one("sum_axes_keepdims", "sum", {"axis": (0, 2), "keepdims": True}, xr, d.sum((0, 2), keepdims=True), "red")
    one("sum_all", "sum", {}, xr, d.sum().reshape(1), "red")
    one("sum_axis_alias", "sum_axis", {"axis": 1}, xr, d.sum(1), "red")
    one("mean_nonadjacent", "mean", {"axis": (1, 3)}, xr, d.mean((1, 3)), "red")
    one("mean_empty_axes", "mean", {"axis": ()}, xr, d.mean().reshape(1), "red")
    one("max_axis", "max", {"axis": (1,)}, xr, d.max(1), "red")
    one("min_keepdims", "min_axis", {"axis": (-1,), "keepdims": True}, xr, d.min(-1, keepdims=True), "red")
    xp = (1 + 0.1 * r(3, 4, 5)).astype(np.float32)
    one("prod", "prod", {"axis": (2,)}, xp, xp.astype(np.float64).prod(2), "red")
    one("norm", "norm", {"axis": (0, 2)}, xr, np.sqrt((d * d).sum((0, 2))), "red")
    x8r = r(3, 2, 5, 1, 3, 2, 7, 3)
    one("sum_rank8_nonadjacent", "sum", {"axis": (0, 2, 5, 7)}, x8r, x8r.astype(np.float64).sum((0, 2, 5, 7)), "red")
    xl = r(3, 3001)
    one("max_rank2_long_row", "max", {"axis": (1,)}, xl, xl.max(1), "red")
    xm = rng.rand(1 << 20).astype(np.float32)                  # one output over 1M values: 256 partial sums of 4096
    one("sum_long_rank1", "sum", {}, xm, xm.astype(np.float64).sum(keepdims=True), "red")
    x6 = r(2, 3, 4, 1, 5, 3)
    one("prod_rank6", "prod", {"axis": (1, 4), "keepdims": True}, (1 + 0.1 * x6).astype(np.float32),
        (1 + 0.1 * x6).astype(np.float32).astype(np.float64).prod((1, 4), keepdims=True), "red")

    # ---- normalisations
    xn = (r(4, 6, 5, 7) * 2 + 1).astype(np.float32)
    dn = xn.astype(np.float64)
    for ax in (-1, 1):
        c = xn.shape[ax]
        g, b = r(c), r(c)
        sh = [1, 1, 1, 1]; sh[ax] = c
        mu, var = dn.mean(ax, keepdims=True), dn.var(ax, keepdims=True)
        one("layernorm_axis%d" % ax, "LayerNorm", {"axis": ax}, xn, (dn - mu) / np.sqrt(var + 1e-5) * g.reshape(sh) + b.reshape(sh), "red",
            params={"gamma": g, "beta": b})
    g, b = r(6), r(6)
    mu, var = dn.mean((2, 3), keepdims=True), dn.var((2, 3), keepdims=True)
    one("instancenorm", "InstanceNorm", {"eps": 1e-3}, xn, (dn - mu) / np.sqrt(var + 1e-3) * g.reshape(1, 6, 1, 1) + b.reshape(1, 6, 1, 1), "red",
        params={"gamma": g, "beta": b})
    for mode, axes in (("instance", (1, 2, 3)), ("channel", (1,)), ("spatial", (2, 3))):
        one("l2norm_" + mode, "L2Normalization", {"mode": mode}, xn, dn / np.sqrt((dn * dn).sum(axes, keepdims=True) + 1e-10), "red")
    for ns in (3, 5):
        sq = dn * dn
        win = np.stack([sq[:, max(c - ns // 2, 0):c + ns // 2 + 1].sum(1) for c in range(6)], 1)
        one("lrn_nsize%d" % ns, "LRN", {"nsize": ns, "alpha": 1e-2, "beta": 0.75, "knorm": 2}, xn, dn * (2 + 1e-2 / ns * win) ** -0.75, "red")

    # ---- elementwise
    xe = r(3, 4, 5)
    xu = (rng.rand(3, 4, 5) * 1.8 - 0.9).astype(np.float32)
    xpos = (rng.rand(3, 4, 5) * 5 + 0.05).astype(np.float32)
    de, du, dp = (v.astype(np.float64) for v in (xe, xu, xpos))
    from scipy.special import erf
    unary = {"sin": (xe, np.sin(de)), "cos": (xe, np.cos(de)), "tan": (xu, np.tan(du)), "arcsin": (xu, np.arcsin(du)), "arccos": (xu, np.arccos(du)),
             "arctan": (xe, np.arctan(de)), "sinh": (xe, np.sinh(de)), "cosh": (xe, np.cosh(de)), "log1p": (xpos, np.log1p(dp)), "expm1": (xe, np.expm1(de)),
             "log2": (xpos, np.log2(dp)), "log10": (xpos, np.log10(dp)), "rsqrt": (xpos, 1 / np.sqrt(dp)), "reciprocal": (xpos, 1 / dp),
             "cbrt": (xe, np.cbrt(de)), "erf": (xe, erf(de))}
    for op, (v, ref) in unary.items():
        one("unary_" + op, op, {}, v, ref, "ulp")
    xh = np.array([-2.5, -1.5, -0.5, 0.5, 1.5, 2.5, -0.0, 0.0, 3.7, -3.7, 1e-3, -2.2], np.float32)
    for op, f in (("floor", np.floor), ("ceil", np.ceil), ("round", lambda v: np.sign(v) * np.floor(np.abs(v) + 0.5)), ("sign", np.sign)):
        one("unary_" + op, op, {}, xh, f(xh.astype(np.float64)), "exact_ew")
    xs1 = r(7)
    one("unary_sin_rank1", "sin", {}, xs1, np.sin(xs1.astype(np.float64)), "ulp")
    p, q = (rng.rand(2, 1, 4) * 3 + 0.1).astype(np.float32), r(3, 1)
    one("broadcast_power", "broadcast_power", {}, p, p.astype(np.float64) ** q.astype(np.float64), "ulp", {"q": q})
    pi, qi = np.round(r(2, 3, 4)), np.round(r(3, 1))
    for op, f in (("broadcast_equal", np.equal), ("broadcast_not_equal", np.not_equal), ("broadcast_greater", np.greater),
                  ("broadcast_greater_equal", np.greater_equal), ("broadcast_lesser", np.less), ("_lesser_equal", np.less_equal)):
        one(op, op, {}, pi, f(pi, qi).astype(np.float64), "exact_ew", {"q": qi})
    one("power_scalar", "_power_scalar", {"scalar": 2.5}, xpos, dp ** 2.5, "ulp")
    one("rpower_scalar", "_rpower_scalar", {"scalar": 1.7}, xe, 1.7 ** de, "ulp")
    one("maximum_scalar", "_maximum_scalar", {"scalar": 0.3}, xe, np.maximum(de, np.float32(0.3)), "exact_ew")
    one("minimum_scalar", "_MinimumScalar", {"scalar": -0.2}, xe, np.minimum(de, np.float32(-0.2)), "exact_ew")
    s2 = np.float32(1.5) * np.float32(1.5)
    one("smooth_l1", "smooth_l1", {"scalar": 1.5}, xe, np.where(np.abs(de) < 1 / s2, 0.5 * s2 * de * de, np.abs(de) - 0.5 / s2), "ulp")
    logits, lab = r(6, 9) * 2, np.array([0, 8, 3, -2, 20, 4.6], np.float32)
    sm = np.exp(logits.astype(np.float64) - logits.max(1, keepdims=True))
    sm /= sm.sum(1, keepdims=True)
    one("softmax_cross_entropy", "softmax_cross_entropy", {}, logits, [-np.log(sm[np.arange(6), cl(lab, 9)]).sum(keepdims=True)], "red", {"label": lab})

    # ---- products
    import torch
    T = lambda a: torch.tensor(np.asarray(a, np.float64))

    def deconv(name, xs, F, k, stride=(1, 1), pad=(0, 0), adj=(0, 0), dil=(1, 1), groups=1, bias=False):
        xd, w = r(*xs), r(xs[1], F // groups, *k) * 0.3
        b = r(F)
        attrs = {"kernel": k, "num_filter": F, "stride": stride, "pad": pad, "adj": adj, "dilate": dil, "num_group": groups, "no_bias": not bias}
        ref = torch.nn.functional.conv_transpose2d(T(xd), T(w), T(b) if bias else None, stride, pad, adj, groups, dil).numpy()
        params = {"w": w, "b": b} if bias else {"w": w}
        add(name, [("Deconvolution", "y", attrs, ["data"] + list(params))], {"data": xd}, ref, "gemm", params)

    deconv("deconv_groups_adj_bias", (2, 4, 3, 4), 6, (3, 2), stride=(2, 2), pad=(1, 0), adj=(1, 0), groups=2, bias=True)
    deconv("deconv_dilated", (1, 2, 3, 3), 3, (2, 2), dil=(2, 1))
    deconv("deconv_stride3_pad_aligned", (3, 8, 8, 8), 16, (4, 4), stride=(3, 3), pad=(2, 1), adj=(2, 1), bias=True)
    deconv("deconv_depthwise", (2, 6, 5, 7), 6, (3, 3), stride=(2, 2), pad=(1, 1), groups=6)
    # DECONV_TWO_CHUNKS: a batch of 8 that the workspace takes in two rounds of products and col2im (test_deconv_two_chunks_case)
    deconv("deconv_two_chunks", DECONV_TWO_CHUNKS["x"], DECONV_TWO_CHUNKS["F"], DECONV_TWO_CHUNKS["k"], pad=(1, 1), bias=True)
    for ta in (False, True):
        for tb in (False, True):
            a_, b_ = r(*((9, 7) if ta else (7, 9))), r(*((5, 9) if tb else (9, 5)))
            ref = (a_.T if ta else a_).astype(np.float64) @ (b_.T if tb else b_).astype(np.float64)
            add("dot_ta%d_tb%d" % (ta, tb), [("dot", "y", {"transpose_a": ta, "transpose_b": tb}, ["a", "b"])], {"a": a_, "b": b_}, ref, "gemm")
    a_, b_ = r(64, 128), r(128, 96)
    add("dot_aligned", [("dot", "y", {}, ["a", "b"])], {"a": a_, "b": b_}, a_.astype(np.float64) @ b_, "gemm")
    return C


CASES = _cases()


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(CASES))
def test_operator_matches_general_executor_and_fp64(name):
    ops, heads, params, inputs, refs, tol = CASES[name]
    dev, host = both(graph(ops, heads), params, inputs)
    try:
        got, want = outputs(dev, inputs), outputs(host, inputs)
        assert len(got) == len(want) == len(refs)
        for g, w, ref in zip(got, want, refs):
            assert g.shape == w.shape == ref.shape, (g.shape, w.shape, ref.shape)
            if tol in ("exact", "exact_ew"):
                assert g.tobytes() == w.tobytes()
                assert np.array_equal(g.astype(np.float64), ref.astype(np.float32).astype(np.float64))
            elif tol == "ulp":
                ulp_close(g, w, 4)
                close(g, ref, 1e-5)
            else:
                rel = 1e-5 if tol == "red" else 1e-4
                close(g, ref, rel)
                close(w, ref, rel)
    finally:
        dev.free(); host.free()


# ------------------------------------------------------------------------------------------------ whole graphs
def _ref64(ops, heads, params, inputs):
    """fp64 evaluation (torch, CPU) of the operators the whole-graph tests use."""
    import torch
    import torch.nn.functional as F
    val = {k: torch.tensor(np.asarray(v, np.float64)) for k, v in list(params.items()) + list(inputs.items())}
    get = lambda i: val[i]
    tup = lambda v: tuple(v) if isinstance(v, (tuple, list)) else (v, v)
    for op, name, a, ins in ops:
        x = get(ins[0])
        if op == "Convolution":
            y = F.conv2d(x, get(ins[1]), get(ins[2]), 1, tup(a.get("pad", 0)))
        elif op == "BatchNorm":
            g, b, m, v = (get(i) for i in ins[1:])
            sh = (1, -1, 1, 1)
            y = (x - m.view(sh)) / torch.sqrt(v.view(sh) + a["eps"]) * g.view(sh) + b.view(sh)
        elif op == "relu":
            y = torch.relu(x)
        elif op == "sigmoid":
            y = torch.sigmoid(x)
        elif op == "Pooling":
            y = F.max_pool2d(x, a["kernel"], a["stride"])
        elif op == "UpSampling":
            y = x.repeat_interleave(a["scale"], 2).repeat_interleave(a["scale"], 3)
        elif op == "Deconvolution":
            y = F.conv_transpose2d(x, get(ins[1]), get(ins[2]) if len(ins) > 2 else None, a.get("stride", 1), a.get("pad", 0), a.get("adj", 0))
        elif op == "Concat":
            y = torch.cat([get(i) for i in ins], a["dim"])
        elif op == "Pad":
            p = a["pad_width"]
            y = F.pad(x, (p[6], p[7], p[4], p[5]), mode="reflect")
        elif op == "InstanceNorm":
            y = F.instance_norm(x, weight=get(ins[1]), bias=get(ins[2]), eps=a["eps"])
        elif op == "LayerNorm":
            ax = a.get("axis", -1)
            mu, var = x.mean(ax, keepdim=True), x.var(ax, unbiased=False, keepdim=True)
            c = x.shape[ax]
            sh = [1] * x.dim(); sh[ax] = c
            y = (x - mu) / torch.sqrt(var + 1e-5) * get(ins[1]).view(sh) + get(ins[2]).view(sh)
        elif op == "SwapAxis":
            y = x.transpose(a["dim1"], a["dim2"])
        elif op == "FullyConnected":
            xx = x if a.get("flatten", True) is False else x.reshape(x.shape[0], -1)
            y = xx @ get(ins[1]).T + get(ins[2])
        elif op == "softmax":
            y = torch.softmax(x, a.get("axis", -1))
        elif op in ("broadcast_mul", "elemwise_mul"):
            y = x * get(ins[1])
        elif op == "elemwise_add":
            y = x + get(ins[1])
        elif op == "broadcast_sub":
            y = x - get(ins[1])
        elif op == "mean":
            y = x.mean(a["axis"], keepdim=a.get("keepdims", False))
        elif op == "slice_axis":
            y = x.narrow(a["axis"], a["begin"], a["end"] - a["begin"])
        elif op == "Flatten":
            y = x.reshape(x.shape[0], -1)
        elif op == "SliceChannel":
            for j, part in enumerate(x.chunk(a["num_outputs"], a["axis"])):
                val["%s:%d" % (name, j)] = part
            continue
        else:
            raise NotImplementedError(op)
        val[name] = y
    return [val[h].numpy() for h in heads]


def _mixed(batch=2):
    """test_c_api_graph.py's general-executor graph: Deconvolution -> SliceChannel -> sigmoid . mul -> LayerNorm -> FullyConnected -> softmax."""
    ops = [("Deconvolution", "up", {"kernel": (2, 2), "stride": (2, 2), "num_filter": 4}, ["data", "up_weight"]),
           ("SliceChannel", "sp", {"num_outputs": 2, "axis": 1}, ["up"]), ("sigmoid", "s", {}, ["sp:0"]), ("broadcast_mul", "gate", {}, ["s", "sp:1"]),
           ("Flatten", "f", {}, ["gate"]), ("LayerNorm", "ln", {"axis": -1}, ["f", "ln_gamma", "ln_beta"]),
           ("FullyConnected", "fc", {"num_hidden": 3}, ["ln", "fc_weight", "fc_bias"]), ("softmax", "prob", {}, ["fc"])]
    rng = np.random.RandomState(11)
    shapes = {"up_weight": (3, 4, 2, 2), "ln_gamma": (128,), "ln_beta": (128,), "fc_weight": (3, 128), "fc_bias": (3,)}
    params = {k: (rng.randn(*s) * 0.5).astype(np.float32) for k, s in shapes.items()}
    return ops, params, rng.rand(batch, 3, 4, 4).astype(np.float32)


def _model(name, batch):
    ops, shapes, shape = SYMBOL_MODELS[name]()
    return ops, symbol_params(shapes), np.random.RandomState(batch).rand(batch, *shape).astype(np.float32)


@pytest.mark.gpu
@pytest.mark.parametrize("model,batch", [("mixed", 2), ("encdec", 1), ("encdec", 8), ("transformer", 1), ("transformer", 8)])
def test_whole_graph_matches_general_executor_and_fp64(model, batch):
    ops, params, x = _mixed(batch) if model == "mixed" else _model(model, batch)
    heads = [ops[-1][1]]
    dev, host = both(graph(ops, heads), params, {"data": x})
    got, want = outputs(dev, {"data": x})[0], outputs(host, {"data": x})[0]
    ref = _ref64(ops, heads, params, {"data": x})[0]
    close(got, ref, 1e-4); close(want, ref, 1e-4); close(got, want.astype(np.float64), 1e-4)
    dev.free(); host.free()


# ------------------------------------------------------------------------------------------------ replay, partial forward, partial outputs
@pytest.mark.gpu
def test_replay_partial_forward_and_partial_outputs():
    ops, params, x = _mixed(2)
    text = graph(ops)
    dev, host = both(text, params, {"data": x})
    a = dev.forward(data=x).out()
    assert a.tobytes() == dev.forward().out().tobytes()                # replay, same input: the same bits
    x2 = np.random.RandomState(9).rand(*x.shape).astype(np.float32)
    b = dev.forward(data=x2).out()
    assert not np.array_equal(a, b)
    close(b, host.forward(data=x2).out().astype(np.float64), 1e-4)
    # one operator at a time: as many steps as the plan has operators, ending in Forward's bytes
    dev.set(data=x)
    _, nops = dev.plan()
    step, left = 0, ctypes.c_int(1)
    while left.value:
        ck(lib().GXPredPartialForward(dev.h, step, ctypes.byref(left)))
        step += 1
        assert left.value == nops - step
    assert step == nops and dev.out().tobytes() == a.tobytes()
    # a secondary output and an internal node by name
    keys = ["sp_output1", "ln"]
    q, qh = both(text, params, {"data": x}, output_keys=keys)
    got, want = outputs(q, {"data": x}), outputs(qh, {"data": x})
    assert len(got) == 2 and got[0].shape == (2, 2, 8, 8)
    for g, w in zip(got, want):
        close(g, w.astype(np.float64), 1e-4)
    ref = _ref64(ops, ["sp:1", "ln"], params, {"data": x})
    close(got[0], ref[0], 1e-4); close(got[1], ref[1], 1e-4)
    for p in (dev, host, q, qh):
        p.free()


@pytest.mark.gpu
def test_replay_reads_new_indices():
    rng = np.random.RandomState(3)
    w, xp = rng.randn(10, 6).astype(np.float32), rng.randn(4, 5).astype(np.float32)
    ops = [("take", "t", {"axis": 0}, ["table", "idx"]), ("pick", "p", {"axis": 1}, ["x", "pidx"]), ("sum", "s", {"axis": (1,)}, ["t"])]
    text = graph(ops, ["s", "p"])
    inputs = {"table": w, "idx": np.array([1, 2, 3], np.float32), "x": xp, "pidx": np.array([0, 1, 2, 3], np.float32)}
    dev, host = both(text, {}, inputs)
    for i in range(3):
        inputs = dict(inputs, idx=rng.randint(-2, 12, 3).astype(np.float32), pidx=rng.randint(-1, 6, 4).astype(np.float32))
        got, want = outputs(dev, inputs), outputs(host, inputs)
        assert got[1].tobytes() == want[1].tobytes()
        close(got[0], want[0].astype(np.float64), 1e-5)
        ref = np.take(w, np.clip(inputs["idx"].astype(np.int64), 0, 9), 0).astype(np.float64).sum(1)
        close(got[0], ref, 1e-5)
    dev.free(); host.free()


# ------------------------------------------------------------------------------------------------ handles
@pytest.mark.gpu
def test_reshape_and_multithread_handles():
    import threading
    ops, params, x = _model("transformer", 4)
    text, blob = graph(ops), save_params(params)
    dev = Pred(text, blob, {"data": x.shape}, 2)
    a = dev.forward(data=x).out()
    r = vp()
    ck(lib().GXPredReshape(1, (cp * 1)(b"data"), (u32 * 2)(0, 3), (u32 * 3)(2, *x.shape[1:]), dev.h, ctypes.byref(r)))
    rp = Pred(None, None, None, None, handle=r)
    assert rp.engine() == 3
    close(rp.forward(data=x[:2]).out(), a[:2].astype(np.float64), 1e-5)
    hs = (vp * 4)()
    ck(lib().GXPredCreateMultiThread(text.encode(), blob, len(blob), 2, 0, 1, (cp * 1)(b"data"), (u32 * 2)(0, 3), (u32 * 3)(*x.shape), 4, hs))
    preds = [Pred(None, None, None, None, handle=vp(hs[i])) for i in range(4)]
    rng = np.random.RandomState(4)
    xs = [rng.rand(*x.shape).astype(np.float32) for _ in preds]
    want = [dev.forward(data=v).out() for v in xs]
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
    for p in preds + [dev, rp]:
        p.free()


@pytest.mark.gpu
def test_create_free_cycles_release_device_memory():
    import torch
    ops, params, x = _model("encdec", 4)
    text, blob = graph(ops), save_params(params)

    def cycle():
        p = Pred(text, blob, {"data": x.shape}, 2)
        assert p.engine() == 3
        p.forward(data=x).out()
        p.free()
    cycle()
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    for _ in range(20):
        cycle()
    torch.cuda.synchronize()
    assert abs(torch.cuda.mem_get_info()[0] - free0) <= 8 << 20


# ------------------------------------------------------------------------------------------------ refusals
def _create(text, shape, dev_type):
    h = vp()
    rc = lib().GXPredCreate(text.encode(), b"", 0, dev_type, 0, 1, (cp * 1)(b"data"), (u32 * 2)(0, len(shape)), (u32 * len(shape))(*shape), ctypes.byref(h))
    if rc == 0:
        ck(lib().GXPredFree(h))
    return rc


@pytest.mark.gpu
def test_refusals():
    # an extent past the kernels' 32-bit range, and a ninth axis: refused at create, before anything is allocated or launched
    wide = graph([("tile", "y", {"reps": (1, 4096)}, ["data"])])
    assert _create(wide, (1, 1 << 20), 2) == -1
    assert "32-bit" in err() and "dev_type 1" in err() and "Python Executor" in err()
    nine = graph([("expand_dims", "e", {"axis": 0}, ["data"]), ("sin", "y", {}, ["e"])])
    assert _create(nine, (2,) * 8, 2) == -1
    assert "at most 8 axes" in err() and "dev_type 1" in err() and "Python Executor" in err()
    # bilinear UpSampling: neither host engine has it, and the device refuses it with the general executor's reason
    bil = graph([("UpSampling", "y", {"scale": 2, "sample_type": "bilinear", "num_args": 1}, ["data"])])
    for dev_type in (1, 2):
        assert _create(bil, (1, 2, 4, 4), dev_type) == -1
        assert "single-input nearest-neighbour UpSampling" in err(), err()
    assert "Python Executor" in err()


# ------------------------------------------------------------------------------------------------ no GPU needed
def test_deconv_two_chunks_case():
    """The Deconvolution case meant to run in two workspace rounds does: the workspace the kernels library sizes holds fewer images than
    the batch, and more than half of it."""
    path = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "geomx_b200", "lib", "libgeomx_kernels.so")
    if not os.path.exists(path):
        pytest.skip("libgeomx_kernels.so not built")
    k = ctypes.CDLL(path)
    k.gx_pred_deconv_workspace.restype = ctypes.c_longlong
    (B, C, H, W), F, (kh, kw) = DECONV_TWO_CHUNKS["x"], DECONV_TWO_CHUNKS["F"], DECONV_TWO_CHUNKS["k"]
    per_image = H * W * ((C + 3) // 4 * 4 + (F * kh * kw + 3) // 4 * 4)
    images = k.gx_pred_deconv_workspace(B, C, H, W, F, kh, kw, 1) // per_image
    assert B // 2 < images < B


def _create_shapes(text, shapes, dev_type):
    h = vp()
    keys = (cp * len(shapes))(*[k.encode() for k in shapes])
    indptr, data = [0], []
    for s in shapes.values():
        data += list(s); indptr.append(len(data))
    rc = lib().GXPredCreate(text.encode(), b"", 0, dev_type, 0, len(shapes), keys, (u32 * len(indptr))(*indptr), (u32 * len(data))(*data), ctypes.byref(h))
    if rc == 0:
        ck(lib().GXPredFree(h))
    return rc, err()


# graphs with a wrong input count or an output index the node does not have: both devices refuse them at create, before the device is
# touched (the planner runs first), so these need no GPU
HOSTILE = {
    "unary_two_inputs": ([("sin", "y", {}, ["data", "other"])], ["y"], {"data": (1,), "other": (1000,)}, "2 inputs in the file, the operator takes 1"),
    "scalar_two_inputs": ([("_power_scalar", "y", {"scalar": 2}, ["data", "other"])], ["y"], {"data": (1,), "other": (1000,)}, "the operator takes 1"),
    "layernorm_one_input": ([("LayerNorm", "y", {}, ["data"])], ["y"], {"data": (3, 4)}, "1 inputs in the file, the operator takes 3"),
    "deconv_one_input": ([("Deconvolution", "y", {"kernel": (2, 2), "num_filter": 2}, ["data"])], ["y"], {"data": (1, 2, 3, 3)}, "the operator takes 2"),
    "where_one_input": ([("where", "y", {}, ["data"])], ["y"], {"data": (3,)}, "the operator takes 3"),
    "take_one_input": ([("take", "y", {}, ["data"])], ["y"], {"data": (3,)}, "the operator takes 2"),
    "dot_one_input": ([("dot", "y", {}, ["data"])], ["y"], {"data": (3, 3)}, "the operator takes 2"),
    "power_one_input": ([("broadcast_power", "y", {}, ["data"])], ["y"], {"data": (3,)}, "the operator takes 2"),
    "head_past_outputs": ([("sin", "y", {}, ["data"])], ["y:1"], {"data": (3,)}, "reads output 1 of y, which has 1 output(s)"),
    "split_head_past_outputs": ([("split", "sp", {"num_outputs": 2}, ["data"])], ["sp:2"], {"data": (2, 4)}, "reads output 2 of sp, which has 2 output(s)"),
    "input_past_outputs": ([("sin", "s", {}, ["data"]), ("cos", "y", {}, ["s:1"])], ["y"], {"data": (3,)}, "reads output 1 of s, which has 1 output(s)"),
}


@pytest.mark.parametrize("name", sorted(HOSTILE))
def test_hostile_graph_is_refused_before_any_launch(name):
    if not os.path.exists(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "geomx_b200", "lib", "libgeomx_capi.so")):
        pytest.skip("libgeomx_capi.so not built")
    ops, heads, shapes, why = HOSTILE[name]
    text = graph(ops, heads)
    rc, msg = _create_shapes(text, shapes, 2)
    assert rc == -1 and why in msg and "dev_type 1" in msg and "Python Executor" in msg, msg
    rc, msg = _create_shapes(text, shapes, 1)
    assert rc == -1, msg
