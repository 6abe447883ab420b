"""``mx.sym`` — a small symbolic graph API with shape inference and an executor, enough for the Module training path.

Parity: ``python/mxnet/symbol/symbol.py`` (``Variable``, composition, ``list_arguments`` / ``list_auxiliary_states`` / ``list_outputs``,
``infer_shape``, ``simple_bind`` / ``bind``, ``tojson`` / ``load_json``) and ``src/executor/graph_executor.cc`` (forward / backward over
a topologically sorted graph, gradient accumulation by ``grad_req``).  The graph is a DAG of :class:`Symbol` nodes; the executor evaluates
it with the same dispatch the imperative API uses (``ops.functional``: native sm_90a kernels on CUDA, PyTorch on CPU) and obtains the
gradients from the autograd tape instead of building a separate backward graph (``src/nnvm/gradient.cc``) — one code path for both front
ends.  Argument naming follows the reference (``<name>_weight``, ``<name>_bias``, ``<name>_gamma``/``_beta``, aux ``_moving_mean``/``_var``,
``softmax_label``)."""
from __future__ import annotations

import json

import numpy as np
import torch

from .base import MXNetError
from .ndarray import NDArray
from .ops import functional as F

__all__ = ["Symbol", "Variable", "var", "Group", "load_json", "FullyConnected", "Convolution", "Activation", "Pooling", "Flatten",
           "BatchNorm", "Dropout", "SoftmaxOutput", "LinearRegressionOutput", "Concat", "elemwise_add", "relu", "softmax", "log_softmax",
           "reshape", "Executor"]

def _auto_name(op, name):
    from .name import NameManager
    return NameManager.current().get(name, op.lower())


def _pair(v, default=None):
    if v is None:
        return default
    return (int(v), int(v)) if np.isscalar(v) else tuple(int(x) for x in v)


class Symbol:
    def __init__(self, op, name, inputs=(), attrs=None, aux=()):
        self.op, self.name, self.inputs, self.attrs, self.aux = op, name, list(inputs), dict(attrs or {}), list(aux)
        from .attribute import AttrScope
        scope = AttrScope.current().get()
        if scope:                                         # user annotations (ctx_group, lr_mult, ...) live under a "__attr__" sub-dict
            self.attrs.setdefault("__attr__", {}).update(scope)

    def list_attr(self):
        return dict(self.attrs.get("__attr__", {}))

    def attr_dict(self):
        return {s.name: s.list_attr() for s in self._topo() if s.attrs.get("__attr__")}

    # ---- composition sugar
    def __add__(self, o): return _binary("_plus", self, o)
    __radd__ = __add__
    def __sub__(self, o): return _binary("_minus", self, o)
    def __mul__(self, o): return _binary("_mul", self, o)
    __rmul__ = __mul__
    def __truediv__(self, o): return _binary("_div", self, o)
    def __rsub__(self, o): return _binary("_plus", -self, o)                      # scalar - symbol
    def __rtruediv__(self, o): return _binary("_mul", _nd_op("reciprocal")(self), o)   # scalar / symbol
    def __getitem__(self, i):
        if self.op == "_nd" and isinstance(i, int) and (i > 0 or self.attrs.get("kwargs", {}).get("num_outputs", 1) > 1 or self.attrs.get("multi")):
            # i-th output of a multi-output imperative op (split / SliceChannel / topk(ret_typ='both') / RNN(state_outputs=True) …)
            self.attrs["multi"] = True
            return Symbol("_item", "%s_output%d" % (self.name, i), [self], {"index": int(i)})
        if self.op != "_group":
            if i in (0, self.list_outputs()[0]):
                return self
            raise IndexError(i)
        return self.inputs[i] if isinstance(i, int) else next(s for s in self.inputs if s.list_outputs()[0] == i)

    def __pow__(self, o): return _nd_op("power")(self, o) if isinstance(o, Symbol) else _nd_op("power")(self, Symbol("_full_like", _auto_name("scalar", None), [self], {"value": float(o)}))
    def __neg__(self): return _binary("_mul", self, -1.0)
    def __copy__(self): return load_json(self.tojson())
    __deepcopy__ = lambda self, memo: load_json(self.tojson())          # noqa: E731

    def get_children(self):
        """Group of the direct inputs of this node (None for variables)."""
        return Group(self.inputs) if self.inputs else None

    def eval(self, ctx=None, **kwargs):
        """Bind with the given NDArrays and run forward once: ``(a + b).eval(a=x, b=y)`` → list of outputs."""
        from .context import cpu
        ex = self.bind(ctx or cpu(), kwargs)
        return ex.forward()

    def infer_shape_partial(self, **shapes):
        """Like ``infer_shape`` but returns ``None`` entries instead of raising when something cannot be inferred."""
        try:
            return self.infer_shape(**shapes)
        except MXNetError:
            args, auxs = self.list_arguments(), self.list_auxiliary_states()
            return [tuple(shapes[a]) if a in shapes else None for a in args], [None] * len(self.list_outputs()), [None] * len(auxs)

    def debug_str(self):
        lines = []
        for s in self._topo():
            if s.op == "null":
                lines.append("Variable:%s" % s.name)
            else:
                lines.append("--------------------\nOp:%s, Name=%s\nInputs:\n%s\nAttrs:%s" % (
                    s.op, s.name, "\n".join("\targ[%d]=%s" % (i, x.name) for i, x in enumerate(s.inputs)), {k: v for k, v in s.attrs.items() if not k.startswith("__")}))
        return "\n".join(lines)

    def gradient(self, wrt):
        raise MXNetError("Symbol.gradient is not available: gradients come from the executor's autograd tape (Executor.backward)")

    def get_backend_symbol(self, backend):
        return self                                           # no graph-partitioning backends: the same graph runs on the native kernels

    # ---- graph walks
    def _topo(self):
        order, seen = [], set()

        def visit(s):
            if id(s) in seen:
                return
            seen.add(id(s))
            for i in s.inputs + s.aux:
                visit(i)
            order.append(s)
        visit(self)
        return order

    def list_arguments(self):
        aux = {id(a) for s in self._topo() for a in s.aux}
        return [s.name for s in self._topo() if s.op == "null" and id(s) not in aux]

    def list_auxiliary_states(self):
        out, seen = [], set()
        for s in self._topo():
            for a in s.aux:
                if id(a) not in seen:
                    seen.add(id(a)); out.append(a.name)
        return out

    def list_outputs(self):
        if self.op == "_group":
            return [o for s in self.inputs for o in s.list_outputs()]
        return [self.name if self.op in ("null", "_item") else self.name + "_output"]          # an _item is already called <node>_output<i>

    def list_inputs(self):
        return self.list_arguments() + self.list_auxiliary_states()

    def get_internals(self):
        return Group([s for s in self._topo() if s.op != "_group"])

    def attr(self, key):
        return self.attrs.get(key)

    # ---- shape inference: run the graph once on zero tensors of the given shapes (meta-free but exact)
    def infer_shape(self, **shapes):
        args, auxs = self.list_arguments(), self.list_auxiliary_states()
        known = {k: tuple(v) for k, v in shapes.items()}
        vals = _ShapeRun(self, known).run()
        arg_shapes = [vals.shapes.get(a) for a in args]
        aux_shapes = [vals.shapes.get(a) for a in auxs]
        outs = [tuple(o.shape) for o in vals.outputs]
        return arg_shapes, outs, aux_shapes

    def infer_type(self, **types):
        args = self.list_arguments()
        return [np.float32] * len(args), [np.float32] * len(self.list_outputs()), [np.float32] * len(self.list_auxiliary_states())

    # ---- binding
    def simple_bind(self, ctx, grad_req="write", group2ctx=None, **shapes):
        from . import ndarray as nd
        arg_shapes, _, aux_shapes = self.infer_shape(**shapes)
        names = self.list_arguments()
        if any(s is None for s in arg_shapes):
            raise MXNetError("cannot infer shapes of %s" % [n for n, s in zip(names, arg_shapes) if s is None])
        # manual model parallelism: a variable annotated with ctx_group (AttrScope) is allocated on the device its group maps to
        place = _placement(self, ctx, group2ctx)
        args = {n: nd.zeros(s, ctx=place.get(n, ctx)) for n, s in zip(names, arg_shapes)}
        req = grad_req if isinstance(grad_req, dict) else {n: grad_req for n in names}
        grads = {n: nd.zeros(s, ctx=place.get(n, ctx)) for n, s in zip(names, arg_shapes) if req.get(n, "null") != "null"}
        aux = {n: nd.zeros(s, ctx=place.get(n, ctx)) for n, s in zip(self.list_auxiliary_states(), aux_shapes)}
        for n, a in aux.items():
            if n.endswith("_moving_var"):
                a[:] = 1.0
        return Executor(self, ctx, args, grads, req, aux, group2ctx)

    def bind(self, ctx, args, args_grad=None, grad_req="write", aux_states=None, group2ctx=None):
        names = self.list_arguments()
        if isinstance(args, (list, tuple)):
            args = dict(zip(names, args))
        if isinstance(args_grad, (list, tuple)):
            args_grad = dict(zip(names, args_grad))
        auxn = self.list_auxiliary_states()
        if isinstance(aux_states, (list, tuple)):
            aux_states = dict(zip(auxn, aux_states))
        req = grad_req if isinstance(grad_req, dict) else {n: (grad_req if args_grad and n in args_grad else "null") for n in names}
        return Executor(self, ctx, dict(args), dict(args_grad or {}), req, dict(aux_states or {}), group2ctx)

    # ---- (de)serialisation: a flat node list in topological order
    def tojson(self, nnvm=False):
        """Graph as JSON.  ``nnvm=True`` writes the reference's dialect (python-repr string attributes, ``[node, output, version]`` input
        triples, ``arg_nodes`` / ``node_row_ptr`` / ``heads``; src/nnvm + nnvm::pass::SaveJSON) so ``-symbol.json`` files can be read by
        MXNet-family tools; ``load_json`` reads both dialects."""
        if nnvm:
            return _to_nnvm_json(self)
        order = self._topo()
        index = {id(s): i for i, s in enumerate(order)}
        nodes = [{"op": s.op, "name": s.name, "attrs": {k: (list(v) if isinstance(v, tuple) else v) for k, v in s.attrs.items()},
                  "inputs": [index[id(i)] for i in s.inputs], "aux": [index[id(a)] for a in s.aux]} for s in order]
        return json.dumps({"nodes": nodes, "heads": [index[id(self)]], "format": "geomx_b200-symbol-1"}, indent=1)

    def save(self, fname, nnvm=False):
        with open(fname, "w") as f:
            f.write(self.tojson(nnvm=nnvm))

    def __repr__(self):
        return "<Symbol %s>" % (self.name if self.op != "_group" else "group [%s]" % ", ".join(self.list_outputs()))


_NNVM_BINARY = {"elemwise_add": "_plus", "_Plus": "_plus", "_plus": "_plus", "_add": "_plus", "elemwise_sub": "_minus", "_Minus": "_minus", "_minus": "_minus",
                "_sub": "_minus", "elemwise_mul": "_mul", "_Mul": "_mul", "_mul": "_mul", "elemwise_div": "_div", "_Div": "_div", "_div": "_div"}
_NNVM_SCALAR = {"_plus_scalar": "_plus", "_PlusScalar": "_plus", "_minus_scalar": "_minus", "_MinusScalar": "_minus", "_mul_scalar": "_mul", "_MulScalar": "_mul",
                "_div_scalar": "_div", "_DivScalar": "_div"}


def _lit(v):
    """python-repr attribute string of the nnvm dialect -> value ("(5, 5)" -> (5, 5), "True" -> True, "relu" -> "relu")."""
    if not isinstance(v, str):
        return v
    import ast
    try:
        return ast.literal_eval(v)
    except (ValueError, SyntaxError):
        return v


def _from_nnvm(d):
    """Build the graph from the reference's JSON dialect (what ``Symbol.save`` of MXNet / GeoMX writes)."""
    built = []
    # nodes with several outputs: output 0 must be taken as an item too (a consumer of the bare node would receive the tuple of all outputs)
    rows = d.get("node_row_ptr") or []
    multi = {i for i in range(len(rows) - 1) if rows[i + 1] - rows[i] > 1}
    for n in d["nodes"]:
        multi.update(e[0] for e in n["inputs"] if len(e) > 1 and e[1])
    multi.update(h[0] for h in d.get("heads", []) if len(h) > 1 and h[1])

    def user_attrs(n, raw):
        a = dict(n.get("attr") or {}) if ("attrs" in n or "param" in n) else {}
        a.update({k: v for k, v in raw.items() if k.startswith("__")})
        return a
    for n in d["nodes"]:
        op, name = n["op"], n["name"]
        raw = n.get("attrs") or n.get("param") or (n.get("attr") if n["op"] != "null" and "param" not in n else None) or {}
        if op == "null":
            raw = n.get("attrs") or n.get("attr") or {}
        kw = {k: _lit(v) for k, v in raw.items() if not k.startswith("__")}
        ins = []
        for e in n["inputs"]:
            src = built[e[0]]
            ins.append(src[e[1]] if (e[1] or e[0] in multi) else src)
        usr = user_attrs(n, raw)
        if op == "null":
            sym = Symbol("null", name, attrs={"__attr__": {k: str(v) for k, v in usr.items()}} if usr else None)
            if "__shape__" in usr:
                sym.attrs["__shape__"] = tuple(_lit(usr["__shape__"]))
        elif op == "FullyConnected":
            sym = Symbol(op, name, ins, {"num_hidden": int(kw["num_hidden"]), "no_bias": bool(kw.get("no_bias", False)), "flatten": bool(kw.get("flatten", True))})
        elif op == "Convolution" and len(tuple(kw["kernel"])) == 2:
            sym = Symbol(op, name, ins, {"kernel": _pair(kw["kernel"]), "num_filter": int(kw["num_filter"]), "stride": _pair(kw.get("stride") or None, (1, 1)),
                                         "pad": _pair(kw.get("pad") or None, (0, 0)), "dilate": _pair(kw.get("dilate") or None, (1, 1)),
                                         "num_group": int(kw.get("num_group", 1)), "no_bias": bool(kw.get("no_bias", False))})
        elif op == "Activation":
            sym = Symbol(op, name, ins, {"act_type": kw["act_type"]})
        elif op == "Pooling" and kw.get("pooling_convention", "valid") == "valid" and kw.get("pool_type", "max") in ("max", "avg") \
                and (kw.get("global_pool") or len(tuple(kw.get("kernel", ()))) == 2):
            sym = Symbol(op, name, ins, {"kernel": _pair(kw.get("kernel") or None, (1, 1)), "pool_type": kw.get("pool_type", "max"),
                                         "stride": _pair(kw.get("stride") or None, (1, 1)), "pad": _pair(kw.get("pad") or None, (0, 0)),
                                         "global_pool": bool(kw.get("global_pool", False))})
        elif op in ("Flatten", "flatten"):
            sym = Symbol("Flatten", name, ins)
        elif op in ("Reshape", "reshape") and "shape" in kw and all(int(v) > 0 or int(v) == -1 for v in kw["shape"]):
            sym = Symbol("Reshape", name, ins, {"shape": tuple(int(v) for v in kw["shape"])})
        elif op == "BatchNorm":
            sym = Symbol(op, name, ins[:3], {"eps": float(kw.get("eps", 1e-3)), "momentum": float(kw.get("momentum", 0.9)), "fix_gamma": bool(kw.get("fix_gamma", True)),
                                             "use_global_stats": bool(kw.get("use_global_stats", False)), "axis": int(kw.get("axis", 1))}, ins[3:5])
        elif op == "Dropout":
            sym = Symbol(op, name, ins, {"p": float(kw.get("p", 0.5))})
        elif op in ("Concat", "concat"):
            sym = Symbol("Concat", name, ins, {"dim": int(kw.get("dim", 1))})
        elif op in ("softmax", "log_softmax"):
            sym = Symbol(op, name, ins, {"axis": int(kw.get("axis", -1))})
        elif op in ("SoftmaxOutput", "Softmax"):
            sym = Symbol("SoftmaxOutput", name, ins, {"grad_scale": float(kw.get("grad_scale", 1.0)), "normalization": kw.get("normalization", "null")})
        elif op == "LinearRegressionOutput":
            sym = Symbol(op, name, ins, {"grad_scale": float(kw.get("grad_scale", 1.0))})
        elif op in _NNVM_BINARY:
            sym = Symbol(_NNVM_BINARY[op], name, ins)
        elif op in _NNVM_SCALAR:
            sym = Symbol(_NNVM_SCALAR[op] + "_scalar", name, ins, {"scalar": float(kw["scalar"])})
        else:                                   # everything else: the imperative operator of that name through the generic bridge
            from . import ndarray as nd
            if not callable(getattr(nd, op, None)):
                raise MXNetError("symbol JSON: operator %s (node %s) is not available" % (op, name))
            kw.pop("num_args", None)
            sym = _nd_op(op)(*ins, name=name, **kw)
        if usr and op != "null":
            sym.attrs.setdefault("__attr__", {}).update({k: str(v) for k, v in usr.items()})
        built.append(sym)
    heads = [built[h[0]][h[1]] if (h[1] or h[0] in multi) else built[h[0]] for h in d["heads"]]
    return heads[0] if len(heads) == 1 else Group(heads)


def _repr_attr(v):
    if isinstance(v, bool):
        return "True" if v else "False"
    if isinstance(v, (list, tuple)):
        return "(" + ", ".join(_repr_attr(x) for x in v) + ("," if len(v) == 1 else "") + ")"
    return str(v)


_TO_NNVM_OP = {"_plus": "elemwise_add", "_minus": "elemwise_sub", "_mul": "elemwise_mul", "_div": "elemwise_div"}


def _to_nnvm_json(sym):
    order = [s for s in sym._topo() if s.op != "_group"]
    index = {id(s): i for i, s in enumerate(order)}
    nodes = []
    for s in order:
        if s.op == "_item":
            continue
        usr = dict(s.attrs.get("__attr__", {}))
        if s.op == "null":
            if s.attrs.get("__shape__") is not None:
                usr["__shape__"] = _repr_attr(s.attrs["__shape__"])
            node = {"op": "null", "name": s.name, "inputs": []}
            if usr:
                node["attrs"] = usr
            nodes.append(node)
            continue
        if s.op == "_nd":
            if s.attrs.get("sym_kwargs"):
                raise MXNetError("tojson(nnvm=True): %s takes tensor keyword arguments, which have no positional order in the nnvm dialect" % s.name)
            op, kw = s.attrs["fn"].split(".")[-1], dict(s.attrs.get("kwargs") or {})
        elif s.op == "_full_like":
            raise MXNetError("tojson(nnvm=True): scalar-broadcast helper nodes cannot be written in the nnvm dialect")
        else:
            op = _TO_NNVM_OP.get(s.op, s.op)
            kw = {k: v for k, v in s.attrs.items() if not k.startswith("__") and v is not None}
            if s.op == "Concat":
                kw["num_args"] = len(s.inputs)
            if s.op == "Pooling" and s.attrs.get("stride") is None:
                kw["stride"] = s.attrs["kernel"]            # here an absent stride means the window; the nnvm default is 1
        attrs = {k: _repr_attr(v) for k, v in kw.items() if v is not None}
        attrs.update(usr)
        ins = []
        for i in list(s.inputs) + list(s.aux):
            ins.append([index[id(i.inputs[0])], int(i.attrs["index"]), 0] if i.op == "_item" else [index[id(i)], 0, 0])
        node = {"op": op, "name": s.name, "inputs": ins}
        if attrs:
            node["attrs"] = attrs
        nodes.append(node)
    # _item nodes were skipped: compact the numbering
    keep = [i for i, s in enumerate(order) if s.op != "_item"]
    renum = {old: new for new, old in enumerate(keep)}
    for n in nodes:
        n["inputs"] = [[renum[e[0]], e[1], e[2]] for e in n["inputs"]]
    heads = sym.inputs if sym.op == "_group" else [sym]
    head_entries = [[renum[index[id(h.inputs[0])]], int(h.attrs["index"]), 0] if h.op == "_item" else [renum[index[id(h)]], 0, 0] for h in heads]
    return json.dumps({"nodes": nodes, "arg_nodes": [i for i, n in enumerate(nodes) if n["op"] == "null"], "node_row_ptr": list(range(len(nodes) + 1)),
                       "heads": head_entries, "attrs": {"mxnet_version": ["int", 10400]}}, indent=2)


def load_json(s):
    d = json.loads(s)
    if "format" not in d and ("arg_nodes" in d or (d.get("nodes") and d["nodes"][0].get("inputs") is not None and d.get("heads") and isinstance(d["heads"][0], list))):
        return _from_nnvm(d)
    built = []
    for n in d["nodes"]:
        attrs = {k: (tuple(v) if isinstance(v, list) else v) for k, v in n["attrs"].items()}
        built.append(Symbol(n["op"], n["name"], [built[i] for i in n["inputs"]], attrs, [built[i] for i in n.get("aux", [])]))
    return built[d["heads"][0]]


def load(fname):
    with open(fname) as f:
        return load_json(f.read())


def Variable(name, shape=None, init=None, lr_mult=None, wd_mult=None, dtype=None, attr=None, **kw):
    """A named input of the graph.  ``init`` (the Initializer ``Module.init_params`` uses for this variable instead of the global one),
    ``lr_mult`` / ``wd_mult``, ``dtype`` and free-form ``attr`` become node attributes (``__init__``, ``__lr_mult__`` ... as in
    python/mxnet/symbol/symbol.py:var), visible through ``list_attr()`` / ``attr_dict()``."""
    user = {str(k): str(v) for k, v in (attr or {}).items()}
    if init is not None:
        user["__init__"] = init if isinstance(init, str) else init.dumps()
    if lr_mult is not None:
        user["__lr_mult__"] = str(lr_mult)
    if wd_mult is not None:
        user["__wd_mult__"] = str(wd_mult)
    if dtype is not None:
        user["__dtype__"] = str(dtype)
    attrs = {}
    if shape:
        attrs["__shape__"] = tuple(shape)
    if user:
        attrs["__attr__"] = user
    return Symbol("null", name, attrs=attrs or None)


var = Variable


def Group(symbols):
    return Symbol("_group", "group", list(symbols))


def _binary(op, a, b):
    if not isinstance(b, Symbol):
        return Symbol(op + "_scalar", _auto_name(op, None), [a], {"scalar": float(b)})
    return Symbol(op, _auto_name(op, None), [a, b])


def _wb(name, no_bias):
    w = Variable(name + "_weight")
    return [w] if no_bias else [w, Variable(name + "_bias")]


def FullyConnected(data, num_hidden, weight=None, bias=None, no_bias=False, flatten=True, name=None):
    name = _auto_name("FullyConnected", name)
    ins = [data, weight or Variable(name + "_weight")] + ([] if no_bias else [bias or Variable(name + "_bias")])
    return Symbol("FullyConnected", name, ins, {"num_hidden": int(num_hidden), "no_bias": bool(no_bias), "flatten": bool(flatten)})


def Convolution(data, kernel, num_filter, stride=None, pad=None, dilate=None, num_group=1, weight=None, bias=None, no_bias=False, name=None):
    name = _auto_name("Convolution", name)
    ins = [data, weight or Variable(name + "_weight")] + ([] if no_bias else [bias or Variable(name + "_bias")])
    return Symbol("Convolution", name, ins, {"kernel": _pair(kernel), "num_filter": int(num_filter), "stride": _pair(stride, (1, 1)),
                                             "pad": _pair(pad, (0, 0)), "dilate": _pair(dilate, (1, 1)), "num_group": int(num_group),
                                             "no_bias": bool(no_bias)})


def Activation(data, act_type="relu", name=None):
    return Symbol("Activation", _auto_name("Activation", name), [data], {"act_type": act_type})


def relu(data, name=None):
    return Activation(data, "relu", name)


def Pooling(data, kernel=(2, 2), pool_type="max", stride=None, pad=None, global_pool=False, name=None):
    return Symbol("Pooling", _auto_name("Pooling", name), [data], {"kernel": _pair(kernel), "pool_type": pool_type, "stride": _pair(stride),
                                                                   "pad": _pair(pad, (0, 0)), "global_pool": bool(global_pool)})


def Flatten(data, name=None):
    return Symbol("Flatten", _auto_name("Flatten", name), [data])


def reshape(data, shape, name=None):
    return Symbol("Reshape", _auto_name("Reshape", name), [data], {"shape": tuple(shape)})


def BatchNorm(data, gamma=None, beta=None, eps=1e-5, momentum=0.9, fix_gamma=False, use_global_stats=False, axis=1, name=None):
    name = _auto_name("BatchNorm", name)
    aux = [Variable(name + "_moving_mean"), Variable(name + "_moving_var")]
    return Symbol("BatchNorm", name, [data, gamma or Variable(name + "_gamma"), beta or Variable(name + "_beta")],
                  {"eps": float(eps), "momentum": float(momentum), "fix_gamma": bool(fix_gamma), "use_global_stats": bool(use_global_stats),
                   "axis": int(axis)}, aux)


def Dropout(data, p=0.5, name=None):
    return Symbol("Dropout", _auto_name("Dropout", name), [data], {"p": float(p)})


def Concat(*data, dim=1, name=None):
    return Symbol("Concat", _auto_name("Concat", name), list(data), {"dim": int(dim)})


def elemwise_add(a, b, name=None):
    return Symbol("_plus", _auto_name("_plus", name), [a, b])


def softmax(data, axis=-1, name=None):
    return Symbol("softmax", _auto_name("softmax", name), [data], {"axis": int(axis)})


def log_softmax(data, axis=-1, name=None):
    return Symbol("log_softmax", _auto_name("log_softmax", name), [data], {"axis": int(axis)})


def SoftmaxOutput(data, label=None, grad_scale=1.0, normalization="null", name=None):
    """Forward: softmax(data).  Backward: (softmax - onehot(label)) * grad_scale, ignoring the head gradient (src/operator/softmax_output-inl.h)."""
    name = _auto_name("SoftmaxOutput", name)
    return Symbol("SoftmaxOutput", name, [data, label or Variable(name + "_label")], {"grad_scale": float(grad_scale), "normalization": normalization})


def LinearRegressionOutput(data, label=None, grad_scale=1.0, name=None):
    name = _auto_name("LinearRegressionOutput", name)
    return Symbol("LinearRegressionOutput", name, [data, label or Variable(name + "_label")], {"grad_scale": float(grad_scale)})


# ------------------------------------------------------------------------------------------------------------------ evaluation
class _SoftmaxOutputFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, label, scale, normalization):
        p = torch.softmax(x, dim=1)
        ctx.save_for_backward(p, label)
        ctx.scale, ctx.norm = scale, normalization
        return p

    @staticmethod
    def backward(ctx, _gy):
        p, label = ctx.saved_tensors
        g = p.clone()
        g.scatter_add_(1, label.long().view(-1, 1), -torch.ones_like(p[:, :1]))
        s = ctx.scale / (p.shape[0] if ctx.norm == "batch" else 1.0)
        return g * s, None, None, None


class _LinRegFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, label, scale):
        ctx.save_for_backward(x, label); ctx.scale = scale
        return x.clone()

    @staticmethod
    def backward(ctx, _gy):
        x, label = ctx.saved_tensors
        return (x - label.view_as(x)) * ctx.scale, None, None


def _eval_node(s, ins, aux, training):
    a = s.attrs
    op = s.op
    q = a.get("__quantized__")
    if q and op in ("FullyConnected", "Convolution"):
        # simulated quantisation (contrib/quantization.py): the layer input is clipped+rounded at the calibrated threshold
        from .contrib.quantization import fake_quantize
        thr = q.get("act_threshold")
        x = ins[0]
        ins = [fake_quantize(x, thr if thr is not None else float(x.abs().max()), "int8" if q["dtype"] == "uint8" and float(x.min()) < 0 else q["dtype"])] + list(ins[1:])
    if op == "FullyConnected":
        return F.dense(ins[0], ins[1], None if a["no_bias"] else ins[2], None, a.get("flatten", True))
    if op == "Convolution":
        return F.conv2d(ins[0], ins[1], None if a["no_bias"] else ins[2], a["stride"], a["pad"], a["dilate"], a["num_group"])
    if op == "Activation":
        return F.activation(ins[0], a["act_type"])
    if op == "Pooling":
        x = ins[0]
        k = tuple(x.shape[2:]) if a["global_pool"] else a["kernel"]
        st = a["stride"] or k
        return F.max_pool2d(x, k, st, a["pad"]) if a["pool_type"] == "max" else F.avg_pool2d(x, k, st, a["pad"])
    if op == "Flatten":
        return F.flatten(ins[0])
    if op == "Reshape":
        return ins[0].reshape(a["shape"])
    if op == "BatchNorm":
        g = torch.ones_like(ins[1]) if a["fix_gamma"] else ins[1]
        return F.batch_norm(ins[0], g, ins[2], aux[0], aux[1], training and not a["use_global_stats"], a["momentum"], a["eps"], a["axis"])
    if op == "Dropout":
        return F.dropout(ins[0], a["p"], training)
    if op == "Concat":
        return torch.cat(ins, dim=a["dim"])
    if op == "softmax":
        return F.softmax(ins[0], a["axis"])
    if op == "log_softmax":
        return F.log_softmax(ins[0], a["axis"])
    if op == "SoftmaxOutput":
        return _SoftmaxOutputFn.apply(ins[0], ins[1], a["grad_scale"], a["normalization"])
    if op == "LinearRegressionOutput":
        return _LinRegFn.apply(ins[0], ins[1], a["grad_scale"])
    if op in ("_plus", "_minus", "_mul", "_div"):
        return {"_plus": torch.add, "_minus": torch.sub, "_mul": torch.mul, "_div": torch.div}[op](ins[0], ins[1])
    if op.endswith("_scalar"):
        return {"_plus": torch.add, "_minus": torch.sub, "_mul": torch.mul, "_div": torch.div}[op[:-7]](ins[0], a["scalar"])
    if op == "_nd":
        return _eval_nd(a, ins)
    if op == "_item":
        if not isinstance(ins[0], tuple):
            raise MXNetError("%s: the producer has a single output" % s.name)
        return ins[0][a["index"]]
    if op == "_full_like":
        return torch.full_like(ins[0], a["value"])
    raise MXNetError("symbol op %s is not implemented" % op)


# ---- generic bridge: every imperative ``mx.nd.<fn>`` / ``mx.nd.contrib.<fn>`` that maps NDArrays to ONE NDArray is also a symbolic op.
# The node stores the function's qualified name and its JSON-able keyword arguments; evaluation calls the imperative function on the
# bound tensors (so gradients come from the same autograd tape).  This is how ``mx.sym.exp`` / ``broadcast_add`` / ``contrib.ROIAlign`` …
# exist without a per-op registration table (the reference generates them from the nnvm registry: python/mxnet/symbol/register.py).
def _resolve_nd(qual):
    from . import ndarray as nd
    obj = nd
    for part in qual.split("."):
        obj = getattr(obj, part)
    return obj


def _eval_nd(a, ins):
    fn = _resolve_nd(a["fn"])
    npos = a["npos"]
    args = [NDArray(t) for t in ins[:npos]]
    kwargs = dict(a.get("kwargs") or {})
    for k, t in zip(a.get("sym_kwargs") or (), ins[npos:]):
        kwargs[k] = NDArray(t)
    out = fn(*args, **kwargs)
    if isinstance(out, (list, tuple)) and a.get("multi"):
        return tuple(o._t for o in out)
    if not isinstance(out, NDArray):
        raise MXNetError("mx.sym.%s: the imperative function returned %s, index the symbol (``sym[i]``) to use one output of a multi-output op" % (a["fn"], type(out).__name__))
    return out._t


# parameter inputs that are created automatically (as ``<name>_<param>`` variables) when the caller does not pass them, and whose shapes
# follow from the attributes / data shape — the bridged counterparts of the reference ops' FListInputNames + FInferShape
_AUTO_PARAMS = {"Embedding": ("weight",), "Deconvolution": ("weight", "bias"), "LayerNorm": ("gamma", "beta"), "InstanceNorm": ("gamma", "beta")}


def _nd_param_shape(a, pname, in_shape):
    fn, kw = a["fn"], a.get("kwargs") or {}
    if fn == "Embedding" and pname == "weight":
        return (int(kw["input_dim"]), int(kw["output_dim"]))
    if fn == "Deconvolution":
        k = tuple(kw["kernel"])
        return (in_shape[1], int(kw["num_filter"]) // int(kw.get("num_group", 1))) + k if pname == "weight" else (int(kw["num_filter"]),)
    if fn == "LayerNorm":
        return (in_shape[int(kw.get("axis", -1))],)
    if fn == "InstanceNorm":
        return (in_shape[1],)
    if fn == "RNN" and pname == "parameters":
        # one flat vector: per layer and direction W_i2h [G*H, C_in] and W_h2h [G*H, H], then as many bias pairs (src/operator/rnn-inl.h)
        H, L, D = int(kw["state_size"]), int(kw.get("num_layers", 1)), 2 if kw.get("bidirectional") else 1
        G = {"rnn_relu": 1, "rnn_tanh": 1, "lstm": 4, "gru": 3}[kw.get("mode", "lstm")]
        total = 0
        for layer in range(L):
            cin = in_shape[2] if layer == 0 else D * H
            total += D * (G * H * (cin + H) + 2 * G * H)
        return (total,)
    if fn == "RNN" and pname in ("state", "state_cell"):
        return ((int(kw.get("num_layers", 1)) * (2 if kw.get("bidirectional") else 1)), in_shape[1], int(kw["state_size"]))
    return None


def _bind_positional(qual, args, kwargs):
    """Bind the positional arguments from the first non-Symbol one on to the imperative function's parameter names, so that
    ``mx.sym.clip(x, 0, 6)``, ``x.clip(0, 6)`` and ``F.clip(x, 0, 6)`` in a traced block mean ``clip(x, a_min=0, a_max=6)`` as in the
    reference's generated ``mx.sym`` functions.  Returns the leading Symbols (still positional) and the keyword arguments."""
    import inspect
    first = next(i for i, x in enumerate(args) if not isinstance(x, Symbol))
    refuse = MXNetError("mx.sym.%s: positional arguments must be Symbols, pass attributes by keyword" % qual)
    try:
        params = list(inspect.signature(_resolve_nd(qual)).parameters.values())
    except (AttributeError, TypeError, ValueError):
        raise refuse from None
    kwargs = dict(kwargs)
    for i in range(first, len(args)):
        if i >= len(params) or any(p.kind != p.POSITIONAL_OR_KEYWORD for p in params[:i + 1]) or params[i].name in kwargs:
            raise refuse
        kwargs[params[i].name] = args[i]
    return list(args[:first]), kwargs


def _nd_op(qual):
    def build(*args, name=None, **kwargs):
        auto = _AUTO_PARAMS.get(qual)
        if auto and len(args) == 1:
            name = _auto_name(qual.lower(), name)
            for pn in auto:
                if pn == "bias" and kwargs.get("no_bias", qual == "Deconvolution"):
                    continue
                if kwargs.get(pn) is None:
                    kwargs[pn] = Variable("%s_%s" % (name, pn))
        pos = [x for x in args if isinstance(x, Symbol)]
        if len(pos) != len(args):
            pos, kwargs = _bind_positional(qual, args, kwargs)
        skw = [k for k, v in kwargs.items() if isinstance(v, Symbol)]
        attrs = {"fn": qual, "npos": len(pos), "sym_kwargs": skw,
                 "kwargs": {k: (list(v) if isinstance(v, tuple) else v) for k, v in kwargs.items() if k not in skw}}
        return Symbol("_nd", _auto_name(qual.split(".")[-1].lower(), name), pos + [kwargs[k] for k in skw], attrs)
    build.__name__ = qual.split(".")[-1]
    build.__doc__ = "Symbolic form of ``mx.nd.%s`` (generic imperative-op bridge)." % qual
    return build


def _namespace(sub, target):
    """``mx.sym.<sub>``: the symbolic forms of the operators in ``mx.nd.<target>`` (reference: python/mxnet/symbol/{contrib,linalg,random,
    sparse,image,op,_internal}.py, generated from the operator registry).  Also importable as ``<package>.symbol.<sub>``."""
    def lookup(item):
        from . import ndarray as nd
        ns = nd
        for part in (target.split(".") if target else ()):
            ns = getattr(ns, part)
        if item.startswith("__") or not callable(getattr(ns, item, None)) or isinstance(getattr(ns, item), type):
            raise AttributeError("mx.sym.%s has no operator %r" % (sub, item))
        return _nd_op((target + "." if target else "") + item)
    from ._alias import submodule
    return submodule(__name__, sub, getattr_fn=lookup, doc="mx.sym.%s operator namespace" % sub)


contrib = _namespace("contrib", "contrib")
linalg = _namespace("linalg", "linalg")
random = _namespace("random", "random")
sparse = _namespace("sparse", "sparse")
image = _namespace("image", "image")
op = _namespace("op", "")
_internal = _namespace("_internal", "_internal")


def __getattr__(item):
    from . import ndarray as nd
    fn = getattr(nd, item, None)
    if item.startswith("_") or fn is None or not callable(fn) or isinstance(fn, type):
        raise AttributeError("module 'mx.sym' has no attribute %r" % item)
    return _nd_op(item)


def _param_shape(s, idx, in_shape):
    """Shape of the idx-th input (a parameter Variable) of node ``s`` given its data shape — the per-op rules of nnvm's InferShape."""
    a = s.attrs
    if s.op == "FullyConnected":
        k = int(np.prod(in_shape[1:])) if a.get("flatten", True) else in_shape[-1]
        return (a["num_hidden"], k) if idx == 1 else (a["num_hidden"],)
    if s.op == "Convolution":
        return (a["num_filter"], in_shape[1] // a["num_group"]) + tuple(a["kernel"]) if idx == 1 else (a["num_filter"],)
    if s.op == "BatchNorm":
        return (in_shape[a["axis"]],)
    if s.op in ("SoftmaxOutput",):
        return (in_shape[0],)
    if s.op == "LinearRegressionOutput":
        return tuple(in_shape)
    return None


class _ShapeRun:
    def __init__(self, sym, known):
        self.sym, self.shapes, self.outputs = sym, dict(known), []

    def run(self):
        vals = {}
        for s in self.sym._topo():
            if s.op == "null":
                shp = self.shapes.get(s.name) or s.attrs.get("__shape__")
                if shp is not None:
                    self.shapes[s.name] = tuple(shp)
                    vals[id(s)] = torch.zeros(tuple(shp))
                continue
            if s.op == "_group":
                continue
            data = vals.get(id(s.inputs[0])) if s.inputs else torch.zeros(())          # creation ops (zeros / ones / arange …) have no inputs
            if data is None:
                raise MXNetError("cannot infer the input shape of %s: provide the shape of %s" % (s.name, s.inputs[0].name))
            for i, inp in enumerate(s.inputs[1:], 1):
                if id(inp) not in vals:
                    if s.op == "_nd":
                        k = i - s.attrs["npos"]
                        shp = _nd_param_shape(s.attrs, s.attrs["sym_kwargs"][k], tuple(data.shape)) if 0 <= k < len(s.attrs["sym_kwargs"]) else None
                    else:
                        shp = _param_shape(s, i, tuple(data.shape))
                    if shp is None:
                        raise MXNetError("cannot infer the shape of %s" % inp.name)
                    self.shapes[inp.name] = shp
                    vals[id(inp)] = torch.zeros(shp)
            for ax in s.aux:
                if id(ax) not in vals:
                    shp = _param_shape(s, 1, tuple(data.shape))
                    self.shapes[ax.name] = shp
                    vals[id(ax)] = torch.ones(shp) if ax.name.endswith("_var") else torch.zeros(shp)
            with torch.no_grad():
                F.use_native(False)
                try:
                    vals[id(s)] = _eval_node(s, [vals[id(i)] for i in s.inputs], [vals[id(x)].clone() for x in s.aux], False)
                finally:
                    F.use_native(True)
        heads = self.sym.inputs if self.sym.op == "_group" else [self.sym]
        missing = [h.name for h in heads if id(h) not in vals]
        if missing:
            raise MXNetError("cannot infer the shape of %s: not enough input shapes given" % missing)
        self.outputs = [vals[id(h)] for h in heads]
        return self


def run_graph(sym, feed, training=False):
    """Evaluate ``sym`` on live tensors: ``feed`` maps every argument / auxiliary-state name to a torch tensor; gradients flow to whatever
    in ``feed`` requires grad.  Used by ``gluon.SymbolBlock``; returns the list of head tensors."""
    vals = {}
    for s in sym._topo():
        if s.op == "null":
            if s.name not in feed:
                raise MXNetError("run_graph: no value for %s" % s.name)
            vals[id(s)] = feed[s.name]
        elif s.op != "_group":
            vals[id(s)] = _eval_node(s, [vals[id(i)] for i in s.inputs], [vals[id(a)] for a in s.aux], training)
    heads = sym.inputs if sym.op == "_group" else [sym]
    return [vals[id(h)] for h in heads]


def _placement(symbol, default_ctx, group2ctx):
    """node name -> Context for every node that carries a ``ctx_group`` annotation present in ``group2ctx`` (reference: the PlaceDevice pass
    of src/executor/graph_executor.cc with _CrossDeviceCopy nodes, src/operator/cross_device_copy.cc)."""
    if not group2ctx:
        return {}
    out = {}
    for s in symbol._topo():
        g = s.attrs.get("__attr__", {}).get("ctx_group")
        if g is not None and g in group2ctx:
            out[s.name] = group2ctx[g]
    return out


class Executor:
    """Bound graph: ``forward(is_train)`` / ``backward(out_grads)`` with ``arg_dict`` / ``grad_dict`` / ``aux_dict`` / ``outputs``.

    ``group2ctx`` (manual model parallelism, ``mx.AttrScope(ctx_group=...)``): every operator runs on the device of its group; an input that
    lives elsewhere is brought over by a differentiable device-to-device copy (NVLink P2P ``cudaMemcpyPeerAsync`` through torch), the
    gradient travels back the same way — the reference inserts ``_CrossDeviceCopy`` nodes for this."""

    def __init__(self, symbol, ctx, args, grads, grad_req, aux, group2ctx=None):
        self._symbol, self._ctx = symbol, ctx
        self._place = _placement(symbol, ctx, group2ctx)
        self.arg_dict, self.grad_dict, self.aux_dict, self._req = args, grads, aux, grad_req
        self.arg_arrays = [args[n] for n in symbol.list_arguments()]
        self.grad_arrays = [grads.get(n) for n in symbol.list_arguments()]
        self.aux_arrays = [aux[n] for n in symbol.list_auxiliary_states()]
        self.outputs = []
        self._heads, self._leaves, self._monitor = None, None, None

    def forward(self, is_train=False, **kwargs):
        for k, v in kwargs.items():
            self.arg_dict[k][:] = v
        vals, leaves = {}, {}
        from . import profiler as _prof
        prof_on = _prof._state["running"] and (_prof._cfg["profile_symbolic"] or _prof._cfg["profile_all"])
        order = self._symbol._topo()
        aux_ids = {id(a) for s in order for a in s.aux}
        with torch.enable_grad() if is_train else torch.no_grad():
            for s in order:
                if s.op == "null":
                    if id(s) in aux_ids:
                        vals[id(s)] = self.aux_dict[s.name]._t
                    else:
                        t = self.arg_dict[s.name]._t.detach()
                        if is_train and self._req.get(s.name, "null") != "null":
                            t = t.requires_grad_(True)
                            leaves[s.name] = t
                        vals[id(s)] = t
                elif s.op != "_group":
                    ins = [vals[id(i)] for i in s.inputs]
                    auxs = [vals[id(a)] for a in s.aux]
                    if self._place:
                        # model parallelism: the node's group decides the device (un-annotated nodes follow their first input); inputs
                        # from another device cross over with a copy that autograd differentiates
                        where = self._place.get(s.name)
                        dev = where.torch_device if where is not None else (ins[0].device if ins else None)
                        if dev is not None:
                            ins = [t.to(dev) if (torch.is_tensor(t) and t.device != dev) else t for t in ins]
                            auxs = [t.to(dev) if (torch.is_tensor(t) and t.device != dev) else t for t in auxs]
                    if prof_on:                                        # one trace event per graph node, like ProfileOperator (threaded_engine.h:336-350)
                        with _prof.scope(s.name, "operator", device=self.arg_arrays[0]._t.is_cuda if self.arg_arrays else False):
                            vals[id(s)] = _eval_node(s, ins, auxs, is_train)
                    else:
                        vals[id(s)] = _eval_node(s, ins, auxs, is_train)
                    if self._monitor is not None:
                        self._monitor(s.name + "_output", NDArray(vals[id(s)].detach()))
        heads = self._symbol.inputs if self._symbol.op == "_group" else [self._symbol]
        self._heads, self._leaves = [vals[id(h)] for h in heads], leaves
        self.outputs = [NDArray(h.detach()) for h in self._heads]
        return self.outputs

    def backward(self, out_grads=None):
        if not self._leaves:
            raise MXNetError("backward needs forward(is_train=True) and at least one argument with grad_req != 'null'")
        heads = [h for h in self._heads if h.requires_grad]
        if out_grads is None:
            gs = [torch.ones_like(h) for h in heads]
        else:
            out_grads = out_grads if isinstance(out_grads, (list, tuple)) else [out_grads]
            gs = [g._t if isinstance(g, NDArray) else g for g in out_grads]
        names = list(self._leaves)
        grads = torch.autograd.grad(heads, [self._leaves[n] for n in names], gs, allow_unused=True)
        for n, g in zip(names, grads):
            if g is None:
                continue
            tgt = self.grad_dict[n]._t
            if self._req.get(n) == "add":
                tgt.add_(g)
            else:
                tgt.copy_(g)

    @property
    def output_dict(self):
        return dict(zip(self._symbol.list_outputs(), self.outputs))

    def set_monitor_callback(self, callback, monitor_all=False):
        """``callback(name, NDArray)`` for every node output of each forward (executor.py:237-260; used by ``mx.monitor.Monitor``)."""
        self._monitor = callback

    def reshape(self, partial_shaping=False, allow_up_sizing=False, **kwargs):
        """New executor for different input shapes sharing every parameter array whose shape did not change (executor.py:380-460)."""
        new = self._symbol.simple_bind(self._ctx, grad_req=self._req, **kwargs)
        for n, a in self.arg_dict.items():
            if n in new.arg_dict and tuple(new.arg_dict[n].shape) == tuple(a.shape) and n not in kwargs:
                new.arg_dict[n] = a
                if n in self.grad_dict and n in new.grad_dict:
                    new.grad_dict[n] = self.grad_dict[n]
        for n, a in self.aux_dict.items():
            if n in new.aux_dict and tuple(new.aux_dict[n].shape) == tuple(a.shape):
                new.aux_dict[n] = a
        new.arg_arrays = [new.arg_dict[n] for n in self._symbol.list_arguments()]
        new.grad_arrays = [new.grad_dict.get(n) for n in self._symbol.list_arguments()]
        new.aux_arrays = [new.aux_dict[n] for n in self._symbol.list_auxiliary_states()]
        return new

    def debug_str(self):
        return self._symbol.debug_str()

    def copy_params_from(self, arg_params, aux_params=None, allow_extra_params=False):
        for k, v in arg_params.items():
            if k in self.arg_dict:
                self.arg_dict[k][:] = v
            elif not allow_extra_params:
                raise MXNetError("unknown argument %s" % k)
        for k, v in (aux_params or {}).items():
            if k in self.aux_dict:
                self.aux_dict[k][:] = v


def pow(base, exp):
    """``mx.sym.pow``: Symbol/scalar base and exponent in any combination."""
    if isinstance(base, Symbol):
        return base ** exp
    if isinstance(exp, Symbol):
        return _nd_op("power")(Symbol("_full_like", _auto_name("scalar", None), [exp], {"value": float(base)}), exp)
    return base ** exp


def _attach_symbol_fluent():
    names = ["abs", "arccos", "arccosh", "arcsin", "arcsinh", "arctan", "arctanh", "argmax", "argmax_channel", "argmin", "argsort", "broadcast_axes",
             "broadcast_like", "broadcast_to", "cbrt", "ceil", "clip", "cos", "cosh", "degrees", "depth_to_space", "diag", "exp", "expand_dims", "expm1",
             "fix", "flatten", "flip", "floor", "log", "log10", "log1p", "log2", "log_softmax", "max", "mean", "min", "nanprod", "nansum", "norm",
             "one_hot", "ones_like", "pad", "pick", "prod", "radians", "rcbrt", "reciprocal", "relu", "repeat", "reshape_like", "rint", "round",
             "rsqrt", "shape_array", "sigmoid", "sign", "sin", "sinh", "size_array", "slice", "slice_axis", "slice_like", "softmax", "softmin", "sort",
             "space_to_depth", "split", "sqrt", "square", "squeeze", "sum", "swapaxes", "take", "tan", "tanh", "tile", "topk", "transpose", "trunc", "zeros_like"]
    for n in names:
        if not hasattr(Symbol, n):
            setattr(Symbol, n, (lambda q: lambda self, *a, **k: _nd_op(q)(self, *a, **k))(n))
    Symbol.reshape = lambda self, *shape, **kw: reshape(self, shape[0] if len(shape) == 1 and isinstance(shape[0], (tuple, list)) else (kw.get("shape") or shape))
    Symbol.astype = lambda self, dtype: _nd_op("cast")(self, dtype=str(dtype))
    Symbol.detach = lambda self: _nd_op("stop_gradient")(self)
    Symbol.copy = lambda self: load_json(self.tojson())
    for n in ("asnumpy", "asscalar", "wait_to_read", "as_in_context", "backward"):
        setattr(Symbol, n, (lambda q: lambda self, *a, **k: (_ for _ in ()).throw(
            NotImplementedError("Symbol.%s: symbols hold no data — bind them (simple_bind / eval) first" % q)))(n))


_attach_symbol_fluent()


# the reference's sub-module paths (python/mxnet/symbol/{symbol,register}.py)
def _register_paths():
    from ._alias import submodule
    g = globals()
    submodule(__name__, "symbol", {k: g[k] for k in ("Symbol", "Variable", "var", "Group", "load", "load_json") if k in g})
    submodule(__name__, "register", {"_nd_op": _nd_op}, doc="operators are bridged from mx.nd on attribute access: nothing to generate")


_register_paths()
