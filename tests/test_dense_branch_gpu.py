"""The dense branch of the classic step (even B <= 32, one rank, paths A-C of ``tests/test_step_paths_gpu.py``).  There the forward kernel
runs the dense chain down to dz3 and stores everything ``dense_wgrad_kernel`` reads, and the tail (``dense_tail_kernel`` from dz3) only turns
dz3 into da2.  So the dense weight gradients branch off right after the forward kernel.  The dense keys' exchange writes W0, which the tail
reads, so it waits for both the weight gradients and the tail: through a programmatic edge from the weight gradients, and a full edge
from the tail on the other branch.

The first test reads these dependencies off the captured graph: the DOT text of ``CUDAGraph.debug_dump``, and the driver's edge types,
which the DOT text does not show.  The second runs one graphed step at lr > 0, where an exchange that overtook the tail would change W0
under it: da2, and with it the conv gradients, would no longer match the weights the step started from."""
import ctypes
import re

import pytest
import torch

import geomx_b200 as mx
from _cnn_ref import GRAD_NAMES, dev, engine, images, nat, rel_err, step_params, step_reference  # noqa: F401  (nat, engine: fixtures)

pytestmark = pytest.mark.gpu

FWD, TAIL, WGRAD, EXCHANGE = "cnn_fwd_dense0_kernel", "dense_tail_kernel", "dense_wgrad_kernel", "hips_fsa_step_single_kernel"
# paths A, B, C at B = 32: the step switches that select them
CLASSIC = {"A": {}, "B": {"GEOMX_CNN_BWD_ONE_LAUNCH": "0"}, "C": {"GEOMX_FUSED_EXCHANGE": "1"}}

_EDGE = re.compile(r'^\s*"([^"]+)"\s*->\s*"([^"]+)"')
_NODE = re.compile(r'^\s*"([^"]+)"\s*\[')
_HANDLE = re.compile(r"node handle \| func handle\} \| \{(0x[0-9A-Fa-f]+)")


def parse_dot(text):
    """cudaGraphDebugDotPrint's output -> ({node: its text}, [(from, to)]).  A node's text runs from its
    definition to the next node or edge line (its label spans several lines)."""
    nodes, edges, cur = {}, [], None
    for line in text.splitlines():
        m = _EDGE.match(line)
        if m:
            edges.append((m.group(1), m.group(2)))
            cur = None
            continue
        m = _NODE.match(line)
        if m:
            cur = m.group(1)
            nodes[cur] = ""
        if cur is not None:
            nodes[cur] += line + "\n"
    return nodes, edges


def edge_types(graph):
    """{(source node handle, destination node handle): dependency type} of every edge of a kept graph, from the driver
    (cuGraphGetEdges_v2: type 0 full, 1 programmatic)."""
    cu = ctypes.CDLL("libcuda.so.1")
    g, n = ctypes.c_void_p(graph.raw_cuda_graph()), ctypes.c_size_t(0)
    assert cu.cuGraphGetEdges_v2(g, None, None, None, ctypes.byref(n)) == 0
    src, dst = (ctypes.c_void_p * n.value)(), (ctypes.c_void_p * n.value)()
    data = (ctypes.c_ubyte * (8 * n.value))()        # CUgraphEdgeData: from_port, to_port, type, 5 reserved bytes
    assert cu.cuGraphGetEdges_v2(g, src, dst, data, ctypes.byref(n)) == 0
    return {(src[i], dst[i]): data[8 * i + 2] for i in range(n.value)}


def handle(node_text):
    return int(_HANDLE.search(node_text).group(1), 16)


def kernel_nodes(nodes, name):
    return [n for n, txt in nodes.items() if name in txt]


def reachable(edges, start):
    succ = {}
    for a, b in edges:
        succ.setdefault(a, []).append(b)
    seen, todo = set(), [start]
    while todo:
        for b in succ.get(todo.pop(), []):
            if b not in seen:
                seen.add(b)
                todo.append(b)
    return seen


@pytest.mark.parametrize("path", list(CLASSIC))
def test_dense_wgrad_forks_after_the_forward_kernel(nat, engine, tmp_path, path):
    B = 32
    eng = engine(B, mx.optimizer.Adam(learning_rate=0.01), env=CLASSIC[path], use_graph=True)
    assert (eng.path.dense, eng.path.wgrad) == ("dz3", "comm"), eng.path
    g = torch.Generator().manual_seed(500)
    eng.x.copy_(images(g, B, "rand")); eng.label.copy_(torch.randint(0, 10, (B,), generator=g).float())
    for _ in range(2):       # the first launch of each kernel configures it (shared memory, cluster occupancy) outside the capture
        eng._body()
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph(keep_graph=True)     # (debug_dump prints the graph it kept)
    graph.enable_debug_mode()
    with torch.cuda.graph(graph):
        eng._body()
    dot = tmp_path / "step.dot"
    graph.debug_dump(str(dot))
    nodes, edges = parse_dot(dot.read_text())
    found = {k: kernel_nodes(nodes, k) for k in (FWD, TAIL, WGRAD)}
    assert all(len(v) == 1 for v in found.values()), found
    fwd, tail, wgrad = found[FWD][0], found[TAIL][0], found[WGRAD][0]
    after_fwd, after_tail, after_wgrad = reachable(edges, fwd), reachable(edges, tail), reachable(edges, wgrad)
    assert wgrad in after_fwd, "dense_wgrad_kernel does not depend on the forward kernel"
    assert wgrad not in after_tail, "dense_wgrad_kernel waits for the tail, which it has no data from"
    # the dense keys' channel: the one exchange launch behind the weight gradients (the conv keys' exchange follows the backward pass)
    dense_kv = [n for n in kernel_nodes(nodes, EXCHANGE) if n in after_wgrad]
    assert len(dense_kv) == 1, (dense_kv, kernel_nodes(nodes, EXCHANGE))
    assert dense_kv[0] in after_tail, "the dense keys' exchange writes W0 while the tail may still read it"
    # forward kernel -> tail stays a programmatic edge: the tail stages W0 while the forward kernel runs.  The DOT text only numbers each
    # node's in-edges (headlabel), so the type comes from the driver, matched by the node handles the DOT text prints
    assert [e for e in edges if e[1] == tail] == [(fwd, tail)], edges
    types = edge_types(graph)
    h = lambda node: handle(nodes[node])
    assert types[(h(fwd), h(tail))] == 1, "forward kernel -> tail is not a programmatic edge"
    # the channel stages its tiles behind the weight gradients (programmatic) and waits for the tail on the other branch (full)
    assert types[(h(wgrad), h(dense_kv[0]))] == 1 and types[(h(tail), h(dense_kv[0]))] == 0, types


def test_graphed_sgd_step_reads_w0_before_the_update(nat, engine):
    """One replay of the captured step with SGD at lr = 0.5, gradients left readable: the loss, logits and all ten gradients match fp64
    computed from the parameters the step started from, and every parameter is then P - lr * G / B (the push scale 1 / B)."""
    B, lr = 32, 0.5
    eng = engine(B, mx.optimizer.SGD(learning_rate=lr, momentum=0.0, wd=0.0), use_graph=True, fused_zero_grad=False)
    assert (eng.path.dense, eng.path.wgrad) == ("dz3", "comm"), eng.path
    g = torch.Generator().manual_seed(501)
    P0 = step_params(g)
    X = images(g, B, "rand")
    y = torch.randint(0, 10, (B,), generator=g).float().to(dev())
    eng.capture()            # its two warm-up steps are real updates: the parameters are set after it
    for p, v in zip(eng.P, P0):
        p.copy_(v)
    eng.fabric.load_master_from_param()
    eng.x.copy_(X); eng.label.copy_(y)
    torch.cuda.synchronize()
    eng.graph.replay()
    torch.cuda.synchronize()
    loss_ref, logits_ref, grads_ref, _ = step_reference(P0, X, y, eng.idx1, eng.idx2)
    errs = {"loss": rel_err(eng.loss, loss_ref), "logits": rel_err(eng.logits, logits_ref)}
    errs.update({n: rel_err(a, b) for n, a, b in zip(GRAD_NAMES, eng.G, grads_ref)})
    bad = {k: v for k, v in errs.items() if not v < 2e-5}
    assert not bad, bad
    for i, (p, p0, grad) in enumerate(zip(eng.P, P0, eng.G)):
        step = lr * (grad / B)
        err = float((p - (p0 - step)).abs().max()) / float(p0.abs().max() + step.abs().max())
        assert err < 1e-6, "parameter %d is not P - lr * G / B (%.2e)" % (i, err)
