"""Short and sample-weighted batches in ``HipsCNNTrainStep.step_async(X, y, sample_weight)``.

A batch of ``n <= B`` rows with weights ``w`` contributes ``(1/n) * sum_i w_i grad_i``: the engine pads it to ``B`` rows and gives row i
the coefficient ``c_i = w_i * B / n`` (0 for padding rows), which the weighted instance of the kernel producing the dlogits applies.  With
``fused_zero_grad=False`` the gradient arena ``G`` after a step holds ``sum_i c_i grad_i``, which is checked against fp64 on every kernel
path of ``test_step_paths_gpu.py``.

Bitwise comparisons between two engines freeze the convolution keys (``lr_mult = 0``): conv0's weight gradient is summed with atomics, so
two runs of the same step differ in its last bits, and through the next forward pass everywhere.  With the convolution weights fixed the
rest of the step is deterministic, and a weighted step that should equal an unweighted one must equal it bit for bit."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import geomx_b200 as mx
from geomx_b200.models.cnn import CNN_PARAM_NAMES
from geomx_b200.parallel import Topology

import _update_ref as U
from _cnn_ref import CASE_IDS, CASES, GRAD_NAMES, PATHS, ROOT, dev, engine, images, nat, step_params, step_reference  # noqa: F401

pytestmark = pytest.mark.gpu

FROZEN_CONV = {0: 0.0, 1: 0.0, 2: 0.0, 3: 0.0}


def coefficients(B, n, w):
    c = torch.zeros(B, dtype=torch.float64)
    c[:n] = (torch.ones(n, dtype=torch.float64) if w is None else w.double()) * B / n
    return c


def frozen(opt):
    """``opt`` with the convolution keys frozen (lr_mult = 0)."""
    opt.set_lr_mult(FROZEN_CONV)
    return opt


def variants(B):
    """(n, weighted) pairs: short batches at n = 1, odd, even and B - 1 (the odd one also weighted), and a weighted full batch."""
    odd = next((k for k in range(B // 2 | 1, 0, -2) if 1 < k < B - 1), None)
    even = next((k for k in range(B // 2, 0, -1) if k % 2 == 0 and k not in (1, B - 1)), None)
    out = [(k, k == odd) for k in sorted({1, B - 1} | {v for v in (odd, even) if v}) if 1 <= k < B]
    return out + [(B, True)]


def same_init(a, b):
    """Give engine ``b`` engine ``a``'s parameters (and, with local updates, its worker weights)."""
    for p, q in zip(b.P, a.P):
        p.copy_(q)
    if b.update == "local":
        b.fabric.param.tensor.copy_(a.fabric.param.tensor)
    b.fabric.load_master_from_param()
    torch.cuda.synchronize()


def state(e):
    """Parameters and optimizer state (master, s0, s1, step count) of every key as host arrays."""
    return {k: v for k, v in e._ckpt_state(with_batch=False).items() if not k.startswith("meta:")}


def assert_same_state(a, b):
    """Every parameter, master weight, step count and the dense keys' optimizer state bit for bit (``==``: +0 equals -0).  The frozen
    conv keys' optimizer state follows their gradients, whose atomic sums differ in the last bits between runs: 1e-5 relative."""
    sa, sb = state(a), state(b)
    assert sa.keys() == sb.keys()
    for k in sa:
        if k.split(":")[0] in ("s0", "s1") and k.split(":")[1] in CNN_PARAM_NAMES[:4]:
            assert U.rel(sb[k], sa[k]) < 1e-5, k
        else:
            assert np.array_equal(sa[k], sb[k]), k


def batch(g, n, kind="rand"):
    return images(g, n, kind).cpu(), torch.randint(0, 10, (n,), generator=g).float()


# ------------------------------------------------------------------------------------------------------------- 1. gradients vs fp64
@pytest.mark.parametrize("path,B,env", CASES, ids=CASE_IDS)
def test_partial_and_weighted_gradients_match_fp64(nat, engine, path, B, env):
    """Short batches (n = 1, odd, even, B - 1) and a weighted full batch on every kernel path: G = sum_i c_i grad_i and the per-sample loss
    against fp64 (2e-5 relative, as the full-batch path tests); the handle reports w_i * loss_i and its mean over n."""
    g = torch.Generator().manual_seed(500 + 3 * B + ord(path))
    P0 = step_params(g)
    eng = engine(B, env=env, use_graph=False, fused_zero_grad=False)
    for p, v in zip(eng.P, P0):
        p.copy_(v)
    eng.fabric.load_master_from_param()
    assert [(n, s) for n, s, _ in eng._steps()] == PATHS[path][3]
    for n, weighted in variants(B):
        X, y = batch(g, n, "patch" if n % 2 else "rand")
        w = (0.2 + 1.8 * torch.rand(n, generator=g)) if weighted else None
        h = eng.step_async(X, y, w)
        lw = h.wait()
        torch.cuda.synchronize()
        Xp = torch.zeros(B, 1, 28, 28); Xp[:n] = X
        yp = torch.zeros(B); yp[:n] = y
        c = coefficients(B, n, w)
        loss_ref, _, grads_ref, _ = step_reference(P0, Xp.to(dev()), yp.to(dev()), eng.idx1, eng.idx2, coef=c)
        errs = {n_: U.rel(a, b) for n_, a, b in zip(GRAD_NAMES, eng.G, grads_ref)}
        lref = loss_ref[:n].cpu() * (1.0 if w is None else w.double())
        errs["loss"] = U.rel(lw, lref)
        errs["item"] = abs(h.item() - float(lref.mean())) / float(lref.abs().mean())
        assert lw.shape == (n,)
        print("\n  path %s B=%-2d n=%-2d %s  %s" % (path, B, n, "w" if weighted else " ", "  ".join("%s %.1e" % kv for kv in errs.items())))
        bad = {k: v for k, v in errs.items() if not v < 2e-5}
        assert not bad, (path, B, n, bad)
        for i, (p, p0) in enumerate(zip(eng.P, P0)):
            assert torch.equal(p, p0), "parameter %d changed by an lr = 0 step" % i


# ------------------------------------------------------------------------------------------------------------- 2. ones are exact
MODES = {
    "server": (32, lambda: mx.optimizer.Adam(learning_rate=0.01, wd=0.01), {}),
    "local": (32, lambda: mx.optimizer.Adam(learning_rate=0.01), {"update": "local"}),
    "hfa": (32, lambda: mx.optimizer.Adam(learning_rate=0.01), {"hfa": (2, 2)}),
    "async": (32, lambda: mx.optimizer.Adam(learning_rate=0.01), {"mode": "dist_async"}),
    "lookahead": (32, lambda: mx.optimizer.Adam(learning_rate=0.01), {"lookahead": True, "loopback": True, "topo": Topology(1, 0, 1, 0)}),
    "gemm": (33, lambda: mx.optimizer.SGD(learning_rate=0.1, momentum=0.9), {}),
}


@pytest.mark.parametrize("mode", list(MODES))
def test_unit_weights_are_bitwise_unweighted(nat, engine, mode):
    """sample_weight = ones(B) replays the weighted graph, and its coefficient 1 must leave every bit as the unweighted step has it:
    parameters, optimizer state and the reported loss, over several steps (conv keys frozen, see the module docstring)."""
    B, opt, kw = MODES[mode]
    g = torch.Generator().manual_seed(11)
    a, b = engine(B, frozen(opt()), **kw), engine(B, frozen(opt()), **kw)
    same_init(a, b)
    la, lb = [], []
    for _ in range(4):
        X, y = batch(g, B)
        la.append(a.step(X, y))
        lb.append(b.step(X, y, torch.ones(B)))
    if a.lookahead:
        la.append(a.flush()); lb.append(b.flush())
    torch.cuda.synchronize()
    assert b._graph_w and not a._graph_w
    assert a.kernels_per_step == b.kernels_per_step
    if a.lookahead:     # flush(): the device mean of an unweighted batch, the host mean of a weighted one
        fa, fb = la.pop(), lb.pop()
        assert abs(fa - fb) <= 1e-5 * abs(fa), (fa, fb)
    assert np.array_equal(np.array(la), np.array(lb), equal_nan=True), (la, lb)
    assert_same_state(a, b)


# ------------------------------------------------------------------------------------------------------------- 3. zero-weight rows
@pytest.mark.parametrize("B", [32, 31, 48])
def test_zero_weight_rows_are_inert(nat, engine, B):
    """Rows of weight 0 contribute exact zeros: other finite images and labels in them leave parameters and optimizer state bitwise equal."""
    g = torch.Generator().manual_seed(21 + B)
    opt = lambda: mx.optimizer.Adam(learning_rate=0.01)
    a, b = engine(B, frozen(opt())), engine(B, frozen(opt()))
    same_init(a, b)
    for _ in range(3):
        X, y = batch(g, B)
        w = torch.rand(B, generator=g) + 0.5
        w[torch.randperm(B, generator=g)[:B // 3]] = 0.0
        X2, y2 = X.clone(), y.clone()
        zero = w == 0
        X2[zero] = torch.rand(int(zero.sum()), 1, 28, 28, generator=g) * 3
        y2[zero] = torch.randint(0, 10, (int(zero.sum()),), generator=g).float()
        la, lb = a.step_async(X, y, w).wait(), b.step_async(X2, y2, w).wait()
        assert torch.equal(la, lb)
    torch.cuda.synchronize()
    assert_same_state(a, b)


# ------------------------------------------------------------------------------------------------------------- 4. a batch-n engine
@pytest.mark.parametrize("B,n,kw", [(32, 12, {}), (48, 31, {}), (32, 7, {"lookahead": True, "loopback": True, "topo": Topology(1, 0, 1, 0)})],
                         ids=["A-n12", "D-n31", "lookahead-n7"])
def test_short_batch_matches_batch_n_engine(nat, engine, B, n, kw):
    """A short batch of n rows on a batch-B engine updates the weights as an engine built for batch n does on the same rows (SGD; fp32
    tolerance: the two run different kernel paths), for three steps."""
    g = torch.Generator().manual_seed(31 + n)
    opt = lambda: mx.optimizer.SGD(learning_rate=0.1, momentum=0.9)
    big, small = engine(B, opt(), **kw), engine(n, opt(), **kw)
    same_init(big, small)
    P0 = [p.clone() for p in big.P]
    for _ in range(3):
        X, y = batch(g, n)
        big.step(X, y); small.step(X, y)
    if big.lookahead:
        big.flush(); small.flush()
    torch.cuda.synchronize()
    errs = [U.rel(pb - p0, ps - p0) for pb, ps, p0 in zip(big.P, small.P, P0)]
    print("\n  B=%d n=%d: displacement rel err %s" % (B, n, " ".join("%.1e" % e for e in errs)))
    assert max(errs) < 1e-4, errs


# ------------------------------------------------------------------------------------------------------------- 5. graphs
def test_weighted_graphs(nat, engine):
    """Weighted steps replay graphs of their own, one per input buffer, with the step's kernel count; a full unweighted step afterwards
    replays the original graph, captured once; set_learning_rate drops both kinds."""
    B = 32
    g = torch.Generator().manual_seed(41)
    eng = engine(B, mx.optimizer.SGD(learning_rate=0.01))
    eng.step(*batch(g, B))
    eng.step(*batch(g, B))
    g0, g1, k = eng.graph, eng._graph_alt, eng.kernels_per_step
    assert g0 is not None and g1 is not None and not eng._graph_w
    for n in (B - 5, 9):
        eng.step(*batch(g, n))
        assert eng.kernels_per_step == k
    assert set(eng._graph_w) == {0, 1}
    gw = dict(eng._graph_w)
    eng.step(*batch(g, B)); eng.step(*batch(g, B))
    eng.step(*batch(g, B), sample_weight=torch.rand(B, generator=g))
    assert eng.graph is g0 and eng._graph_alt is g1 and eng._graph_w == gw
    eng.set_learning_rate(0.02)
    assert eng.graph is None and not eng._graph_w
    eng.step(*batch(g, 3))
    assert eng._graph_w and eng.kernels_per_step == k


# ------------------------------------------------------------------------------------------------------------- 6. look-ahead checkpoint
def test_lookahead_short_batch_checkpoint(nat, engine, tmp_path):
    """A short, weighted batch primed last before flush(): a save_states / load_states round trip resumes it bitwise (conv keys frozen),
    the file holds batch:weight, and a file saved with a full unweighted primed batch does not."""
    B = 32
    g = torch.Generator().manual_seed(51)
    kw = dict(lookahead=True, loopback=True, topo=Topology(1, 0, 1, 0))
    opt = lambda: mx.optimizer.Adam(learning_rate=0.01)
    a = engine(B, frozen(opt()), **kw)
    for _ in range(2):
        a.step(*batch(g, B))
    full = str(tmp_path / "full.params")
    a.save_states(full)
    assert "batch:weight" not in mx.nd.load(full)
    X, y = batch(g, 13)
    w = torch.rand(13, generator=g) + 0.5
    a.step(X, y, w)
    short = str(tmp_path / "short.params")
    a.save_states(short)
    c = mx.nd.load(short)["batch:weight"].asnumpy()
    assert c.shape == (1, B) and np.array_equal(c[0, 13:], np.zeros(B - 13, np.float32))
    assert np.allclose(c[0, :13], w.numpy() * B / 13, rtol=1e-6)
    b = engine(B, frozen(opt()), **kw)
    b.load_states(short)
    la, lb = a.flush(), b.flush()
    torch.cuda.synchronize()
    assert la == la and abs(la - lb) <= 1e-6 * abs(la), (la, lb)
    assert_same_state(a, b)


def test_lookahead_short_batch_before_flush_trains(nat, engine):
    """The last, short batch of a look-ahead run is trained by flush() with its own coefficients: the same weights (within fp32) as an
    engine without look-ahead after the same batches."""
    B = 32
    g = torch.Generator().manual_seed(61)
    opt = lambda: mx.optimizer.SGD(learning_rate=0.1)
    la = engine(B, opt(), lookahead=True, loopback=True, topo=Topology(1, 0, 1, 0))
    plain = engine(B, opt(), loopback=True, topo=Topology(1, 0, 1, 0))
    same_init(la, plain)
    P0 = [p.clone() for p in la.P]
    batches = [batch(g, B), batch(g, B), batch(g, 5)]
    for X, y in batches:
        la.step(X, y); plain.step(X, y)
    loss = la.flush()
    torch.cuda.synchronize()
    errs = [U.rel(p - p0, q - p0) for p, q, p0 in zip(la.P, plain.P, P0)]
    assert max(errs) < 1e-4 and loss == loss, (errs, loss)


# ------------------------------------------------------------------------------------------------------------- 7. errors
def test_refusals_enqueue_nothing(nat, engine):
    from geomx_b200.ops import native
    B = 8
    eng = engine(B, use_graph=False)
    X, y = batch(torch.Generator().manual_seed(71), B + 1)
    eng.step(X[:B], y[:B])
    torch.cuda.synchronize()
    before = (native.launch_count, eng.steps_done, eng._pipeline()["n"])
    for args in ((X[:0], y[:0]), (X, y), (X[:4], y[:5]), (X[:4], y[:4], torch.ones(5)), (X[:B], y[:B], torch.ones(B - 1))):
        with pytest.raises(ValueError):
            eng.step_async(*args)
    assert (native.launch_count, eng.steps_done, eng._pipeline()["n"]) == before


# ------------------------------------------------------------------------------------------------------------- 8. several ranks
def _ngpus():
    return torch.cuda.device_count() if torch.cuda.is_available() else 0


@pytest.mark.multigpu
@pytest.mark.skipif(_ngpus() < 2, reason="needs >= 2 GPUs")
def test_two_ranks_short_and_full(tmp_path):
    """Rank 0 passes a short, weighted batch and rank 1 a full one in the same step: the update is the fp64 sum of both contributions."""
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", "29731", os.path.join(ROOT, "tools", "partial_batch_check.py")]
    r = subprocess.run(cmd, cwd=ROOT, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=300)
    assert r.returncode == 0 and "PARTIAL_BATCH_CHECK PASS" in r.stdout, r.stdout[-3000:]
