"""``HipsCNNTrainStep.save_states`` / ``load_states`` on the GPU: a saved engine loads into a fresh one bit for bit, the first update
after the load is the fp64 reference's update from the saved state, dropping any piece of the state on load is caught, and a resumed run
tracks an uninterrupted one.  Gradients stay readable (``fused_zero_grad=False``).  The two engines are not compared bit for bit after a
step: conv0's weight gradient is summed with atomics."""
import gc
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import geomx_b200 as mx
from geomx_b200.models.cnn import CNN_PARAM_NAMES, STEP_SWITCHES

import _optim_ref as R
import _update_ref as U

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TOL = R.DISP_TOL
# MPQ + DGT re-ranks every 4 steps: once before the save (after step 4) and once among the steps after the load (before step 8)
N_BEFORE, K_AFTER = 5, 3
# The resumed wire-format runs are compared with the uninterrupted run across K_AFTER + 1 steps.  Two uninterrupted MPQ + DGT runs of the
# same seed and batches already differ there: conv0's weight gradient is summed with atomics, and the fp16 / fp8 wire rounding and the
# re-ranking amplify its last-bit differences (measured on an H100 over five runs: 6e-7 .. 9.7e-4).  The bound is 5x the largest.
WIRE_RUN_TOL = 5e-3

OPTS = {
    "adam": lambda: mx.optimizer.Adam(learning_rate=0.01, wd=0.01),
    "sgd": lambda: mx.optimizer.SGD(learning_rate=0.1, momentum=0.9, wd=0.01),
    "sgd0": lambda: mx.optimizer.SGD(learning_rate=0.1),
    "dcasgd": lambda: mx.optimizer.DCASGD(learning_rate=0.1, momentum=0.9, lamda=40.0, wd=0.01),
    "ftrl": lambda: mx.optimizer.Ftrl(learning_rate=0.01, lamda1=1e-5, beta=1e-6),
}
# name -> (B, step switches, optimizer, engine kwargs, graph).  The wire-format cases (Bi-Sparse, MPQ + DGT) are checked against the
# uninterrupted engine's next update; the others against the fp64 reference.
CASES = {
    "channel-adam-graph": (32, {}, "adam", {}, True),
    "ll-loopback-adam": (32, {"GEOMX_STEP_OVERLAP": "0"}, "adam", dict(loopback=True), False),
    "local-adam": (32, {}, "adam", dict(update="local"), False),
    "bsc-sgd": (32, {"GEOMX_STEP_OVERLAP": "0"}, "sgd", dict(loopback=True, bsc_threshold=0.01, size_lower_bound=100000), False),
    "mpq-dgt-sgd": (32, {"GEOMX_STEP_OVERLAP": "0"}, "sgd0", dict(loopback=True, wire_dtype="mpq", dgt=True, dgt_rerank_every=4,
                                                                  size_lower_bound=10000), False),
    "async-adam": (32, {}, "adam", dict(mode="dist_async"), False),
    "lookahead-adam-graph": (32, {}, "adam", dict(lookahead=True), True),
    "b64-sgd-graph": (64, {}, "sgd", {}, True),
    "dcasgd": (32, {}, "dcasgd", {}, False),
    "ftrl": (32, {}, "ftrl", {}, False),
}
WIRE = ("bsc-sgd", "mpq-dgt-sgd")


@pytest.fixture
def clean_env(monkeypatch):
    for k in STEP_SWITCHES + ("GEOMX_FABRIC_PROTOCOL", "GEOMX_FABRIC_DIRECT", "DMLC_K", "ADAPTIVE_K_FLAG"):
        monkeypatch.delenv(k, raising=False)
    return monkeypatch


def _cleanup():
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def _make(name, seed=0):
    from geomx_b200.parallel import Topology
    B, _, kind, kw, graph = CASES[name]
    torch.manual_seed(seed)
    return mx.models.HipsCNNTrainStep(batch_size=B, optimizer=OPTS[kind](), topo=Topology(1, 0, 1, 0 if kw.get("loopback") else 1),
                                      use_graph=graph, fused_zero_grad=False, **kw)


def _batches(B, n, seed=11):
    g = torch.Generator().manual_seed(seed)
    return [(torch.rand(B, 1, 28, 28, generator=g).cuda(), torch.randint(0, 10, (B,), generator=g).float().cuda()) for _ in range(n)]


def _master(eng):
    return eng.Wl if eng.update == "local" else eng.fabric.w


def _keys(eng, t):
    return [eng.layout.view(t, i).detach().cpu().clone() for i in range(10)]


def _device_state(eng):
    """Every device tensor that load_states restores (clones)."""
    f = eng.fabric
    ts = {"P%d" % i: p for i, p in enumerate(eng.P)}
    if eng.update == "local":
        ts.update(Wl=eng.Wl, s0l=eng.s0l, s1l=eng.s1l, step=eng.opt_state[:1])
    else:
        ts.update(w=f.w, s0=f.s0, s1=f.s1)
        if eng.mode == "dist_async":
            ts["step"] = f.flags.tensor[f.off["async_step"]: f.off["async_step"] + f.tiles]
        else:
            ts["step"] = torch.stack([f.state[n][2] for n in (list(f.channels) or ["fsa"])])
    if f.bsc_u is not None:
        ts.update(bsc_u=f.bsc_u, bsc_v=f.bsc_v)
    if f.dgt_contrib is not None:
        ts.update(dgt_contrib=f.dgt_contrib, tile_order=f.tile_order, tile_fmt=f.tile_fmt)
    if eng.lookahead and eng._primed:
        ts.update(x=eng.x_cur, label=eng.label_cur, a2=eng.a2)
    return {k: v.detach().clone() for k, v in ts.items()}


def _load_file(path):
    return {k: v.asnumpy() for k, v in mx.nd.load(path).items()}


def _save_file(path, d):
    mx.nd.save(path, {k: mx.nd.NDArray(torch.from_numpy(np.ascontiguousarray(v))) for k, v in d.items()})
    return path


def _reference(eng, saved, grads):
    """fp64 update of every key from the saved state and the engine's own gradient sums of the step after the load."""
    spec = eng._local_spec if eng.update == "local" else eng.fabric.opt_spec
    h = R.hyper(spec)
    out = []
    for i, n in enumerate(CNN_PARAM_NAMES):
        w = torch.from_numpy(saved["master:" + n]).double()
        s0, s1 = torch.from_numpy(saved["s0:" + n]).double(), torch.from_numpy(saved["s1:" + n]).double()
        t = int(saved["step:" + n].max()) + 1
        R.update(h, w, grads[i].double() * (1.0 / eng.B), s0, s1, t)
        out.append(w)
    return out


def _mutations(name, saved):
    """name -> the entry prefixes whose load is skipped (the loading engine keeps its own values there), or None for the primed batch."""
    kind = CASES[name][2]
    out = {}
    if kind != "sgd0":
        out["skip s0"] = ("s0:",)
    if kind in ("adam", "dcasgd", "ftrl"):
        out["skip s1"] = ("s1:",)
    if kind == "adam":
        out["reset the step count"] = ("step:",)
    if "bsc_u:4.weight" in saved:
        out["skip the Bi-Sparse residual"] = ("bsc_u:", "bsc_v:")
    if "dgt:order" in saved:
        out["skip the DGT order"] = ("dgt:order", "dgt_fmt:")
    if "batch:x" in saved:
        out["forget the primed batch"] = None
    return out


@pytest.mark.parametrize("name", list(CASES))
def test_save_load_resume(clean_env, tmp_path, name):
    B, env, kind, kw, graph = CASES[name]
    for k, v in env.items():
        clean_env.setenv(k, v)
    batches = _batches(B, N_BEFORE + 1 + K_AFTER)
    a = _make(name, seed=1)
    for X, y in batches[:N_BEFORE]:
        a.step(X, y)
    if name == "b64-sgd-graph":
        a.set_learning_rate(0.05)          # a constant lr other than the optimizer's: the load applies it
    path = str(tmp_path / "ckpt.params")
    a.save_states(path)
    want = _device_state(a)
    meta = (a.opt_step, a.learning_rate, a.steps_done)
    saved = _load_file(path)
    if graph:
        # a load without an lr change leaves the captured graph and the launch count as they are
        g, kps = a.graph, a.kernels_per_step
        a.load_states(path)
        assert a.graph is g and a.kernels_per_step == kps
        assert all(torch.equal(v, want[k]) for k, v in _device_state(a).items())

    # round trip into a fresh engine: bit for bit
    b = _make(name, seed=2)
    b.load_states(path)
    got = _device_state(b)
    assert set(got) == set(want)
    diff = [k for k in want if not torch.equal(got[k], want[k])]
    assert not diff, (name, diff)
    assert (b.opt_step, b.learning_rate, b.steps_done) == meta, ((b.opt_step, b.learning_rate, b.steps_done), meta)

    # the live weights interoperate with build_cnn()
    net = mx.models.build_cnn()
    net.load_parameters(path, ignore_extra=True)
    assert all(torch.equal(p.data()._t.cpu(), q.cpu()) for p, q in zip(net.collect_params().values(), a.P))

    # the first update after the load: keys whose tiles are all fp32 against the fp64 reference from the saved state; keys with fp16 / fp8 /
    # Bi-Sparse tiles against the uninterrupted engine's update
    M_saved = [torch.from_numpy(saved["master:" + n]) for n in CNN_PARAM_NAMES]
    X, y = batches[N_BEFORE]
    twin = _make(name, seed=1) if name in WIRE else None        # a second uninterrupted run: the run-to-run spread of this config
    if twin is not None:
        for Xk, yk in batches[:N_BEFORE]:
            twin.step(Xk, yk)
    a.step(X, y)
    b.step(X, y)
    torch.cuda.synchronize()
    M_a, M_b = _keys(a, _master(a)), _keys(b, _master(b))
    fp64 = _reference(b, saved, [g.detach().cpu() for g in b.G])
    fp32_keys = _fp32_keys(saved)
    ref = [fp64[i] if i in fp32_keys else M_a[i].double() for i in range(10)]
    e_next = R.displacement_err(M_b, M_saved, ref, stores=1)
    print("\n  %-22s next update %.1e (%d keys against fp64)" % (name, e_next, len(fp32_keys)), end="")
    assert e_next < TOL, (name, e_next)

    # K more steps (MPQ + DGT: across a re-rank): the resumed run tracks the uninterrupted one
    if twin is not None:
        twin.step(X, y)
    for Xk, yk in batches[N_BEFORE + 1:]:
        for e in (a, b, twin):
            if e is not None:
                e.step(Xk, yk)
    torch.cuda.synchronize()
    P_saved = [torch.from_numpy(saved[n]) for n in CNN_PARAM_NAMES]
    P_a = [p.cpu().double() for p in a.P]
    e_run = R.displacement_err([p.cpu() for p in b.P], P_saved, P_a, stores=K_AFTER + 1)
    spread = R.displacement_err([p.cpu() for p in twin.P], P_saved, P_a, stores=K_AFTER + 1) if twin is not None else 0.0
    lookahead = b.lookahead
    print("  | resumed run %.1e (two uninterrupted runs: %.1e)" % (e_run, spread), end="")
    assert not b.fabric.check_protocol_errors()
    del a, b, twin
    _cleanup()

    # every piece of the state that a load could drop changes that update far beyond the tolerance
    for mut, prefixes in _mutations(name, saved).items():
        c = _make(name, seed=3)
        if prefixes is None:
            bad = {k: v for k, v in saved.items() if not k.startswith("batch:")}
        else:
            fresh_state = c._ckpt_state(with_batch=False)
            bad = {k: (fresh_state[k] if k.startswith(prefixes) else v) for k, v in saved.items()}
        c.load_states(_save_file(str(tmp_path / "bad.params"), bad))
        c.step(X, y)
        torch.cuda.synchronize()
        e = R.displacement_err(_keys(c, _master(c)), M_saved, ref)
        print("  | %s %.1e" % (mut, e), end="")
        assert e > 100 * TOL, (name, mut, e)
        del c
        _cleanup()
    if "dgt:order" in saved:
        _check_rerank_after_load(name, saved, path, tmp_path, X, y)
    print()
    assert e_run < (WIRE_RUN_TOL if name in WIRE else 10 * TOL if lookahead else TOL), (name, e_run)


def _fp32_keys(saved):
    """Indices of the keys whose tiles all travel as fp32 (after the saved DGT demotions, if any)."""
    out = []
    for i, n in enumerate(CNN_PARAM_NAMES):
        fm = saved.get("dgt_fmt:" + n)
        if fm is None:
            from geomx_b200.parallel.arena import ArenaLayout
            from geomx_b200.models.cnn import CNN_PARAM_SHAPES
            sl = ArenaLayout.build(list(enumerate(CNN_PARAM_SHAPES))).slots[i]
            fm = saved["meta:wire_formats"][sl.offset // 1024: sl.offset // 1024 + sl.tiles]
        if (fm == 0).all():
            out.append(i)
    return out


def _check_rerank_after_load(name, saved, path, tmp_path, X, y):
    """The re-ranking consumes the restored contributions: right after a load it gives the ranking that the saved contributions give
    (fp64 host ranking of _update_ref.dgt_formats); with the contributions dropped on load it gives another, and the update after it
    lands far outside the tolerance."""
    code = {0: "fp32", 1: "fp16", 2: "bsc", 3: "fp8"}
    base = [code[int(v)] for v in saved["meta:wire_formats"]]
    contrib = np.concatenate([saved["dgt_contrib:" + n] for n in CNN_PARAM_NAMES])
    order, _, fmts = U.dgt_formats(base, torch.from_numpy(contrib), 0.8)
    d = _make(name, seed=4)
    d.load_states(path)
    d.fabric.dgt_rerank()
    assert torch.equal(d.fabric.tile_order.cpu().long(), order), "re-ranking after the load differs from the saved contributions' ranking"
    assert [code[int(v)] for v in d.fabric.tile_fmt.cpu()] == fmts
    c = _make(name, seed=3)
    fresh = c._ckpt_state(with_batch=False)
    bad = {k: (fresh[k] if k.startswith("dgt_contrib:") else v) for k, v in saved.items()}
    c.load_states(_save_file(str(tmp_path / "bad.params"), bad))
    c.fabric.dgt_rerank()
    moved = int((c.fabric.tile_fmt != d.fabric.tile_fmt).sum())
    for e in (c, d):
        e.step(X, y)
    torch.cuda.synchronize()
    M_saved = [torch.from_numpy(saved["master:" + n]) for n in CNN_PARAM_NAMES]
    err = R.displacement_err(_keys(c, _master(c)), M_saved, [m.double() for m in _keys(d, _master(d))])
    print("  | skip dgt_contrib %.1e (%d tiles re-formatted)" % (err, moved), end="")
    assert err > 100 * TOL, (name, err)
    del c, d
    _cleanup()


def test_batch_size_may_differ_but_wire_format_must_match(clean_env, tmp_path):
    from geomx_b200.parallel import Topology
    a = mx.models.HipsCNNTrainStep(batch_size=32, optimizer=OPTS["adam"](), topo=Topology(1, 0, 1, 1), use_graph=False, fused_zero_grad=False)
    for X, y in _batches(32, 2):
        a.step(X, y)
    path = str(tmp_path / "b32.params")
    a.save_states(path)
    b = mx.models.HipsCNNTrainStep(batch_size=64, optimizer=OPTS["adam"](), topo=Topology(1, 0, 1, 1), use_graph=False)
    assert b.direct_conv and a.direct_conv and b.path != a.path
    b.load_states(path)
    assert b.opt_step == a.opt_step and all(torch.equal(p, q) for p, q in zip(a.P, b.P))
    assert np.isfinite(b.step(*_batches(64, 1)[0]))
    del a, b
    _cleanup()

    h = mx.models.HipsCNNTrainStep(batch_size=32, optimizer=OPTS["adam"](), topo=Topology(1, 0, 1, 0), use_graph=False, loopback=True,
                                   wire_dtype="fp16")
    h.save_states(path)
    f = mx.models.HipsCNNTrainStep(batch_size=32, optimizer=OPTS["adam"](), topo=Topology(1, 0, 1, 0), use_graph=False, loopback=True)
    before = [p.clone() for p in f.P]
    with pytest.raises(ValueError, match="meta:wire_formats"):
        f.load_states(path)
    assert all(torch.equal(p, q) for p, q in zip(before, f.P))
    s = mx.models.HipsCNNTrainStep(batch_size=32, optimizer=OPTS["sgd"](), topo=Topology(1, 0, 1, 0), use_graph=False, loopback=True,
                                   wire_dtype="fp16")
    with pytest.raises(ValueError, match="meta:opt_kind"):
        s.load_states(path)
    del h, f, s
    _cleanup()


def _ngpus():
    return torch.cuda.device_count() if torch.cuda.is_available() else 0


@pytest.mark.multigpu
@pytest.mark.skipif(_ngpus() < 2, reason="needs >= 2 GPUs")
@pytest.mark.parametrize("direction", ["2to1", "1to2", "lookahead"])
def test_resume_on_another_number_of_ranks(tmp_path, direction):
    """2 ranks save and 1 rank resumes, or the reverse; the resumed engine's first update is the fp64 reference's from the saved state.
    ``lookahead``: 2 look-ahead ranks save and 2 resume, each priming its own saved batch."""
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", str(29701 + ["2to1", "1to2", "lookahead"].index(direction)), os.path.join(ROOT, "tools", "engine_checkpoint_check.py"), direction,
           str(tmp_path / "ckpt.params")]
    r = subprocess.run(cmd, cwd=ROOT, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=300)
    assert r.returncode == 0 and "CKPT_CHECK PASS" in r.stdout, r.stdout[-3000:]
