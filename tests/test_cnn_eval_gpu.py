"""Inference of the demo CNN in one launch (cnn_eval_kernel, csrc/kernels/cnn_direct.cu) and the engine API on top of it
(HipsCNNTrainStep.evaluate / evaluate_async / predict).  Every output buffer is longer than N and pre-filled with NaN or a sentinel, so a
slice never written, or a write past N, shows up.  Checked: the kernel against an fp64 forward at batch sizes that cover one image, odd
batches (the last cluster's missing image) and the whole test-set size; launch-to-launch determinism; labels outside [0, 10); predict-only
launches; the engine against fp64 and against the Gluon net re-homed onto it, in every update / graph / look-ahead mode and for every input
kind; and that evaluation writes nothing the training step owns."""
import math

import pytest
import torch

import geomx_b200 as mx
from _cnn_ref import conv_forward_ref, dense_chain_ref, engine, nat, rel_err  # noqa: F401  (nat, engine: fixtures)

pytestmark = pytest.mark.gpu

PAD = 64                    # sentinel elements after the N outputs of every buffer
SENT = -7                   # int32 sentinel of pred / correct


def _params(seed):
    """The ten parameters of the demo CNN.  The conv and dense0 biases are negative, so that an all-zero image has a2 = 0 and a3 = 0."""
    g = torch.Generator().manual_seed(seed)
    r = lambda *s, scale: torch.randn(*s, generator=g) * scale
    P = [r(16, 1, 5, 5, scale=0.3), -r(16, scale=0.1).abs(), r(32, 16, 5, 5, scale=0.08), -r(32, scale=0.1).abs(),
         r(256, 512, scale=0.05), -r(256, scale=0.1).abs(), r(128, 256, scale=0.08), r(128, scale=0.1), r(10, 128, scale=0.1), r(10, scale=0.1)]
    return [p.cuda() for p in P]


def _images(N, seed, zero_rows=()):
    g = torch.Generator().manual_seed(seed)
    x = torch.full((N + PAD, 1, 28, 28), float("nan"))
    x[:N] = torch.rand(N, 1, 28, 28, generator=g)
    for i in zero_rows:
        x[i] = 0.0
    y = torch.randint(0, 10, (N,), generator=g).float()
    return x.cuda(), y.cuda()


def ref_forward(x, P):
    """fp64 forward of the demo CNN: (a2, a3, logits)."""
    _, a2, _ = conv_forward_ref(x.double(), *[p.double() for p in P[:4]])
    d = dense_chain_ref(P[4:], a2=a2)
    return a2.flatten(1), d["a3"], d["logits"]


def _outputs(N):
    return {"logits": torch.full((N + PAD, 10), float("nan"), device="cuda"), "loss": torch.full((N + PAD,), float("nan"), device="cuda"),
            "pred": torch.full((N + PAD,), SENT, dtype=torch.int32, device="cuda"),
            "correct": torch.full((N + PAD,), SENT, dtype=torch.int32, device="cuda")}


def _run(nat, x, P, label, N):
    out = _outputs(N)
    nat.cnn_eval(x[:N], *P, label, out["logits"][:N], out["loss"][:N], out["pred"][:N], out["correct"][:N])
    torch.cuda.synchronize()
    return out


def _check_padding(out, N):
    assert torch.isnan(out["logits"][N:]).all() and torch.isnan(out["loss"][N:]).all(), (N, "written past N")
    assert (out["pred"][N:] == SENT).all() and (out["correct"][N:] == SENT).all(), (N, "written past N")


def _check_against_fp64(logits, loss, pred, correct, label, ref_logits, what):
    err = rel_err(logits, ref_logits)
    assert err <= 1e-5, (what, "logits", err)
    ref_loss = -torch.log_softmax(ref_logits, dim=1).gather(1, label.long().view(-1, 1)).view(-1)
    assert float((loss.double() - ref_loss).abs().max()) <= 1e-4, (what, "loss")
    top2 = ref_logits.topk(2, dim=1).values
    clear = (top2[:, 0] - top2[:, 1]) > 1e-3
    assert torch.equal(pred.long()[clear], ref_logits.argmax(1)[clear]), (what, "pred")
    assert torch.equal(correct, (pred.long() == label.long()).int()), (what, "correct")


# ---------------------------------------------------------------------------------------------------------------- kernel
@pytest.mark.parametrize("N", [1, 2, 3, 31, 32, 33, 1000, 10000])
def test_cnn_eval_matches_fp64(nat, N):
    zero_rows = (1, N - 1) if N >= 3 else ()
    P = _params(40 + N)
    x, y = _images(N, 1000 + N, zero_rows)
    out = _run(nat, x, P, y, N)
    _check_padding(out, N)
    for k in ("logits", "loss"):
        assert not torch.isnan(out[k][:N]).any(), (N, k, "element never written")
    a2, a3, ref = ref_forward(x[:N], P)
    for i in zero_rows:
        assert (a2[i] <= 0).all() and (a3[i] <= 0).all(), "precondition: an all-zero image has no positive a2 / a3"
    _check_against_fp64(out["logits"][:N], out["loss"][:N], out["pred"][:N], out["correct"][:N], y, ref, N)


def test_cnn_eval_two_launches_bit_identical(nat):
    N = 1001
    P = _params(3)
    x, y = _images(N, 4)
    a, b = _run(nat, x, P, y, N), _run(nat, x, P, y, N)
    for k in a:
        assert torch.equal(a[k][:N], b[k][:N]), (k, "differs between launches on the same inputs")


def test_cnn_eval_rejects_labels_outside_the_classes(nat):
    N = 37
    P = _params(5)
    x, y = _images(N, 6)
    bad = {0: -1.0, 3: 10.0, 5: 2.5, 8: float("nan"), 13: float("inf"), 17: float("-inf"), 21: 3e9, 25: -3e9, 30: 1e30, 36: 9.999}
    for i, v in bad.items():
        y[i] = v
    out = _run(nat, x, P, y, N)
    _check_padding(out, N)
    idx = torch.tensor(sorted(bad), device="cuda")
    assert torch.isnan(out["loss"][idx]).all(), out["loss"][idx]
    assert (out["correct"][idx] == 0).all(), out["correct"][idx]
    good = torch.ones(N, dtype=torch.bool, device="cuda")
    good[idx] = False
    _, _, ref = ref_forward(x[:N], P)
    assert not torch.isnan(out["loss"][:N][good]).any()
    _check_against_fp64(out["logits"][:N][good], out["loss"][:N][good], out["pred"][:N][good], out["correct"][:N][good], y[good], ref[good],
                        "valid labels among invalid ones")
    assert rel_err(out["logits"][:N], ref) <= 1e-5          # a bad label changes neither the logits nor the prediction of its row
    assert torch.equal(out["pred"][:N], _run(nat, x, P, None, N)["pred"][:N])


def test_cnn_eval_without_labels_writes_logits_and_predictions_only(nat):
    N = 33
    P = _params(7)
    x, y = _images(N, 8)
    full = _run(nat, x, P, y, N)
    out = _run(nat, x, P, None, N)
    assert torch.isnan(out["loss"]).all() and (out["correct"] == SENT).all(), "loss / correct written without labels"
    _check_padding(out, N)
    assert torch.equal(out["logits"][:N], full["logits"][:N]) and torch.equal(out["pred"][:N], full["pred"][:N])


def test_cnn_eval_refuses_an_empty_batch(nat):
    P = _params(9)
    out = _outputs(0)
    before = nat.launch_count
    with pytest.raises(ValueError):
        nat.cnn_eval(torch.empty(0, 1, 28, 28, device="cuda"), *P, None, out["logits"][:0], None, out["pred"][:0], None)
    assert nat.launch_count == before


# ---------------------------------------------------------------------------------------------------------------- engine
def _engine(engine, net=None, update="server", use_graph=True, lookahead=False):
    return engine(32, mx.optimizer.Adam(learning_rate=0.01), net=net, use_graph=use_graph, update=update, lookahead=lookahead)


def _train_batches(n, seed):
    g = torch.Generator().manual_seed(seed)
    return [(torch.rand(32, 1, 28, 28, generator=g).pin_memory(), torch.randint(0, 10, (32,), generator=g).float().pin_memory()) for _ in range(n)]


def _as_input(t, kind):
    return {"host": lambda: t.clone(), "pinned": lambda: t.clone().pin_memory(), "cuda": lambda: t.cuda(),
            "ndarray": lambda: mx.nd.array(t, ctx=mx.gpu(0))}[kind]()


@pytest.mark.parametrize("update,use_graph,lookahead,x_kind,y_kind", [
    ("server", True, False, "pinned", "float"),
    ("server", False, False, "host", "int"),
    ("server", True, True, "cuda", "int"),
    ("server", False, True, "pinned", "float"),
    ("local", True, False, "cuda", "float"),
    ("local", False, False, "ndarray", "int"),
])
def test_engine_evaluate_and_predict_score_the_live_weights(nat, engine, update, use_graph, lookahead, x_kind, y_kind):
    torch.manual_seed(31)
    net = mx.models.build_cnn()
    net.initialize(init=mx.init.Xavier(), ctx=mx.gpu(0))
    net(mx.nd.array(torch.zeros(1, 1, 28, 28), ctx=mx.gpu(0)))          # deferred shapes -> parameters
    eng = _engine(engine, net, update, use_graph, lookahead)
    batches = _train_batches(20, 32)
    for X, y in batches[:-1]:
        eng.step(X, y)
    N = 333
    g = torch.Generator().manual_seed(33)
    Xe, ye = torch.rand(N, 1, 28, 28, generator=g), torch.randint(0, 10, (N,), generator=g)
    Xin = _as_input(Xe.reshape(N, 784) if x_kind == "host" else Xe, x_kind)     # both image layouts
    yin = _as_input(ye.float() if y_kind == "float" else ye, x_kind)
    # the last step and the evaluation are enqueued back to back: the evaluation must see that step's update (with look-ahead, the last
    # completed one: the launch also ran the convolutions of the next batch, which change no weight)
    eng.step_async(*batches[-1])
    handle = eng.evaluate_async(Xin, yin)
    logits = eng.predict(Xin)
    mean_loss, acc = handle.item()
    torch.cuda.synchronize()
    P = [torch.from_numpy(p).cuda() for p in eng.params_numpy()]
    _, _, ref = ref_forward(Xe.cuda(), P)
    assert logits.shape == (N, 10) and logits.is_cuda
    assert rel_err(logits, ref) <= 1e-5, rel_err(logits, ref)
    ref_loss = -torch.log_softmax(ref, 1).gather(1, ye.cuda().view(-1, 1)).view(-1)
    assert abs(mean_loss - float(ref_loss.mean())) <= 1e-4, (mean_loss, float(ref_loss.mean()))
    top2 = ref.topk(2, dim=1).values
    unclear = int(((top2[:, 0] - top2[:, 1]) <= 1e-3).sum())
    ref_hits = int((ref.argmax(1).cpu() == ye).sum())
    hits = round(acc * N)
    assert abs(acc * N - hits) < 1e-6 and abs(hits - ref_hits) <= unclear, (acc, ref_hits, unclear)
    # the Gluon net re-homed onto the engine reads the same live weights through the generic layer-by-layer path
    gl = torch.from_numpy(net(mx.nd.array(Xe, ctx=mx.gpu(0))).asnumpy()).cuda()
    assert rel_err(logits, gl) <= 1e-4, rel_err(logits, gl)
    # same inputs, same bits
    assert eng.evaluate(Xin, yin) == (mean_loss, acc)
    assert torch.equal(eng.predict(Xin), logits)


def _engine_tensors(eng):
    t = {"P%d" % i: p for i, p in enumerate(eng.P)}
    t.update({"G%d" % i: g for i, g in enumerate(eng.G)})
    for name in ("xin", "a1", "idx1", "col1", "z2", "a2", "idx2", "a3", "a4", "loss", "logits", "dz4", "dz3", "da2", "dl", "dz2rows", "dcol1",
                 "da1", "label_cur", "x_cur", "loss_host", "Wl", "s0l", "s1l", "opt_state"):
        if getattr(eng, name, None) is not None:
            t[name] = getattr(eng, name)
    f = eng.fabric
    t.update({"fabric.param": f.param.tensor, "fabric.grad": f.grad.tensor})
    for name in ("w", "s0", "s1"):
        if getattr(f, name, None) is not None:
            t["fabric." + name] = getattr(f, name)
    t.update({"fabric.state." + k: v for k, v in f.state.items()})
    return t


def _bits(t):
    return t.detach().contiguous().view(-1).view(torch.uint8).clone()


@pytest.mark.parametrize("update,lookahead", [("server", True), ("server", False), ("local", False)])
def test_evaluation_leaves_training_alone(nat, engine, update, lookahead):
    torch.manual_seed(41)
    eng = _engine(engine, None, update, True, lookahead)
    for X, y in _train_batches(5, 42):
        eng.step(X, y)
    torch.cuda.synchronize()
    kps = eng.kernels_per_step
    before = {k: _bits(v) for k, v in _engine_tensors(eng).items()}
    g = torch.Generator().manual_seed(43)
    Xe, ye = torch.rand(1001, 1, 28, 28, generator=g).cuda(), torch.randint(0, 10, (1001,), generator=g).float().cuda()
    launches = nat.launch_count
    for i in range(3):
        eng.evaluate(Xe[:1001 - i], ye[:1001 - i])
        assert nat.launch_count == launches + i + 1, "one native launch per evaluate"
    eng.predict(Xe)
    assert nat.launch_count == launches + 4
    torch.cuda.synchronize()
    for k, v in _engine_tensors(eng).items():
        assert torch.equal(_bits(v), before[k]), (k, "written by evaluation")
    assert eng.kernels_per_step == kps


def test_engine_evaluate_rejects_mismatched_inputs(nat, engine):
    eng = _engine(engine, None, "server", False, False)
    with pytest.raises(ValueError):
        eng.evaluate(torch.rand(4, 1, 28, 27), torch.zeros(4))
    with pytest.raises(ValueError):
        eng.evaluate(torch.rand(4, 784), torch.zeros(5))
    with pytest.raises(ValueError):
        eng.predict(torch.rand(0, 784))
    assert math.isfinite(eng.evaluate(torch.rand(3, 784), torch.zeros(3))[0])
