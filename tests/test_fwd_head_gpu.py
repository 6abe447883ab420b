"""The training head of the forward kernel: at even batches <= 32 the classic step runs cnn_fwd_dense0_kernel with its head outputs
(csrc/kernels/cnn_direct.cu: dense1, the classifier, softmax-CE, dz4 and dz3 in the clusters of two images) and dense_tail_kernel from dz3
(csrc/kernels/mlp_chain.cu: da2 = dz3 W0 only).  These tests check the head against fp64, including confidently classified samples, the
from-dz3 tail against fp64, the new pair against the pair that goes through a3, launch-to-launch determinism, and which pair the captured
step runs with and without look-ahead.  Every output is pre-filled with NaN, so that an element never written shows up."""
import pytest
import torch

import geomx_b200 as mx
from _cnn_ref import D0, D1, D2, dense_chain_ref, engine, nan, nat, rel_err  # noqa: F401  (nat, engine: fixtures)

pytestmark = pytest.mark.gpu

C = 10
HEAD_OUT = ("loss", "logits", "a4", "dz4", "dz3", "dl")


def _inputs(B, seed, w2_scale=0.1):
    """Images, the ten parameters in CNN_PARAM_SHAPES order and labels.  A large w2_scale spreads the logits far apart, so that most samples
    are classified with a probability near 1 (dlogits near 0 for the right class, near -1 for a confident wrong one)."""
    g = torch.Generator().manual_seed(seed)
    r = lambda *s, scale=1.0: (torch.randn(*s, generator=g) * scale).cuda()
    x = torch.rand(B, 1, 28, 28, generator=g).cuda()
    P = [r(16, 1, 5, 5, scale=0.3), r(16, scale=0.1), r(32, 16, 5, 5, scale=0.08), r(32, scale=0.1),
         r(D1, D0, scale=0.05), r(D1, scale=0.1), r(D2, D1, scale=0.08), r(D2, scale=0.1), r(C, D2, scale=w2_scale), r(C, scale=0.1)]
    y = torch.randint(0, C, (B,), generator=g).float().cuda()
    return x, P, y


def _conv_outputs(B):
    return [nan(B, 16, 12, 12), nan(B, 16, 12, 12, dtype=torch.uint8), nan(B, 32, 4, 4), nan(B, 32, 4, 4, dtype=torch.uint8)]


def _head_outputs(B):
    return {"loss": nan(B), "logits": nan(B, C), "a4": nan(B, D2), "dz4": nan(B, D2), "dz3": nan(B, D1), "dl": nan(B, 16)}


def _run_head(nat, x, P, y):
    B = x.shape[0]
    conv, a3, out = _conv_outputs(B), nan(B, D1), _head_outputs(B)
    assert nat.cnn_fwd_dense0(x, *P[:6], *conv, a3, wd1=P[6], bd1=P[7], wd2=P[8], bd2=P[9], label=y, **out)
    torch.cuda.synchronize()
    out["a3"], out["a2"] = a3, conv[2]
    return out


@pytest.mark.parametrize("B", [2, 8, 32])
@pytest.mark.parametrize("w2_scale", [0.1, 3.0], ids=["spread", "confident"])
def test_fwd_head_matches_fp64(nat, B, w2_scale):
    x, P, y = _inputs(B, 800 + B, w2_scale)
    got = _run_head(nat, x, P, y)
    assert torch.equal(got["dl"][:, C:], torch.zeros_like(got["dl"][:, C:])), (B, "dlogits beyond the classes")
    got["dl"] = got["dl"][:, :C]
    # the dense chain from a2 (a2 itself from the kernel, which the convolution tests check bit for bit against cnn_fwd)
    ref = dense_chain_ref(P[4:], y, a2=got["a2"])
    if w2_scale > 1:
        p_max = torch.softmax(ref["logits"], 1).max(1).values
        assert (p_max > 0.999).float().mean() > 0.5, "most samples must be classified confidently"
    for name in ("a3", "a4", "loss", "logits", "dl", "dz4", "dz3"):
        g, want = got[name], ref[name]
        assert not torch.isnan(g).any(), (B, name, "element never written")
        err = rel_err(g, want)
        assert err < (1e-6 if name == "a3" else 1e-5), (B, w2_scale, name, err)


def _run_tail(nat, dz3, w0, from_dz3, a3=None, P=None, y=None):
    """from_dz3: dz3 is the input and every other operand NaN (none may be read); otherwise the chain from a3, whose dz3 output replaces
    the given one in the result"""
    B = dz3.shape[0]
    dx, out = nan(B, D0), _head_outputs(B)
    if from_dz3:
        del out["dz3"]
        args = (nan(B, D1), w0, nan(D2, D1), nan(D2), nan(C, D2), nan(C), nan(B))
        assert nat.dense_tail(*args, out["loss"], out["logits"], dx, out["a4"], out["dz4"], dz3, out["dl"], from_dz3=True)
    else:
        assert nat.dense_tail(a3, w0, P[6], P[7], P[8], P[9], y, out["loss"], out["logits"], dx, out["a4"], out["dz4"], out["dz3"], out["dl"])
    torch.cuda.synchronize()
    out["dx"] = dx
    return out


@pytest.mark.parametrize("B", [1, 8, 32])
def test_dense_tail_from_dz3_matches_fp64(nat, B):
    g = torch.Generator().manual_seed(900 + B)
    dz3 = (torch.randn(B, D1, generator=g) * (torch.rand(B, D1, generator=g) > 0.4)).cuda()   # masked by a ReLU: many zeros
    w0 = (torch.randn(D1, D0, generator=g) * 0.05).cuda()
    out = _run_tail(nat, dz3, w0, True)
    assert not torch.isnan(out["dx"]).any(), (B, "dx element never written")
    assert rel_err(out["dx"], dense_chain_ref([w0] + [None] * 5, dz3=dz3)["dx"]) < 1e-6, B
    # nothing but dx is written in this mode
    for name in HEAD_OUT:
        if name != "dz3":
            assert torch.isnan(out[name]).all(), (B, name, "written by the from-dz3 tail")


@pytest.mark.parametrize("B", [2, 32])
def test_new_pair_matches_the_pair_through_a3(nat, B):
    x, P, y = _inputs(B, 950 + B)
    head = _run_head(nat, x, P, y)
    new = _run_tail(nat, head["dz3"], P[4], True)
    conv, a3 = _conv_outputs(B), nan(B, D1)
    assert nat.cnn_fwd_dense0(x, *P[:6], *conv, a3)
    torch.cuda.synchronize()
    assert torch.equal(a3, head["a3"]), B
    old = _run_tail(nat, nan(B, D1), P[4], False, a3=a3, P=P, y=y)
    for name in HEAD_OUT:
        err = rel_err(head[name], old[name])
        assert err < 1e-5, (B, name, err)
    assert rel_err(new["dx"], old["dx"]) < 1e-5, B


def test_head_and_tail_three_launches_bit_identical(nat):
    B = 32
    x, P, y = _inputs(B, 31)
    first = _run_head(nat, x, P, y)
    dx = _run_tail(nat, first["dz3"], P[4], True)["dx"]
    for _ in range(2):
        again = _run_head(nat, x, P, y)
        for name, t in again.items():
            assert torch.equal(first[name], t), (name, "differs between launches on the same inputs")
        assert torch.equal(dx, _run_tail(nat, first["dz3"], P[4], True)["dx"]), "dx differs between launches"


@pytest.mark.parametrize("lookahead", [False, True])
def test_captured_step_pair(nat, engine, monkeypatch, lookahead):
    """B = 32: the classic step runs the forward kernel with its head and the tail from dz3; the look-ahead step keeps the pair through a3
    (its launch ends with the next batch's forward kernel, which would overwrite the loss and logits the host has not read yet)."""
    seen = {"fwd": [], "tail": []}
    fwd, tail = nat.cnn_fwd_dense0, nat.dense_tail
    monkeypatch.setattr(nat, "cnn_fwd_dense0", lambda *a, **k: (seen["fwd"].append(k.get("a4") is not None), fwd(*a, **k))[1])
    monkeypatch.setattr(nat, "dense_tail", lambda *a, **k: (seen["tail"].append(bool(k.get("from_dz3"))), tail(*a, **k))[1])
    B = 32
    g = torch.Generator().manual_seed(901)
    X, y = torch.rand(B, 1, 28, 28, generator=g), torch.randint(0, 10, (B,), generator=g).float()
    eng = engine(B, mx.optimizer.Adam(learning_rate=0.01), use_graph=True, lookahead=lookahead)
    l0 = eng.step(X.pin_memory(), y.pin_memory())
    for _ in range(5):
        l1 = eng.step(X.pin_memory(), y.pin_memory())
    if lookahead:
        l1 = eng.flush()
    assert seen["fwd"] and seen["tail"], seen
    assert set(seen["fwd"]) == {not lookahead} and set(seen["tail"]) == {not lookahead}, seen
    if not lookahead:
        assert eng.kernels_per_step == 6, eng.kernels_per_step
        assert l0 == l0 and l1 < l0, (l0, l1)
