"""The demo CNN's fp64 reference and the harness its GPU tests share.

The reference takes the two max-pool arg-max decisions from the kernels (``idx1`` / ``idx2``): a window whose two largest candidates agree to
fp32 rounding can legitimately go either way.  ``check_routing`` checks those decisions separately against the fp64 first maximum, wherever
the window is not such a near-tie.  Exact ties (the zero background of the demo's images makes every conv0 window there a four-way tie) must
resolve to the first position, like torch's max-pool.

The dense chain (dense0 -> ReLU -> dense1 -> ReLU -> classifier -> softmax-CE) is written once, in ``dense_chain_ref``, and can start where
each kernel does: at a2 (the dense-chain cluster kernel), at a3 (``dense_tail_kernel``) or at dz3 (its from-dz3 mode).
"""
import gc
import math
import os
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as F

import geomx_b200 as mx
from geomx_b200.models.cnn import DENSE_KV, DENSE_WGRAD, DIRECT_FWD, EXCH, FUSED_BWD, GEMM_FWD, MLP, ONE_GRID, STEP_SWITCHES

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
D0, D1, D2 = 512, 256, 128          # a2 (flattened), a3, a4


# ---------------------------------------------------------------------------------------------------------------- harness
@pytest.fixture(scope="module")
def nat():
    """The native library.  TF32 is off for torch's own matmuls and convolutions, so that every test file runs with the same settings
    whichever files ran before it in the process."""
    from geomx_b200.ops import native
    native.require()
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    return native


def dev():
    return torch.device("cuda", 0)


def rel_err(a, b):
    return float((a.double() - b.double()).norm() / (b.double().norm() + 1e-30))


def nan(*shape, dtype=torch.float32):
    """An output buffer pre-filled so that an element never written shows up: NaN, or 255 for the uint8 arg-max maps."""
    if dtype == torch.uint8:
        return torch.full(shape, 255, dtype=dtype, device=dev())
    return torch.full(shape, float("nan"), dtype=dtype, device=dev())


def cleanup():
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


@pytest.fixture
def engine(monkeypatch):
    """A factory of training engines for one test: the step switches (and GEOMX_MLP_CLUSTER) are cleared first, ``env`` is applied before
    each engine is built, and every engine built is released at teardown.  The engine runs on one rank with SGD at lr = 0 unless told
    otherwise."""
    from geomx_b200.parallel import Topology
    for k in STEP_SWITCHES + ("GEOMX_MLP_CLUSTER",):
        monkeypatch.delenv(k, raising=False)
    built = []

    def make(B, optimizer=None, env=None, **kw):
        for k, v in (env or {}).items():
            monkeypatch.setenv(k, v)
        kw.setdefault("topo", Topology(1, 0, 1, 1))
        built.append(mx.models.HipsCNNTrainStep(batch_size=B, optimizer=optimizer or mx.optimizer.SGD(learning_rate=0.0), **kw))
        return built[-1]

    yield make
    built.clear()
    cleanup()


def run_in_fresh_interpreter(env, code, expect_kernel, expect_instance):
    """Run ``code`` (which may import ``_cnn_ref``) in a new interpreter with ``env`` added, under the CUDA profiler; every launch of a
    kernel whose name contains ``expect_kernel`` must be the template instance ``expect_instance``.  For choices the native library caches
    per process, such as GEOMX_MLP_CLUSTER."""
    script = "\n".join([
        "import sys",
        "sys.path[:0] = [%r, %r]" % (ROOT, os.path.join(ROOT, "tests")),
        "import torch",
        "from geomx_b200.ops import native",
        "import _cnn_ref as ref",
        "native.require()",
        "with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:",
        "\n".join("    " + line for line in code.strip().splitlines()),
        "names = {e.key for e in prof.key_averages() if %r in e.key}" % expect_kernel,
        "assert names and all(%r in n for n in names), names" % expect_instance,
        "print('fresh interpreter ok', sorted(names))",
    ])
    r = subprocess.run([sys.executable, "-c", script], env=dict(os.environ, **env), cwd=ROOT, stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                       text=True, timeout=600)
    assert r.returncode == 0 and "fresh interpreter ok" in r.stdout, r.stdout[-4000:]
    print("\n  " + r.stdout.strip().splitlines()[-1])


# ---------------------------------------------------------------------------------------------------------------- fp64 reference
def windows(z):
    """(B, C, H, W) -> (B, C, H/2, W/2, 4): the four candidates of every 2x2 pooling window, position k = 2*dy + dx (the kernels' idx)."""
    B, C, H, W = z.shape
    return z.reshape(B, C, H // 2, 2, W // 2, 2).permute(0, 1, 2, 4, 3, 5).reshape(B, C, H // 2, W // 2, 4)


def pool_at(z, idx):
    """Max-pool of ``z`` routed by the given arg-max positions (differentiable: the gradient goes to the chosen position only); with
    ``idx=None`` the plain fp64 maximum."""
    if idx is None:
        return windows(z).amax(-1)
    return windows(z).gather(-1, idx.long().unsqueeze(-1)).squeeze(-1)


def route(g, idx):
    """Pooled gradient (B, C, h, w) -> pre-pool map (B, C, 2h, 2w) with the value at the arg-max position of each window."""
    B, C, h, w = g.shape
    out = torch.zeros(B, C, 2 * h, 2 * w, dtype=g.dtype, device=g.device)
    for k in range(4):
        out[:, :, (k >> 1)::2, (k & 1)::2] = torch.where(idx == k, g, torch.zeros_like(g))
    return out


def check_routing(what, idx, z, zabs, bias):
    """Compare a kernel's max-pool arg-max ``idx`` with the first maximum of the fp64 pre-bias map ``z`` (bias is per channel, so it does
    not change the order).  ``zabs`` = the same convolution of |input| with |weights|: the scale of the fp32 rounding error of ``z``.

    Windows whose pooled value is not clearly positive get no gradient whichever position is taken, and are skipped.  Windows whose top
    candidates differ by more than fp64 rounding but by at most 1e-6 of the scale are near-ties: fp32 may order them either way; they are
    skipped and counted.  Every other window must match, exact ties included (first position wins).  Returns (near-ties, exact ties)."""
    cand = windows(z)
    scale = windows(zabs).amax(-1) + bias.abs().view(1, -1, 1, 1)
    top = cand.amax(-1)
    gap = top.unsqueeze(-1) - cand
    exact = gap <= 1e-12 * scale.unsqueeze(-1)                  # candidates equal to the maximum up to fp64 rounding
    near = ((~exact) & (gap <= 1e-6 * scale.unsqueeze(-1))).any(-1)
    first = torch.full(top.shape, 3, dtype=torch.long, device=z.device)
    for k in (2, 1, 0):
        first = torch.where(exact[..., k], torch.full_like(first, k), first)
    live = (top + bias.view(1, -1, 1, 1)) > 1e-6 * scale
    checked = live & ~near
    bad = checked & (idx.long() != first)
    assert not bool(bad.any()), "%s: %d of %d windows disagree with the fp64 first maximum (first at %s)" % (
        what, int(bad.sum()), int(checked.sum()), bad.nonzero()[0].tolist())
    n_near = int((live & near).sum())
    assert n_near <= max(4, int(1e-4 * checked.numel())), "%s: %d near-tie windows" % (what, n_near)
    return n_near, int((checked & (exact.sum(-1) > 1)).sum())


def conv_forward_ref(x, w0, b0, w1, b1, idx1=None, idx2=None):
    """fp64 conv0 -> ReLU -> pool -> conv1 -> ReLU -> pool, pooled at the kernels' arg-max positions, which are checked as well (returned:
    a1, a2 and the two check_routing counts).  Without positions, pooled at the fp64 maximum and nothing is checked."""
    z1 = F.conv2d(x, w0)
    a1 = torch.relu(pool_at(z1, idx1) + b0.view(1, -1, 1, 1))
    z2 = F.conv2d(a1, w1)
    a2 = torch.relu(pool_at(z2, idx2) + b1.view(1, -1, 1, 1))
    if idx1 is None:
        return a1, a2, None
    with torch.no_grad():
        r1 = check_routing("idx1", idx1, z1, F.conv2d(x.abs(), w0.abs()), b0)
        r2 = check_routing("idx2", idx2, z2, F.conv2d(a1.abs(), w1.abs()), b1)
    return a1, a2, r1 + r2


def dense_chain_ref(W, y=None, a2=None, a3=None, dz3=None, coef=None):
    """fp64 dense chain of the demo CNN with W = (w0, b0, w1, b1, w2, b2), started at a2, at a3 or at dz3 (the parameters the start does
    not read may be None).  Returns the intermediates the kernels store: a3, a4, loss (per sample), logits, dl (dlogits), dz4, dz3, and
    dx = dz3 W0 (da2); "grads" = the six parameter gradients (dW0 and db0 need a2).  The gradients are those of sum_i coef_i loss_i
    (coef = None: all ones).  Without labels, only the forward values."""
    w0, b0, w1, b1, w2, b2 = [None if t is None else t.detach().double() for t in W]
    out = {}
    if dz3 is None:
        for t in (w1, b1, w2, b2):
            t.requires_grad_(y is not None)
        if a3 is None:
            a2 = a2.detach().double().flatten(1)
            a3 = torch.relu(F.linear(a2, w0, b0))
        a3 = a3.detach().double().requires_grad_(y is not None)
        z4 = F.linear(a3, w1, b1)
        a4 = torch.relu(z4)
        logits = F.linear(a4, w2, b2)
        out = {"a3": a3.detach(), "a4": a4.detach(), "logits": logits.detach()}
        if y is None:
            return out
        z4.retain_grad()
        logits.retain_grad()
        loss = F.cross_entropy(logits, y.long(), reduction="none")
        (loss.sum() if coef is None else (loss * coef.to(loss)).sum()).backward()
        dz3 = a3.grad * (a3.detach() > 0)
        out.update(loss=loss.detach(), dl=logits.grad, dz4=z4.grad, dz3=dz3)
        out["grads"] = [None, None, w1.grad, b1.grad, w2.grad, b2.grad]
        if a2 is not None:
            out["grads"][:2] = [dz3.T @ a2, dz3.sum(0)]
    out["dx"] = dz3.double() @ w0
    return out


def step_reference(P, x, y, idx1, idx2, coef=None):
    """The whole step in fp64: per-sample loss, logits and the 10 parameter gradients of sum_i coef_i loss_i (coef = None: the plain sum
    over the batch), and the check_routing counts of both poolings."""
    ps = [p.detach().double().requires_grad_(True) for p in P[:4]]
    _, a2, ties = conv_forward_ref(x.double(), *ps, idx1, idx2)
    d = dense_chain_ref(P[4:], y, a2=a2, coef=coef)
    a2.backward(d["dx"].view_as(a2))
    return d["loss"], d["logits"], [p.grad for p in ps] + d["grads"], ties


# ---------------------------------------------------------------------------------------------------------------- data
def images(g, B, kind):
    """'rand': uniform noise.  'patch': a zero background with a 12x12 random patch in the middle, like the demo's digits: every conv0
    window in the background is an exact four-way tie."""
    x = torch.rand(B, 1, 28, 28, generator=g)
    if kind == "patch":
        bg = torch.zeros_like(x)
        bg[:, :, 8:20, 8:20] = x[:, :, 8:20, 8:20]
        x = bg
    return x.to(dev())


def conv_params(g, regime="default"):
    """conv0 / conv1 weights and biases.  'posbias': b0 > 0, so the background ties of 'patch' images have a positive pooled value and
    carry gradient; 'full': b1 = +5 (a2 > 0 everywhere: every per-window list of the data-gradient kernel holds 32 entries); 'empty':
    b1 = -5 (a2 = 0 everywhere, empty lists); 'dead0': b0 = -5 (a1 = 0 everywhere: every pixel skips its gradient sum)."""
    w0 = torch.randn(16, 1, 5, 5, generator=g) * 0.2
    b0 = torch.randn(16, generator=g) * 0.1
    w1 = torch.randn(32, 16, 5, 5, generator=g) * 0.05
    b1 = torch.randn(32, generator=g) * 0.1
    if regime == "posbias":
        b0 = 0.05 + 0.1 * torch.rand(16, generator=g)
    elif regime == "full":
        b1 = torch.full((32,), 5.0)
    elif regime == "empty":
        b1 = torch.full((32,), -5.0)
    elif regime == "dead0":
        b0 = torch.full((16,), -5.0)
    return [t.to(dev()) for t in (w0, b0, w1, b1)]


def step_params(g):
    P = conv_params(g, "posbias")
    for n_out, n_in in ((D1, D0), (D2, D1), (10, D2)):
        P += [(torch.randn(n_out, n_in, generator=g) / math.sqrt(n_in)).to(dev()), (torch.randn(n_out, generator=g) * 0.1).to(dev())]
    return P


# ---------------------------------------------------------------------------------------------------------------- the step's kernel paths
# The step's kernel paths A-G (tests/test_step_paths_gpu.py lists what selects each): the ordered (launch, stream) lists of the step on one
# rank (overlapped channels: the dense keys' exchange on the comm stream)
WGRAD_KV = (DENSE_WGRAD + " + " + DENSE_KV, "comm")
GEMM_CONV_FWD = [(GEMM_FWD[0], "main"), (GEMM_FWD[1], "main")]
GEMM_CONV_BWD = [("pool+relu bwd -> rows", "main"), ("dWc1 gemm (split-K)", "side"), ("dcol1 gemm", "main"), ("conv0 wgrad + col2im", "main")]
GEMM_HEAD = [("dense0 gemm", "main"), ("dense1 gemm", "main"), ("head fwd+bwd", "main"), ("dW1 gemm", "side"), ("dz3 gemm (mask,colsum)", "main"),
             ("dW0 gemm", "side"), ("da2 gemm", "main")]

# path -> (direct_conv, fused_mlp, fused_exchange, the step's (launch, stream) list)
PATHS = {
    "A": (True, True, False, [(DIRECT_FWD, "main"), (MLP, "main"), WGRAD_KV, (ONE_GRID, "main"), (EXCH, "join")]),
    "B": (True, True, False, [(DIRECT_FWD, "main"), (MLP, "main"), WGRAD_KV, ("conv1 wgrad (direct, sparse)", "side"),
                              ("conv1 dgrad + conv0 wgrad (direct)", "main"), (EXCH, "join")]),
    "C": (True, True, True, [(DIRECT_FWD, "main"), (MLP, "main"), WGRAD_KV, (FUSED_BWD, "main")]),
    "D": (True, False, False, [(DIRECT_FWD, "main")] + GEMM_HEAD + [(DENSE_KV, "comm"), (ONE_GRID, "main"), (EXCH, "join")]),
    "E": (False, True, False, GEMM_CONV_FWD + [(MLP, "main"), WGRAD_KV] + GEMM_CONV_BWD + [(EXCH, "join")]),
    "F": (False, True, False, GEMM_CONV_FWD + [(MLP, "main"), WGRAD_KV] + GEMM_CONV_BWD + [(EXCH, "join")]),
    "G": (False, False, False, GEMM_CONV_FWD + GEMM_HEAD + [(DENSE_KV, "comm")] + GEMM_CONV_BWD + [(EXCH, "join")]),
}
CASES = [("A", 2, {}), ("A", 32, {}),
         ("B", 32, {"GEOMX_CNN_BWD_ONE_LAUNCH": "0"}),
         ("C", 32, {"GEOMX_FUSED_EXCHANGE": "1"}),
         ("D", 48, {}), ("D", 64, {}), ("D", 32, {"GEOMX_FUSED_MLP": "0"}),
         ("E", 1, {}), ("E", 31, {}), ("E", 32, {"GEOMX_DIRECT_CONV": "0"}),
         ("F", 32, {"GEOMX_DIRECT_CONV": "0", "GEOMX_NO_POOL_FUSION": "1"}),
         ("G", 33, {}), ("G", 96, {})]
CASE_IDS = ["%s-B%d" % (p, b) for p, b, _ in CASES]
GRAD_NAMES = ["dw0", "db0", "dw1", "db1", "dW2", "db2", "dW3", "db3", "dW4", "db4"]


# ---------------------------------------------------------------------------------------------------------------- dense-chain kernels
# The checks the cluster-size tests also run in a fresh interpreter (GEOMX_MLP_CLUSTER=8), with their data.
MLP_NAMES = ("loss", "logits", "dx", "dw0", "db0", "dw1", "db1", "dw2", "db2")


def mlp_chain_inputs(B, C, seed, margin=None):
    """a2 (non-negative with many zeros, like pooled conv activations), the six dense parameters and labels.  ``margin`` (the classifier
    head's tests): the class biases spread evenly over [0, margin] in a random order, and every other label the last class."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    r = lambda *s, scale=1.0: (torch.randn(*s, generator=g) * scale).cuda()
    x = r(B, D0).relu()
    w = [r(D1, D0, scale=0.05), r(D1, scale=0.1), r(D2, D1, scale=0.08), r(D2, scale=0.1), r(C, D2, scale=0.1), r(C, scale=0.1)]
    y = torch.randint(0, C, (B,), generator=g).cuda()
    if margin is not None:
        if margin:
            g = torch.Generator(device="cpu").manual_seed(seed + 1)
            w[5] = (torch.randperm(C, generator=g).float() * (margin / max(C - 1, 1))).cuda()
        y[::2] = C - 1      # the last class, in the partly filled column tile when C is not a multiple of 4
    return x, w, y


def mlp_chain_run(nat, x, w, y):
    """One mlp_chain launch with every output pre-filled with NaN; the outputs in MLP_NAMES order."""
    B, C = x.shape[0], w[4].shape[0]
    outs = [nan(B), nan(B, C), nan(B, D0), nan(D1, D0), nan(D1), nan(D2, D1), nan(D2), nan(C, D2), nan(C)]
    loss, logits, dx, dw0, db0, dw1, db1, dw2, db2 = outs
    assert nat.mlp_chain(x, *w, y.float(), loss, logits, dw0, db0, dw1, db1, dw2, db2, dx)
    torch.cuda.synchronize()
    return outs


def check_mlp_chain(nat, B, C, seed, margin=None):
    """Every output against fp64: relative error < 1e-5, or with ``margin`` (the head's tests, where C = 1 makes every gradient exactly
    zero) an absolute floor of 1e-6 added to the 1e-5 relative bound."""
    x, w, y = mlp_chain_inputs(B, C, seed, margin)
    got = mlp_chain_run(nat, x, w, y)
    d = dense_chain_ref(w, y, a2=x)
    for name, g, ref in zip(MLP_NAMES, got, [d["loss"], d["logits"], d["dx"]] + d["grads"]):
        assert not torch.isnan(g).any(), (B, C, margin, name, "element never written")
        if margin is None:
            err = rel_err(g, ref)
            assert err < 1e-5, (B, C, name, err)
        else:
            err, scale = float((g.double() - ref).norm()), float(ref.norm())
            assert err <= 1e-5 * scale + 1e-6, (B, C, margin, name, err, scale)


def check_mlp_chain_repeatable(nat, B, C, seed, margin=None, launches=3):
    x, w, y = mlp_chain_inputs(B, C, seed, margin)
    first = mlp_chain_run(nat, x, w, y)
    for _ in range(launches - 1):
        for name, a, b in zip(MLP_NAMES, first, mlp_chain_run(nat, x, w, y)):
            assert torch.equal(a, b), (B, C, name, "differs between launches on the same inputs")


def dense_tail_inputs(B, C, seed):
    """a3 (a ReLU output: non-negative with many zeros), [w0, w1, b1, w2, b2] and labels."""
    g = torch.Generator().manual_seed(seed)
    r = lambda *s, scale=1.0: (torch.randn(*s, generator=g) * scale).cuda()
    a3 = r(B, D1).relu()
    w = [r(D1, D0, scale=0.05), r(D2, D1, scale=0.08), r(D2, scale=0.1), r(C, D2, scale=0.1), r(C, scale=0.1)]
    y = torch.randint(0, C, (B,), generator=g).cuda()
    return a3, w, y


def dense_tail_run(nat, a3, w, y):
    B, C = a3.shape[0], w[3].shape[0]
    out = {"loss": nan(B), "logits": nan(B, C), "dx": nan(B, D0), "a4": nan(B, D2), "dz4": nan(B, D2), "dz3": nan(B, D1), "dl": nan(B, 16)}
    assert nat.dense_tail(a3, *w, y.float(), out["loss"], out["logits"], out["dx"], out["a4"], out["dz4"], out["dz3"], out["dl"])
    torch.cuda.synchronize()
    return out


def check_dense_tail(nat, B, C, seed):
    a3, w, y = dense_tail_inputs(B, C, seed)
    got = dense_tail_run(nat, a3, w, y)
    assert torch.equal(got["dl"][:, C:], torch.zeros_like(got["dl"][:, C:])), (B, C, "dlogits beyond the classes")
    got["dl"] = got["dl"][:, :C]
    ref = dense_chain_ref([w[0], None] + w[1:], y, a3=a3)
    for name, g in got.items():
        assert not torch.isnan(g).any(), (B, C, name, "element never written")
        err = rel_err(g, ref[name])
        assert err < 1e-5, (B, C, name, err)


def check_dense_tail_repeatable(nat, B, C, seed, launches=3):
    a3, w, y = dense_tail_inputs(B, C, seed)
    first = dense_tail_run(nat, a3, w, y)
    for _ in range(launches - 1):
        for name, t in dense_tail_run(nat, a3, w, y).items():
            assert torch.equal(first[name], t), (B, C, name, "differs between launches on the same inputs")
