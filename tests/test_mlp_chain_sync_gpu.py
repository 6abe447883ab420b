"""The dense-chain cluster kernel (csrc/kernels/mlp_chain.cu) hands every layer's output to the other CTAs of its cluster with st.async and
per-buffer transaction barriers instead of cluster-wide barriers.  These tests check what that hand-off must preserve: every output against
fp64 autograd at the batch sizes it covers, at both cluster sizes, with every output buffer pre-filled with NaN (a slice that is never
written, or read before it has landed, shows up), and bit-identical results from launch to launch (every sum has a fixed order)."""
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
D0, D1, D2 = 512, 256, 128


def _inputs(B, C, seed):
    g = torch.Generator(device="cpu").manual_seed(seed)
    r = lambda *s, scale=1.0: (torch.randn(*s, generator=g) * scale).cuda()
    x = r(B, D0).relu()                                   # pooled conv activations are non-negative with many zeros
    w = [r(D1, D0, scale=0.05), r(D1, scale=0.1), r(D2, D1, scale=0.08), r(D2, scale=0.1), r(C, D2, scale=0.1), r(C, scale=0.1)]
    y = torch.randint(0, C, (B,), generator=g).cuda()
    return x, w, y


def _reference(x, w, y):
    import torch.nn.functional as F
    ps = [t.double().requires_grad_(True) for t in [x] + w]
    h = torch.relu(F.linear(ps[0], ps[1], ps[2])); h = torch.relu(F.linear(h, ps[3], ps[4])); lg = F.linear(h, ps[5], ps[6])
    loss = F.cross_entropy(lg, y, reduction="none")
    loss.sum().backward()
    return [loss.detach(), lg.detach(), ps[0].grad] + [p.grad for p in ps[1:]]


def _run(nat, x, w, y):
    B, C = x.shape[0], w[4].shape[0]
    e = lambda *s: torch.full(s, float("nan"), device="cuda")
    outs = [e(B), e(B, C), e(B, D0), e(D1, D0), e(D1), e(D2, D1), e(D2), e(C, D2), e(C)]
    loss, logits, dx, dw0, db0, dw1, db1, dw2, db2 = outs
    assert nat.mlp_chain(x, *w, y.float(), loss, logits, dw0, db0, dw1, db1, dw2, db2, dx)
    torch.cuda.synchronize()
    return outs


NAMES = ("loss", "logits", "dx", "dw0", "db0", "dw1", "db1", "dw2", "db2")


def check_against_fp64(nat, B, C, seed):
    x, w, y = _inputs(B, C, seed)
    got = _run(nat, x, w, y)
    for name, g, ref in zip(NAMES, got, _reference(x, w, y)):
        assert not torch.isnan(g).any(), (B, C, name, "element never written")
        err = float((g.double() - ref).norm() / (ref.norm() + 1e-30))
        assert err < 1e-5, (B, C, name, err)


def check_repeatable(nat, B, C, seed, launches=3):
    x, w, y = _inputs(B, C, seed)
    first = _run(nat, x, w, y)
    for _ in range(launches - 1):
        for name, a, b in zip(NAMES, first, _run(nat, x, w, y)):
            assert torch.equal(a, b), (B, C, name, "differs between launches on the same inputs")


@pytest.fixture(scope="module")
def nat():
    from geomx_b200.ops import native
    native.require()
    return native


@pytest.mark.parametrize("B", [1, 20, 32])
@pytest.mark.parametrize("C", [10, 16])
def test_mlp_chain_cluster16_matches_fp64(nat, B, C):
    check_against_fp64(nat, B, C, seed=100 + B + C)


@pytest.mark.parametrize("B", [1, 32])
def test_mlp_chain_three_launches_bit_identical(nat, B):
    check_repeatable(nat, B, 10, seed=7 + B)


_CLUSTER8 = """
import sys
sys.path.insert(0, {root!r}); sys.path.insert(0, {tests!r})
import torch
from geomx_b200.ops import native
import test_mlp_chain_sync_gpu as t
native.require()
with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
    for B in (1, 20, 32):
        t.check_against_fp64(native, B, 10, seed=200 + B)
    t.check_repeatable(native, 32, 10, seed=9)
names = {{e.key for e in prof.key_averages() if "mlp_chain_kernel" in e.key}}
assert names and all("128, 8>" in n for n in names), names
print("cluster-8 ok", sorted(names))
"""


def test_mlp_chain_cluster8_matches_fp64():
    """GEOMX_MLP_CLUSTER=8 (the portable cluster size); the choice is cached per process, hence a fresh interpreter."""
    env = dict(os.environ, GEOMX_MLP_CLUSTER="8")
    code = _CLUSTER8.format(root=ROOT, tests=os.path.join(ROOT, "tests"))
    r = subprocess.run([sys.executable, "-c", code], env=env, cwd=ROOT, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True,
                       timeout=600)
    assert r.returncode == 0 and "cluster-8 ok" in r.stdout, r.stdout[-4000:]
