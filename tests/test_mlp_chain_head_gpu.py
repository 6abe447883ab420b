"""The classifier head of the dense-chain cluster kernel (csrc/kernels/mlp_chain.cu) computes the 32 x C logits as 4x4 register tiles, runs
softmax-CE on the four lanes that hold a row, and every CTA then computes the whole dz4 itself instead of receiving it.  These tests cover
what that layout has to get right: class counts that are not a multiple of four (C = 1, 3, 13) with the last class as a label, batches that
fill the last 4-row tile only partly (B = 7, 31: the padded rows must add nothing to any output), logit margins up to 60, and
bit-identical outputs from launch to launch at both cluster sizes.  Outputs are pre-filled with NaN and checked against fp64 autograd."""
import os
import subprocess
import sys

import pytest
import torch

import test_mlp_chain_sync_gpu as sync

pytestmark = pytest.mark.gpu


def _inputs(B, C, seed, margin):
    x, w, y = sync._inputs(B, C, seed)
    if margin:
        # class biases spread evenly over [0, margin] in a random order: the logits of a row differ by up to about `margin`
        g = torch.Generator(device="cpu").manual_seed(seed + 1)
        w[5] = (torch.randperm(C, generator=g).float() * (margin / max(C - 1, 1))).cuda()
    y[::2] = C - 1      # the last class, in the partly filled column tile when C is not a multiple of 4
    return x, w, y


def check_against_fp64(nat, B, C, seed, margin):
    x, w, y = _inputs(B, C, seed, margin)
    got = sync._run(nat, x, w, y)
    for name, g, ref in zip(sync.NAMES, got, sync._reference(x, w, y)):
        assert not torch.isnan(g).any(), (B, C, margin, name, "element never written")
        # with C = 1 every gradient is exactly zero: the absolute floor keeps that case meaningful
        err, scale = float((g.double() - ref).norm()), float(ref.norm())
        assert err <= 1e-5 * scale + 1e-6, (B, C, margin, name, err, scale)


def check_repeatable(nat, B, C, seed, margin, launches=3):
    x, w, y = _inputs(B, C, seed, margin)
    first = sync._run(nat, x, w, y)
    for _ in range(launches - 1):
        for name, a, b in zip(sync.NAMES, first, sync._run(nat, x, w, y)):
            assert torch.equal(a, b), (B, C, name, "differs between launches on the same inputs")


@pytest.fixture(scope="module")
def nat():
    from geomx_b200.ops import native
    native.require()
    return native


@pytest.mark.parametrize("margin", [0, 60])
@pytest.mark.parametrize("C", [1, 3, 13])
@pytest.mark.parametrize("B", [7, 31])
def test_mlp_chain_head_matches_fp64(nat, B, C, margin):
    check_against_fp64(nat, B, C, seed=300 + 3 * B + C, margin=margin)


@pytest.mark.parametrize("B,C", [(31, 13), (7, 3)])
def test_mlp_chain_head_three_launches_bit_identical(nat, B, C):
    check_repeatable(nat, B, C, seed=400 + B, margin=60)


_CLUSTER8 = """
import sys
sys.path.insert(0, {root!r}); sys.path.insert(0, {tests!r})
import torch
from geomx_b200.ops import native
import test_mlp_chain_head_gpu as t
native.require()
with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
    for B in (7, 31):
        for C in (1, 3, 13):
            t.check_against_fp64(native, B, C, seed=500 + B + C, margin=60)
    t.check_repeatable(native, 31, 13, seed=9, margin=60)
names = {{e.key for e in prof.key_averages() if "mlp_chain_kernel" in e.key}}
assert names and all("128, 8>" in n for n in names), names
print("cluster-8 ok", sorted(names))
"""


def test_mlp_chain_head_cluster8():
    """GEOMX_MLP_CLUSTER=8 (the portable cluster size); the choice is cached per process, hence a fresh interpreter."""
    env = dict(os.environ, GEOMX_MLP_CLUSTER="8")
    code = _CLUSTER8.format(root=sync.ROOT, tests=os.path.join(sync.ROOT, "tests"))
    r = subprocess.run([sys.executable, "-c", code], env=env, cwd=sync.ROOT, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True,
                       timeout=600)
    assert r.returncode == 0 and "cluster-8 ok" in r.stdout, r.stdout[-4000:]
