"""CPU checks of the generic operator path's fp64 references and host dispatch predicates (``tests/_generic_ref.py``), which
``tests/test_generic_ops_gpu.py`` uses to judge the kernels and to assert which kernel ran."""
import math

import torch

import _generic_ref as R
from geomx_b200.ops import _native_api as NA


def _tf32(t):
    """Round to TF32 (10-bit mantissa, round to nearest) the way the plain tf32 mode feeds the tensor core."""
    b = t.float().view(torch.int32)
    b = (b + 0x1000) & ~0x1FFF
    return b.view(torch.float32)


def test_gemm_bounds_accept_fp32_and_reject_tf32():
    """The element-wise and norm-wise bounds hold for an fp32 product and fail for the TF32 product at every K the GPU tests use."""
    g = torch.Generator().manual_seed(0)
    for M, N, K in ((7, 33, 1), (33, 7, 7), (129, 127, 129), (16, 40, 1090), (16, 144, 25088)):
        A = torch.randn(M, K, generator=g)
        B = torch.randn(N, K, generator=g)
        ref, scale = R.gemm_ref(A, B)
        D = A @ B.t()
        assert R.gemm_elem_excess(D, ref, scale, K) < 1 and R.rel_err(D, ref) < R.gemm_norm_bound(K)
        Dt = _tf32(A).double() @ _tf32(B).double().t()
        assert R.rel_err(Dt, ref) > 3 * R.gemm_norm_bound(K), (M, N, K, R.rel_err(Dt, ref))


def test_gemm_block_n_heuristic_covers_every_width():
    sms = 132
    assert R.gemm_block_n(128, 16, False, sms) == 16
    assert R.gemm_block_n(128, 16, True, sms) == 32           # an MN-major B tile is made of 32-wide boxes
    assert R.gemm_block_n(127, 768, False, sms) == 32
    assert R.gemm_block_n(1533, 127, False, sms) == 64
    assert R.gemm_block_n(3071, 129, False, sms) == 128
    assert R.gemm_splits(285, 2) == (9, 5, 2) and R.gemm_splits(285, 7) == (9, 2, 5) and R.gemm_splits(285, 50) == (9, 1, 9)


def test_maxpool_reference_takes_the_first_maximum():
    x = torch.tensor([[[[1.0, 1.0], [1.0, 1.0]], [[0.0, 2.0], [2.0, 0.0]]]]).reshape(1, 2, 2, 2)
    v, idx = R.maxpool2x2_ref(x)
    assert idx.flatten().tolist() == [0, 1] and v.flatten().tolist() == [1.0, 2.0]
    x = torch.full((1, 1, 2, 2), float("-inf"))
    v, idx = R.maxpool2x2_ref(x)
    assert idx.item() == 0 and v.item() == float("-inf")
    d = R.maxpool2x2_route(torch.tensor([[[[3.0]]]]), torch.tensor([[[[2]]]], dtype=torch.uint8))
    assert d.flatten().tolist() == [0.0, 0.0, 3.0, 0.0]


def test_bn_reference_fixed_statistics_gradient():
    """With fixed statistics dx = dy·γ·rsqrt(rv+eps); the batch-statistics formula on the same statistics is far from it."""
    g = torch.Generator().manual_seed(1)
    x = torch.randn(8, 3, 5, 5, generator=g) * 1.7 + 0.6
    dy = torch.randn(8, 3, 5, 5, generator=g) + 0.3
    gamma, beta = torch.rand(3, generator=g) + 0.5, torch.randn(3, generator=g)
    rm, rv = torch.randn(3, generator=g), torch.rand(3, generator=g) + 0.5
    y, dx, dg, db, _, _ = R.bn_ref(x, gamma, beta, rm, rv, False, 1e-5, dy)
    inv = 1.0 / torch.sqrt(rv.double() + 1e-5)
    assert torch.allclose(dx, dy.double() * (gamma.double() * inv).view(1, 3, 1, 1))
    assert torch.allclose(db, dy.double().sum((0, 2, 3)))
    assert torch.allclose(dg, (dy.double() * (x.double() - rm.double().view(1, 3, 1, 1)) * inv.view(1, 3, 1, 1)).sum((0, 2, 3)))
    bad = R.bn_dx_batch_formula(x, dy, gamma, rm, inv)
    assert R.rel_err(bad, dx) > 0.05
    # with batch statistics the same formula is the exact gradient
    y, dx, *_ = R.bn_ref(x, gamma, beta, rm, rv, True, 1e-5, dy)
    m = x.double().mean((0, 2, 3)); v = x.double().var((0, 2, 3), unbiased=False)
    assert R.rel_err(R.bn_dx_batch_formula(x, dy, gamma, m, 1.0 / torch.sqrt(v + 1e-5)), dx) < 1e-12


def test_bn_split_form_predicate():
    assert not R.bn_split_form(2, 3, 25) and R.bn_split_form(16, 4, 256) and R.bn_split_form(9, 5, 529)
    assert not R.bn_split_form(300, 3, 15)                    # N·HW >= 4096 but HW < 16
    assert not R.bn_split_form(4096, 6, 1)                    # [N, C] input
    assert not R.bn_split_form(256, 16385, 16)                # more channels than the accumulators hold


def test_depthwise_predicate_keeps_backward_in_shared_memory():
    """The old dispatch test looked at the input plane only; with padding the output plane, which the input- and filter-gradient kernels
    stage, can be larger.  A 152x152 plane with a 31x31 filter and padding 15 passed it, and its filter gradient needs 224 KB."""
    x, w = (1, 2, 152, 152), (2, 1, 31, 31)
    assert (152 * 152 + 31 * 31) * 8 <= 190 * 1024               # the old predicate accepted it
    sm = NA.depthwise_smem(152, 152, 31, 31, (1, 1), (30, 30))
    assert sm["wgrad"] > NA.DW_SMEM_LIMIT
    assert not NA.depthwise_supported(x, w, (1, 1), (30, 30))
    assert NA.depthwise_supported(x, w, (1, 1), (15, 15))
    assert NA.depthwise_supported((1, 1, 161, 151), (1, 1, 3, 3), (1, 1), (1, 1))       # just inside the plane limit
    assert not NA.depthwise_supported((1, 1, 161, 152), (1, 1, 3, 3), (1, 1), (1, 1))
    assert not NA.depthwise_supported((1, 1, 4, 4), (1, 1, 7, 7), (1, 1), (0, 0))       # empty output
    # every accepted shape fits all three kernels
    for H, W, K, p, s in ((100, 100, 3, 60, 1), (150, 150, 9, 8, 1), (120, 90, 5, 4, 2), (155, 155, 7, 6, 1)):
        ok = NA.depthwise_supported((1, 1, H, W), (1, 1, K, K), (s, s), (p, p))
        sm = NA.depthwise_smem(H, W, K, K, (s, s), (p, p))
        assert not ok or max(sm.values()) <= NA.DW_SMEM_LIMIT
