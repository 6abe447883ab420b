"""The generic operator path (every Gluon / Module / Symbol model except the fused demo CNN) against fp64, at every kernel its host code
selects: the wgmma GEMM and its CUDA-core fallback, im2col / col2im (tiled and general), depthwise convolution, ReLU, 2x2 max-pool and
BatchNorm (one-CTA and split forms, batch and fixed statistics), and one small Gluon network end to end.

ReLU masks and pooling arg-maxes are discrete, so gradients are compared with an fp64 reference routed through the kernel's own decisions;
tolerances are then fp32-tight.  Each section computes the plausible wrong result (its mutation) on the same data and shows that it fails
the tolerance, and every threshold-selected path is asserted by recomputing the host predicate (``tests/_generic_ref.py``)."""
import math

import pytest
import torch
import torch.nn.functional as F

import _generic_ref as R
import geomx_b200 as mx

pytestmark = pytest.mark.gpu

rel_err = R.rel_err


@pytest.fixture(scope="module")
def nat():
    from geomx_b200.ops import native
    native.require()
    assert native.gemm_precision() == "3xtf32"
    return native


@pytest.fixture(scope="module")
def OF():
    from geomx_b200.ops import functional
    functional.use_native(True)
    return functional


def dev():
    return torch.device("cuda", 0)


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def offset_view(shape, off, gen=None, fill=None):
    """A contiguous CUDA fp32 tensor of ``shape`` that starts ``off`` floats into its storage."""
    n = math.prod(shape)
    base = torch.randn(n + off, device=dev(), generator=gen) if fill is None else torch.full((n + off,), fill, device=dev())
    v = base[off:off + n].view(shape)
    assert v.is_contiguous() and v.data_ptr() % 16 == 4 * off % 16
    return v


# ====================================================================================================================== A. GEMM
def _operands(M, N, K, a_mn, b_mn, g):
    A = torch.randn(M, K, device=dev(), generator=g)
    B = torch.randn(N, K, device=dev(), generator=g)
    return (A.t().contiguous() if a_mn else A), (B.t().contiguous() if b_mn else B)


def _run_gemm(nat, A, B, D, simt, **kw):
    nat.gemm(A, B, D, force_simt=simt, **kw)
    torch.cuda.synchronize()
    return D


# odd leading dimensions take the CUDA-core kernel even on the wgmma entry; the last five shapes satisfy TMA in every major
TAILS = [(1, 1, 1), (7, 33, 7), (33, 7, 129), (127, 129, 33), (129, 127, 127), (7, 1, 300), (1, 129, 64),
         (200, 72, 100), (128, 132, 36), (132, 8, 68), (4, 36, 100), (260, 12, 1028)]


@pytest.mark.parametrize("simt", [False, True], ids=["wgmma", "simt"])
@pytest.mark.parametrize("a_mn,b_mn", [(False, False), (False, True), (True, False), (True, True)])
def test_gemm_majors_and_tails(nat, simt, a_mn, b_mn):
    """All four operand majors, partial tiles in M, N and K, on the 3xTF32 wgmma kernel and on the CUDA-core kernel.  Mutation: the plain
    TF32 product (one MMA per K step) fails the norm-wise bound at every shape that runs on the wgmma kernel."""
    g = torch.Generator(device=dev()).manual_seed(1)
    on_tma = 0
    for M, N, K in TAILS:
        A, B = _operands(M, N, K, a_mn, b_mn, g)
        tma = R.gemm_tma_ok(A.data_ptr(), A.stride(0), B.data_ptr(), B.stride(0), K)
        on_tma += tma
        D = torch.full((M, N), float("nan"), device=dev())
        _run_gemm(nat, A, B, D, simt, a_mn=a_mn, b_mn=b_mn)
        ref, scale = R.gemm_ref(A, B, a_mn, b_mn)
        ex = R.gemm_elem_excess(D, ref, scale, K)
        assert ex < 1 and rel_err(D, ref) < R.gemm_norm_bound(K), (M, N, K, ex, rel_err(D, ref))
        if not simt and tma and K >= 7:
            nat.set_gemm_precision("tf32")
            try:
                Dt = _run_gemm(nat, A, B, torch.zeros(M, N, device=dev()), False, a_mn=a_mn, b_mn=b_mn)
            finally:
                nat.set_gemm_precision("3xtf32")
            assert rel_err(Dt, ref) > 3 * R.gemm_norm_bound(K), ("tf32 mutation passes", M, N, K, rel_err(Dt, ref))
    assert on_tma >= 5


def test_gemm_every_tile_width_and_trimmed_boxes(nat):
    """block_n 16 / 32 / 64 / 128 from gemm_tf32_impl's heuristic (recomputed from the SM count), the MN-major B minimum of 32, single-tile
    problems whose TMA boxes are trimmed (mt == 1 with M % 8 != 0, nt == 1)."""
    n_sm = sms()
    g = torch.Generator(device=dev()).manual_seed(2)
    seen = set()
    cases = [(128, 16, 40, False, False, 16), (7, 13, 40, False, False, 16), (128, 16, 40, False, True, 32), (127, 768, 36, False, False, 32),
             (1532, 128, 68, True, True, 64), (3071, 129, 72, False, False, 128), (33, 20, 100, False, True, 32), (12, 4, 36, True, True, 32)]
    for M, N, K, a_mn, b_mn, want in cases:
        bn = R.gemm_block_n(M, N, b_mn, n_sm)
        assert bn == want, (M, N, b_mn, bn, want)
        seen.add(bn)
        A, B = _operands(M, N, K, a_mn, b_mn, g)
        assert R.gemm_tma_ok(A.data_ptr(), A.stride(0), B.data_ptr(), B.stride(0), K), "this case must run on the wgmma kernel"
        D = torch.full((M, N), float("nan"), device=dev())
        _run_gemm(nat, A, B, D, False, a_mn=a_mn, b_mn=b_mn)
        ref, scale = R.gemm_ref(A, B, a_mn, b_mn)
        assert R.gemm_elem_excess(D, ref, scale, K) < 1, (M, N, K, a_mn, b_mn)
    assert seen == {16, 32, 64, 128}


@pytest.mark.parametrize("split_k", [1, 2, 3, 5, 7, 50])
def test_gemm_split_k(nat, split_k):
    """Split-K onto a non-zero D: an odd number of K blocks, split boundaries that are not multiples of the 3xTF32 chunk (ACC_CHUNK_KB = 4),
    more splits than K blocks.  Mutation: a lost split (one K slice missing) is far outside the bound."""
    g = torch.Generator(device=dev()).manual_seed(3)
    for M, N, K, a_mn, b_mn in ((33, 40, 284, False, False), (16, 144, 1090, True, True), (129, 8, 300, False, True)):
        num_kb, per, eff = R.gemm_splits(K, split_k)
        A, B = _operands(M, N, K, a_mn, b_mn, g)
        assert R.gemm_tma_ok(A.data_ptr(), A.stride(0), B.data_ptr(), B.stride(0), K)
        D0 = torch.randn(M, N, device=dev(), generator=g)
        D = _run_gemm(nat, A, B, D0.clone(), False, a_mn=a_mn, b_mn=b_mn, split_k=split_k, accumulate=True)
        ref, scale = R.gemm_ref(A, B, a_mn, b_mn)
        ref = ref + D0.double()
        ex = R.gemm_elem_excess(D, ref, scale + D0.double().abs(), K)
        assert ex < 1, (M, N, K, split_k, eff, ex)
        if eff > 1:
            Ad = (A.t() if a_mn else A).double(); Bd = (B.t() if b_mn else B).double()
            k1 = min(K, per * R.BLOCK_K)
            lost = D0.double() + Ad[:, k1:] @ Bd[:, k1:].t()          # the first split's slice dropped
            assert R.gemm_elem_excess(lost.float(), ref, scale, K) > 10
    # the chunked accumulation crosses a split boundary off the chunk grid for these parameters
    assert any(R.gemm_splits(K, split_k)[1] % R.ACC_CHUNK_KB for K in (284, 1090, 300)) or split_k in (1, 50)


@pytest.mark.parametrize("simt", [False, True], ids=["wgmma", "simt"])
@pytest.mark.parametrize("bias,relu,mask,colsum", [(True, False, False, False), (True, True, False, False), (False, False, True, True),
                                                    (True, True, True, True), (True, False, False, True), (False, True, True, False)])
def test_gemm_epilogues(nat, simt, bias, relu, mask, colsum):
    """alpha != 1 with every epilogue combination on partial row tiles (M = 129, 127); the column sum with the mask applied.  Mutation: a
    column sum taken before the mask."""
    g = torch.Generator(device=dev()).manual_seed(4)
    for M, N, K in ((129, 40, 68), (127, 33, 132)):
        A, B = _operands(M, N, K, False, False, g)
        assert R.gemm_tma_ok(A.data_ptr(), A.stride(0), B.data_ptr(), B.stride(0), K)
        bv = torch.randn(N, device=dev(), generator=g) if bias else None
        mk = torch.randn(M, N, device=dev(), generator=g) if mask else None
        cs = torch.zeros(N, device=dev()) if colsum else None
        D = torch.full((M, N), float("nan"), device=dev())
        _run_gemm(nat, A, B, D, simt, alpha=0.37, bias=bv, relu=relu, mask=mk, colsum=cs)
        ref, scale = R.gemm_ref(A, B, alpha=0.37, bias=bv, relu=relu, mask=mk)
        assert R.gemm_elem_excess(D, ref, scale, K) < 1, (M, N, K)
        if colsum:
            rs = ref.sum(0)
            err = (cs.double() - rs).abs()
            bound = R.GEMM_ELEM_C * math.sqrt(K) * R.U32 * scale.sum(0) + 4 * math.sqrt(M) * R.U32 * ref.abs().sum(0) + 1e-30
            assert float((err / bound).max()) < 1, float((err / bound).max())
            if mask:
                pre = R.gemm_ref(A, B, alpha=0.37, bias=bv, relu=relu)[0].sum(0)
                assert float(((pre - rs).abs() / bound).max()) > 10


@pytest.mark.parametrize("simt", [False, True], ids=["wgmma", "simt"])
@pytest.mark.parametrize("hw", [9, 20, 36, 64])
def test_gemm_nchw_store(nat, simt, hw):
    """NCHW scatter with hw not a multiple of 32 (and 9: not of 4); with bias and ReLU.  Mutation: the [pixel][channel] layout."""
    g = torch.Generator(device=dev()).manual_seed(5)
    n_img, C, K = 5, 13, 40
    A = torch.randn(n_img * hw, K, device=dev(), generator=g); B = torch.randn(C, K, device=dev(), generator=g)
    bv = torch.randn(C, device=dev(), generator=g)
    Y = torch.full((n_img, C, hw), float("nan"), device=dev())
    _run_gemm(nat, A, B, Y, simt, bias=bv, relu=True, store_nchw_hw=hw)
    ref, scale = R.gemm_ref(A, B, bias=bv, relu=True)
    to_nchw = lambda t: t.reshape(n_img, hw, C).permute(0, 2, 1)
    assert R.gemm_elem_excess(Y, to_nchw(ref), to_nchw(scale), K) < 1
    assert rel_err(Y.reshape(-1), ref.reshape(-1)) > 0.1


@pytest.mark.parametrize("simt", [False, True], ids=["wgmma", "simt"])
def test_gemm_operand_layouts(nat, simt):
    """Padded leading dimensions (ld > K) on both operands and the output; operands offset by one float, which the wgmma kernel refuses (TMA
    needs 16-byte bases) so the call takes the CUDA-core kernel with the same result."""
    g = torch.Generator(device=dev()).manual_seed(6)
    M, N, K = 70, 45, 37
    Ap = torch.randn(M, K + 7, device=dev(), generator=g)[:, :K]
    Bp = torch.randn(N, K + 11, device=dev(), generator=g)[:, :K]
    Dp = torch.full((M, N + 5), float("nan"), device=dev())
    _run_gemm(nat, Ap, Bp, Dp[:, :N], simt, lda=Ap.stride(0), ldb=Bp.stride(0), ldd=Dp.stride(0))
    ref, scale = R.gemm_ref(Ap, Bp)
    assert R.gemm_elem_excess(Dp[:, :N], ref, scale, K) < 1 and bool(torch.isnan(Dp[:, N:]).all())
    Bq = torch.randn(N, K + 3, device=dev(), generator=g)[:, :K]            # ld = 40: aligned rows
    A1 = offset_view((M, K + 3), 1, g)[:, :K]
    assert not R.gemm_tma_ok(A1.data_ptr(), A1.stride(0), Bq.data_ptr(), Bq.stride(0), K)
    A2 = torch.empty(M, K + 3, device=dev())[:, :K]
    A2.copy_(A1)
    assert R.gemm_tma_ok(A2.data_ptr(), A2.stride(0), Bq.data_ptr(), Bq.stride(0), K)
    D1 = _run_gemm(nat, A1, Bq, torch.empty(M, N, device=dev()), simt)
    D2 = _run_gemm(nat, A2, Bq, torch.empty(M, N, device=dev()), simt)
    ref, scale = R.gemm_ref(A1, Bq)
    assert R.gemm_elem_excess(D1, ref, scale, K) < 1 and R.gemm_elem_excess(D2, ref, scale, K) < 1


def test_gemm_conv_weight_gradient_large_k(nat):
    """The weight-gradient GEMM of Conv2dFn: dW[Co, C·9] = rows[N·OH·OW, Co]ᵀ · col[N·OH·OW, C·9], K = 25 088, split-K as Conv2dFn picks it,
    accumulated onto zeros.  Mutation: the plain TF32 product."""
    g = torch.Generator(device=dev()).manual_seed(7)
    Kc, Co, Kd = 25088, 16, 144
    rows = torch.randn(Kc, Co, device=dev(), generator=g); col = torch.randn(Kc, Kd, device=dev(), generator=g)
    kb = (Kc + 31) // 32
    split = max(1, min(32, kb // 4))
    dw = torch.zeros(Co, Kd, device=dev())
    _run_gemm(nat, rows, col, dw, False, a_mn=True, b_mn=True, M=Co, N=Kd, K=Kc, lda=Co, ldb=Kd, ldd=Kd, split_k=split, accumulate=True)
    ref, scale = R.gemm_ref(rows, col, True, True)
    assert R.gemm_elem_excess(dw, ref, scale, Kc) < 1 and rel_err(dw, ref) < R.gemm_norm_bound(Kc), rel_err(dw, ref)
    nat.set_gemm_precision("tf32")
    try:
        dt = _run_gemm(nat, rows, col, torch.zeros(Co, Kd, device=dev()), False, a_mn=True, b_mn=True, split_k=split, accumulate=True)
    finally:
        nat.set_gemm_precision("3xtf32")
    assert rel_err(dt, ref) > 3 * R.gemm_norm_bound(Kc), rel_err(dt, ref)


@pytest.mark.parametrize("simt", [False, True], ids=["wgmma", "simt"])
def test_gemm_empty_k_writes_the_epilogue(nat, simt):
    """K = 0: D = epi(alpha · 0) on both kernels, i.e. relu(bias), bias or 0 (the wgmma entry hands the call to the CUDA-core kernel), and
    accumulate adds the bias."""
    M, N = 9, 20
    A = torch.empty(M, 0, device=dev()); B = torch.empty(N, 0, device=dev())
    bv = torch.randn(N, device=dev())
    D = _run_gemm(nat, A, B, torch.full((M, N), float("nan"), device=dev()), simt, bias=bv, relu=True)
    assert torch.equal(D, bv.clamp_min(0).expand(M, N))
    D = _run_gemm(nat, A, B, torch.full((M, N), float("nan"), device=dev()), simt)
    assert torch.equal(D, torch.zeros(M, N, device=dev()))
    D0 = torch.randn(M, N, device=dev())
    D = _run_gemm(nat, A, B, D0.clone(), simt, bias=bv, accumulate=True)
    assert torch.equal(D, D0 + bv)


# ====================================================================================================================== B. convolution
# (N, C, H, W, Co, KH, KW, stride, padding, bias, relu, x_grad)
CONV_CASES = [
    (2, 4, 9, 11, 8, 3, 3, (1, 1), (0, 0), True, True, True),       # tiled im2col + tiled col2im
    (3, 3, 10, 10, 6, 3, 3, (1, 1), (0, 0), True, True, True),      # K = 27 (RGB 3x3): general im2col, tiled col2im
    (2, 5, 9, 7, 7, 3, 5, (1, 2), (2, 0), True, False, True),       # 3x5, asymmetric stride / padding, Co odd (CUDA-core GEMMs)
    (1, 6, 8, 8, 8, 1, 1, (2, 1), (0, 1), False, True, True),       # 1x1, N = 1, C = 6, no bias
    (2, 4, 80, 80, 4, 3, 3, (1, 1), (0, 0), True, True, True),      # 6400-pixel plane: general im2col and col2im
    (4, 8, 12, 12, 16, 5, 5, (1, 1), (0, 0), None, False, True),    # bias None, ReLU off
    (2, 3, 7, 9, 5, 3, 5, (2, 2), (1, 2), True, True, False),       # x without requires_grad
    (1, 4, 40, 40, 8, 3, 3, (1, 1), (0, 0), True, False, True),     # tiled im2col, general col2im (slab > 160 KB)
    (2, 5, 6, 6, 3, 2, 2, (2, 2), (1, 1), True, True, True),        # stride 2 and padding 1, C = 5
]


@pytest.mark.parametrize("case", CONV_CASES, ids=[str(i) for i in range(len(CONV_CASES))])
def test_conv2d_forward_and_gradients(nat, OF, case):
    """OF.conv2d -> Conv2dFn (im2col + wgmma / CUDA-core GEMM with NCHW store, col2im, split-K weight gradient, channel-sum bias gradient)
    against fp64 with the kernel's ReLU mask.  Mutations: the filter read with KH and KW exchanged, and the filter's last column tap
    dropped, both fail the forward tolerance."""
    N, C, H, W, Co, KH, KW, st, pd, has_b, relu, xg = case
    g = torch.Generator(device=dev()).manual_seed(10)
    x = torch.randn(N, C, H, W, device=dev(), generator=g)
    w = torch.randn(Co, C, KH, KW, device=dev(), generator=g) * 0.2
    b = torch.randn(Co, device=dev(), generator=g) if has_b else None
    xr = x.clone().requires_grad_(xg); wr = w.clone().requires_grad_(True); br = b.clone().requires_grad_(True) if has_b else None
    y = OF.conv2d(xr, wr, br, st, pd, act="relu" if relu else None)
    gy = torch.randn(y.shape, device=dev(), generator=g)
    y.backward(gy)
    torch.cuda.synchronize()
    z = R.conv_ref(x, w, b, st, pd)
    yref = z.clamp_min(0) if relu else z
    assert rel_err(y.detach(), yref) < 2e-6, rel_err(y.detach(), yref)
    if KH != KW:
        wt = w.reshape(Co, C, KW, KH).transpose(2, 3).contiguous()
        assert rel_err(F.conv2d(x.double(), wt.double(), None if b is None else b.double(), st, pd), z) > 0.1
    wd = w.clone(); wd[..., -1] = 0
    assert rel_err(R.conv_ref(x, wd, b, st, pd), z) > 1e-3
    dz = torch.where(y.detach() > 0, gy, torch.zeros_like(gy)) if relu else gy
    dx, dw, db = R.conv_grads_ref(x, w, dz, st, pd, has_b)
    assert rel_err(wr.grad, dw) < 1e-5, rel_err(wr.grad, dw)
    if has_b:
        assert rel_err(br.grad, db) < 1e-5
    if xg:
        assert rel_err(xr.grad, dx) < 1e-5, rel_err(xr.grad, dx)
    else:
        assert xr.grad is None


def test_conv_cases_reach_every_im2col_and_col2im_kernel():
    tiled_i = {R.im2col_tiled(C, H, W, KH, KW, st, pd) for (N, C, H, W, Co, KH, KW, st, pd, *_) in CONV_CASES}
    tiled_c = {R.col2im_tiled(C, H, W, KH, KW, st, pd) for (N, C, H, W, Co, KH, KW, st, pd, *_) in CONV_CASES}
    assert tiled_i == {True, False} and tiled_c == {True, False}
    general_causes = set()
    for (N, C, H, W, Co, KH, KW, st, pd, *_) in CONV_CASES:
        if (C * KH * KW) % 4:
            general_causes.add("K")
        if st != (1, 1):
            general_causes.add("stride")
        if pd != (0, 0):
            general_causes.add("padding")
        if 4 * H * W * 4 > 96 * 1024:
            general_causes.add("plane")
    assert general_causes == {"K", "stride", "padding", "plane"}


# ====================================================================================================================== C. depthwise
# (N, C, H, W, KH, KW, stride, padding)
DW_CASES = [
    (3, 4, 9, 11, 3, 5, (1, 1), (1, 2)),        # non-square kernel
    (2, 5, 13, 7, 3, 3, (2, 1), (2, 2)),        # stride (2, 1), padding k-1
    (2, 3, 11, 9, 4, 4, (2, 2), (0, 0)),        # odd H != W, last window hangs off the edge
    (4, 6, 8, 8, 1, 1, (1, 1), (0, 0)),         # 1x1
    (64, 96, 10, 10, 3, 3, (1, 1), (1, 1)),     # N·C = 6144 planes
    (1, 2, 161, 151, 3, 3, (1, 1), (1, 1)),     # plane just inside the dispatch predicate
]


@pytest.mark.parametrize("case", DW_CASES, ids=[str(i) for i in range(len(DW_CASES))])
def test_depthwise_forward_and_gradients(nat, OF, case):
    """groups == channels through DepthwiseConv2dFn against fp64 with the kernel's ReLU mask; the forward's acceptance implies the input-
    and filter-gradient kernels accept too.  Mutation: the filter transposed (KH <-> KW read order)."""
    N, C, H, W, KH, KW, st, pd = case
    assert nat.depthwise_supported((N, C, H, W), (C, 1, KH, KW), st, pd)
    assert max(nat.depthwise_smem(H, W, KH, KW, st, pd).values()) <= nat.DW_SMEM_LIMIT
    g = torch.Generator(device=dev()).manual_seed(11)
    x = torch.randn(N, C, H, W, device=dev(), generator=g)
    w = torch.randn(C, 1, KH, KW, device=dev(), generator=g) * 0.3
    b = torch.randn(C, device=dev(), generator=g)
    xr, wr, br = (t.clone().requires_grad_(True) for t in (x, w, b))
    y = OF.conv2d(xr, wr, br, st, pd, groups=C, act="relu")
    gy = torch.randn(y.shape, device=dev(), generator=g)
    y.backward(gy)
    torch.cuda.synchronize()
    z = F.conv2d(x.double(), w.double(), b.double(), st, pd, groups=C)
    assert rel_err(y.detach(), z.clamp_min(0)) < 2e-6
    wt = w.reshape(C, 1, KW, KH).transpose(2, 3)
    if KH != KW or KH > 1:
        zt = F.conv2d(x.double(), wt.double() if KH != KW else w.double().transpose(2, 3), b.double(), st, pd, groups=C)
        assert rel_err(zt, z) > 1e-2
    dz = torch.where(y.detach() > 0, gy, torch.zeros_like(gy))
    dx, dw, db = R.depthwise_grads_ref(x, w, dz, st, pd)
    for got, ref, name in ((xr.grad, dx, "dx"), (wr.grad, dw, "dw"), (br.grad, db, "db")):
        assert rel_err(got, ref) < 1e-5, (name, rel_err(got, ref))


# ====================================================================================================================== D. dense
@pytest.mark.parametrize("units", [1, 10, 33, 256])
@pytest.mark.parametrize("in_units", [1, 7, 784])
@pytest.mark.parametrize("B", [1, 3, 257])
def test_dense(nat, OF, units, in_units, B):
    """DenseFn (y = x·Wᵀ + b, dx = dy·W, dW = dyᵀ·x, db = colsum) against fp64 with the kernel's ReLU mask; ReLU and bias alternate over
    the grid.  Mutation: the plain TF32 product fails the forward tolerance once in_units > 1."""
    relu = (units + in_units + B) % 2 == 0
    has_b = units != 33
    g = torch.Generator(device=dev()).manual_seed(12)
    x = torch.randn(B, in_units, device=dev(), generator=g)
    w = torch.randn(units, in_units, device=dev(), generator=g) / math.sqrt(in_units)
    b = torch.randn(units, device=dev(), generator=g) if has_b else None
    xr, wr = x.clone().requires_grad_(True), w.clone().requires_grad_(True)
    br = b.clone().requires_grad_(True) if has_b else None
    y = OF.dense(xr, wr, br, "relu" if relu else None)
    gy = torch.randn(y.shape, device=dev(), generator=g)
    y.backward(gy)
    torch.cuda.synchronize()
    ref, scale = R.gemm_ref(x, w, bias=b, relu=relu)
    assert R.gemm_elem_excess(y.detach(), ref, scale, in_units) < 1
    dz = torch.where(y.detach() > 0, gy, torch.zeros_like(gy)) if relu else gy
    dx, dxs = R.gemm_ref(dz, w, b_mn=True)
    dw, dws = R.gemm_ref(dz, x, a_mn=True, b_mn=True)
    assert R.gemm_elem_excess(xr.grad, dx, dxs, units) < 1 and R.gemm_elem_excess(wr.grad, dw, dws, B) < 1
    if has_b:
        assert rel_err(br.grad, dz.double().sum(0)) < 4 * math.sqrt(B) * R.U32 + 1e-7
    if in_units == 784 and units == 256 and B == 257:
        nat.set_gemm_precision("tf32")
        try:
            yt = OF.dense(x, w, b, "relu" if relu else None)
            torch.cuda.synchronize()
        finally:
            nat.set_gemm_precision("3xtf32")
        assert rel_err(yt, ref) > 3 * R.gemm_norm_bound(in_units), rel_err(yt, ref)


def test_dense_4d_input_and_offset_view(nat, OF):
    """A 4-D input is flattened; an input that starts one float into its storage takes the CUDA-core GEMMs (TMA refuses it) with the
    same result."""
    g = torch.Generator(device=dev()).manual_seed(13)
    w = torch.randn(10, 48, device=dev(), generator=g) * 0.2; b = torch.randn(10, device=dev(), generator=g)
    x4 = torch.randn(5, 3, 4, 4, device=dev(), generator=g).requires_grad_(True)
    xo = offset_view((5, 48), 1, g).requires_grad_(True)
    assert not R.gemm_tma_ok(xo.data_ptr(), 48, w.data_ptr(), 48, 48)
    for xr in (x4, xo):
        wr, br = w.clone().requires_grad_(True), b.clone().requires_grad_(True)
        y = OF.dense(xr, wr, br, "relu")
        gy = torch.randn(y.shape, device=dev(), generator=g)
        y.backward(gy)
        torch.cuda.synchronize()
        x2 = xr.detach().reshape(5, 48)
        ref, scale = R.gemm_ref(x2, w, bias=b, relu=True)
        assert R.gemm_elem_excess(y.detach(), ref, scale, 48) < 1
        dz = torch.where(y.detach() > 0, gy, torch.zeros_like(gy))
        dx, dxs = R.gemm_ref(dz, w, b_mn=True)
        dw, dws = R.gemm_ref(dz, x2, a_mn=True, b_mn=True)
        assert xr.grad.shape == xr.shape
        assert R.gemm_elem_excess(xr.grad.reshape(5, 48), dx, dxs, 10) < 1 and R.gemm_elem_excess(wr.grad, dw, dws, 5) < 1


# ====================================================================================================================== E. ReLU
@pytest.mark.parametrize("n", [1, 3, 4, 5, 1023, 1024, 1025, 4097])
def test_relu_sizes_and_offsets_bit_exact(nat, OF, n):
    """relu_fwd / relu_bwd at every size around the 4-element vector step, on views that start 0-3 floats into their storage (input,
    gradient and output), bit-exact against fp64.  fmaxf maps NaN to 0 like the reference's mshadow_op::relu (torch.relu propagates it);
    that is pinned here.  Mutation: a kernel that skips the unaligned head (leaves the output untouched) is caught by the NaN-filled output."""
    g = torch.Generator(device=dev()).manual_seed(14)
    for off_x in range(4):
        for off_g in range(4):
            x = offset_view((n,), off_x, g)
            x[0] = -0.0
            if n > 2:
                x[1] = 0.0; x[2] = float("nan")
            xr = x.detach().clone() if off_x == 0 else x
            xr.requires_grad_(True)
            y = OF.activation(xr, "relu")
            gy = offset_view((n,), off_g, g)
            y.backward(gy)
            torch.cuda.synchronize()
            xd = x.detach().double()
            yref = torch.where(xd > 0, xd, torch.zeros_like(xd))              # NaN -> 0, -0.0 -> 0
            assert torch.equal(y.detach().double(), yref), (n, off_x, off_g)
            assert torch.equal(xr.grad.double(), torch.where(xd > 0, gy.double(), torch.zeros_like(xd))), (n, off_x, off_g)
            # all three pointers unaligned, straight through the wrappers
            out = offset_view((n,), (off_x + off_g) % 4, fill=float("nan"))
            nat.relu_fwd(x.detach(), out=out)
            dxo = offset_view((n,), (off_x + 3) % 4, fill=float("nan"))
            nat.relu_bwd(out, gy, out=dxo)
            torch.cuda.synchronize()
            assert torch.equal(out.double(), yref) and torch.equal(dxo.double(), torch.where(yref > 0, gy.double(), torch.zeros_like(xd)))


def test_relu_backward_of_cat_slices_into_dense(nat, OF):
    """torch.cat backward hands DenseFn(relu=True) gradient slices that start 5 floats into the cat's gradient; relu_bwd reads them
    unaligned, and the input, weight and bias gradients must be the fp64 ones."""
    g = torch.Generator(device=dev()).manual_seed(15)
    w = torch.randn(5, 12, device=dev(), generator=g) * 0.3; b = torch.randn(5, device=dev(), generator=g)
    x1, x2 = torch.randn(1, 12, device=dev(), generator=g), torch.randn(3, 12, device=dev(), generator=g)
    wr, br = w.clone().requires_grad_(True), b.clone().requires_grad_(True)
    x1r, x2r = x1.clone().requires_grad_(True), x2.clone().requires_grad_(True)
    y1, y2 = OF.dense(x1r, wr, br, "relu"), OF.dense(x2r, wr, br, "relu")
    z = torch.cat([y1, y2], 0)
    gz = torch.randn(z.shape, device=dev(), generator=g)
    assert gz[1:].data_ptr() % 16 != 0
    z.backward(gz)
    torch.cuda.synchronize()
    X = torch.cat([x1, x2], 0)
    Y = torch.cat([y1, y2], 0).detach()
    dz = torch.where(Y > 0, gz, torch.zeros_like(gz))
    dx, dxs = R.gemm_ref(dz, w, b_mn=True)
    dw, dws = R.gemm_ref(dz, X, a_mn=True, b_mn=True)
    assert R.gemm_elem_excess(torch.cat([x1r.grad, x2r.grad], 0), dx, dxs, 5) < 1
    assert R.gemm_elem_excess(wr.grad, dw, dws, 4) < 1
    assert rel_err(br.grad, dz.double().sum(0)) < 1e-6


# ====================================================================================================================== F. max-pool
def _pool_inputs(g):
    yield "noise", torch.randn(3, 4, 8, 10, device=dev(), generator=g)
    yield "constant", torch.full((2, 3, 6, 6), 0.75, device=dev())
    yield "relu zeros", torch.randn(4, 5, 12, 12, device=dev(), generator=g).clamp_min(0)
    x = torch.randn(2, 2, 4, 6, device=dev(), generator=g)
    x[0, 0] = float("-inf"); x[1, 1, :2, :2] = float("-inf"); x[1, 0, 0, 1] = float("-inf")
    yield "-inf", x
    yield "2x2", torch.randn(7, 3, 2, 2, device=dev(), generator=g)
    yield "odd pooled columns", torch.randn(3, 2, 6, 6, device=dev(), generator=g)
    yield "large NC", torch.randn(256, 300, 4, 6, device=dev(), generator=g)
    yield "offset view", offset_view((2, 3, 4, 6), 1, g)


def test_maxpool2x2(nat, OF):
    """MaxPool2x2Fn against fp64 2x2/2 pooling with the FIRST maximum winning: pooled values and arg-max bit-exact, the gradient routed to
    it.  Mutation: the last maximum winning differs on the tied planes."""
    g = torch.Generator(device=dev()).manual_seed(16)
    ties_seen = False
    for name, x in _pool_inputs(g):
        xr = x.detach().clone() if name != "offset view" else x
        xr.requires_grad_(True)
        y = OF.max_pool2d(xr, (2, 2), (2, 2))
        gy = torch.randn(y.shape, device=dev(), generator=g)
        y.backward(gy)
        torch.cuda.synchronize()
        vref, iref = R.maxpool2x2_ref(x.detach())
        assert torch.equal(y.detach().double(), vref), name
        dref = R.maxpool2x2_route(gy, iref)
        assert torch.equal(xr.grad.double(), dref), name
        N, C, H, W = x.shape
        win = x.detach().double().reshape(N, C, H // 2, 2, W // 2, 2).permute(0, 1, 2, 4, 3, 5).reshape(N, C, H // 2, W // 2, 4)
        last = 3 - torch.argmax((win == vref.unsqueeze(-1)).flip(-1).to(torch.uint8), dim=-1)
        if not torch.equal(last.to(torch.uint8), iref):
            ties_seen = True
            assert not torch.equal(R.maxpool2x2_route(gy, last.to(torch.uint8)), xr.grad.double()), name
    assert ties_seen


# ====================================================================================================================== G. BatchNorm
# (shape, training)
BN_SHAPES = [(2, 3, 5, 5), (16, 4, 16, 16), (9, 5, 23, 23), (300, 3, 3, 5), (64, 6), (256, 16385, 4, 4), (40, 7, 12, 10)]


def _bn_case(shape, g, mean=0.6, std=1.7):
    C = shape[1]
    x = torch.randn(*shape, device=dev(), generator=g) * std + mean
    gamma = torch.rand(C, device=dev(), generator=g) + 0.5
    beta = torch.randn(C, device=dev(), generator=g)
    rm = torch.randn(C, device=dev(), generator=g) * 0.3 + mean
    rv = (torch.rand(C, device=dev(), generator=g) + 0.5) * std * std
    dy = torch.randn(*shape, device=dev(), generator=g) + 0.3
    return x, gamma, beta, rm, rv, dy


def _hw(shape):
    return math.prod(shape[2:]) if len(shape) > 2 else 1


@pytest.mark.parametrize("training", [True, False], ids=["batch_stats", "fixed_stats"])
@pytest.mark.parametrize("shape", BN_SHAPES, ids=["x".join(map(str, s)) for s in BN_SHAPES])
def test_batchnorm(nat, OF, shape, training):
    """OF.batch_norm -> BatchNormFn on both kernel forms (one-CTA: N·HW < 4096 or HW < 16 or C > 16384; split otherwise), HW % 4 zero and
    not, [N, C] input; forward, running statistics and the three gradients against fp64.  Mutation (fixed statistics): the batch-statistics
    input gradient, which the backward kernels applied in every mode before, fails by orders of magnitude."""
    g = torch.Generator(device=dev()).manual_seed(17)
    N, C, HW = shape[0], shape[1], _hw(shape)
    x, gamma, beta, rm, rv, dy = _bn_case(shape, g)
    rm0, rv0 = rm.clone(), rv.clone()
    xr, gr, br = (t.clone().requires_grad_(True) for t in (x, gamma, beta))
    if R.bn_split_form(N, C, HW):
        OF.batch_norm(x[:1].expand(*shape).contiguous(), gamma, beta, rm.clone(), rv.clone(), True)    # allocate this stream's accumulators
        assert nat.bn_workspace_ready()
    y = OF.batch_norm(xr, gr, br, rm, rv, training, momentum=0.9, eps=1e-5)
    y.backward(dy)
    torch.cuda.synchronize()
    yref, dx, dg, db, bmean, bvar = R.bn_ref(x, gamma, beta, rm0, rv0, training, 1e-5, dy)
    assert rel_err(y.detach(), yref) < 5e-6, rel_err(y.detach(), yref)
    assert rel_err(xr.grad, dx) < 2e-5, ("dx", rel_err(xr.grad, dx))
    assert rel_err(gr.grad, dg) < 1e-5 and rel_err(br.grad, db) < 1e-5, (rel_err(gr.grad, dg), rel_err(br.grad, db))
    if training:
        assert rel_err(rm, 0.9 * rm0.double() + 0.1 * bmean) < 2e-6 and rel_err(rv, 0.9 * rv0.double() + 0.1 * bvar) < 2e-6
    else:
        assert torch.equal(rm, rm0) and torch.equal(rv, rv0)
        bad = R.bn_dx_batch_formula(x, dy, gamma, rm0, torch.rsqrt(rv0.double() + 1e-5))
        assert rel_err(bad, dx) > 100 * 2e-5, rel_err(bad, dx)


def test_batchnorm_shapes_cover_both_forms():
    forms = {(R.bn_split_form(s[0], s[1], _hw(s)), _hw(s) % 4 == 0) for s in BN_SHAPES}
    assert forms == {(True, True), (True, False), (False, True), (False, False)}
    assert any(s[1] > R.BN_MAX_C for s in BN_SHAPES) and any(len(s) == 2 for s in BN_SHAPES)


@pytest.mark.parametrize("layer", ["gluon", "nd"])
def test_batchnorm_use_global_stats_through_the_layers(nat, layer):
    """gluon.nn.BatchNorm(use_global_stats=True) under autograd.record() and nd.BatchNorm(use_global_stats=True): the input gradient is
    dy·γ·rsqrt(rv+eps) and the running statistics stay untouched (both kernel forms)."""
    g = torch.Generator(device=dev()).manual_seed(18)
    for shape in ((4, 3, 6, 6), (16, 3, 16, 16)):
        x, gamma, beta, rm, rv, dy = _bn_case(shape, g)
        X = mx.nd.array(x, ctx=mx.gpu(0)); X.attach_grad()
        if layer == "gluon":
            net = mx.gluon.nn.BatchNorm(use_global_stats=True, in_channels=3)
            net.initialize(ctx=mx.gpu(0))
            for p, v in ((net.gamma, gamma), (net.beta, beta), (net.running_mean, rm), (net.running_var, rv)):
                p.set_data(mx.nd.array(v, ctx=mx.gpu(0)))
            with mx.autograd.record():
                Y = net(X)
            stats = (net.running_mean.data()._t, net.running_var.data()._t)
            eps = 1e-5
        else:
            G, Bt, RM, RV = (mx.nd.array(v, ctx=mx.gpu(0)) for v in (gamma, beta, rm, rv))
            G.attach_grad(); Bt.attach_grad()
            with mx.autograd.record():
                Y = mx.nd.BatchNorm(X, G, Bt, RM, RV, eps=1e-3, fix_gamma=False, use_global_stats=True)
            stats = (RM._t, RV._t)
            eps = 1e-3
        Y.backward(mx.nd.array(dy, ctx=mx.gpu(0)))
        torch.cuda.synchronize()
        yref, dx, dg, db, _, _ = R.bn_ref(x, gamma, beta, rm, rv, False, eps, dy)
        assert rel_err(Y._t, yref) < 5e-6 and rel_err(X.grad._t, dx) < 2e-5, (layer, shape, rel_err(X.grad._t, dx))
        if layer == "nd":
            assert rel_err(G.grad._t, dg) < 1e-5 and rel_err(Bt.grad._t, db) < 1e-5
        assert torch.equal(stats[0], rm) and torch.equal(stats[1], rv)


def test_batchnorm_second_stream_and_graph_capture(nat, OF):
    """The split form's accumulators re-arm on a second stream; the first BatchNorm on a stream that is being captured into a CUDA graph
    cannot allocate them, runs the one-CTA form and gives the same numbers; replaying the graph repeats them."""
    g = torch.Generator(device=dev()).manual_seed(19)
    shape = (16, 6, 16, 16)
    assert R.bn_split_form(shape[0], shape[1], _hw(shape))
    x, gamma, beta, rm, rv, dy = _bn_case(shape, g)
    yref, *_ , bmean, bvar = R.bn_ref(x, gamma, beta, rm, rv, True, 1e-5, dy)
    s2 = torch.cuda.Stream()
    s2.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s2):
        for _ in range(3):
            y2 = OF.batch_norm(x, gamma, beta, rm.clone(), rv.clone(), True)
        assert nat.bn_workspace_ready()
    torch.cuda.synchronize()
    assert rel_err(y2, yref) < 5e-6
    fresh = None
    for prio in (0, -1):
        for _ in range(40):
            s = torch.cuda.Stream(priority=prio)
            if not nat.bn_workspace_ready(s):
                fresh = s
                break
        if fresh is not None:
            break
    assert fresh is not None, "every pooled stream already holds BatchNorm accumulators"
    rmc, rvc = rm.clone(), rv.clone()
    static_x = x.clone()
    graph = torch.cuda.CUDAGraph()
    fresh.wait_stream(torch.cuda.current_stream())
    with torch.cuda.graph(graph, stream=fresh):
        yg = OF.batch_norm(static_x, gamma, beta, rmc, rvc, True, momentum=0.0)
    assert not nat.bn_workspace_ready(fresh)
    graph.replay()
    torch.cuda.synchronize()
    assert rel_err(yg, yref) < 5e-6 and rel_err(rvc, bvar) < 2e-6 and rel_err(rmc, bmean) < 2e-6
    static_x.mul_(2.0)
    graph.replay()
    torch.cuda.synchronize()
    assert rel_err(rvc, 4 * bvar) < 2e-6


@pytest.mark.parametrize("offset", [0.0, 100.0, 1000.0])
@pytest.mark.parametrize("shape", [(4, 4, 28, 28), (16, 4, 28, 28)], ids=["one_cta", "split"])
def test_batchnorm_statistics_of_offset_data(nat, shape, offset):
    """Batch statistics of data whose |mean|/std is 0, 100 and 1000, both forms, against fp64, under ONE tolerance: saved mean within
    2e-6·std + 16u·|mean| (the one-CTA form sums x in fp32), variance and inverse standard deviation within 1e-5 relative, y within fp32 rounding of its terms.

    The split form used to accumulate Σx and Σx² in fp32 and form E[x²] − mean²; it now subtracts a per-channel pivot (x[0, c, 0]) first.
    Worst relative variance error over the four channels, measured on an H100 80GB HBM3 (power limit 700 W):
    offset 0 / 100 / 1000: one-CTA 7.5e-8 / 8.8e-8 / 1.1e-7, split 2.7e-8 / 3.4e-8 / 3.5e-8 (inverse std <= 1e-7 everywhere);
    the split form without the pivot: 2.7e-8 / 4.1e-4 / 1.3e-2, i.e. 40x and 1300x outside the tolerance."""
    g = torch.Generator(device=dev()).manual_seed(20)
    N, C, HW = shape[0], shape[1], _hw(shape)
    x = torch.randn(*shape, device=dev(), generator=g) + offset * torch.tensor([1.0, -1.0, 0.5, 1.0], device=dev()).view(1, C, 1, 1)
    gamma = torch.rand(C, device=dev(), generator=g) + 0.5; beta = torch.randn(C, device=dev(), generator=g)
    rm, rv = torch.zeros(C, device=dev()), torch.ones(C, device=dev())
    if R.bn_split_form(N, C, HW):
        nat.bn_fwd(x, gamma, beta, rm.clone(), rv.clone(), True, 0.0, 1e-5)
        assert nat.bn_workspace_ready()
    y, sm, si = nat.bn_fwd(x, gamma, beta, rm, rv, True, 0.0, 1e-5)
    torch.cuda.synchronize()
    xd = x.double()
    mean = xd.mean((0, 2, 3)); var = xd.var((0, 2, 3), unbiased=False); inv = 1.0 / torch.sqrt(var + 1e-5)
    std = var.sqrt()
    e_mean = float(((sm.double() - mean).abs() / (2e-6 * std + 16 * R.U32 * mean.abs())).max())
    e_var = float(((rv.double() - var).abs() / var).max())
    e_inv = float(((si.double() - inv).abs() / inv).max())
    a = gamma.double() * inv
    yref = (xd - mean.view(1, C, 1, 1)) * a.view(1, C, 1, 1) + beta.double().view(1, C, 1, 1)
    ybound = 8 * R.U32 * (xd.abs() * a.view(1, C, 1, 1) + beta.double().abs().view(1, C, 1, 1) + (mean.abs() * a).view(1, C, 1, 1)) \
        + 2e-6 * (yref - beta.double().view(1, C, 1, 1)).abs()
    e_y = float(((y.double() - yref).abs() / ybound).max())
    print("MEASURED bn offset %g %s: mean %.3g (of bound) var %.3g inv %.3g y %.3g (of bound)"
          % (offset, "split" if R.bn_split_form(N, C, HW) else "one-CTA", e_mean, e_var, e_inv, e_y))
    assert e_mean < 1 and e_var < 1e-5 and e_inv < 1e-5 and e_y < 1, (offset, shape, e_mean, e_var, e_inv, e_y)
    assert torch.equal(rm, sm)


# ====================================================================================================================== H. network
@pytest.mark.parametrize("global_stats", [False, True])
def test_small_gluon_network_end_to_end(nat, OF, global_stats):
    """Conv2D(3->5, 3x3, pad 1) -> BatchNorm -> ReLU -> MaxPool2D -> Dense(10) -> softmax-CE on the GPU kernels: loss and every parameter
    gradient against the same network evaluated in fp64 with use_native(False); running statistics updated (or, with global statistics,
    untouched) as the fp64 network does."""
    mx.random.seed(3); torch.manual_seed(3)
    net = mx.gluon.nn.HybridSequential()
    net.add(mx.gluon.nn.Conv2D(5, 3, padding=1, in_channels=3), mx.gluon.nn.BatchNorm(use_global_stats=global_stats, in_channels=5),
            mx.gluon.nn.Activation("relu"), mx.gluon.nn.MaxPool2D(2, 2), mx.gluon.nn.Dense(10))
    net.initialize(mx.init.Xavier(), ctx=mx.gpu(0))
    g = torch.Generator(device=dev()).manual_seed(21)
    x = torch.randn(8, 3, 12, 12, device=dev(), generator=g)
    label = torch.randint(0, 10, (8,), device=dev(), generator=g).float()
    net(mx.nd.array(x, ctx=mx.gpu(0)))
    bn = net[1]
    bn.running_mean.set_data(mx.nd.array(torch.randn(5, device=dev(), generator=g) * 0.1, ctx=mx.gpu(0)))
    bn.running_var.set_data(mx.nd.array(torch.rand(5, device=dev(), generator=g) + 0.5, ctx=mx.gpu(0)))
    params = [p for p in net.collect_params().values()]
    before = {p.name: p.data()._t.detach().clone() for p in params}
    loss_fn = mx.gluon.loss.SoftmaxCrossEntropyLoss()
    with mx.autograd.record():
        loss = loss_fn(net(mx.nd.array(x, ctx=mx.gpu(0))), mx.nd.array(label, ctx=mx.gpu(0)))
    loss.backward()
    torch.cuda.synchronize()
    conv, dense = net[0], net[4]
    P = {k: before[p.name].double().requires_grad_(True)
         for k, p in (("cw", conv.weight), ("cb", conv.bias), ("g", bn.gamma), ("b", bn.beta), ("dw", dense.weight), ("db", dense.bias))}
    rm, rv = before[bn.running_mean.name].double(), before[bn.running_var.name].double()
    OF.use_native(False)
    try:
        with torch.enable_grad():
            h0 = OF.conv2d(x.double(), P["cw"], P["cb"], (1, 1), (1, 1))
            h = OF.batch_norm(h0, P["g"], P["b"], rm, rv, not global_stats, 0.9, 1e-5)
            h = OF.max_pool2d(OF.activation(h, "relu"), (2, 2), (2, 2))
            lref = OF.softmax_cross_entropy(OF.dense(h, P["dw"], P["db"]), label.double())
            *grads, dh0 = torch.autograd.grad(lref.sum(), list(P.values()) + [h0])
            gref = dict(zip(P, grads))
    finally:
        OF.use_native(True)
    assert rel_err(loss._t, lref.detach()) < 1e-5, rel_err(loss._t, lref.detach())
    for k, p in (("cw", conv.weight), ("cb", conv.bias), ("g", bn.gamma), ("b", bn.beta), ("dw", dense.weight), ("db", dense.bias)):
        if k == "cb" and not global_stats:
            # batch statistics remove the conv bias: its gradient is zero up to the rounding of a sum of the conv output's gradients
            err = float((p.grad()._t.double() - gref[k]).abs().max())
            assert err <= 2e-5 * float(dh0.abs().sum((0, 2, 3)).min()), (k, err)
            continue
        assert rel_err(p.grad()._t, gref[k]) < 2e-5, (k, rel_err(p.grad()._t, gref[k]))
    if global_stats:
        assert torch.equal(bn.running_mean.data()._t, before[bn.running_mean.name]) and torch.equal(bn.running_var.data()._t, before[bn.running_var.name])
    else:
        assert rel_err(bn.running_mean.data()._t, rm) < 1e-5 and rel_err(bn.running_var.data()._t, rv) < 1e-5
