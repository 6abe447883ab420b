"""fp64 references and host dispatch predicates of the generic operator path (``ops/functional.py`` -> ``ops/autograd_fns.py`` ->
``gemm_wgmma.cu``, ``conv_pool.cu``, ``depthwise_conv.cu``, ``batchnorm.cu``), shared by ``test_generic_ops.py`` (CPU) and
``test_generic_ops_gpu.py``.  Every predicate restates the host code it names so that a test can assert which kernel ran."""
import math

import torch
import torch.nn.functional as F

U32 = 2.0 ** -24                    # unit roundoff of fp32
GEMM_ELEM_C = 16                    # |D - A·Bᵀ| <= GEMM_ELEM_C · √K · u · (|A|·|B|ᵀ) element-wise (plus the epilogue's own rounding)
GEMM_NORM_C = 8                     # ||D - A·Bᵀ||_F <= GEMM_NORM_C · √K · u · ||A·Bᵀ||_F


# ------------------------------------------------------------------------------------------------------------------------ GEMM
BLOCK_M, BLOCK_K, ACC_CHUNK_KB = 128, 32, 4


def gemm_block_n(M, N, b_mn, sms):
    """Tile width gemm_tf32_impl picks (gemm_wgmma.cu: narrow tiles for small problems, 128 once they alone fill every SM)."""
    mt = -(-M // BLOCK_M)
    block_n = 16
    for bn in (128, 64, 32, 16):
        if mt * -(-N // bn) >= 24 or bn == 16:
            block_n = bn
            break
    if mt * -(-N // 128) >= sms:
        block_n = 128
    if b_mn and block_n < 32:
        block_n = 32
    return block_n


def gemm_tma_ok(A_ptr, lda, B_ptr, ldb, K):
    """gemm_tf32_impl's refusal test: False sends the call to the CUDA-core kernel (TMA needs 16-byte aligned bases and strides)."""
    return K > 0 and lda % 4 == 0 and ldb % 4 == 0 and A_ptr % 16 == 0 and B_ptr % 16 == 0


def gemm_splits(K, split_k):
    """(K blocks, K blocks per split, effective splits) as gemm_tf32_impl derives them."""
    num_kb = -(-K // BLOCK_K)
    s = max(1, min(split_k, num_kb))
    per = -(-num_kb // s)
    return num_kb, per, -(-num_kb // per)


def gemm_ref(A, B, a_mn=False, b_mn=False, alpha=1.0, bias=None, relu=False, mask=None):
    """fp64 D = epi(alpha · A·Bᵀ) from the operands as the kernel reads them; also |alpha|·|A|·|B|ᵀ + |bias| (the element-wise error scale)."""
    Ad = (A.t() if a_mn else A).double()
    Bd = (B.t() if b_mn else B).double()
    D = alpha * (Ad @ Bd.t())
    scale = abs(alpha) * (Ad.abs() @ Bd.abs().t())
    if bias is not None:
        D = D + bias.double()
        scale = scale + bias.double().abs()
    if relu:
        D = D.clamp_min(0.0)
    if mask is not None:
        D = torch.where(mask > 0, D, torch.zeros_like(D))
    return D, scale


def gemm_elem_excess(D, ref, scale, K):
    """max of |D - ref| / bound (> 1 fails), bound = GEMM_ELEM_C·√K·u·scale + 2u·|ref| (alpha and bias roundings) + tiny."""
    bound = GEMM_ELEM_C * math.sqrt(max(K, 1)) * U32 * scale + 2 * U32 * ref.abs() + 1e-30
    return float(((D.double() - ref).abs() / bound).max())


def gemm_norm_bound(K):
    return GEMM_NORM_C * math.sqrt(max(K, 1)) * U32


def rel_err(a, b):
    return float((a.double() - b.double()).norm() / (b.double().norm() + 1e-300))


# ------------------------------------------------------------------------------------------------------------------------ convolution
def im2col_tiled(C, H, W, KH, KW, stride, padding):
    """gx_im2col: the shared-memory tiled kernel needs stride 1, no padding, ldc == K (K % 4 == 0) and 4 planes in 96 KB."""
    K = C * KH * KW
    ldc = (K + 3) // 4 * 4
    return tuple(stride) == (1, 1) and tuple(padding) == (0, 0) and ldc == K and 4 * H * W * 4 <= 96 * 1024


def col2im_tiled(C, H, W, KH, KW, stride, padding):
    """gx_col2im: the tiled kernel needs stride 1, no padding and a [OH·OW][4·KH·KW] slab in 160 KB."""
    OH, OW = H - KH + 1, W - KW + 1
    return tuple(stride) == (1, 1) and tuple(padding) == (0, 0) and OH * OW * 4 * KH * KW * 4 <= 160 * 1024


def conv_ref(x, w, b, stride, padding):
    return F.conv2d(x.double(), w.double(), None if b is None else b.double(), stride, padding)


def conv_grads_ref(x, w, dz, stride, padding, has_bias):
    """fp64 dx, dw, db of a convolution for the pre-activation gradient dz (already routed through the kernel's ReLU mask)."""
    xd, wd, dzd = x.double(), w.double(), dz.double()
    dx = torch.nn.grad.conv2d_input(xd.shape, wd, dzd, stride, padding)
    dw = torch.nn.grad.conv2d_weight(xd, wd.shape, dzd, stride, padding)
    db = dzd.sum((0, 2, 3)) if has_bias else None
    return dx, dw, db


def depthwise_grads_ref(x, w, dz, stride, padding):
    xd = x.double().requires_grad_(True)
    wd = w.double().requires_grad_(True)
    y = F.conv2d(xd, wd, None, stride, padding, groups=x.shape[1])
    dx, dw = torch.autograd.grad(y, (xd, wd), dz.double())
    return dx, dw, dz.double().sum((0, 2, 3))


# ------------------------------------------------------------------------------------------------------------------------ pooling
def maxpool2x2_ref(x):
    """fp64 2x2/2 max-pool with the FIRST maximum of each window winning (window order (0,0), (0,1), (1,0), (1,1)): values and arg-max."""
    N, C, H, W = x.shape
    win = x.double().reshape(N, C, H // 2, 2, W // 2, 2).permute(0, 1, 2, 4, 3, 5).reshape(N, C, H // 2, W // 2, 4)
    best = win.max(-1).values
    hit = win == best.unsqueeze(-1)
    first = torch.argmax(hit.to(torch.uint8), dim=-1)          # argmax returns the first maximal index
    return best, first.to(torch.uint8)


def maxpool2x2_route(dy, idx):
    """Scatter the pooled gradient to the arg-max position of every window (fp64)."""
    N, C, PH, PW = dy.shape
    out = torch.zeros(N, C, 2 * PH, 2 * PW, dtype=torch.float64, device=dy.device)
    for k in range(4):
        out[:, :, (k >> 1)::2, (k & 1)::2] = torch.where(idx == k, dy.double(), torch.zeros((), dtype=torch.float64, device=dy.device))
    return out


# ------------------------------------------------------------------------------------------------------------------------ BatchNorm
BN_MAX_C = 16384


def bn_split_form(N, C, HW):
    """gx_bn_fwd / gx_bn_bwd take the (channel, slice)-grid statistics kernel + streaming apply kernel for feature maps, else one CTA per
    channel (the split form also needs the per-stream accumulators, which the first launch inside a graph capture cannot allocate)."""
    return N * HW >= 4096 and HW >= 16 and C <= BN_MAX_C


def bn_ref(x, gamma, beta, rm, rv, training, eps, dy):
    """fp64 BatchNorm forward and gradients.  training: batch statistics (population variance); otherwise the running statistics, which
    are constants.  Returns y, dx, dgamma, dbeta, batch mean, batch variance."""
    C = x.shape[1]
    dims = [0] + list(range(2, x.dim()))
    shp = [1, C] + [1] * (x.dim() - 2)
    xd = x.double().requires_grad_(True)
    gd = gamma.double().requires_grad_(True)
    bd = beta.double().requires_grad_(True)
    bmean = xd.detach().mean(dims)
    bvar = ((xd.detach() - bmean.view(shp)) ** 2).mean(dims)
    if training:
        mean = xd.mean(dims, keepdim=True)
        var = ((xd - mean) ** 2).mean(dims, keepdim=True)
    else:
        mean, var = rm.double().view(shp), rv.double().view(shp)
    y = (xd - mean) / torch.sqrt(var + eps) * gd.view(shp) + bd.view(shp)
    dx, dg, db = torch.autograd.grad(y, (xd, gd, bd), dy.double())
    return y.detach(), dx, dg, db, bmean, bvar


def bn_dx_batch_formula(x, dy, gamma, mean, invstd):
    """The batch-statistics input gradient k·(dy − mean(dy) − x̂·mean(dy·x̂)) with the given mean / invstd (fp64): what a kernel that ignores
    fixed statistics computes."""
    C = x.shape[1]
    dims = [0] + list(range(2, x.dim()))
    shp = [1, C] + [1] * (x.dim() - 2)
    xh = (x.double() - mean.double().view(shp)) * invstd.double().view(shp)
    g = dy.double()
    k = gamma.double().view(shp) * invstd.double().view(shp)
    return k * (g - g.mean(dims, keepdim=True) - xh * (g * xh).mean(dims, keepdim=True))
