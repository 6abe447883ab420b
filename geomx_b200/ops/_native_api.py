"""Python wrappers over the C ABI of ``libgeomx_kernels.so``.  All functions take raw CUDA ``torch.Tensor`` s, launch on
the current stream and return nothing (or the output tensor); shapes/dtypes are asserted here, not in the kernels."""
from __future__ import annotations

import ctypes
import math
from typing import NamedTuple

import torch

from . import native as _n

_DT = {torch.float32: 0, torch.float16: 1, torch.bfloat16: 2}


def _lib():
    return _n.require()


def _s():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _p(t):
    return ctypes.c_void_p(0 if t is None else t.data_ptr())


def _ck(rc, what):
    _n.launch_count += 1
    if rc != 0:
        raise RuntimeError("%s failed (rc=%d)" % (what, rc))


def _f32c(t):
    assert t.is_cuda and t.dtype == torch.float32 and t.is_contiguous(), "expected contiguous CUDA fp32 tensor"
    return t


def _aligned(t, nbytes):
    """``t`` itself when its data starts on an ``nbytes`` boundary, else an aligned copy (for kernels with vector accesses and no scalar
    path; a contiguous view such as ``x[1:]`` can start anywhere)."""
    return t if t.data_ptr() % nbytes == 0 else t.clone()


# --------------------------------------------------------------------------------------------------------------- GEMM
def set_gemm_precision(mode):
    """Process-wide multiply precision of the wgmma GEMM: ``"3xtf32"`` (default; fp32-accurate: hi/lo split of both operands, three MMAs per
    K step, fp32 accumulation — matches the reference's fp32 SGEMM, linalg_impl.h:196-214) or ``"tf32"`` (one MMA, 10-bit mantissa)."""
    return _lib().gx_gemm_set_precision(1 if str(mode).lower() in ("tf32", "1", "fast") else 3)


def gemm_precision():
    return "tf32" if _lib().gx_gemm_get_precision() == 1 else "3xtf32"


def gemm(A, B, D, a_mn=False, b_mn=False, bias=None, mask=None, colsum=None, relu=False, accumulate=False,
         store_nchw_hw=0, alpha=1.0, split_k=1, M=None, N=None, K=None, lda=None, ldb=None, ldd=None, force_simt=False):
    """D[M,N] = epi(alpha * A·Bᵀ).  A is [M,K] (K-major) or [K,M] (MN-major, ``a_mn``); B is [N,K] or [K,N] (``b_mn``).
    ``split_k > 1`` adds the partial products of K slices into D (so D must hold zeros, or the value to accumulate onto); it cannot be
    combined with ``relu`` (raises RuntimeError)."""
    if M is None:
        M = A.shape[1] if a_mn else A.shape[0]
    if K is None:
        K = A.shape[0] if a_mn else A.shape[1]
    if N is None:
        N = B.shape[1] if b_mn else B.shape[0]
    lda = A.stride(0) if lda is None else lda
    ldb = B.stride(0) if ldb is None else ldb
    if ldd is None:
        ldd = D.stride(0) if (store_nchw_hw == 0 and D.dim() >= 2) else N
    ldmask = mask.stride(0) if mask is not None else 0
    lib = _lib()
    rc = -1
    if not force_simt:
        rc = lib.gx_gemm_tf32(_p(A), lda, int(a_mn), _p(B), ldb, int(b_mn), M, N, K, _p(D), ldd, _p(bias), _p(mask), ldmask,
                              _p(colsum), int(relu), int(accumulate), 1 if store_nchw_hw else 0, int(store_nchw_hw), float(alpha),
                              int(split_k), _s())
    if rc == -1:  # TMA alignment not satisfied -> CUDA-core fallback kernel (same contract)
        rc = lib.gx_gemm_simt(_p(A), lda, int(a_mn), _p(B), ldb, int(b_mn), M, N, K, _p(D), ldd, _p(bias), _p(mask), ldmask,
                              _p(colsum), int(relu), int(accumulate), 1 if store_nchw_hw else 0, int(store_nchw_hw), float(alpha), _s())
    _ck(rc, "gemm")
    return D


def gemm_pool(A, B, pooled, idx, OH, OW, bias=None, relu=True, a_mn=False, b_mn=False, alpha=1.0):
    """Convolution-as-GEMM with bias + ReLU + 2x2/2 max-pool fused into the GEMM epilogue.  ``A``: [images*OH*OW, K] im2col rows,
    ``B``: [N, K] filters; writes ``pooled`` [images, N, OH/2, OW/2] and ``idx`` (uint8 arg-max).  Returns False when the geometry does not
    fit the in-warp pooling (caller falls back to gemm + maxpool2x2_fwd)."""
    M = A.shape[1] if a_mn else A.shape[0]
    K = A.shape[0] if a_mn else A.shape[1]
    N = B.shape[1] if b_mn else B.shape[0]
    rc = _lib().gx_gemm_tf32_pool(_p(A), A.stride(0), int(a_mn), _p(B), B.stride(0), int(b_mn), M, N, K, _p(pooled), _p(bias), int(relu), OH * OW, OW,
                                  _p(idx), float(alpha), _s())
    if rc == -1:
        return False
    _ck(rc, "gemm_pool")
    return True


def mlp_chain(x, w0, b0, w1, b1, w2, b2, label, loss, logits, dw0, db0, dw1, db1, dw2, db2, dx):
    """Dense(D1,relu) -> Dense(D2,relu) -> Dense(C) -> softmax-CE, forward and backward (csrc/kernels/mlp_chain.cu): the cluster launch of
    :func:`mlp_chain_data`, then :func:`dense_wgrad`, both on the current stream, with scratch tensors of their own.
    Returns False when the shapes are not the compiled 512 -> 256 -> 128 -> C<=16, batch <= 32 (callers then use the per-layer kernels)."""
    B = x.shape[0]
    e = lambda *s: torch.empty(*s, dtype=torch.float32, device=x.device)
    a3, a4, dz4, dz3, dl = e(B, w0.shape[0]), e(B, w1.shape[0]), e(B, w1.shape[0]), e(B, w0.shape[0]), e(B, 16)
    if not mlp_chain_data(x, w0, b0, w1, b1, w2, b2, label, loss, logits, dx, a3, a4, dz4, dz3, dl):
        return False
    dense_wgrad(x, a3, a4, dz4, dz3, dl, dw0, db0, dw1, db1, dw2, db2)
    return True


def _weight(weight, B):
    assert weight is None or (weight.shape == (B,) and weight.is_cuda and weight.dtype == torch.float32 and weight.is_contiguous())
    return _p(weight)


def mlp_chain_data(x, w0, b0, w1, b1, w2, b2, label, loss, logits, dx, a3, a4, dz4, dz3, dl, weight=None):
    """The data path of the dense chain in ONE cluster launch: per-sample loss, logits and dx; it also stores what :func:`dense_wgrad` reads:
    a3 [B,D1], a4 [B,D2], dz4 [B,D2], dz3 [B,D1] and the dlogits dl [B,16].  ``weight`` [B] (fp32): the dlogits of row b are scaled by
    ``weight[b]`` before anything is derived from them (the weighted instance of the kernel); the loss is not.  Returns False for shapes
    other than 512 -> 256 -> 128 -> C<=16, batch <= 32."""
    B, D0 = x.shape
    D1, D2, C = w0.shape[0], w1.shape[0], w2.shape[0]
    rc = _lib().gx_mlp_chain(_p(x), _p(w0), _p(b0), _p(w1), _p(b1), _p(w2), _p(b2), _p(label), _p(loss), _p(logits), _p(dx),
                             _p(a3), _p(a4), _p(dz4), _p(dz3), _p(dl), _weight(weight, B), B, D0, D1, D2, C, _s())
    if rc == -1:
        return False
    _ck(rc, "mlp_chain")
    return True


def dense_tail(a3, w0, w1, b1, w2, b2, label, loss, logits, dx, a4, dz4, dz3, dl, from_dz3=False, weight=None):
    """The data path of the dense chain from a3 [B,D1] on (what :func:`cnn_fwd_dense0` computed), in ONE cluster launch: per-sample loss,
    logits and dx [B,D0]; it also stores a4, dz4, dz3 and the dlogits dl [B,16] for :func:`dense_wgrad` (a3 is already in memory).  ``w0``
    [D1,D0] is read for dx only.  ``from_dz3=True``: dz3 [B,D1] is the input (what :func:`cnn_fwd_dense0`'s training head computed) and the
    launch computes dx = dz3 · w0 only; the other buffers are neither read nor written.  ``weight`` [B] (not with ``from_dz3``, whose dz3
    already carries it) scales the dlogits as in :func:`mlp_chain_data`.  Returns False for shapes other than 512 -> 256 -> 128 -> C<=16,
    batch <= 32."""
    B, D1 = dz3.shape
    D0, D2, C = w0.shape[1], w1.shape[0], w2.shape[0]
    assert w0.shape[0] == D1 and dx.shape == (B, D0) and dl.shape == (B, 16) and dz3.is_contiguous()
    assert weight is None or not from_dz3, "from_dz3: the weights are applied where dz3 is computed"
    rc = _lib().gx_dense_tail(_p(a3), _p(w0), _p(w1), _p(b1), _p(w2), _p(b2), _p(label), _p(loss), _p(logits), _p(dx), _p(a4), _p(dz4), _p(dz3),
                              _p(dl), _weight(weight, B), B, D0, D1, D2, C, int(bool(from_dz3)), _s())
    if rc == -1:
        return False
    _ck(rc, "dense_tail")
    return True


def capture_demote_joined_edges():
    """While the current stream is being captured into a CUDA graph: the launch just captured on it keeps its programmatic edge from the
    launch before it on this stream, and waits for the streams it joined through full edges.  Returns the number of edges changed (0 when
    the stream is not capturing)."""
    rc = _lib().gx_capture_demote_joined_edges(_s())
    if rc < 0:
        raise RuntimeError("gx_capture_demote_joined_edges failed")
    return rc


def dense_wgrad(x, a3, a4, dz4, dz3, dl, dw0, db0, dw1, db1, dw2, db2):
    """The dense chain's weight and bias gradients (overwritten) from what :func:`mlp_chain_data` stored: dW0 = dz3ᵀ·x, dW1 = dz4ᵀ·a3,
    dW2 = dlᵀ·a4 and their column sums, one launch."""
    B, D0 = x.shape
    D1, D2, C = a3.shape[1], a4.shape[1], dw2.shape[0]
    assert dl.shape == (B, 16) and all(t.shape[0] == B for t in (a3, a4, dz4, dz3))
    rc = _lib().gx_dense_wgrad(_p(x), _p(a3), _p(a4), _p(dz4), _p(dz3), _p(dl), _p(dw0), _p(db0), _p(dw1), _p(db1), _p(dw2), _p(db2),
                               B, D0, D1, D2, C, _s())
    _ck(rc, "dense_wgrad")


# --------------------------------------------------------------------------------------------------------------- demo-CNN direct convolutions
def cnn_fwd(x, w0, b0, w1, b1, a1, idx1, a2, idx2, carry=None, x_keep=None):
    """Conv(16,k5)+ReLU+MaxPool2 -> Conv(32,k5)+ReLU+MaxPool2 of the demo CNN in one launch (csrc/kernels/cnn_direct.cu), fp32 FMA.
    ``carry=(src, dst)``: also copy the small fp32 vector ``src`` to ``dst`` (the labels of a look-ahead step, see models/cnn.py);
    ``x_keep``: also store a copy of the image batch there (its backward pass runs after the next batch has arrived in ``x``)."""
    src, dst = carry if carry is not None else (None, None)
    _ck(_lib().gx_cnn_fwd(_p(x), _p(w0), _p(b0), _p(w1), _p(b1), _p(a1), _p(idx1), _p(a2), _p(idx2), _p(src), _p(dst),
                          0 if src is None else src.numel(), _p(x_keep), x.shape[0], _s()), "cnn_fwd")


def cnn_fwd_dense0(x, w0, b0, w1, b1, wd, bd, a1, idx1, a2, idx2, a3, carry=None, x_keep=None, *, wd1=None, bd1=None, wd2=None, bd2=None,
                   label=None, loss=None, logits=None, a4=None, dz4=None, dz3=None, dl=None, weight=None):
    """:func:`cnn_fwd` followed by the first dense layer in the same launch: also a3 [B,256] = relu(a2.view(B,512) · wdᵀ + bd), with
    wd [256,512].  ``carry`` / ``x_keep`` as in :func:`cnn_fwd`.  Runs clusters of two images: returns False without launching for odd B or
    B > 32.

    With ``a4`` given, the same launch also runs the rest of the dense chain's row-separable part (the training head): dense1 (``wd1``
    [128,256], ``bd1``), the classifier (``wd2`` [10,128], ``bd2``) and softmax-CE against ``label`` [B] (float class ids), and the data
    gradients down to dz3.  It writes loss [B], logits [B,10] (skipped when None), a4 [B,128], dz4 [B,128], dz3 [B,256] and the dlogits
    dl [B,16] (classes >= 10 zero): what :func:`dense_tail` with ``from_dz3=True`` and :func:`dense_wgrad` read.  ``weight`` [B] (with the
    head only) scales the dlogits of row b by ``weight[b]`` before dz4 and dz3 are derived from them (the weighted instance of the kernel);
    the loss is not."""
    B = x.shape[0]
    assert weight is None or a4 is not None, "weight scales the training head's dlogits"
    assert wd.shape == (256, 512) and a3.shape == (B, 256) and a3.is_contiguous()
    head = (wd1, bd1, wd2, bd2, label, loss, logits, a4, dz4, dz3, dl)
    if a4 is not None:
        assert wd1.shape == (128, 256) and wd2.shape == (10, 128) and label.numel() == B and loss.numel() == B
        assert all(t.is_contiguous() for t in (wd1, wd2, a4, dz4, dz3, dl))
        assert a4.shape == (B, 128) and dz4.shape == (B, 128) and dz3.shape == (B, 256) and dl.shape == (B, 16)
        assert logits is None or (logits.shape == (B, 10) and logits.is_contiguous())
    src, dst = carry if carry is not None else (None, None)
    rc = _lib().gx_cnn_fwd_dense0(_p(x), _p(w0), _p(b0), _p(w1), _p(b1), _p(wd), _p(bd), _p(a1), _p(idx1), _p(a2), _p(idx2), _p(a3), _p(src),
                                  _p(dst), 0 if src is None else src.numel(), _p(x_keep),
                                  *(_p(t) if a4 is not None else None for t in head), _weight(weight, B), B, _s())
    if rc == -1:
        return False
    _ck(rc, "cnn_fwd_dense0")
    return True


def cnn_eval(x, w0, b0, w1, b1, wd0, bd0, wd1, bd1, wd2, bd2, label, logits, loss, pred, correct):
    """Inference of the whole demo CNN for N >= 1 images in one launch (cnn_eval_kernel, csrc/kernels/cnn_direct.cu), fp32 FMA: x [N,1,28,28]
    or [N,784], the ten parameters in ``CNN_PARAM_SHAPES`` order.  Writes logits [N,10] fp32 (skipped when None) and pred [N] int32 (arg-max);
    with ``label`` [N] fp32 (class ids) also loss [N] fp32 (softmax-CE; NaN for a label that is not an integer in [0, 10)) and correct [N]
    int32 (1 where pred == label).  ``label=None`` (predict only) leaves ``loss`` / ``correct`` unwritten; they may be None then."""
    N = x.shape[0]
    if N < 1:
        raise ValueError("cnn_eval needs at least one image")
    shapes = [(16, 1, 5, 5), (16,), (32, 16, 5, 5), (32,), (256, 512), (256,), (128, 256), (128,), (10, 128), (10,)]
    for t, s in zip((w0, b0, w1, b1, wd0, bd0, wd1, bd1, wd2, bd2), shapes):
        assert t.numel() == math.prod(s), ("parameter shape", tuple(t.shape), s)
        _f32c(t)
    assert x.numel() == N * 784, ("images must be [N,1,28,28] or [N,784]", tuple(x.shape))
    _f32c(x)
    outs = [(pred, torch.int32, (N,))]
    if logits is not None:
        outs.append((logits, torch.float32, (N, 10)))
    if label is not None:
        outs += [(label, torch.float32, (N,)), (loss, torch.float32, (N,)), (correct, torch.int32, (N,))]
    for t, dt, s in outs:
        assert t is not None and t.is_cuda and t.dtype == dt and t.is_contiguous() and t.numel() == math.prod(s), \
            ("expected contiguous CUDA %s of %d elements" % (dt, math.prod(s)), None if t is None else (t.dtype, tuple(t.shape)))
    _ck(_lib().gx_cnn_eval(_p(x), _p(w0), _p(b0), _p(w1), _p(b1), _p(wd0), _p(bd0), _p(wd1), _p(bd1), _p(wd2), _p(bd2), _p(label), _p(logits),
                           _p(loss), _p(pred), _p(correct), N, _s()), "cnn_eval")


def cnn_bwd(x, w1, a1, idx1, a2, idx2, da2, dw0, db0):
    """conv1 data gradient + pool/ReLU backward of both layers + conv0 weight / bias gradient (accumulated with atomics into dw0 / db0)."""
    _ck(_lib().gx_cnn_bwd(_p(x), _p(w1), _p(a1), _p(idx1), _p(a2), _p(idx2), _p(da2), _p(dw0), _p(db0), x.shape[0], _s()), "cnn_bwd")


def cnn_bwd_all(x, w1, a1, idx1, a2, idx2, da2, dw0, db0, dw1, db1):
    """The whole convolution backward pass (``cnn_bwd`` + ``cnn_wgrad1``) as one heterogeneous-grid launch."""
    _ck(_lib().gx_cnn_bwd_all(_p(x), _p(w1), _p(a1), _p(idx1), _p(a2), _p(idx2), _p(da2), _p(dw0), _p(db0), _p(dw1), _p(db1), x.shape[0], _s()),
        "cnn_bwd_all")


def cnn_bwd_all_geometry(B):
    """How ``cnn_bwd_all`` runs at batch ``B``: a dict of its grid (CTAs), dynamic shared memory, the two bodies' shared memory, CTAs resident
    per SM and clusters of two resident on the whole idle device (occupancy queries), registers per thread, and how many of its last CTAs
    record (start, end, SM) in the debug buffer.  None for batches it does not cover."""
    import ctypes
    out = (ctypes.c_int * 8)()
    rc = _lib().gx_cnn_bwd_all_geometry(int(B), out)
    if rc == -1:
        return None
    _ck(rc, "cnn_bwd_all_geometry")
    keys = ("grid", "smem", "dgrad_smem", "wgrad_smem", "ctas_per_sm", "clusters", "regs", "stamped_ctas")
    return dict(zip(keys, list(out)))


def cnn_bwd_exchange(x, w1, a1, idx1, a2, idx2, da2, dw0, db0, dw1, db1, params, tile_list, n_active):
    """``cnn_bwd_all`` whose last CTAs also perform the exchange of the conv keys (``params``: the channel's FabricParams block from
    ``HipsFabric.channel_fused_args``): convolution backward + push + server tiers + optimizer + pull in one launch."""
    import ctypes
    _ck(_lib().gx_cnn_bwd_exchange(_p(x), _p(w1), _p(a1), _p(idx1), _p(a2), _p(idx2), _p(da2), _p(dw0), _p(db0), _p(dw1), _p(db1), x.shape[0],
                                   ctypes.byref(params), _p(tile_list), int(n_active), _s()), "cnn_bwd_exchange")


def cnn_wgrad1(a1, a2, idx2, da2, dw1, db1):
    """conv1 weight / bias gradient (overwrites dw1 / db1).  Returns False for batch sizes the kernel does not cover (odd or > 64)."""
    rc = _lib().gx_cnn_wgrad1(_p(a1), _p(a2), _p(idx2), _p(da2), _p(dw1), _p(db1), a1.shape[0], _s())
    if rc == -1:
        return False
    _ck(rc, "cnn_wgrad1")
    return True


# --------------------------------------------------------------------------------------------------------------- depthwise convolution
DW_SMEM_LIMIT = 200 * 1024       # ensure_smem in depthwise_conv.cu


def depthwise_smem(H, W, KH, KW, stride, padding):
    """Dynamic shared memory (bytes) of the forward, input-gradient and filter-gradient kernels, or None when the output is empty."""
    OH, OW = conv_out_hw(H, W, KH, KW, stride[0], stride[1], padding[0], padding[1])
    if OH < 1 or OW < 1:
        return None
    return dict(fwd=(H * W + KH * KW) * 4, dgrad=(OH * OW + KH * KW) * 4, wgrad=(H * W + OH * OW) * 4)


def depthwise_supported(x_shape, w_shape, stride, padding):
    """Whether a depthwise layer runs on the kernels: the input plane is at most ~95 KB (forward: plane + filter in shared memory) and the
    input- and filter-gradient kernels, whose footprints grow with the OUTPUT plane (padding), fit as well, so that backward never refuses
    a shape the forward accepted."""
    H, W = x_shape[2], x_shape[3]
    KH, KW = w_shape[2], w_shape[3]
    sm = depthwise_smem(H, W, KH, KW, stride, padding)
    return sm is not None and (H * W + KH * KW) * 8 <= 190 * 1024 and max(sm.values()) <= DW_SMEM_LIMIT


def depthwise_fwd(x, w, bias, y, stride, padding, relu=False):
    N, C, H, W = x.shape
    rc = _lib().gx_depthwise_fwd(_p(x), _p(w), _p(bias), _p(y), N, C, H, W, w.shape[2], w.shape[3], stride[0], stride[1], padding[0], padding[1],
                                 int(relu), _s())
    if rc == -1:
        return False
    _ck(rc, "depthwise_fwd")
    return True


def depthwise_dgrad(dy, w, dx, stride, padding):
    N, C, H, W = dx.shape
    _ck(_lib().gx_depthwise_dgrad(_p(dy), _p(w), _p(dx), N, C, H, W, w.shape[2], w.shape[3], stride[0], stride[1], padding[0], padding[1], _s()),
        "depthwise_dgrad")


def depthwise_wgrad(x, dy, dw, db, stride, padding):
    N, C, H, W = x.shape
    _ck(_lib().gx_depthwise_wgrad(_p(x), _p(dy), _p(dw), _p(db), N, C, H, W, dw.shape[2], dw.shape[3], stride[0], stride[1], padding[0], padding[1],
                                  _s()), "depthwise_wgrad")


# --------------------------------------------------------------------------------------------------------------- conv / pool
def conv_out_hw(H, W, KH, KW, sh, sw, ph, pw):
    return (H + 2 * ph - KH) // sh + 1, (W + 2 * pw - KW) // sw + 1


def conv_supported(x, w, stride, padding):
    return x.dim() == 4 and w.dim() == 4 and x.shape[1] == w.shape[1]


def im2col(x, KH, KW, stride=(1, 1), padding=(0, 0), out=None):
    N, C, H, W = x.shape
    OH, OW = conv_out_hw(H, W, KH, KW, stride[0], stride[1], padding[0], padding[1])
    K = C * KH * KW
    ldc = (K + 3) // 4 * 4
    if out is None:
        out = torch.empty(N * OH * OW, ldc, dtype=torch.float32, device=x.device)
    _ck(_lib().gx_im2col(_p(_f32c(x)), _p(out), N, C, H, W, KH, KW, stride[0], stride[1], padding[0], padding[1], ldc, _s()), "im2col")
    return out


def col2im(dcol, x_shape, KH, KW, stride=(1, 1), padding=(0, 0), out=None):
    N, C, H, W = x_shape
    if out is None:
        out = torch.empty(x_shape, dtype=torch.float32, device=dcol.device)
    _ck(_lib().gx_col2im(_p(dcol), _p(out), N, C, H, W, KH, KW, stride[0], stride[1], padding[0], padding[1], dcol.stride(0), _s()), "col2im")
    return out


def nchw_to_rows(x, out=None):
    N, C = x.shape[0], x.shape[1]
    HW = x.numel() // (N * C)
    if out is None:
        out = torch.empty(N * HW, C, dtype=torch.float32, device=x.device)
    _ck(_lib().gx_nchw_to_rows(_p(_f32c(x)), _p(out), N, C, HW, _s()), "nchw_to_rows")
    return out


def colsum(x, out=None, accumulate=False):
    R, Cc = x.shape
    if out is None:
        out = torch.empty(Cc, dtype=torch.float32, device=x.device)
    _ck(_lib().gx_colsum(_p(x), _p(out), R, Cc, x.stride(0), int(accumulate), _s()), "colsum")
    return out


def chansum_nchw(x, out=None):
    N, C = x.shape[0], x.shape[1]
    HW = x.numel() // (N * C)
    if out is None:
        out = torch.empty(C, dtype=torch.float32, device=x.device)
    _ck(_lib().gx_chansum_nchw(_p(_f32c(x)), _p(out), N, C, HW, _s()), "chansum")
    return out


def relu_fwd(x, out=None):
    out = torch.empty_like(x) if out is None else out
    _ck(_lib().gx_relu_fwd(_p(_f32c(x)), _p(out), x.numel(), _s()), "relu_fwd")
    return out


def relu_bwd(y, dy, out=None):
    out = torch.empty_like(dy) if out is None else out
    _ck(_lib().gx_relu_bwd(_p(_f32c(y)), _p(_f32c(dy)), _p(out), y.numel(), _s()), "relu_bwd")
    return out


def maxpool2x2_fwd(x, out=None, idx=None):
    N, C, H, W = x.shape
    if out is None:
        out = torch.empty(N, C, H // 2, W // 2, dtype=torch.float32, device=x.device)
    if idx is None:
        idx = torch.empty(N, C, H // 2, W // 2, dtype=torch.uint8, device=x.device)
    _ck(_lib().gx_maxpool2x2_fwd(_p(_aligned(_f32c(x), 8)), _p(out), _p(idx), N * C, H, W, _s()), "maxpool_fwd")
    return out, idx


def maxpool2x2_bwd(dy, idx, x_shape, out=None):
    N, C, H, W = x_shape
    if out is None:
        out = torch.empty(x_shape, dtype=torch.float32, device=dy.device)
    assert out.data_ptr() % 8 == 0, "maxpool2x2_bwd writes float2 pairs"
    _ck(_lib().gx_maxpool2x2_bwd(_p(_f32c(dy)), _p(idx), _p(out), N * C, H, W, _s()), "maxpool_bwd")
    return out


def pool_relu_bwd_rows(dpooled, pooled, idx, dz_rows, dbias):
    N, C, PH, PW = pooled.shape
    _ck(_lib().gx_pool_relu_bwd_rows(_p(dpooled), _p(pooled), _p(idx), _p(dz_rows), _p(dbias), N, C, PH, PW, _s()), "pool_relu_bwd_rows")


def conv_relu_pool_fwd(x, w, b, y, idx):
    N, Cin, H, W = x.shape
    Cout, _, KH, KW = w.shape
    _ck(_lib().gx_conv_relu_pool_fwd(_p(x), _p(w), _p(b), _p(y), _p(idx), N, Cin, H, W, Cout, KH, KW, _s()), "conv_relu_pool_fwd")


def conv_relu_pool_wgrad(x, dpooled, pooled, idx, dw, db, w_shape):
    N, Cin, H, W = x.shape
    Cout, _, KH, KW = w_shape
    _ck(_lib().gx_conv_relu_pool_wgrad(_p(x), _p(dpooled), _p(pooled), _p(idx), _p(dw), _p(db), N, Cin, H, W, Cout, KH, KW, _s()),
        "conv_relu_pool_wgrad")


def conv_relu_pool_im2col_fwd(x, w, b, y, idx, col, KH2, KW2):
    N, Cin, H, W = x.shape
    Cout, _, KH, KW = w.shape
    _ck(_lib().gx_conv_relu_pool_im2col_fwd(_p(x), _p(w), _p(b), _p(y), _p(idx), _p(col), N, Cin, H, W, Cout, KH, KW, KH2, KW2, col.stride(0), _s()),
        "conv_relu_pool_im2col_fwd")


def conv_relu_pool_wgrad_col2im(x, dcol, pooled, idx, dw, db, w_shape, KH2, KW2):
    N, Cin, H, W = x.shape
    Cout, _, KH, KW = w_shape
    _ck(_lib().gx_conv_relu_pool_wgrad_col2im(_p(x), _p(dcol), _p(pooled), _p(idx), _p(dw), _p(db), N, Cin, H, W, Cout, KH, KW, KH2, KW2, dcol.stride(0), _s()),
        "conv_relu_pool_wgrad_col2im")


# --------------------------------------------------------------------------------------------------------------- loss / head
def softmax_ce_fwd(logits, label, out=None):
    R, Cc = logits.shape
    out = torch.empty(R, dtype=torch.float32, device=logits.device) if out is None else out
    _ck(_lib().gx_softmax_ce_fwd(_p(_f32c(logits)), _p(_f32c(label)), _p(out), R, Cc, _s()), "softmax_ce_fwd")
    return out


def softmax_ce_bwd(logits, label, dloss, out=None):
    R, Cc = logits.shape
    out = torch.empty_like(logits) if out is None else out
    _ck(_lib().gx_softmax_ce_bwd(_p(logits), _p(label), _p(dloss), _p(out), R, Cc, _s()), "softmax_ce_bwd")
    return out


def head_fwd_bwd(a, W, bias, label, loss, logits, dW, db, da, dbias_prev, relu_mask=True, weight=None):
    """Classifier head forward and backward in one launch (csrc/kernels/loss_head.cu).  ``weight`` [B] (fp32): the dlogits of sample b are
    scaled by ``weight[b]`` before dW, db, da and dbias_prev are derived from them (the weighted instance of the kernel); the loss is not."""
    B, K = a.shape
    Cc = W.shape[0]
    _ck(_lib().gx_head_fwd_bwd(_p(a), _p(W), _p(bias), _p(label), _p(loss), _p(logits), _p(dW), _p(db), _p(da), _p(dbias_prev),
                               _weight(weight, B), B, K, Cc, int(relu_mask), _s()), "head_fwd_bwd")


# --------------------------------------------------------------------------------------------------------------- optimizers

# learning-rate schedule kinds of the kernels (SchedKind in csrc/kernels/optim.cuh); the dicts come from LRScheduler.device_spec()
SCHED_KIND = {None: 0, "none": 0, "factor": 1, "multifactor": 2, "poly": 3, "cosine": 4}
SCHED_MAX_MILESTONES = 16


class LrSchedule(ctypes.Structure):
    """Mirror of ``LrSchedule`` (csrc/kernels/optim.cuh), the last member of ``OptHyper``."""
    _fields_ = [("kind", ctypes.c_int), ("warmup_steps", ctypes.c_int), ("warmup_linear", ctypes.c_int), ("warmup_begin_lr", ctypes.c_float),
                ("step", ctypes.c_int), ("factor", ctypes.c_float), ("stop_factor_lr", ctypes.c_float), ("num_milestones", ctypes.c_int),
                ("milestones", ctypes.c_int * SCHED_MAX_MILESTONES), ("max_update", ctypes.c_int), ("final_lr", ctypes.c_float),
                ("pwr", ctypes.c_float)]


def pack_schedule(sched):
    """``LRScheduler.device_spec()`` dict (or None: constant lr) -> :class:`LrSchedule`."""
    s = LrSchedule()
    if sched is None:
        return s
    ms = [int(m) for m in sched.get("milestones", [])]
    if len(ms) > SCHED_MAX_MILESTONES:
        raise ValueError("a device schedule holds at most %d milestones, got %d" % (SCHED_MAX_MILESTONES, len(ms)))
    s.kind = SCHED_KIND[sched["kind"]]
    s.warmup_steps, s.warmup_linear = int(sched["warmup_steps"]), int(sched["warmup_mode"] == "linear")
    s.warmup_begin_lr = float(sched["warmup_begin_lr"])
    s.step, s.factor, s.stop_factor_lr = int(sched["step"]), float(sched["factor"]), float(sched["stop_factor_lr"])
    s.num_milestones = len(ms)
    for i, m in enumerate(ms):
        s.milestones[i] = m
    s.max_update, s.final_lr, s.pwr = int(sched["max_update"]), float(sched["final_lr"]), float(sched["pwr"])
    return s


class OptHyper(ctypes.Structure):
    """Mirror of ``OptHyper`` (csrc/kernels/optim.cuh): the field order is ABI.  :data:`OPT_HYPER_LAYOUT` holds the offsets that optim.cuh
    pins with static_asserts."""
    _fields_ = ([(n, ctypes.c_float) for n in ("lr", "wd", "rescale", "clip", "momentum", "beta1", "beta2", "eps", "lamda", "wd_lh",
                                               "clip_weights", "gamma1", "rho", "beta", "lamda1")]
                + [("kind", ctypes.c_int), ("sched", LrSchedule)])


OPT_HYPER_LAYOUT = dict(wd_lh=36, lamda1=56, kind=60, sched=64, size=172, sched_size=108)
assert all(getattr(OptHyper, k).offset == v for k, v in OPT_HYPER_LAYOUT.items() if k not in ("size", "sched_size"))
assert ctypes.sizeof(OptHyper) == OPT_HYPER_LAYOUT["size"] and ctypes.sizeof(LrSchedule) == OPT_HYPER_LAYOUT["sched_size"]


class OptKindInfo(NamedTuple):
    code: int               # OptKind in csrc/kernels/optim.cuh
    fields: tuple           # (OptHyper field, spec() key, default) of the kind's own hyper-parameters
    clip_zero_off: bool     # clip_gradient 0 means "no clipping": the reference passes the clip to the operator only when it is truthy
    s1_is_weight: bool      # the state slot s1 starts as the weight (DCASGD's previous weight); every other state starts at 0


# The optimizers the update kernels run, by ``Optimizer.spec()['name']``.  The state slots of a kind, and how its class's create_state()
# lays them out, are the same thing (state_slots): sgd / nag / signum: mom (None without momentum); adam: (m, v); dcasgd: (mom or None,
# previous weight); rmsprop: (n,); adagrad: history; adadelta: (acc_g, acc_delta); ftrl: (z, n).
_MOM = (("momentum", "momentum", 0.0),)
OPT_KINDS = {
    "sgd": OptKindInfo(0, _MOM, False, False),
    "adam": OptKindInfo(1, (("beta1", "beta1", 0.9), ("beta2", "beta2", 0.999), ("eps", "epsilon", 1e-8)), False, False),
    "dcasgd": OptKindInfo(2, _MOM + (("lamda", "lamda", 0.04),), False, True),
    "nag": OptKindInfo(3, _MOM, False, False),
    "signum": OptKindInfo(4, _MOM + (("wd_lh", "wd_lh", 0.0),), True, False),
    "rmsprop": OptKindInfo(5, (("gamma1", "gamma1", 0.9), ("eps", "epsilon", 1e-8), ("clip_weights", "clip_weights", -1.0)), True, False),
    "adagrad": OptKindInfo(6, (("eps", "epsilon", 1e-7),), False, False),
    "adadelta": OptKindInfo(7, (("rho", "rho", 0.9), ("eps", "epsilon", 1e-5)), False, False),
    "ftrl": OptKindInfo(8, (("beta", "beta", 1.0), ("lamda1", "lamda1", 0.01)), True, False),
}
OPT_KIND = {k: v.code for k, v in OPT_KINDS.items()}


def pack_hyper(spec):
    """``Optimizer.spec()`` dict -> :class:`OptHyper`, the kernels' view of it (its ``lr_schedule``, if any, included).  ``None``: no
    optimizer (the fabric stores the aggregated gradient)."""
    h = OptHyper()
    if spec is None:
        h.kind, h.lr, h.clip, h.rescale = -1, 0.0, -1.0, 1.0
        return h
    info = OPT_KINDS[spec["name"]]
    clip = spec.get("clip_gradient", -1.0)
    if clip is None or (info.clip_zero_off and not clip):
        clip = -1.0
    h.kind = info.code
    h.lr, h.wd, h.rescale, h.clip = spec["lr"], spec["wd"], spec["rescale_grad"], clip
    for field, key, default in info.fields:
        setattr(h, field, spec.get(key, default))
    h.sched = pack_schedule(spec.get("lr_schedule"))
    return h


def state_slots(state):
    """The tensors ``(s0, s1)`` (None: no such slot) of an optimizer state as ``create_state`` of a native kind returns it."""
    from ..ndarray import NDArray
    if state is None or isinstance(state, NDArray):
        state = (state,)
    state = tuple(state) + (None,) * (2 - len(state))
    return tuple(None if s is None else s._t for s in state)


def arena_opt(kind, w, g, s0, s1, n, tile_mult, lr, wd, rescale, clip, momentum, b1, b2, eps, lamda, step_state, g_zero=None, schedule=None):
    """Fused arena optimizer; ``lr`` is the base lr of ``schedule`` (an ``LRScheduler.device_spec()`` dict, or an :class:`LrSchedule` that
    :func:`pack_schedule` made from one), which the kernel evaluates at the device step count ``step_state[0] + 1``; ``schedule=None``:
    constant lr."""
    if schedule is not None and not isinstance(schedule, LrSchedule):
        schedule = pack_schedule(schedule)
    sched = None if schedule is None else ctypes.byref(schedule)
    _ck(_lib().gx_arena_opt(OPT_KIND[kind], _p(w), _p(g), _p(s0), _p(s1), n, _p(tile_mult), lr, wd, rescale, clip, momentum, b1, b2, eps,
                            lamda, _p(step_state), _p(g_zero), sched, _s()), "arena_opt")


def single_opt(kind, w, g, s0, s1, lr_t, wd, rescale, clip, momentum=0.0, b1=0.9, b2=0.999, eps=1e-8, lamda=0.04):
    _ck(_lib().gx_single_opt(OPT_KIND[kind], _p(w), _p(g), _p(s0), _p(s1), w.numel(), lr_t, wd, rescale, clip, momentum, b1, b2, eps, lamda, _s()),
        "single_opt")


def arena_opt_h(hyper, w, g, s0, s1, n, tile_mult, step_state, g_zero=None):
    """:func:`arena_opt` for any kind of :data:`OPT_KINDS`: ``hyper`` is the :class:`OptHyper` that :func:`pack_hyper` made from a spec."""
    _ck(_lib().gx_arena_opt_h(ctypes.byref(hyper), _p(w), _p(g), _p(s0), _p(s1), n, _p(tile_mult), _p(step_state), _p(g_zero), _s()),
        "arena_opt")


def single_opt_h(hyper, w, g, s0, s1, lr_t):
    """:func:`single_opt` for any kind; ``lr_t`` is the step's lr (Adam: bias-corrected)."""
    _ck(_lib().gx_single_opt_h(ctypes.byref(hyper), _p(w), _p(g), _p(s0), _p(s1), w.numel(), lr_t, _s()), "single_opt")


def adam_update(w, g, m, v, lr_t, b1, b2, eps, wd, rescale, clip):
    single_opt("adam", w, g.contiguous(), m, v, lr_t, wd, rescale, clip, 0.0, b1, b2, eps)


class _TensorEntry(ctypes.Structure):
    _fields_ = [("w", ctypes.c_void_p), ("g", ctypes.c_void_p), ("s0", ctypes.c_void_p), ("s1", ctypes.c_void_p),
                ("n", ctypes.c_longlong), ("lr_mult", ctypes.c_float), ("wd_mult", ctypes.c_float)]


_mt_cache = {}


def multi_tensor_update(optimizer, updater, idxs, ws, gs):
    """One launch for the whole parameter list (Trainer fused path), for an optimizer whose ``spec()`` names a kind of :data:`OPT_KINDS`."""
    from ..ndarray import NDArray
    spec = optimizer.spec()
    kind = spec["name"]
    for i, w in zip(idxs, ws):
        if i not in updater.states:
            updater.states[i] = optimizer.create_state_multi_precision(i, NDArray(w))
            updater.states_synced[i] = True
    optimizer._update_count(idxs)
    t = optimizer._index_update_count[idxs[0]]
    lr = optimizer.learning_rate
    lr_t = lr * math.sqrt(1.0 - spec["beta2"] ** t) / (1.0 - spec["beta1"] ** t) if kind == "adam" else lr
    key = (id(updater), tuple(w.data_ptr() for w in ws), tuple(g.data_ptr() for g in gs))
    ent = _mt_cache.get(key)
    if ent is None:
        arr = (_TensorEntry * len(ws))()
        for j, (i, w, g) in enumerate(zip(idxs, ws, gs)):
            s0, s1 = state_slots(updater.states[i])
            p = optimizer.param_dict.get(i)
            arr[j] = _TensorEntry(w.data_ptr(), g.data_ptr(), 0 if s0 is None else s0.data_ptr(), 0 if s1 is None else s1.data_ptr(),
                                  w.numel(), p.lr_mult if p is not None else 1.0, p.wd_mult if p is not None else 1.0)
        host = torch.frombuffer(bytearray(bytes(arr)), dtype=torch.uint8)
        dev = host.to(ws[0].device)
        ent = (dev, max(w.numel() for w in ws), len(ws))
        if len(_mt_cache) > 64:
            _mt_cache.clear()
        _mt_cache[key] = ent
    dev, max_n, cnt = ent
    h = pack_hyper(dict(spec, lr=lr_t))
    _ck(_lib().gx_multi_tensor_opt_h(ctypes.byref(h), _p(dev), cnt, max_n, lr_t, _s()), "multi_tensor_opt")
    return True


def nary_sum(out, parts):
    assert 1 <= len(parts) <= 8
    arr = (ctypes.c_void_p * len(parts))(*[p.data_ptr() for p in parts])
    _ck(_lib().gx_nary_sum(_p(out), arr, len(parts), out.numel(), _s()), "nary_sum")
    return out


def scale_cast(x, out_dtype, scale=1.0, out=None):
    out = torch.empty(x.shape, dtype=out_dtype, device=x.device) if out is None else out
    _ck(_lib().gx_scale_cast(_p(x.contiguous()), _DT[x.dtype], _p(out), _DT[out.dtype], float(scale), x.numel(), _s()), "scale_cast")
    return out


# --------------------------------------------------------------------------------------------------------------- compression
def quantize_2bit(grad, residual, out, thr):
    _ck(_lib().gx_quantize_2bit(_p(_f32c(grad)), _p(residual), _p(out), grad.numel(), thr, _s()), "quantize_2bit")


def dequantize_2bit(packed, out, thr, accumulate=False):
    _ck(_lib().gx_dequantize_2bit(_p(packed), _p(out), out.numel(), thr, int(accumulate), _s()), "dequantize_2bit")


class _BscSeg(ctypes.Structure):
    _fields_ = [("grad", ctypes.c_void_p), ("u", ctypes.c_void_p), ("v", ctypes.c_void_p), ("out", ctypes.c_void_p),
                ("n", ctypes.c_longlong), ("k", ctypes.c_int), ("sample", ctypes.c_int), ("k_sample", ctypes.c_int)]


def _segs_to_dev(segs, device):
    arr = (_BscSeg * len(segs))(*segs)
    assert ctypes.sizeof(_BscSeg) == _lib().gx_bsc_seg_size()
    return torch.frombuffer(bytearray(bytes(arr)), dtype=torch.uint8).to(device)


def bsc_segment(grad, u, v, out, k, sample, k_sample):
    return _BscSeg(grad.data_ptr() if grad is not None else 0, 0 if u is None else u.data_ptr(), 0 if v is None else v.data_ptr(),
                   out.data_ptr(), (grad if grad is not None else v).numel(), k, sample, k_sample)


def bsc_compress_batch(seg_table_dev, num, momentum=0.9):
    _ck(_lib().gx_bsc_compress_batch(_p(seg_table_dev), num, momentum, _s()), "bsc_compress")


def bsc_pull_compress_batch(seg_table_dev, num):
    _ck(_lib().gx_bsc_pull_compress_batch(_p(seg_table_dev), num, _s()), "bsc_pull_compress")


def bsc_compress(grad, u, v, out, k, sample, k_sample, momentum=0.9):
    tab = _segs_to_dev([bsc_segment(_f32c(grad), u, v, out, k, sample, k_sample)], grad.device)
    bsc_compress_batch(tab, 1, momentum)
    return out


def bsc_pull_compress(dense, out, k):
    tab = _segs_to_dev([bsc_segment(_f32c(dense), None, None, out, k, 0, 0)], dense.device)
    bsc_pull_compress_batch(tab, 1)
    return out


def bsc_decompress(zipped, out, accumulate=False):
    _ck(_lib().gx_bsc_decompress(_p(zipped), _p(out), out.numel(), zipped.numel() // 2, int(accumulate), _s()), "bsc_decompress")
    return out


def fp8_block_quantize(x, residual, q, scale):
    _ck(_lib().gx_fp8_block_quantize(_p(_f32c(x)), _p(residual), _p(q), _p(scale), x.numel(), _s()), "fp8_quantize")


def fp8_block_dequantize(q, scale, out, accumulate=False):
    _ck(_lib().gx_fp8_block_dequantize(_p(q), _p(scale), _p(out), out.numel(), int(accumulate), _s()), "fp8_dequantize")


def dgt_contrib(g, contrib, block_elems, alpha, first):
    _ck(_lib().gx_dgt_contrib(_p(g), _p(contrib), g.numel(), block_elems, alpha, int(first), _s()), "dgt_contrib")


# --------------------------------------------------------------------------------------------------------------- row-sparse helpers
def unique_i64(ids):
    """Sorted unique of a CUDA int64 vector (CUB radix sort + select; the count is read back, as UniqueImplGPU does)."""
    ids = ids.reshape(-1).contiguous()
    n = ids.numel()
    if n == 0:
        return ids
    lib = _lib()
    ws = torch.empty(int(lib.gx_unique_i64_workspace(n)) + 16, dtype=torch.uint8, device=ids.device)
    tmp, out = torch.empty_like(ids), torch.empty_like(ids)
    cnt = torch.zeros(1, dtype=torch.int32, device=ids.device)
    _ck(lib.gx_unique_i64(_p(ids), n, _p(tmp), _p(out), _p(cnt), _p(ws), ws.numel(), _s()), "unique_i64")
    return out[:int(cnt.item())]


def gather_rows(src, ids, out=None):
    L = src.numel() // src.shape[0]
    out = torch.empty((ids.numel(),) + tuple(src.shape[1:]), dtype=src.dtype, device=src.device) if out is None else out
    _ck(_lib().gx_gather_rows(_p(_f32c(src)), _p(ids.contiguous()), _p(out), ids.numel(), L, _s()), "gather_rows")
    return out


def scatter_rows(dst, ids, rows, add=False):
    L = dst.numel() // dst.shape[0]
    _ck(_lib().gx_scatter_rows(_p(_f32c(dst)), _p(ids.contiguous()), _p(_f32c(rows)), ids.numel(), L, int(add), _s()), "scatter_rows")
    return dst


# --------------------------------------------------------------------------------------------------------------- batch norm
def bn_fwd(x, gamma, beta, rm, rv, training, momentum, eps):
    N, C = x.shape[0], x.shape[1]
    HW = x.numel() // (N * C)
    x = _aligned(_f32c(x), 16)            # the feature-map kernels stream x with 128-bit loads
    y = torch.empty_like(x)
    sm = torch.empty(C, dtype=torch.float32, device=x.device)
    si = torch.empty(C, dtype=torch.float32, device=x.device)
    _ck(_lib().gx_bn_fwd(_p(_f32c(x)), _p(gamma), _p(beta), _p(rm), _p(rv), _p(y), _p(sm), _p(si), N, C, HW, int(training), momentum, eps, _s()),
        "bn_fwd")
    return y, sm, si


def bn_workspace_ready(stream=None):
    """Whether the split form's accumulators exist for ``stream`` (default: the current stream) on the current device."""
    s = torch.cuda.current_stream() if stream is None else stream
    return bool(_lib().gx_bn_workspace_ready(ctypes.c_void_p(s.cuda_stream)))


def bn_bwd(x, dy, gamma, sm, si, fixed_stats=False):
    """Input, scale and shift gradients of :func:`bn_fwd`.  ``sm`` / ``si``: the mean and inverse standard deviation the forward pass
    normalised with.  ``fixed_stats``: they were the running statistics (inference mode, ``use_global_stats``), constants with respect to x,
    so dx = dy * gamma * si; otherwise they were the batch's own and dx carries the terms of their dependence on x."""
    N, C = x.shape[0], x.shape[1]
    HW = x.numel() // (N * C)
    x, dy = _aligned(_f32c(x), 16), _aligned(_f32c(dy), 16)
    dx = torch.empty_like(x)
    dg = torch.empty(C, dtype=torch.float32, device=x.device)
    dbt = torch.empty(C, dtype=torch.float32, device=x.device)
    _ck(_lib().gx_bn_bwd(_p(x), _p(dy), _p(gamma), _p(sm), _p(si), _p(dx), _p(dg), _p(dbt), N, C, HW, int(bool(fixed_stats)), _s()), "bn_bwd")
    return dx, dg, dbt
