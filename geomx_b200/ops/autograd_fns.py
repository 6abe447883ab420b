"""``torch.autograd.Function`` nodes that put the hand-written sm_90a kernels on torch's tape (the generic Gluon path).

Forward/backward decomposition (all GEMMs on wgmma via ``native.gemm``; reference op semantics cited in ``functional.py``):
  Dense    y = x·Wᵀ+b          dx = dy·W (B MN-major)        dW = dyᵀ·x (A,B MN-major)        db = colsum(dy)
  Conv2d   col = im2col(x);  y = col·Wᵀ+b → NCHW store      dcol = dy_rows·W → col2im        dW = dy_rowsᵀ·col   db = chansum(dy)
"""
from __future__ import annotations

import torch

from . import native


class ReluFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x):
        y = native.relu_fwd(x.contiguous())
        ctx.save_for_backward(y)
        return y

    @staticmethod
    def backward(ctx, dy):
        (y,) = ctx.saved_tensors
        return native.relu_bwd(y, dy.contiguous())


class DenseFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, w, b, relu):
        x = x.contiguous(); w = w.contiguous()
        y = torch.empty(x.shape[0], w.shape[0], dtype=torch.float32, device=x.device)
        native.gemm(x, w, y, bias=b, relu=relu)
        ctx.save_for_backward(x, w, y if relu else None)
        ctx.relu, ctx.has_bias = relu, b is not None
        return y

    @staticmethod
    def backward(ctx, dy):
        x, w, y = ctx.saved_tensors
        dy = dy.contiguous()
        if ctx.relu:
            dy = native.relu_bwd(y, dy)
        dx = dw = db = None
        if ctx.needs_input_grad[0]:
            dx = torch.empty_like(x)
            native.gemm(dy, w, dx, b_mn=True)            # [B,U]·[U,I]
        if ctx.needs_input_grad[1]:
            dw = torch.empty_like(w)
            native.gemm(dy, x, dw, a_mn=True, b_mn=True)  # dyᵀ[U,B]·x[B,I]
        if ctx.has_bias and ctx.needs_input_grad[2]:
            db = native.colsum(dy)
        return dx, dw, db, None


class Conv2dFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, w, b, stride, padding, relu):
        x = x.contiguous(); w = w.contiguous()
        N, C, H, W = x.shape
        Co, _, KH, KW = w.shape
        OH, OW = native.conv_out_hw(H, W, KH, KW, stride[0], stride[1], padding[0], padding[1])
        col = native.im2col(x, KH, KW, stride, padding)          # [(n,oh,ow)][ldc]
        K = C * KH * KW
        y = torch.empty(N, Co, OH, OW, dtype=torch.float32, device=x.device)
        w2 = w.reshape(Co, K)
        native.gemm(col, w2, y, bias=b, relu=relu, store_nchw_hw=OH * OW, M=N * OH * OW, N=Co, K=K, lda=col.stride(0), ldb=K)
        ctx.save_for_backward(col, w, y if relu else None)
        ctx.cfg = (x.shape, stride, padding, relu, b is not None)
        return y

    @staticmethod
    def backward(ctx, dy):
        col, w, y = ctx.saved_tensors
        xs, stride, padding, relu, has_bias = ctx.cfg
        N, C, H, W = xs
        Co, _, KH, KW = w.shape
        K = C * KH * KW
        dy = dy.contiguous()
        if relu:
            dy = native.relu_bwd(y, dy)
        rows = native.nchw_to_rows(dy)                           # [(n,oh,ow)][Co]
        dx = dw = db = None
        if ctx.needs_input_grad[0]:
            dcol = torch.empty(rows.shape[0], col.stride(0), dtype=torch.float32, device=dy.device)
            native.gemm(rows, w.reshape(Co, K), dcol, b_mn=True, M=rows.shape[0], N=K, K=Co, lda=Co, ldb=K, ldd=dcol.stride(0))
            dx = native.col2im(dcol, xs, KH, KW, stride, padding)
        if ctx.needs_input_grad[1]:
            dw = torch.zeros(Co, K, dtype=torch.float32, device=dy.device)
            kb = (rows.shape[0] + 31) // 32
            native.gemm(rows, col, dw, a_mn=True, b_mn=True, M=Co, N=K, K=rows.shape[0], lda=Co, ldb=col.stride(0), ldd=K,
                        split_k=max(1, min(32, kb // 4)), accumulate=True)
            dw = dw.reshape(w.shape)
        if has_bias and ctx.needs_input_grad[2]:
            db = native.chansum_nchw(dy)
        return dx, dw, db, None, None, None


class DepthwiseConv2dFn(torch.autograd.Function):
    """groups == channels convolution through csrc/kernels/depthwise_conv.cu (reference: src/operator/nn/depthwise_convolution_tf.cuh:76-754)."""

    @staticmethod
    def forward(ctx, x, w, b, stride, padding, relu):
        x = x.contiguous(); w = w.contiguous()
        N, C, H, W = x.shape
        OH, OW = native.conv_out_hw(H, W, w.shape[2], w.shape[3], stride[0], stride[1], padding[0], padding[1])
        y = torch.empty(N, C, OH, OW, dtype=torch.float32, device=x.device)
        if not native.depthwise_fwd(x, w, b, y, stride, padding, relu):
            raise RuntimeError("depthwise plane does not fit shared memory")
        ctx.save_for_backward(x, w, y if relu else None)
        ctx.cfg = (stride, padding, relu, b is not None)
        return y

    @staticmethod
    def backward(ctx, dy):
        x, w, y = ctx.saved_tensors
        stride, padding, relu, has_bias = ctx.cfg
        dy = dy.contiguous()
        if relu:
            dy = native.relu_bwd(y, dy)
        dx = dw = db = None
        if ctx.needs_input_grad[0]:
            dx = torch.empty_like(x)
            native.depthwise_dgrad(dy, w, dx, stride, padding)
        if ctx.needs_input_grad[1] or (has_bias and ctx.needs_input_grad[2]):
            dw = torch.zeros_like(w)
            db = torch.zeros(w.shape[0], dtype=torch.float32, device=dy.device) if has_bias else None
            native.depthwise_wgrad(x, dy, dw, db, stride, padding)
        return dx, dw, db, None, None, None


class MaxPool2x2Fn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x):
        y, idx = native.maxpool2x2_fwd(x.contiguous())
        ctx.save_for_backward(idx)
        ctx.xs = tuple(x.shape)
        return y

    @staticmethod
    def backward(ctx, dy):
        (idx,) = ctx.saved_tensors
        return native.maxpool2x2_bwd(dy.contiguous(), idx, ctx.xs)


class SoftmaxCEFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, logits, label):
        logits = logits.contiguous()
        lab = label.to(torch.float32).contiguous()
        loss = native.softmax_ce_fwd(logits, lab)
        ctx.save_for_backward(logits, lab)
        return loss

    @staticmethod
    def backward(ctx, dloss):
        logits, lab = ctx.saved_tensors
        return native.softmax_ce_bwd(logits, lab, dloss.contiguous()), None


class BatchNormFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, gamma, beta, rm, rv, training, momentum, eps):
        x = x.contiguous()
        y, sm, si = native.bn_fwd(x, gamma, beta, rm, rv, training, momentum, eps)
        if not training:
            sm = rm.clone(); si = torch.rsqrt(rv + eps)
        ctx.save_for_backward(x, gamma, sm, si)
        ctx.fixed_stats = not training
        return y

    @staticmethod
    def backward(ctx, dy):
        x, gamma, sm, si = ctx.saved_tensors
        dx, dg, db = native.bn_bwd(x, dy.contiguous(), gamma, sm, si, fixed_stats=ctx.fixed_stats)
        return dx, dg, db, None, None, None, None, None
