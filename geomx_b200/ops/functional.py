"""Operator dispatch used by the Gluon layers.

Every op takes and returns raw ``torch.Tensor`` s.  On a CUDA tensor the op runs the
hand-written sm_90a kernel (``geomx_b200/ops/native.py`` → ``csrc/kernels/*.cu``) wrapped
in a ``torch.autograd.Function``; on CPU (no GPU in the authoring sandbox, CPU workers in
BASELINE config 1) it runs the plain PyTorch fp32 definition, which is also the numerics
oracle of ``tests/test_kernels_gpu.py``.

Parity (operator semantics): Convolution ``src/operator/nn/convolution-inl.h:165-206``,
FullyConnected ``src/operator/nn/fully_connected-inl.h:71-173``, Pooling ``src/operator/nn/pool.cuh``,
Activation ``src/operator/nn/activation-inl.h``, BatchNorm ``src/operator/nn/batch_norm.cu``,
softmax / log_softmax ``src/operator/nn/softmax-inl.h``, pick
``src/operator/tensor/broadcast_reduce_op_index.cu``.

If a CUDA tensor arrives and the native library is missing, ops raise — a silent eager
fallback on a GPU box would hide a broken build.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

from . import native

__all__ = ["conv2d", "dense", "max_pool2d", "avg_pool2d", "activation", "batch_norm", "softmax_cross_entropy",
           "log_softmax", "softmax", "dropout", "flatten", "use_native", "layer_norm"]

_FORCE_TORCH = False


def use_native(flag: bool):
    """Testing hook: force the PyTorch definitions even on CUDA (the NCCL+cuBLAS 'oracle' arm)."""
    global _FORCE_TORCH
    _FORCE_TORCH = not flag


def _nat(x: torch.Tensor) -> bool:
    if not x.is_cuda or _FORCE_TORCH:
        return False
    native.require()  # raises loudly when the .so is missing on a GPU box
    return True


def _act(y, act):
    if act is None:
        return y
    if act == "relu":
        return torch.relu(y)
    if act == "sigmoid":
        return torch.sigmoid(y)
    if act == "tanh":
        return torch.tanh(y)
    if act == "softrelu":
        return F.softplus(y)
    if act == "softsign":
        return F.softsign(y)
    raise ValueError("unknown activation %s" % act)


def activation(x, act):
    if act == "relu" and _nat(x) and x.dtype == torch.float32:
        from .autograd_fns import ReluFn
        return ReluFn.apply(x)
    return _act(x, act)


def conv2d(x, w, b=None, stride=(1, 1), padding=(0, 0), dilation=(1, 1), groups=1, act=None):
    """NCHW convolution with optional fused bias + activation."""
    if (_nat(x) and x.dtype == torch.float32 and groups == 1 and tuple(dilation) == (1, 1)
            and act in (None, "relu") and native.conv_supported(x, w, stride, padding)):
        from .autograd_fns import Conv2dFn
        return Conv2dFn.apply(x, w, b, tuple(stride), tuple(padding), act == "relu")
    if (_nat(x) and x.dtype == torch.float32 and x.dim() == 4 and groups == x.shape[1] == w.shape[0] and w.shape[1] == 1 and tuple(dilation) == (1, 1)
            and act in (None, "relu") and native.depthwise_supported(x.shape, w.shape, stride, padding)):
        from .autograd_fns import DepthwiseConv2dFn            # depthwise: one CTA per (image, channel) plane, filter + plane in shared memory
        return DepthwiseConv2dFn.apply(x, w, b, tuple(stride), tuple(padding), act == "relu")
    return _act(F.conv2d(x, w, b, stride, padding, dilation, groups), act)


def dense(x, w, b=None, act=None, flatten=True):
    """``y = act(x · wᵀ + b)``; ``w`` is (units, in_units) like MXNet's FullyConnected."""
    if flatten and x.dim() > 2:
        x = x.reshape(x.shape[0], -1)
    if _nat(x) and x.dtype == torch.float32 and x.dim() == 2 and act in (None, "relu"):
        from .autograd_fns import DenseFn
        return DenseFn.apply(x, w, b, act == "relu")
    return _act(F.linear(x, w, b), act)


def max_pool2d(x, kernel, stride=None, padding=(0, 0), ceil_mode=False):
    stride = stride or kernel
    if (_nat(x) and x.dtype == torch.float32 and tuple(kernel) == (2, 2) and tuple(stride) == (2, 2)
            and tuple(padding) == (0, 0) and x.shape[2] % 2 == 0 and x.shape[3] % 2 == 0):
        from .autograd_fns import MaxPool2x2Fn
        return MaxPool2x2Fn.apply(x)
    return F.max_pool2d(x, kernel, stride, padding, ceil_mode=ceil_mode)


def avg_pool2d(x, kernel, stride=None, padding=(0, 0), ceil_mode=False, count_include_pad=True):
    return F.avg_pool2d(x, kernel, stride or kernel, padding, ceil_mode=ceil_mode, count_include_pad=count_include_pad)


def batch_norm(x, gamma, beta, running_mean, running_var, training, momentum=0.9, eps=1e-5, axis=1):
    """MXNet BatchNorm: ``running = momentum*running + (1-momentum)*batch`` (note: opposite of torch)."""
    if _nat(x) and x.dtype == torch.float32 and axis == 1 and x.dim() in (2, 4):
        from .autograd_fns import BatchNormFn
        return BatchNormFn.apply(x, gamma, beta, running_mean, running_var, bool(training), float(momentum), float(eps))
    if axis != 1:
        x = x.transpose(1, axis)
    if training:
        # the running variance tracks the POPULATION variance of the batch, as the reference's kernels do (src/operator/nn/batch_norm.cu:355-362,
        # contrib/sync_batch_norm-inl.h:392) — torch's own running update would use the unbiased estimate
        with torch.no_grad():
            dims = [0] + list(range(2, x.dim()))
            xf = x.float()
            mean = xf.mean(dims)
            var = (xf * xf).mean(dims).sub_(mean * mean).clamp_min_(0.0)
            running_mean.mul_(momentum).add_(mean.to(running_mean.dtype), alpha=1.0 - momentum)
            running_var.mul_(momentum).add_(var.to(running_var.dtype), alpha=1.0 - momentum)
        y = F.batch_norm(x, None, None, gamma, beta, True, 0.0, eps)
    else:
        y = F.batch_norm(x, running_mean, running_var, gamma, beta, False, 0.0, eps)
    return y.transpose(1, axis) if axis != 1 else y


def layer_norm(x, gamma, beta, axis=-1, eps=1e-5):
    if axis not in (-1, x.dim() - 1):
        x = x.transpose(axis, -1)
        return F.layer_norm(x, x.shape[-1:], gamma, beta, eps).transpose(axis, -1)
    return F.layer_norm(x, x.shape[-1:], gamma, beta, eps)


def log_softmax(x, axis=-1):
    return torch.log_softmax(x, dim=axis)


def softmax(x, axis=-1):
    return torch.softmax(x, dim=axis)


def softmax_cross_entropy(logits, label, sparse_label=True, axis=-1):
    """Per-sample ``-log_softmax(logits)[label]`` (``python/mxnet/gluon/loss.py:304-318``)."""
    if sparse_label and axis in (-1, logits.dim() - 1) and logits.dim() == 2 and _nat(logits) \
            and logits.dtype == torch.float32 and logits.shape[1] <= 1024:
        from .autograd_fns import SoftmaxCEFn
        return SoftmaxCEFn.apply(logits, label)
    lp = torch.log_softmax(logits, dim=axis)
    if sparse_label:
        return -torch.gather(lp, axis, label.long().unsqueeze(axis)).squeeze(axis)
    return -(lp * label).sum(dim=axis)


def dropout(x, p, training):
    return F.dropout(x, p, training)


def flatten(x):
    return x.reshape(x.shape[0], -1)
