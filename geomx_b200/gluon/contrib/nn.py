"""``mx.gluon.contrib.nn.SyncBatchNorm`` — batch normalisation whose statistics span every rank of the job.

Parity: ``python/mxnet/gluon/contrib/nn/basic_layers.py`` SyncBatchNorm over ``src/operator/contrib/sync_batch_norm-inl.h:79-455`` (the reference
shares host-memory accumulators between the GPU threads of ONE process and meets at a barrier).  Here one process drives one GPU, so the
per-channel (count, sum, sum of squares) — and in the backward pass (sum dy, sum dy·x̂) — are all-reduced across the process group
(NCCL over NVLink on CUDA, gloo on CPU); with a single rank the layer degenerates to BatchNorm."""
from __future__ import annotations

import torch

from ... import autograd
from ...ndarray import NDArray
from ..nn.basic_layers import BatchNorm

__all__ = ["SyncBatchNorm", "Concurrent", "HybridConcurrent", "Identity", "SparseEmbedding", "PixelShuffle2D"]


def _all_reduce(t):
    import torch.distributed as dist
    if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
        dist.all_reduce(t)
    return t


class _SyncBNFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, gamma, beta, running_mean, running_var, momentum, eps):
        C = x.shape[1]
        dims = [0] + list(range(2, x.dim()))
        xf = x.float()
        stats = torch.cat([xf.sum(dims), (xf * xf).sum(dims), torch.full((1,), float(x.numel() // C), device=x.device)])
        _all_reduce(stats)
        n = stats[-1]
        mean = stats[:C] / n
        var = (stats[C:2 * C] / n - mean * mean).clamp_min_(0.0)
        with torch.no_grad():
            running_mean.mul_(momentum).add_(mean.to(running_mean.dtype), alpha=1 - momentum)
            running_var.mul_(momentum).add_(var.to(running_var.dtype), alpha=1 - momentum)      # population variance (sync_batch_norm-inl.h:392)
        inv = torch.rsqrt(var + eps)
        shape = [1, C] + [1] * (x.dim() - 2)
        xhat = (xf - mean.view(shape)) * inv.view(shape)
        ctx.save_for_backward(xhat, gamma, inv, n)
        return (xhat * gamma.float().view(shape) + beta.float().view(shape)).to(x.dtype)

    @staticmethod
    def backward(ctx, dy):
        xhat, gamma, inv, n = ctx.saved_tensors
        C = xhat.shape[1]
        dims = [0] + list(range(2, xhat.dim()))
        shape = [1, C] + [1] * (xhat.dim() - 2)
        dyf = dy.float()
        local = torch.cat([dyf.sum(dims), (dyf * xhat).sum(dims)])
        dbeta, dgamma = local[:C].clone(), local[C:].clone()
        _all_reduce(local)                                   # the normalisation couples every sample of the GLOBAL batch
        sdy, sdyx = local[:C] / n, local[C:] / n
        dx = (dyf - sdy.view(shape) - xhat * sdyx.view(shape)) * (gamma.float() * inv).view(shape)
        return dx.to(dy.dtype), dgamma.to(gamma.dtype), dbeta.to(gamma.dtype), None, None, None, None


class SyncBatchNorm(BatchNorm):
    def __init__(self, in_channels=0, num_devices=None, momentum=0.9, epsilon=1e-5, center=True, scale=True, use_global_stats=False, **kwargs):
        super().__init__(axis=1, momentum=momentum, epsilon=epsilon, center=center, scale=scale, use_global_stats=use_global_stats,
                         in_channels=in_channels, **kwargs)
        self._num_devices = num_devices

    def hybrid_forward(self, F, x, gamma, beta, running_mean, running_var):
        if not (autograd.is_training() and not self._use_global):
            return super().hybrid_forward(F, x, gamma, beta, running_mean, running_var)
        return NDArray(_SyncBNFn.apply(x._t, gamma._t, beta._t, running_mean._t, running_var._t, self._momentum, self._eps))


from ..block import Block, HybridBlock  # noqa: E402
from ..nn.basic_layers import HybridSequential, Sequential  # noqa: E402


class Concurrent(Sequential):
    """Feeds the same input to every child and concatenates the outputs along ``axis``
    (``gluon/contrib/nn/basic_layers.py:30-60``)."""

    def __init__(self, axis=-1, prefix=None, params=None):
        super().__init__(prefix=prefix, params=params); self.axis = axis

    def forward(self, x):
        return NDArray(torch.cat([blk(x)._t for blk in self._children.values()], dim=self.axis))


class HybridConcurrent(HybridSequential):
    def __init__(self, axis=-1, prefix=None, params=None):
        super().__init__(prefix=prefix, params=params); self.axis = axis

    def forward(self, x):
        from ...symbol import Symbol
        if isinstance(x, Symbol):                     # export traces hybrid_forward
            return HybridBlock.forward(self, x)
        return NDArray(torch.cat([blk(x)._t for blk in self._children.values()], dim=self.axis))

    def hybrid_forward(self, F, x):
        return F.concat(*[blk(x) for blk in self._children.values()], dim=self.axis)


class Identity(HybridBlock):
    """Pass-through block, useful as a branch of ``Concurrent`` for residual structures."""

    def hybrid_forward(self, F, x):
        return x


class SparseEmbedding(Block):
    """Embedding whose gradient is ``row_sparse``: only the rows that were looked up travel to the parameter server
    (``gluon/contrib/nn/basic_layers.py:115-160``; see ``kv.row_sparse_pull`` and the sparse wire of the TCP plane)."""

    def __init__(self, input_dim, output_dim, dtype="float32", weight_initializer=None, **kwargs):
        super().__init__(**kwargs)
        with self.name_scope():
            self.weight = self.params.get("weight", shape=(input_dim, output_dim), init=weight_initializer, dtype=dtype,
                                          grad_stype="row_sparse", stype="row_sparse")

    def forward(self, x):
        return NDArray(torch.nn.functional.embedding(x._t.long(), self.weight.data(x.context)._t))


class PixelShuffle2D(HybridBlock):
    """``(N, C·f1·f2, H, W) → (N, C, H·f1, W·f2)`` sub-pixel upsampling."""

    def __init__(self, factor, **kwargs):
        super().__init__(**kwargs)
        self._f = (factor, factor) if isinstance(factor, int) else tuple(factor)

    def hybrid_forward(self, F, x):
        f1, f2 = self._f
        N, C, H, W = x._t.shape
        t = x._t.reshape(N, C // (f1 * f2), f1, f2, H, W).permute(0, 1, 4, 2, 5, 3)
        return NDArray(t.reshape(N, C // (f1 * f2), H * f1, W * f2))
