"""Gradient compression: 2-bit (with residual), Bi-Sparse (BSC), fp16/bf16 and block-scaled fp8 transport.

Parity (behavioural contract, reference ``src/kvstore/gradient_compression.{h,cc}``, ``-inl.h``):

* **2bit** ``Quantize`` (:118-153, kernel ``-inl.h:40-81``): ``residual += grad``; 16 values → one 32-bit word,
  byte ``(i&15)>>2``, bit pair chosen by ``posbits {0xc0,0x30,0x0c,0x03}`` / ``negbits {0x80,0x20,0x08,0x02}``
  (11 = +thr, 10 = −thr, 00 = 0); ``residual -= ±thr`` where sent.  ``Dequantize`` (:155-189) expands to ±thr/0.
  Compressed size ``ceil(N/16)`` words (:111-116).  The byte layout is reproduced bit-exactly so a reference
  payload decodes here and vice versa.
* **BSC** ``BSCompress`` (:191-269): ``u = 0.9u + g; v += u``; boundary = k-th largest ``|v|`` over a random
  sample (``sample = N·0.005`` if ``N·0.005·thr ≥ 10`` else ``10/thr``; ``k_sample = sample·thr``); keep the first
  ``k = ⌊N·thr⌋`` entries *in index order* with ``|v| ≥ boundary``; payload ``[vals(k) ‖ idx(k) as float]``, padded
  with ``(-65530, -1)``; ``u, v`` zeroed at sent indices.  ``BSCPullCompress`` (:271-308): keep non-zeros in index
  order up to ``⌊N·thr·mult⌋``.  ``BSCDecompress`` (:310-336): zero-fill then scatter entries with ``idx ≥ 0``.
  The reference samples with ``std::shuffle(seed=42)`` on the CPU; that is not reproducible on a GPU, so the
  contract here is (a) ≤ k entries, (b) every sent ``|v| ≥ boundary``, (c) error-feedback state zeroed exactly at
  sent indices, (d) sentinel padding — sampling is a deterministic stride (SURVEY §7.4-3).
* **fp16 / MPQ**: script-level casts in the reference; here also a transport dtype of the fused push kernel.
* **fp8 block-scaled** (new, H100): e4m3 payload + one fp32 scale per 128-value block, with error feedback.

This module is the CPU implementation *and* the numerics oracle; on CUDA tensors the same functions dispatch to
``csrc/kernels/compress.cu``.
"""
from __future__ import annotations


import torch

from ..base import MXNetError

__all__ = ["GradientCompression", "quantize_2bit", "dequantize_2bit", "bsc_compress", "bsc_pull_compress",
           "bsc_decompress", "bsc_sizes", "fp8_block_quantize", "fp8_block_dequantize", "BSC_PAD_VAL", "BSC_PAD_IDX"]

BSC_PAD_VAL = -65530.0
BSC_PAD_IDX = -1.0
BSC_MOMENTUM = 0.9
BSC_MAX_N = 1 << 24       # indices travel as float32, which holds every integer exactly only up to 2^24
_POS = (0xC0, 0x30, 0x0C, 0x03)
_NEG = (0x80, 0x20, 0x08, 0x02)


def _flat(t):
    """A read-only input as a contiguous float32 vector (fp16 / bf16 gradients are cast, as the reference's scripts cast them)."""
    return t.reshape(-1).float().contiguous()


def _state(t, what):
    """A tensor the codec updates or fills in place: flattening a non-contiguous one would copy it, and the update would be lost."""
    if t is not None and not t.is_contiguous():
        raise MXNetError("%s must be contiguous" % what)


def _bsc_check(n):
    if n > BSC_MAX_N:
        raise MXNetError("Bi-Sparse compression supports at most 2^24 = %d elements per tensor (indices are sent as float32), got %d"
                         % (BSC_MAX_N, n))


def _use_native(t):
    if not t.is_cuda:
        return False
    from ..ops import native
    native.require()
    return True


# ------------------------------------------------------------------------------------------------------------
# 2-bit
# ------------------------------------------------------------------------------------------------------------
def compressed_size_2bit(n: int) -> int:
    return (n + 15) // 16


def quantize_2bit(grad: torch.Tensor, residual: torch.Tensor, threshold: float) -> torch.Tensor:
    """Returns ``ceil(N/16)`` packed words stored as float32 (the reference ships them as a float array)."""
    n = grad.numel()
    _state(residual, "residual")
    if _use_native(grad):
        from ..ops import native
        out = torch.empty(compressed_size_2bit(n), dtype=torch.float32, device=grad.device)
        native.quantize_2bit(_flat(grad), residual.reshape(-1), out, float(threshold))
        return out
    g = _flat(grad); r = residual.reshape(-1)
    r.add_(g)
    pos = r >= threshold
    neg = (r <= -threshold) & ~pos
    r.sub_(pos.to(r.dtype) * threshold).add_(neg.to(r.dtype) * threshold)
    pad = compressed_size_2bit(n) * 16 - n
    code = (pos.to(torch.uint8) * 3 + neg.to(torch.uint8) * 2)
    if pad:
        code = torch.cat([code, torch.zeros(pad, dtype=torch.uint8)])
    code = code.reshape(-1, 4)                       # 4 values per byte, value j -> bits (7-2j, 6-2j)
    byte = (code[:, 0] << 6) | (code[:, 1] << 4) | (code[:, 2] << 2) | code[:, 3]
    return byte.contiguous().view(torch.float32).clone()


def dequantize_2bit(packed: torch.Tensor, n: int, threshold: float, out: torch.Tensor | None = None) -> torch.Tensor:
    if out is None:
        out = torch.empty(n, dtype=torch.float32, device=packed.device)
    _state(out, "out")
    if _use_native(packed):
        from ..ops import native
        native.dequantize_2bit(packed, out.reshape(-1), float(threshold))
        return out
    byte = packed.contiguous().view(torch.uint8)
    code = torch.stack([(byte >> 6) & 3, (byte >> 4) & 3, (byte >> 2) & 3, byte & 3], dim=1).reshape(-1)[:n]
    res = torch.zeros(n, dtype=torch.float32)
    res[code == 3] = threshold
    res[code == 2] = -threshold
    out.reshape(-1).copy_(res)
    return out


# ------------------------------------------------------------------------------------------------------------
# Bi-Sparse
# ------------------------------------------------------------------------------------------------------------
def bsc_sizes(n: int, threshold: float):
    """(k = zipped size, sample_size, k_sample) exactly as the reference computes them (int truncation)."""
    k = int(float(n) * threshold)
    sample = int(n * 0.005) if n * 0.005 * threshold >= 10 else int(10 / threshold)
    sample = max(1, min(sample, n))
    k_sample = min(sample, max(1, int(sample * threshold)))
    return k, sample, k_sample


def _sample_boundary(v_abs: torch.Tensor, sample: int, k_sample: int) -> torch.Tensor:
    n = v_abs.numel()
    stride = max(1, n // sample)
    s = v_abs[::stride][:sample]
    k_sample = min(k_sample, s.numel())
    return torch.topk(s, k_sample).values[-1]


def bsc_compress(grad: torch.Tensor, u: torch.Tensor, v: torch.Tensor, threshold: float,
                 out: torch.Tensor | None = None) -> torch.Tensor:
    """Momentum-corrected sampled-threshold sparsifier.  Returns ``[vals(k) ‖ idx(k)]`` float32 (size 2k)."""
    n = grad.numel()
    _bsc_check(n)
    _state(u, "u"); _state(v, "v"); _state(out, "out")
    k, sample, k_sample = bsc_sizes(n, threshold)
    if out is None:
        out = torch.empty(2 * k, dtype=torch.float32, device=grad.device)
    g = _flat(grad); u = u.reshape(-1); v = v.reshape(-1)
    if k == 0:
        u.mul_(BSC_MOMENTUM).add_(g); v.add_(u)
        return out
    if _use_native(grad):
        from ..ops import native
        native.bsc_compress(g, u, v, out, k, sample, k_sample, BSC_MOMENTUM)
        return out
    u.mul_(BSC_MOMENTUM).add_(g)
    v.add_(u)
    va = v.abs()
    boundary = _sample_boundary(va, sample, k_sample)
    idx = torch.nonzero(va >= boundary).reshape(-1)[:k]
    m = idx.numel()
    out[:k] = BSC_PAD_VAL
    out[k:] = BSC_PAD_IDX
    out[:m] = v[idx]
    out[k:k + m] = idx.to(torch.float32)
    v[idx] = 0
    u[idx] = 0
    return out


def bsc_pull_compress(dense: torch.Tensor, threshold: float, multiplier: int, out: torch.Tensor | None = None) -> torch.Tensor:
    n = dense.numel()
    _bsc_check(n)
    _state(out, "out")
    k = int(float(n) * threshold * multiplier)
    if out is None:
        out = torch.empty(2 * k, dtype=torch.float32, device=dense.device)
    if k == 0:
        return out
    d = _flat(dense)
    if _use_native(dense):
        from ..ops import native
        native.bsc_pull_compress(d, out, k)
        return out
    idx = torch.nonzero(d != 0).reshape(-1)[:k]
    m = idx.numel()
    out[:k] = BSC_PAD_VAL
    out[k:] = BSC_PAD_IDX
    out[:m] = d[idx]
    out[k:k + m] = idx.to(torch.float32)
    return out


def bsc_decompress(zipped: torch.Tensor, n: int, out: torch.Tensor | None = None, accumulate: bool = False) -> torch.Tensor:
    """Scatter ``[vals ‖ idx]`` into a dense length-``n`` tensor (zero-filled unless ``accumulate``)."""
    if out is None:
        out = torch.zeros(n, dtype=torch.float32, device=zipped.device)
        accumulate = True
    _state(out, "out")
    if _use_native(zipped):
        from ..ops import native
        native.bsc_decompress(zipped, out.reshape(-1), accumulate)
        return out
    k = zipped.numel() // 2
    o = out.reshape(-1)
    if not accumulate:
        o.zero_()
    vals, idx = zipped[:k], zipped[k:2 * k]
    keep = idx >= 0
    ii = idx[keep].long()
    if accumulate:
        o.index_add_(0, ii, vals[keep])
    else:
        o[ii] = vals[keep]
    return out


# ------------------------------------------------------------------------------------------------------------
# block-scaled fp8 (e4m3, 128-value blocks)
# ------------------------------------------------------------------------------------------------------------
FP8_BLOCK = 128
FP8_MAX = 448.0


def fp8_block_quantize(x: torch.Tensor, residual: torch.Tensor | None = None):
    """x (+ residual) → (e4m3 payload uint8[N_pad], fp32 scales[N_pad/128]); residual receives the rounding error."""
    n = x.numel()
    nb = (n + FP8_BLOCK - 1) // FP8_BLOCK
    _state(residual, "residual")
    if _use_native(x):
        from ..ops import native
        q = torch.empty(nb * FP8_BLOCK, dtype=torch.uint8, device=x.device)
        s = torch.empty(nb, dtype=torch.float32, device=x.device)
        native.fp8_block_quantize(_flat(x), residual.reshape(-1) if residual is not None else None, q, s)
        return q, s
    xf = _flat(x)
    if residual is not None:
        xf = xf + residual.reshape(-1)
    pad = nb * FP8_BLOCK - n
    xp = torch.cat([xf, torch.zeros(pad)]) if pad else xf
    blk = xp.reshape(nb, FP8_BLOCK)
    amax = blk.abs().amax(dim=1)
    scale = torch.where(amax > 0, amax / FP8_MAX, torch.ones_like(amax))
    q8 = (blk / scale[:, None]).to(torch.float8_e4m3fn)
    if residual is not None:
        deq = (q8.float() * scale[:, None]).reshape(-1)[:n]
        residual.reshape(-1).copy_(xf - deq)
    return q8.view(torch.uint8).reshape(-1), scale


def fp8_block_dequantize(q: torch.Tensor, scale: torch.Tensor, n: int, out: torch.Tensor | None = None) -> torch.Tensor:
    if out is None:
        out = torch.empty(n, dtype=torch.float32, device=q.device)
    _state(out, "out")
    if _use_native(q):
        from ..ops import native
        native.fp8_block_dequantize(q, scale, out.reshape(-1))
        return out
    blk = q.view(torch.float8_e4m3fn).float().reshape(-1, FP8_BLOCK) * scale[:, None]
    out.reshape(-1).copy_(blk.reshape(-1)[:n])
    return out


# ------------------------------------------------------------------------------------------------------------
# parameter object shipped to servers
# ------------------------------------------------------------------------------------------------------------
class GradientCompression:
    """``type ∈ {none, 2bit, bsc}`` + ``threshold``; ``EncodeParams``/``DecodeParams`` = ``"type,threshold"``."""

    TYPES = {"none": 0, "2bit": 1, "bsc": 2}

    def __init__(self):
        self.type = "none"
        self.threshold = 0.5
        self._residual = {}

    @property
    def active(self):
        return self.type == "2bit"

    def set_params(self, params):
        t = params.get("type", "none")
        if t not in self.TYPES:
            raise MXNetError("Unknown type for gradient compression %s" % t)
        thr = float(params.get("threshold", 0.5))
        if t != "none" and not thr > 0:
            raise MXNetError("threshold must be greater than 0")
        self.type, self.threshold = t, thr

    def get_type_str(self):
        return str(self.TYPES[self.type])

    def encode_params(self):
        return "%d,%s" % (self.TYPES[self.type], repr(self.threshold))

    def decode_params(self, s):
        a, b = s.split(",")
        rev = {v: k for k, v in self.TYPES.items()}
        self.type, self.threshold = rev[int(a)], float(b)

    def get_compression_factor(self):
        if self.type == "2bit":
            return 16
        raise MXNetError("Unsupported compression type: %s" % self.type)

    def get_compressed_size(self, n):
        f = self.get_compression_factor()
        return (n + f - 1) // f

    def quantize(self, slot, grad):
        r = self._residual.get(slot)
        if r is None or r.numel() != grad.numel() or r.device != grad.device:
            r = torch.zeros(grad.numel(), dtype=torch.float32, device=grad.device); self._residual[slot] = r
        return quantize_2bit(grad, r, self.threshold)

    def dequantize(self, packed, n):
        return dequantize_2bit(packed, n, self.threshold)
