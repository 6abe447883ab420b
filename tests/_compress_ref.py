"""Plain numpy references of the gradient-compression codecs (``csrc/kernels/compress.cu``), written from the reference's documented
formats and not from ``kvstore/compression.py``.

* 2-bit: value j of a 16-value word goes in byte j>>2, bit pair ``posbits {c0,30,0c,03}`` (+thr) / ``negbits {80,20,08,02}`` (-thr).  The
  residual update is one fp32 add and one fp32 subtract, so words and residuals are exact.
* fp8 block: a table of all 256 e4m3 codes, round to nearest, ties to even, saturating at +-448; the scale is fp32(amax) / 448 in fp32.
* Bi-Sparse: ``bsc_replay`` checks one compress launch from the state before and after it, so fp32 differences cannot compound over rounds.
* DGT: the per-block EMA of mean |g| in fp64.
"""
import numpy as np

POS = (0xC0, 0x30, 0x0C, 0x03)
NEG = (0x80, 0x20, 0x08, 0x02)
PAD_VAL, PAD_IDX = np.float32(-65530.0), np.float32(-1.0)
F32 = np.float32


def f32(x):
    return np.asarray(x, dtype=np.float32)


def bits(x):
    return np.ascontiguousarray(x).view(np.uint32)


def ulp_err(got, exact):
    """|got - exact| in fp32 ulps of the exact (fp64) value."""
    exact = np.asarray(exact, dtype=np.float64)
    u = np.spacing(np.abs(exact).astype(np.float32)).astype(np.float64)
    return float(np.max(np.abs(np.asarray(got, dtype=np.float64) - exact) / u, initial=0.0))


def fma32(a, b, c):
    """fp32 a*b + c with one rounding (what the GPU's FFMA computes).  a*b is exact in fp64; a sum that fp64 rounds onto an fp32 midpoint is
    resolved by the sign of fp64's own rounding error."""
    p = np.asarray(a, np.float64) * np.asarray(b, np.float64)
    c = np.asarray(c, np.float64)
    s = p + c
    bb = s - p
    e = (p - (s - bb)) + (c - bb)
    r = s.astype(np.float32)
    up, dn = np.nextafter(s, np.inf).astype(np.float32), np.nextafter(s, -np.inf).astype(np.float32)
    return np.where(e > 0, up, np.where(e < 0, dn, r)).astype(np.float32)


# ---------------------------------------------------------------------------------------------------------------- 2-bit
def quantize_2bit(grad, residual, thr, posbits=POS, negbits=NEG):
    """Returns (uint32 words, new residual); ``grad`` and ``residual`` are fp32 arrays, ``thr`` the threshold as the kernel gets it (fp32)."""
    thr = F32(thr)
    r = f32(residual) + f32(grad)
    pos = r >= thr
    neg = ~pos & (r <= -thr)
    r = np.where(pos, r - thr, np.where(neg, r + thr, r)).astype(np.float32)
    n = r.size
    words = (n + 15) // 16
    code = np.zeros(words * 16, np.uint8)
    code[:n] = np.where(pos, 3, np.where(neg, 2, 0))
    code = code.reshape(words, 16)
    out = np.zeros((words, 4), np.uint8)
    for j in range(16):
        out[:, j >> 2] |= np.where(code[:, j] == 3, posbits[j & 3], np.where(code[:, j] == 2, negbits[j & 3], 0)).astype(np.uint8)
    return out.reshape(-1).view("<u4").astype(np.uint32), r


def dequantize_2bit(words, n, thr, out=None):
    thr = F32(thr)
    b = np.ascontiguousarray(words, dtype="<u4").view(np.uint8).reshape(-1, 4)
    v = np.zeros(b.shape[0] * 16, np.float32)
    for j in range(16):
        byte = b[:, j >> 2]
        v[j::16] = np.where(byte & POS[j & 3] == POS[j & 3], thr, np.where(byte & POS[j & 3] == NEG[j & 3], -thr, F32(0)))
    v = v[:n]
    return v if out is None else (f32(out) + v).astype(np.float32)


# ---------------------------------------------------------------------------------------------------------------- fp8 e4m3 block
def e4m3_table():
    """Value of each of the 256 e4m3 (fn) codes in fp64: 1 sign, 4 exponent (bias 7), 3 mantissa bits; S.1111.111 is NaN, no infinity."""
    c = np.arange(256)
    s, e, m = c >> 7, (c >> 3) & 15, c & 7
    mag = np.where(e == 0, m / 8.0 * 2.0 ** -6, (1 + m / 8.0) * 2.0 ** (e - 7.0))
    val = np.where(s == 1, -mag, mag)
    val[(c & 0x7F) == 0x7F] = np.nan
    return val


_MAGS = e4m3_table()[:127]          # codes 0x00 .. 0x7E: 0 .. 448, increasing


def to_e4m3(x):
    """fp32 -> e4m3 code: round to nearest, ties to the even code, saturate at +-448 (NaN -> 0x7F with the sign)."""
    x = f32(x)
    ax = np.abs(x.astype(np.float64))
    hi = np.clip(np.searchsorted(_MAGS, ax, side="left"), 1, 126)
    lo = hi - 1
    mid = (_MAGS[lo] + _MAGS[hi]) / 2
    code = np.where(ax < mid, lo, np.where(ax > mid, hi, np.where(lo % 2 == 0, lo, hi)))
    code = np.where(ax >= 448.0, 126, code)
    code = np.where(np.isnan(ax), 0x7F, code)
    return (code | (np.signbit(x).astype(np.int64) << 7)).astype(np.uint8)


def fp8_quantize(x, residual=None, scale_div=448.0):
    """Returns (codes uint8[nb*128], scales fp32[nb], v = x + residual (fp32), exact residual v - q*s in fp64)."""
    x = f32(x)
    n = x.size
    # the kernel adds a zero residual when there is none, so -0.0 becomes +0.0 (code 0x00, not 0x80)
    v = (x + (np.float32(0) if residual is None else f32(residual))).astype(np.float32)
    nb = (n + 127) // 128
    vp = np.zeros(nb * 128, np.float32)
    vp[:n] = v
    blk = vp.reshape(nb, 128)
    amax = np.abs(blk).max(axis=1) if nb else np.zeros(0, np.float32)
    scale = np.where(amax > 0, amax / F32(scale_div), F32(1)).astype(np.float32)
    q = to_e4m3((blk / scale[:, None]).astype(np.float32)).reshape(-1)
    deq = e4m3_table()[q].reshape(nb, 128) * scale[:, None].astype(np.float64)
    return q, scale, v, v.astype(np.float64) - deq.reshape(-1)[:n]


def fp8_dequantize(q, scale, n, out=None):
    qv = e4m3_table()[q[:n]].astype(np.float32)
    s = np.repeat(f32(scale), 128)[:n]
    if out is None:
        return (qv * s).astype(np.float32)
    return fma32(qv, s, out)                 # the kernel's out + q*s is one FFMA


# ---------------------------------------------------------------------------------------------------------------- Bi-Sparse
def bsc_sizes(n, thr):
    """k, sample, k_sample as the reference computes them (int truncation; k_sample at most the sample)."""
    k = int(float(n) * thr)
    sample = int(n * 0.005) if n * 0.005 * thr >= 10 else int(10 / thr)
    sample = max(1, min(sample, n))
    return k, sample, min(sample, max(1, int(sample * thr)))


def bsc_replay(g, u0, v0, u1, v1, out, k, sample, k_sample, ge=True):
    """One compress launch, from the state before (u0, v0) and after (u1, v1, out).  Returns the errors in ulps of u and of v before the
    reset, and raises AssertionError on any exact condition.  ``ge=False`` keeps |v| > boundary instead (a mutation check)."""
    n = g.size
    vals, idx = out[:k], out[k:2 * k]
    sent = idx >= 0
    m = int(sent.sum())
    assert np.all(sent[:m]) and not np.any(sent[m:]), "padding not at the end"
    assert np.all(bits(vals[m:]) == bits(np.full(k - m, PAD_VAL, np.float32))) and np.all(idx[m:] == PAD_IDX), "padding"
    ii = idx[:m].astype(np.int64)
    assert np.all(ii.astype(np.float32) == idx[:m]), "index not an integer"
    # v before the reset: the sent values at the sent indices, v1 elsewhere
    v_pre = v1.copy()
    v_pre[ii] = vals[:m]
    u_exact = np.float64(np.float32(0.9)) * u0.astype(np.float64) + g.astype(np.float64)
    u_unsent = np.ones(n, bool)
    u_unsent[ii] = False
    eu = ulp_err(u1[u_unsent], u_exact[u_unsent])
    v_exact = v0.astype(np.float64) + fma32(np.float32(0.9), u0, g).astype(np.float64)
    ev = ulp_err(v_pre, v_exact)
    # boundary: the k_sample-th largest |v| over the strided sample
    stride = max(1, n // sample)
    s = np.abs(v_pre[np.arange(sample, dtype=np.int64) * stride])
    boundary = np.sort(s)[::-1][k_sample - 1]
    keep = np.abs(v_pre) >= boundary if ge else np.abs(v_pre) > boundary
    want = np.flatnonzero(keep)[:k]
    assert m == want.size and np.array_equal(ii, want), "sent set: %d sent, %d expected" % (m, want.size)
    assert np.all(bits(u1[ii]) == 0) and np.all(bits(v1[ii]) == 0), "state not reset at the sent indices"
    return eu, ev


def bsc_pull(dense, k):
    """Non-zeros in index order (-0.0 is zero, NaN is not), at most k, padded."""
    dense = f32(dense)
    ii = np.flatnonzero(dense != 0)[:k]
    out = np.empty(2 * k, np.float32)
    out[:k], out[k:] = PAD_VAL, PAD_IDX
    out[:ii.size] = dense[ii]
    out[k:k + ii.size] = ii
    return out


def bsc_decompress(z, n, out=None):
    k = z.size // 2
    res = np.zeros(n, np.float32) if out is None else f32(out).copy()
    idx = z[k:]
    ok = idx >= 0
    ii = idx[ok].astype(np.int64)
    res[ii] = (res[ii] + z[:k][ok]).astype(np.float32)
    return res


# ---------------------------------------------------------------------------------------------------------------- DGT
def dgt_contrib(g, prev, block_elems, alpha, first, tail=0):
    """``tail`` adds to the length the last block is divided by (a mutation check: it must be its own length)."""
    n = g.size
    nb = (n + block_elems - 1) // block_elems
    a = np.abs(g.astype(np.float64))
    sums = np.add.reduceat(a, np.arange(nb) * block_elems) if nb else np.zeros(0)
    lens = np.minimum(block_elems, n - np.arange(nb) * block_elems).astype(np.float64)
    lens[-1:] += tail
    mean = sums / lens
    return mean if first else alpha * prev.astype(np.float64) + (1 - alpha) * mean
