"""The gradient-compression kernels (``csrc/kernels/compress.cu``) against the independent references of ``_compress_ref.py``.

* 2-bit words, residuals and dequantised values bit for bit, at sizes that reach the grid-stride loop, with values at +-thr and one ulp off.
* fp8 block payload, scales, padding and dequantised values bit for bit; the residual to 1 ulp (the kernel computes v - q*s as one FFMA).
* Bi-Sparse compress replayed launch by launch: u and v to 1 ulp of fp64, the boundary, sent set, padding and state reset exactly; a batched
  launch equals each segment's own launch bit for bit.  Pull-compress and decompress exactly.
* DGT contribution to 1e-6 relative of fp64.
* The KVStore entry points that use these kernels on one GPU, over several rounds with their residuals.
* Each check is shown to reject a deliberately broken reference replayed on the recorded GPU outputs.
The largest error of each family is printed (``-s``).
"""
import numpy as np
import pytest
import torch

import geomx_b200 as mx
from geomx_b200 import runtime
from geomx_b200.base import MXNetError
from geomx_b200.kvstore import compression as gc
from geomx_b200.ops import _native_api as api

import _compress_ref as CR
from _cnn_ref import dev, nat  # noqa: F401  (nat: fixture)
from _update_harness import clean_env  # noqa: F401  (fixture)

pytestmark = pytest.mark.gpu
needs_c = pytest.mark.skipif(not runtime.available(), reason="native runtime not built")


def cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev())


def host(t):
    return t.detach().cpu().numpy()


def u32(t):
    return np.ascontiguousarray(host(t) if isinstance(t, torch.Tensor) else t).view(np.uint32)


# ---------------------------------------------------------------------------------------------------------------- 2-bit
def grad_2bit(n, thr, rng):
    """Random values, with values at exactly +-thr, one ulp either side, +-0 and magnitudes far above thr at both ends."""
    t = np.float32(thr)
    special = np.float32([t, -t, np.nextafter(t, 0), np.nextafter(t, 1), -np.nextafter(t, 0), -np.nextafter(t, 1), 0.0, -0.0,
                          1e3 * t, -1e3 * t, 7 * t, -7 * t, 2 * t, -2 * t])
    g = (rng.randn(n) * 1.5 * thr).astype(np.float32)
    m = min(n, 48)
    g[:m] = np.resize(special, m)
    if n > 96:
        g[-m:] = np.resize(special[::-1], m)
    return g


@pytest.mark.parametrize("thr", [0.5, 0.1, 1e-3])
@pytest.mark.parametrize("n", [1, 15, 16, 17, 1000, 65537, 5000003])
def test_2bit_bit_exact(nat, n, thr):
    """Four rounds carrying the residual; dequantised by overwriting and by accumulating into a random ``out``.  5,000,003 values is past
    the 1184-CTA grid of both kernels (303,104 words per pass of the quantiser)."""
    rng = np.random.RandomState(n % 9973)
    res, res_ref = torch.zeros(n, device=dev()), np.zeros(n, np.float32)
    for rnd in range(4):
        g = grad_2bit(n, thr, rng)
        q = gc.quantize_2bit(cuda(g), res, thr)
        words, res_ref = CR.quantize_2bit(g, res_ref, thr)
        got = u32(q)
        assert np.array_equal(got, words), (n, thr, rnd, int((got != words).sum()))
        assert np.array_equal(u32(res), u32(res_ref)), (n, thr, rnd)
        if n % 16:
            unused = sum(0xC0 >> (2 * (j & 3)) << (8 * (j >> 2)) for j in range(n % 16, 16))
            assert int(got[-1]) & unused == 0
        d = gc.dequantize_2bit(q, n, thr)
        assert np.array_equal(u32(d), u32(CR.dequantize_2bit(words, n, thr)))
        out0 = rng.randn(n).astype(np.float32)
        out = cuda(out0)
        nat.dequantize_2bit(q, out, thr, accumulate=True)
        assert np.array_equal(u32(out), u32(CR.dequantize_2bit(words, n, thr, out=out0)))


# ---------------------------------------------------------------------------------------------------------------- fp8 block
def fp8_data(n, rng):
    """Random blocks, and full blocks cycling through: all zeros; one outlier among tiny values (e4m3 subnormals, values that underflow to 0);
    exact rounding ties between codes (scale 1/8, values at code midpoints / 8); values at exactly +-amax (+-448 s) among +-0; an fp32-denormal
    amax."""
    x = (rng.randn(n) * 3).astype(np.float32)
    mags = CR.e4m3_table()[:127]
    mids = ((mags[:-1] + mags[1:]) / 2).astype(np.float32)
    for b in range(n // 128):
        blk = slice(b * 128, (b + 1) * 128)
        kind = b % 6
        if kind == 0:
            x[blk] = 0
        elif kind == 1:
            x[blk] = (rng.randn(128) * 10.0 ** rng.uniform(-7, -1, 128)).astype(np.float32)
            x[b * 128 + rng.randint(128)] = 37.5
        elif kind == 2:
            x[blk] = mids[rng.randint(0, 126, 128)] * np.float32(0.125) * np.where(rng.rand(128) < 0.5, -1, 1).astype(np.float32)
            x[b * 128] = 56.0                          # amax 56: scale exactly 1/8
        elif kind == 3:
            a = np.float32(rng.uniform(0.1, 9))
            x[blk] = np.where(rng.rand(128) < 0.5, -a, a) * (rng.rand(128) < 0.5)
            x[b * 128] = a
        elif kind == 4:
            x[blk] = (rng.randn(128) * 1e-40).astype(np.float32)
    return x


@pytest.mark.parametrize("n", [0, 1, 127, 128, 129, 1000, (1 << 20) + 5])
def test_fp8_block_bit_exact(nat, n):
    rng = np.random.RandomState(n % 7919)
    worst = 0.0
    for with_res in (False, True):
        x = fp8_data(n, rng)
        r0 = (rng.randn(n) * 0.01).astype(np.float32)
        res = cuda(r0) if with_res else None
        q, s = gc.fp8_block_quantize(cuda(x), res)
        qr, sr, v, exact = CR.fp8_quantize(x, r0 if with_res else None)
        nb = (n + 127) // 128
        assert q.numel() == nb * 128 and s.numel() == nb
        assert np.array_equal(host(q), qr), (n, with_res, int((host(q) != qr).sum()))
        assert np.array_equal(u32(s), u32(sr))
        assert not host(q)[n:].any()                                      # padding bytes
        if with_res:
            e = CR.ulp_err(host(res), exact)
            worst = max(worst, e)
            assert e <= 1.0, (n, e)
        assert np.array_equal(u32(gc.fp8_block_dequantize(q, s, n)), u32(CR.fp8_dequantize(qr, sr, n)))
        out0 = rng.randn(n).astype(np.float32)
        out = cuda(out0)
        nat.fp8_block_dequantize(q, s, out, accumulate=True)
        assert np.array_equal(u32(out), u32(CR.fp8_dequantize(qr, sr, n, out=out0)))
    print("\n  fp8 n=%d: residual within %.2f ulp" % (n, worst), end="")


# ---------------------------------------------------------------------------------------------------------------- DGT
@pytest.mark.parametrize("block_elems", [1024, 1000])
@pytest.mark.parametrize("n", [0, 1, 1023, 1024, 1025, 300000])
def test_dgt_contribution(nat, n, block_elems):
    """One launch with ``first`` (the previous contribution, NaN, must be ignored), then three rounds of the EMA at alpha = 0.3; each round
    from the kernel's own previous contribution.  The last block may be partial: it is divided by its own length."""
    rng = np.random.RandomState(n + block_elems)
    nb = (n + block_elems - 1) // block_elems
    contrib = torch.full((nb,), float("nan"), device=dev())
    worst = 0.0
    for rnd in range(4):
        g = (rng.randn(n) * rng.uniform(0.1, 10)).astype(np.float32)
        prev = host(contrib).copy()
        nat.dgt_contrib(cuda(g), contrib, block_elems, 0.3, rnd == 0)
        ref = CR.dgt_contrib(g, prev, block_elems, 0.3, rnd == 0)
        if nb:
            e = float(np.max(np.abs(host(contrib) - ref) / np.abs(ref)))
            worst = max(worst, e)
            assert e <= 1e-6, (n, block_elems, rnd, e)
    print("\n  DGT n=%d block %d: rel err %.1e" % (n, block_elems, worst), end="")


# ---------------------------------------------------------------------------------------------------------------- Bi-Sparse
SEGMENTS = [(50, 0.5), (1023, 1.0), (4096, 0.05), (4097, 0.5), (131072, 0.01), (1000003, 0.05)]


def bsc_grad(n, thr, regime, rng):
    k, sample, _ = CR.bsc_sizes(n, thr)
    at_sample = np.zeros(n, bool)
    at_sample[np.arange(sample, dtype=np.int64) * max(1, n // sample)] = True
    if regime == "random":
        return rng.randn(n).astype(np.float32)
    if regime == "integer":                              # heavy ties at the boundary
        return rng.randint(-3, 4, n).astype(np.float32)
    if regime == "zeros":                                # boundary 0: the first k are sent, zeros included
        return np.zeros(n, np.float32)
    if regime == "sparse":                               # large only where sampled: fewer than k reach the boundary, the rest is padding
        return np.where(at_sample, rng.randn(n) * 10, rng.randn(n) * 1e-3).astype(np.float32)
    # dense: small where sampled, large elsewhere: far more than k reach the boundary, the first k span several 4096-value chunks
    return np.where(at_sample, rng.randn(n) * 1e-3, rng.randn(n) * 10).astype(np.float32)


def bsc_segments(items):
    """items: [(g, u, v, out, (k, sample, k_sample))] -> a device table for one batched launch."""
    return api._segs_to_dev([api.bsc_segment(g, u, v, out, *sz) for g, u, v, out, sz in items], dev())


def bsc_check(g, u0, v0, u, v, out, sz, ge=True):
    return CR.bsc_replay(g, u0, v0, host(u), host(v), host(out), *sz, ge=ge)


@pytest.mark.parametrize("regime", ["random", "integer", "zeros", "sparse", "dense"])
def test_bsc_compress_batched(nat, regime):
    """Six segments in one launch, three rounds: every segment replayed against the reference, and equal bit for bit to its own launch."""
    rng = np.random.RandomState(["random", "integer", "zeros", "sparse", "dense"].index(regime))
    state = []
    for n, thr in SEGMENTS:
        u0 = (rng.randn(n) * 0.1).astype(np.float32) if regime != "zeros" else np.zeros(n, np.float32)
        state.append((cuda(u0), cuda(u0 * 2)))
    eu = ev = 0.0
    padded = spread = 0
    for rnd in range(3):
        items, before = [], []
        for (n, thr), (u, v) in zip(SEGMENTS, state):
            sz = CR.bsc_sizes(n, thr)
            g = bsc_grad(n, thr, regime, rng)
            out = torch.full((2 * sz[0],), float("nan"), device=dev())
            items.append((cuda(g), u, v, out, sz))
            before.append((g, host(u).copy(), host(v).copy()))
        api.bsc_compress_batch(bsc_segments(items), len(items))
        for (gd, u, v, out, sz), (g, u0, v0) in zip(items, before):
            a, b = bsc_check(g, u0, v0, u, v, out, sz)
            eu, ev = max(eu, a), max(ev, b)
            assert a <= 1.0 and b <= 1.0, (regime, rnd, g.size, a, b)
            idx = host(out)[sz[0]:]
            padded += int((idx < 0).any())
            spread += int(idx.max() >= 3 * 4096)
            u1, v1, o1 = cuda(u0), cuda(v0), torch.full_like(out, float("nan"))
            api.bsc_compress_batch(bsc_segments([(gd, u1, v1, o1, sz)]), 1)
            for x, y in ((out, o1), (u, u1), (v, v1)):
                assert np.array_equal(u32(x), u32(y)), (regime, rnd, g.size)
    if regime == "sparse":
        assert padded >= 3 * len(SEGMENTS) - 2        # every round of (almost) every segment padded
    if regime == "dense":
        assert spread >= 3                            # the 1 M segment's k entries run over many compaction chunks
    print("\n  Bi-Sparse %-7s: u %.2f ulp, v %.2f ulp" % (regime, eu, ev), end="")


@pytest.mark.parametrize("n", [10_000_000, 12_000_000, 1 << 24])
def test_bsc_compress_large(nat, n):
    """The sample (0.5% of n, up to 83,886 values) no longer has to fit in shared memory: these sizes used to be refused on CUDA."""
    rng = np.random.RandomState(n % 1000)
    thr = 0.01
    sz = CR.bsc_sizes(n, thr)
    u, v = torch.zeros(n, device=dev()), torch.zeros(n, device=dev())
    for rnd in range(2):
        g = rng.randn(n).astype(np.float32)
        u0, v0 = host(u).copy(), host(v).copy()
        out = gc.bsc_compress(cuda(g), u, v, thr)
        a, b = bsc_check(g, u0, v0, u, v, out, sz)
        assert a <= 1.0 and b <= 1.0, (n, a, b)
    with pytest.raises(MXNetError, match="2\\^24"):
        gc.bsc_compress(torch.zeros((1 << 24) + 1, device=dev()), u, v, thr)


def test_bsc_threshold_above_one(nat):
    """k_sample > sample (threshold 2): the boundary is the smallest sampled |v|, as in the reference, not 0 (which sent everything)."""
    rng = np.random.RandomState(5)
    n, thr = 1000, 2.0
    sz = CR.bsc_sizes(n, thr)
    g = rng.randn(n).astype(np.float32)
    u, v = torch.zeros(n, device=dev()), torch.zeros(n, device=dev())
    out = gc.bsc_compress(cuda(g), u, v, thr)
    bsc_check(g, np.zeros(n, np.float32), np.zeros(n, np.float32), u, v, out, sz)
    assert int((host(out)[sz[0]:] >= 0).sum()) < n


def test_bsc_pull_compress_and_decompress(nat):
    rng = np.random.RandomState(11)

    def dense(n, zeros):
        d = rng.randn(n).astype(np.float32)
        d[rng.rand(n) < zeros] = 0.0
        d[rng.rand(n) < 0.05] = -0.0                    # not sent
        d[rng.rand(n) < 0.01] = np.nan                  # sent
        d[-1] = 1.5
        return d

    ds = [dense(5000, 0.7), dense(300000, 0.5), np.zeros(7, np.float32), dense(4097, 0.0)]
    cnt = [int((d != 0).sum()) for d in ds]
    ks = [cnt[0] + 100, cnt[1] // 3, 3, 2 * 4096]       # above / below the count; all padding; everything sent over two chunks
    outs = [torch.full((2 * k,), 7.0, device=dev()) for k in ks]
    gs = [cuda(d) for d in ds]
    api.bsc_pull_compress_batch(api._segs_to_dev([api.bsc_segment(g, None, None, o, k, 0, 0) for g, o, k in zip(gs, outs, ks)], dev()), len(ds))
    for d, o, k in zip(ds, outs, ks):
        assert np.array_equal(u32(o), u32(CR.bsc_pull(d, k))), (d.size, k)
    z = gc.bsc_pull_compress(gs[1], 0.01, 3)
    assert np.array_equal(u32(z), u32(CR.bsc_pull(ds[1], int(300000 * 0.01 * 3))))
    # decompress: sentinels skipped, index n-1 reached, overwrite and accumulate, k = 0
    d = ds[0].copy()
    d[np.isnan(d)] = 2.0
    zp = CR.bsc_pull(d, cnt[0] + 100)
    assert zp[len(zp) // 2:].max() == d.size - 1 and zp.min() == -65530.0
    out0 = rng.randn(d.size).astype(np.float32)
    for acc in (False, True):
        out = cuda(out0)
        gc.bsc_decompress(cuda(zp), d.size, out=out, accumulate=acc)
        assert np.array_equal(u32(out), u32(CR.bsc_decompress(zp, d.size, out0 if acc else None)))
        out = cuda(out0)
        gc.bsc_decompress(torch.zeros(0, device=dev()), d.size, out=out, accumulate=acc)
        assert np.array_equal(host(out), out0 if acc else np.zeros_like(out0))


# ---------------------------------------------------------------------------------------------------------------- edges of the entry points
def test_empty_tensors_and_input_checks(nat):
    """n = 0 launches nothing (a zero-CTA grid is a launch error); non-contiguous state is refused; an fp16 gradient is cast as on the CPU."""
    e = torch.zeros(0, device=dev())
    q, s = gc.fp8_block_quantize(e, torch.zeros(0, device=dev()))
    assert q.numel() == 0 and s.numel() == 0 and gc.fp8_block_dequantize(q, s, 0).numel() == 0
    nat.dgt_contrib(e, torch.zeros(0, device=dev()), 1024, 0.3, True)
    api.bsc_compress_batch(e, 0)
    api.bsc_pull_compress_batch(e, 0)
    assert gc.quantize_2bit(e, torch.zeros(0, device=dev()), 0.5).numel() == 0
    torch.cuda.synchronize()
    g = torch.randn(1000, device=dev())
    st = torch.zeros(1000, 2, device=dev())[:, 0]
    for call in (lambda: gc.quantize_2bit(g, st, 0.5), lambda: gc.bsc_compress(g, st, torch.zeros_like(g), 0.5),
                 lambda: gc.bsc_compress(g, torch.zeros_like(g), st, 0.5), lambda: gc.fp8_block_quantize(g, st)):
        with pytest.raises(MXNetError, match="contiguous"):
            call()
    h = g.half()
    r1, r2 = torch.zeros_like(g), torch.zeros_like(g)
    assert torch.equal(gc.quantize_2bit(h, r1, 0.5).view(torch.int32), gc.quantize_2bit(h.float(), r2, 0.5).view(torch.int32))
    assert torch.equal(r1, r2)
    u1, v1, u2, v2 = (torch.zeros_like(g) for _ in range(4))
    assert torch.equal(gc.bsc_compress(h, u1, v1, 0.05), gc.bsc_compress(h.float(), u2, v2, 0.05)) and torch.equal(v1, v2)
    assert all(torch.equal(a, b) for a, b in zip(gc.fp8_block_quantize(h), gc.fp8_block_quantize(h.float())))


# ---------------------------------------------------------------------------------------------------------------- wire compatibility
@needs_c
def test_wire_compatible_with_native_cpu_codec(nat):
    """GPU 2-bit words and residuals equal the CPU codec's and the native C++ codec's; a GPU Bi-Sparse payload decodes identically there."""
    C = runtime.C()
    comp = C.GradientCompression()
    comp.set_params("2bit", 0.5)
    rng = np.random.RandomState(3)
    n = 100003
    r_gpu, r_cpu, r_c = torch.zeros(n, device=dev()), torch.zeros(n), np.zeros(n, np.float32)
    for _ in range(3):
        g = grad_2bit(n, 0.5, rng)
        q_gpu = gc.quantize_2bit(cuda(g), r_gpu, 0.5)
        q_cpu = gc.quantize_2bit(torch.from_numpy(g), r_cpu, 0.5)
        q_c = comp.quantize_2bit(g, r_c)
        assert np.array_equal(u32(q_gpu), u32(q_cpu)) and np.array_equal(u32(q_gpu), q_c.view(np.uint32))
        assert np.array_equal(u32(r_gpu), u32(r_cpu)) and np.array_equal(u32(r_gpu), u32(r_c))
    u, v = torch.zeros(n, device=dev()), torch.zeros(n, device=dev())
    for _ in range(2):
        z = gc.bsc_compress(cuda(rng.randn(n).astype(np.float32)), u, v, 0.01)
        zz = host(z)
        assert np.array_equal(u32(gc.bsc_decompress(z, n)), u32(C.GradientCompression.bsc_decompress(zz, n)))


# ---------------------------------------------------------------------------------------------------------------- KVStore entry points
def test_kvstore_device_2bit_reduce(nat):
    """``kv.create('device')`` with 2-bit: two arrays on gpu(0) pushed for one key take CommDevice's compressed reduce, one residual per
    source; a single-source push stays uncompressed (comm.h:506)."""
    kv = mx.kv.create("device")
    kv.set_gradient_compression({"type": "2bit", "threshold": 0.5})
    shape = (300, 71)
    n = 300 * 71
    kv.init(3, mx.nd.zeros(shape, ctx=mx.gpu(0)))
    out = mx.nd.zeros(shape, ctx=mx.gpu(0))
    rng = np.random.RandomState(8)
    res = [np.zeros(n, np.float32), np.zeros(n, np.float32)]
    for rnd in range(5):
        gs = [(rng.randn(n) * 0.4).astype(np.float32) for _ in range(2)]
        kv.push(3, [mx.nd.array(cuda(g.reshape(shape)), ctx=mx.gpu(0)) for g in gs])
        kv.pull(3, out=out)
        deq = []
        for i in range(2):
            w, res[i] = CR.quantize_2bit(gs[i], res[i], 0.5)
            deq.append(CR.dequantize_2bit(w, n, 0.5).astype(np.float64))
        got = host(out._t).reshape(-1).astype(np.float64)
        assert np.array_equal(got, deq[0] + deq[1]), rnd          # multiples of 0.5: the fp32 sum is exact
        assert np.abs(got - (gs[0] + gs[1])).max() > 0.1            # and it is not the uncompressed sum
    g = (rng.randn(n) * 0.4).astype(np.float32)
    kv.push(3, mx.nd.array(cuda(g.reshape(shape)), ctx=mx.gpu(0)))
    kv.pull(3, out=out)
    assert np.array_equal(host(out._t).reshape(-1), g)


def _twobit_sgd_ref(w0, grads, thr, lr, scale):
    """fp64 weights after SGD on the 2-bit dequantised gradients (residual carried per key in fp32, bit-exact)."""
    w = [x.astype(np.float64).reshape(-1) for x in w0]
    res = [np.zeros(x.size, np.float32) for x in w0]
    for gr in grads:
        for i, g in enumerate(gr):
            q, res[i] = CR.quantize_2bit(g.reshape(-1), res[i], thr)
            w[i] = w[i] - lr * scale * CR.dequantize_2bit(q, g.size, thr).astype(np.float64)
    return w


def test_kvstore_fabric_2bit_sgd(nat, clean_env):
    """``kv.create('dist_sync')`` on one GPU (the in-process fabric KVStore) with 2-bit compression and SGD, four rounds."""
    clean_env.delenv("WORLD_SIZE", raising=False)
    clean_env.delenv("RANK", raising=False)
    clean_env.setenv("GEOMX_FABRIC", "auto")
    from geomx_b200.parallel.fabric_kvstore import KVStoreFabric
    kv = mx.kv.create("dist_sync")
    assert isinstance(kv, KVStoreFabric), type(kv)
    kv.set_optimizer(mx.optimizer.SGD(learning_rate=0.1))
    kv.set_gradient_compression({"type": "2bit", "threshold": 0.25})
    rng = np.random.RandomState(4)
    shapes = [(1000,), (50, 37), (3,)]
    W0 = [rng.randn(*s).astype(np.float32) for s in shapes]
    arrs = [mx.nd.array(cuda(w), ctx=mx.gpu(0)) for w in W0]
    for i, a in enumerate(arrs):
        kv.init(i, a)
    grads = []
    outs = [mx.nd.zeros(s, ctx=mx.gpu(0)) for s in shapes]
    for rnd in range(4):
        gr = [(rng.randn(*s) * 0.3).astype(np.float32) for s in shapes]
        grads.append(gr)
        for i, g in enumerate(gr):
            kv.push(i, mx.nd.array(cuda(g), ctx=mx.gpu(0)))
        for i in range(len(shapes)):
            kv.pull(i, out=outs[i])
        ref = _twobit_sgd_ref(W0, grads, 0.25, 0.1, 1.0)
        err = max(float(np.abs(host(o._t).reshape(-1) - r).max()) for o, r in zip(outs, ref))
        assert err < 1e-6, (rnd, err)
    plain = [w.astype(np.float64).reshape(-1) - 0.1 * sum(gr[i].reshape(-1).astype(np.float64) for gr in grads) for i, w in enumerate(W0)]
    assert max(float(np.abs(a - b).max()) for a, b in zip(plain, ref)) > 1e-2       # the check can tell compressed from plain pushes
    print("\n  fabric KVStore 2-bit + SGD: %.1e" % err, end="")


def test_trainer_2bit_compression(nat, clean_env):
    """``gluon.Trainer(kvstore='dist_sync', compression_params={'type': '2bit'})`` on a small Dense net: the recorded gradients replayed
    through the reference give the weights the trainer ends with."""
    clean_env.delenv("WORLD_SIZE", raising=False)
    clean_env.delenv("RANK", raising=False)
    clean_env.setenv("GEOMX_FABRIC", "auto")
    mx.random.seed(2)
    net = mx.gluon.nn.HybridSequential()
    net.add(mx.gluon.nn.Dense(16, in_units=12, activation="relu"), mx.gluon.nn.Dense(3, in_units=16))
    net.initialize(mx.init.Xavier(), ctx=mx.gpu(0))
    params = list(net.collect_params().values())
    W0 = [host(p.data()._t).copy() for p in params]
    B, lr, thr = 8, 0.5, 0.05
    tr = mx.gluon.Trainer(net.collect_params(), "sgd", {"learning_rate": lr}, kvstore="dist_sync",
                          compression_params={"type": "2bit", "threshold": thr})
    loss_fn = mx.gluon.loss.L2Loss()
    rng = np.random.RandomState(6)
    grads = []
    for _ in range(5):
        x = mx.nd.array(cuda(rng.randn(B, 12).astype(np.float32)), ctx=mx.gpu(0))
        y = mx.nd.array(cuda(rng.randn(B, 3).astype(np.float32)), ctx=mx.gpu(0))
        with mx.autograd.record():
            loss = loss_fn(net(x), y)
        loss.backward()
        grads.append([host(p.grad()._t).copy() for p in params])
        tr.step(B)
    ref = _twobit_sgd_ref(W0, grads, thr, lr, 1.0 / B)
    got = [host(p.data()._t).reshape(-1) for p in params]
    err = max(float(np.abs(a - b).max()) for a, b in zip(got, ref))
    assert err < 1e-5, err
    print("\n  Trainer 2-bit: %.1e" % err, end="")


# ---------------------------------------------------------------------------------------------------------------- the checks catch bugs
def test_mutations_fall_outside(nat):
    """Recorded GPU outputs replayed through deliberately broken references: swapped pos/neg bits, '>' for '>=' at the Bi-Sparse boundary,
    the DGT tail block divided by one more than its length, an fp8 scale of amax/447.  Each must fail its check."""
    rng = np.random.RandomState(9)
    g = grad_2bit(1000, 0.1, rng)
    q = gc.quantize_2bit(cuda(g), torch.zeros(1000, device=dev()), 0.1)
    assert np.array_equal(u32(q), CR.quantize_2bit(g, np.zeros(1000, np.float32), 0.1)[0])
    assert not np.array_equal(u32(q), CR.quantize_2bit(g, np.zeros(1000, np.float32), 0.1, posbits=CR.NEG, negbits=CR.POS)[0])

    n, thr = 4097, 0.05
    sz = CR.bsc_sizes(n, thr)
    g = rng.randint(-3, 4, n).astype(np.float32)
    u, v = torch.zeros(n, device=dev()), torch.zeros(n, device=dev())
    out = gc.bsc_compress(cuda(g), u, v, thr)
    z0 = np.zeros(n, np.float32)
    bsc_check(g, z0, z0, u, v, out, sz)
    with pytest.raises(AssertionError, match="sent set"):
        bsc_check(g, z0, z0, u, v, out, sz, ge=False)

    n, be = 1025, 1000
    g = rng.randn(n).astype(np.float32)
    c = torch.zeros(2, device=dev())
    nat.dgt_contrib(cuda(g), c, be, 0.3, True)
    good, bad = CR.dgt_contrib(g, None, be, 0.3, True), CR.dgt_contrib(g, None, be, 0.3, True, tail=1)
    assert np.max(np.abs(host(c) - good) / good) <= 1e-6 < np.max(np.abs(host(c) - bad) / bad)

    x = fp8_data(1000, rng)
    q, s = gc.fp8_block_quantize(cuda(x))
    qr, sr, _, _ = CR.fp8_quantize(x, scale_div=447.0)
    assert not np.array_equal(u32(s), u32(sr)) and not np.array_equal(host(q), qr)
