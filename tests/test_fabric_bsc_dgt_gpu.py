"""The fused exchange's Bi-Sparse tiles and its DGT re-ranking on one GPU, against the fp64 reference of ``tests/_update_ref.py``.

Everything here runs the multi-rank LL packet kernel in loop-back (``HipsFabric(..., loopback=True)``) on one GPU:

  a. crafted tiles, one round from zero state: ``u = v = g * push_scale`` exactly (a power-of-two push scale), so the selection (K largest
     |v|, ties to the lowest index) is fully determined and the pulled sparse aggregate, ``bsc_u`` and ``bsc_v`` must match bit for bit;
  b. five rounds on an arena that mixes Bi-Sparse, fp16, fp8 and fp32 keys, without a server optimizer and with SGD / Adam / DCASGD, and
     masked rounds.  After round 1 the kernel's fp32 ``u`` / ``v`` may differ from fp64 in the last bits, and a near-tie at the K-th
     magnitude can legitimately go the other way; so each round the kernel's selection (the entries it cleared in ``bsc_v``) is checked to
     be a top-K of the reference's |v| within SEL_SLACK, and the reference then adopts it;
  c. the packet-buffer limit, channels that contain Bi-Sparse tiles, DGT contributions / re-ranking / demotion / tile order;
  d. the training engine in the bench's ``bsc`` and ``mpq_dgt`` configurations, and the re-rank schedule of eager and graphed engines.

Measured errors are printed (``-s``).
"""
import numpy as np
import pytest
import torch

import geomx_b200 as mx

import _update_ref as R
from _cnn_ref import cleanup, dev, nat  # noqa: F401  (nat: fixture)
from _update_harness import A_LOCAL, FAB_SPECS, KEY_MULTS, KEY_SIZES, PUSH_SCALE, SWITCHES, TOL, _batches, _clip_for, _opt, half_ulps

pytestmark = pytest.mark.gpu

# the update paths' switches and the Bi-Sparse / DGT ones
BSC_SWITCHES = SWITCHES + ("ADAPTIVE_K_FLAG", "DMLC_K", "DMLC_K_MIN", "DGT_CONTRIBUTION_ALPHA")
# Relative slack of a kernel's Bi-Sparse selection against the reference's |v| at the K-th magnitude (see R.selection_slack): fp32 u / v
# carry a few ulps of rounding per round (relative ~1e-7 after five rounds), so a real near-tie may fall either way; 1e-5 is far below
# what a wrong rule (ties to the high index, a stale residual) produces on these tiles.
SEL_SLACK = 1e-5


@pytest.fixture
def clean_env(monkeypatch):
    for k in BSC_SWITCHES:
        monkeypatch.delenv(k, raising=False)
    return monkeypatch


def bits(t):
    return t.detach().float().cpu().contiguous().view(torch.int32)


MIX_FMTS = ["fp32", "bsc", "fp16", "bsc", "fp8", "bsc"]


def _fabric(sizes, fmts, spec, thr=0.01, mults=None, push_scale=PUSH_SCALE):
    from geomx_b200.parallel import ArenaLayout, HipsFabric, Topology
    layout = ArenaLayout.build([(i, (n,)) for i, n in enumerate(sizes)], mults=mults)
    f = HipsFabric(layout, Topology(1, 0, 1, 0), dev(), spec, loopback=True)
    assert f.protocol == "ll"
    f.set_push_scale(push_scale)
    f.set_wire_formats({i: m for i, m in enumerate(fmts)}, bsc_threshold=thr)
    return f


def _key(f, t, i):
    """Key i of arena tensor ``t``, tile-padded."""
    sl = f.layout.slots[i]
    return t[sl.offset:sl.offset + sl.tiles * 1024]


def _push(f, grads):
    for i, x in enumerate(grads):
        f.grad_view(i).copy_(x)


def _adopt(f, checked):
    """A ``bsc_select`` for ``UpdateRef.step``: the kernel's selection of a tile is where its (post-round) ``bsc_v`` is 0 and the reference's
    v is not; it is checked to be a top-K of the reference's |v| (the worst slack goes to ``checked``) and then adopted."""
    kv = f.bsc_v.cpu()

    def select(i, t, vt):
        sl = f.layout.slots[i]
        a = sl.offset + t * 1024
        sel = torch.nonzero((kv[a:a + 1024] == 0) & (vt != 0)).flatten()
        s = R.selection_slack(vt, sel, f.bsc_k)
        checked.append(s)
        assert s <= SEL_SLACK, (i, t, s)
        return sel
    return select


def _bsc_state_err(f, ref):
    """Worst norm-relative error of bsc_u / bsc_v over the keys that have Bi-Sparse tiles."""
    e = 0.0
    for i in range(len(ref.w)):
        if "bsc" in ref.tile_fmts(i):
            e = max(e, R.rel(_key(f, f.bsc_u, i), ref.u[i]), R.rel(_key(f, f.bsc_v, i), ref.v[i]))
    return e


# ============================================================================================================ a. crafted tiles, bit for bit
def _crafted_tiles(K, gen):
    """(name, tile) pairs, 1024 float32 values each, whose selection at this K is fully determined."""
    rs = lambda n: torch.where(torch.rand(n, generator=gen) < 0.5, -1.0, 1.0)
    perm = lambda: torch.randperm(1024, generator=gen)
    out = []
    # exact ties at the K-th magnitude: K-3 distinct larger values, 40 entries of magnitude 5, the rest smaller
    t = torch.rand(1024, generator=gen) * 2.0
    p = perm()
    top = max(0, K - 3)
    t[p[:top]] = 10.0 + torch.arange(top, dtype=torch.float32) * 0.25
    t[p[top:top + 40]] = 5.0
    out.append(("ties", t * rs(1024)))
    # magnitudes that share their top 24 bits: only the last radix pass separates them (duplicates among the 256 patterns tie as well)
    b = (0x3F9A5A00 | torch.randint(0, 256, (1024,), generator=gen)).to(torch.int32)
    out.append(("low-byte", b.view(torch.float32) * rs(1024)))
    # K-th and (K+1)-th magnitude one ulp apart
    t = torch.rand(1024, generator=gen) * 0.5
    p = perm()
    t[p[:K - 1]] = 2.0 + torch.rand(K - 1, generator=gen)
    t[p[K - 1]] = 1.0
    t[p[K]] = float(np.nextafter(np.float32(1.0), np.float32(0.0)))
    out.append(("one-ulp", t * rs(1024)))
    # mixed signs and +-0
    t = torch.randn(1024, generator=gen)
    z = torch.rand(1024, generator=gen) < 0.3
    t[z] = 0.0
    t[z & (torch.rand(1024, generator=gen) < 0.5)] = -0.0
    out.append(("signed-zeros", t))
    # all zeros (some negative) and fewer than K non-zeros
    t = torch.zeros(1024)
    t[perm()[:100]] = -0.0
    out.append(("all-zero", t))
    t = torch.zeros(1024)
    t[perm()[:K // 2]] = torch.randn(K // 2, generator=gen)
    out.append(("sparse", t))
    return out


@pytest.mark.parametrize("K", [1, 10, 20, 512])
def test_bsc_crafted_tiles_bit_exact(nat, clean_env, K):
    """One round from zero state per K, no server optimizer, push scale 1/2: the pulled sparse aggregate (parameter arena), the global
    owner's stored aggregate and ``bsc_u`` / ``bsc_v`` equal the reference bit for bit; at most K non-zeros per tile; the padding of the
    partial last tiles (keys of 1025 and 1000 floats) stays zero in the parameter arena and in u / v; no protocol error."""
    gen = torch.Generator().manual_seed(K)
    tiles = _crafted_tiles(K, gen)
    sizes = [1024] * len(tiles) + [1025, 1000]
    f = _fabric(sizes, ["bsc"] * len(sizes), None, thr=K / 1024, push_scale=0.5)
    try:
        assert f.bsc_k == K
        for rnd in range(2):             # two crafted rounds, the state cleared in between
            grads = [t.clone() for _, t in tiles] + [torch.randn(1025, generator=gen), torch.randn(1000, generator=gen)]
            if rnd == 1:
                grads = [g.flip(0) for g in grads]
            f.bsc_u.zero_()
            f.bsc_v.zero_()
            _push(f, grads)
            f.fsa_step()
            torch.cuda.synchronize()
            assert not f.check_protocol_errors()
            ref = R.UpdateRef(None, [torch.zeros(n) for n in sizes], push_scale=0.5, fmts=["bsc"] * len(sizes), round_after_scale=True, bsc_k=K)
            ref.step(grads)
            P = ref.params()
            for i in range(len(sizes)):
                name = tiles[i][0] if i < len(tiles) else "partial-%d" % sizes[i]
                assert torch.equal(bits(f.param_view(i)), bits(P[i])), (K, name, "pulled aggregate")
                assert torch.equal(f.layout.view(f.w, i).cpu().double(), ref.w[i]), (K, name, "stored aggregate")
                assert torch.equal(bits(_key(f, f.bsc_u, i)), bits(ref.u[i])), (K, name, "bsc_u")
                assert torch.equal(bits(_key(f, f.bsc_v, i)), bits(ref.v[i])), (K, name, "bsc_v")
                nz = (_key(f, f.param.tensor, i) != 0).view(-1, 1024).sum(1)
                assert int(nz.max()) <= K, (K, name)
            for sl in f.layout.slots:
                a, b = sl.offset + sl.numel, sl.offset + sl.tiles * 1024
                for t in (f.param.tensor, f.w, f.bsc_u, f.bsc_v):
                    assert bool((t[a:b] == 0).all()), "padding of key %d" % sl.key
    finally:
        del f
        cleanup()


# ============================================================================================================ b. rounds against the reference
def _grads(gen, sizes=KEY_SIZES):
    out = []
    for n in sizes:
        x = torch.randn(n, generator=gen) * 0.01 * 32
        x[torch.rand(n, generator=gen) < 0.05] = 0.0
        out.append(x)
    return out


@pytest.mark.parametrize("kind", [None, "sgd", "adam", "dcasgd"])
def test_bsc_mixed_rounds(nat, clean_env, kind):
    """Five rounds on keys of 1 .. 70 000 floats with Bi-Sparse, fp16, fp8 and fp32 keys and multipliers.  No server optimizer: the stored
    and the pulled aggregate (sparse for Bi-Sparse keys, halves for fp16 / fp8).  SGD / Adam / DCASGD: master weights and both state slots
    (displacement tolerance), dense pulls (fp32 and Bi-Sparse keys exact copies of the master weights, fp16 / fp8 keys fp16 of it).  Every
    round: ``bsc_u`` / ``bsc_v``, the step count, a valid selection."""
    spec = FAB_SPECS.get(kind)
    f = _fabric(KEY_SIZES, MIX_FMTS, spec, mults=KEY_MULTS)
    try:
        gen = torch.Generator().manual_seed(5 + len(kind or ""))
        W0 = [torch.randn(n, generator=gen) * 0.1 for n in KEY_SIZES]
        for i, w in enumerate(W0):
            f.param_view(i).copy_(w)
        f.load_master_from_param()
        ref = R.UpdateRef(spec, W0, mults=KEY_MULTS, push_scale=PUSH_SCALE, fmts=MIX_FMTS, round_after_scale=True, bsc_k=f.bsc_k)
        worst = [0.0] * 4
        for k in range(1, 6):
            grads = _grads(gen)
            _push(f, grads)
            f.fsa_step()
            torch.cuda.synchronize()
            checked = []
            ref.step(grads, bsc_select=_adopt(f, checked))
            assert f.opt_step == k and not f.check_protocol_errors()
            W = [f.layout.view(f.w, i) for i in range(len(KEY_SIZES))]
            Pk = [f.param_view(i) for i in range(len(KEY_SIZES))]
            e_uv = _bsc_state_err(f, ref)
            if spec is None:
                e_w = max(R.rel(W[i], ref.w[i]) for i in range(len(KEY_SIZES)))
                e_p = max(R.rel(Pk[i], p) for i, p in enumerate(ref.params()))
                e_s = 0.0
                for i in range(len(KEY_SIZES)):
                    if MIX_FMTS[i] == "bsc":
                        assert int((_key(f, f.param.tensor, i) != 0).view(-1, 1024).sum(1).max()) <= f.bsc_k
            else:
                e_w = R.displacement_err(W, W0, ref.w, stores=k)
                e_s = max(max(R.rel(f.layout.view(f.s0, i), ref.s0[i]), R.rel(f.layout.view(f.s1, i), ref.s1[i]) if kind != "sgd" else 0.0)
                          for i in range(len(KEY_SIZES)))
                half = [i for i, m in enumerate(MIX_FMTS) if m in ("fp16", "fp8")]
                assert all(torch.equal(Pk[i], W[i].half().float()) for i in half), "fp16 pull != fp16(master)"
                assert all(torch.equal(Pk[i], W[i]) for i in range(len(KEY_SIZES)) if i not in half), "pull != master"
                # a pulled fp16 element may sit one fp16 step off where its fp8 gradient rounded across a tie differently (as in
                # test_update_paths_gpu.py: at most 2)
                e_p = 0.0
                assert max(half_ulps(Pk[i], ref.w[i]) for i in half) <= 2.0
            worst = [max(a, b) for a, b in zip(worst, (e_w, e_s, e_uv, max(checked)))]
            assert e_w < TOL and e_s < TOL and e_uv < TOL and e_p < TOL, (kind, k, e_w, e_s, e_uv, e_p)
        print("\n  bsc rounds %-6s  w %.1e  state %.1e  u/v %.1e  selection slack %.1e" % ((kind or "none",) + tuple(worst)))
    finally:
        del f
        cleanup()


def test_bsc_masked_rounds(nat, clean_env):
    """Masked rounds (``tile_active``) with Adam: the keys of the round follow the reference, every other key keeps w, s0, s1, the parameters
    and its Bi-Sparse u / v bit-identical.  The active sets only shrink (the fabric's Adam step count is per channel)."""
    spec = FAB_SPECS["adam"]
    f = _fabric(KEY_SIZES, MIX_FMTS, spec, mults=KEY_MULTS)
    try:
        gen = torch.Generator().manual_seed(77)
        W0 = [torch.randn(n, generator=gen) * 0.1 for n in KEY_SIZES]
        for i, w in enumerate(W0):
            f.param_view(i).copy_(w)
        f.load_master_from_param()
        ref = R.UpdateRef(spec, W0, mults=KEY_MULTS, push_scale=PUSH_SCALE, fmts=MIX_FMTS, round_after_scale=True, bsc_k=f.bsc_k)
        for k, active in enumerate([None, [0, 1, 2, 3, 4, 5], [1, 3, 4, 5], [3, 5], [5]], 1):
            grads = _grads(gen)
            _push(f, grads)
            before = [t.clone() for t in (f.w, f.s0, f.s1, f.param.tensor, f.bsc_u, f.bsc_v)]
            if active is None:
                f.fsa_step()
            else:
                mask = torch.zeros(f.tiles, dtype=torch.uint8)
                for i in active:
                    sl = f.layout.slots[i]
                    mask[sl.offset // 1024: sl.offset // 1024 + sl.tiles] = 1
                f.tile_active.copy_(mask.to(dev()))
                f.fsa_step(masked=True)
            torch.cuda.synchronize()
            ref.step(grads, active, bsc_select=_adopt(f, []))
            for i in set(range(len(KEY_SIZES))) - set(active if active is not None else range(len(KEY_SIZES))):
                sl = f.layout.slots[i]
                a, b = sl.offset, sl.offset + sl.tiles * 1024
                for old, new in zip(before, (f.w, f.s0, f.s1, f.param.tensor, f.bsc_u, f.bsc_v)):
                    assert torch.equal(old[a:b], new[a:b]), "inactive key %d changed in round %d" % (i, k)
            W = [f.layout.view(f.w, i) for i in range(len(KEY_SIZES))]
            e = (R.displacement_err(W, W0, ref.w, stores=k), _bsc_state_err(f, ref))
            assert max(e) < TOL, (k, e)
        print("\n  bsc masked rounds: w %.1e  u/v %.1e" % e)
    finally:
        del f
        cleanup()


# ============================================================================================================ c. limits, channels, DGT
def test_bsc_limits(nat, clean_env):
    """``floor(1024 * thr) * num_parties`` above 512 packets is refused; 512 is accepted; a tiny threshold gives K = 1 (one non-zero per
    tile of the pulled aggregate)."""
    f = _fabric([5000], ["fp32"], None)
    try:
        with pytest.raises(RuntimeError):
            f.set_wire_formats({0: "bsc"}, bsc_threshold=513 / 1024)
        f.set_wire_formats({0: "bsc"}, bsc_threshold=0.5)
        assert f.bsc_k == 512
        f.set_wire_formats({0: "bsc"}, bsc_threshold=1e-6)
        assert f.bsc_k == 1
        f.bsc_u.zero_(); f.bsc_v.zero_()
        g = torch.randn(5000, generator=torch.Generator().manual_seed(1))
        f.grad_view(0).copy_(g)
        f.fsa_step()
        torch.cuda.synchronize()
        nz = (f.param.tensor != 0).view(-1, 1024).sum(1)
        assert nz.tolist() == [1] * 5 and not f.check_protocol_errors()
        ref = R.UpdateRef(None, [torch.zeros(5000)], push_scale=PUSH_SCALE, fmts=["bsc"], round_after_scale=True, bsc_k=1)
        ref.step([g])
        assert torch.equal(bits(f.param_view(0)), bits(ref.params()[0]))
    finally:
        del f
        cleanup()


@pytest.mark.parametrize("replicate", [True, False])
def test_bsc_channel_falls_back_to_ll(nat, clean_env, replicate):
    """A channel with Bi-Sparse tiles cannot take the direct protocol: it runs the LL kernel on its tiles, and its rounds equal
    ``fsa_step`` on a twin fabric bit for bit (weights, state, parameters, u / v); a replicated such channel cannot run in a compute kernel's
    tail (``channel_fused_args`` is None)."""
    spec = FAB_SPECS["adam"]
    fa = _fabric(KEY_SIZES, MIX_FMTS, spec, mults=KEY_MULTS)
    fb = _fabric(KEY_SIZES, MIX_FMTS, spec, mults=KEY_MULTS)
    try:
        assert fa.ll_d is not None
        fa.add_channel("c", list(range(len(KEY_SIZES))), replicate=replicate)
        assert not fa._channel_formats_direct_ok(fa.channels["c"])
        assert fa.channel_fused_args("c") is None
        gen = torch.Generator().manual_seed(8)
        W0 = [torch.randn(n, generator=gen) * 0.1 for n in KEY_SIZES]
        for f in (fa, fb):
            for i, w in enumerate(W0):
                f.param_view(i).copy_(w)
            f.load_master_from_param()
        for _ in range(4):
            grads = _grads(gen)
            _push(fa, grads)
            _push(fb, grads)
            fa.channel_step("c")
            fb.fsa_step()
            torch.cuda.synchronize()
            for a, b in ((fa.w, fb.w), (fa.s0, fb.s0), (fa.s1, fb.s1), (fa.param.tensor, fb.param.tensor), (fa.bsc_u, fb.bsc_u), (fa.bsc_v, fb.bsc_v)):
                assert torch.equal(a, b)
        assert fa.opt_step == fb.opt_step == 4
        assert not fa.check_protocol_errors()
    finally:
        del fa, fb
        cleanup()


def _dgt_fabric(spec, k):
    f = _fabric(KEY_SIZES, MIX_FMTS, spec, mults=KEY_MULTS)
    f.enable_dgt(k=k, alpha=0.3)
    return f


def _flat_fmts(ref):
    return [x for i in range(len(ref.w)) for x in ref.tile_fmts(i)]


def _set_ref_fmts(ref, flat):
    pos = 0
    for i in range(len(ref.w)):
        T = ref.u[i].numel() // 1024
        ref.fmts[i] = list(flat[pos:pos + T])
        pos += T


CODE = {"fp32": 0, "fp16": 1, "bsc": 2, "fp8": 3}


@pytest.mark.parametrize("adaptive", [False, True])
def test_dgt_rerank_and_rounds(nat, clean_env, adaptive):
    """DGT with Adam on the mixed arena, three blocks of rounds with a re-rank after each of the first two:

    * the contributions (Bi-Sparse tiles: of the decompressed aggregate) are the fp64 EMA of the mean |aggregate| per tile;
    * ``dgt_rerank()`` returns them, makes ``tile_order`` a permutation non-increasing in them, sizes the important set as the reference
      does (fixed K, or ``ADAPTIVE_K_FLAG=1`` with ``DMLC_K_MIN``), demotes the unimportant fp32 / fp16 tiles to fp8 and leaves Bi-Sparse
      and important tiles at their base format;
    * the rounds after a re-rank match the reference with those per-tile formats;
    * a twin fabric with the same formats but the identity tile order computes the same bits."""
    if adaptive:
        clean_env.setenv("ADAPTIVE_K_FLAG", "1")
        clean_env.setenv("DMLC_K_MIN", "0.05")
    # fixed: 5 % of the 79 tiles important; adaptive: the prefix with 60 % of the contribution, at least 5 % of the tiles.  The one-float
    # fp32 key and (at fixed K) the fp16 key rank below the dense fp8 key, so something is demoted
    spec = FAB_SPECS["adam"]
    k = 0.6 if adaptive else 0.05
    fa, fb = _dgt_fabric(spec, k), _dgt_fabric(spec, k)
    try:
        gen = torch.Generator().manual_seed(9 + adaptive)
        W0 = [torch.randn(n, generator=gen) * 0.1 for n in KEY_SIZES]
        for f in (fa, fb):
            for i, w in enumerate(W0):
                f.param_view(i).copy_(w)
            f.load_master_from_param()
        ref = R.UpdateRef(spec, W0, mults=KEY_MULTS, push_scale=PUSH_SCALE, fmts=list(MIX_FMTS), round_after_scale=True, bsc_k=fa.bsc_k)
        base = _flat_fmts(ref)
        ema = torch.zeros(fa.tiles, dtype=torch.float64)
        worst = [0.0, 0.0, 0.0]
        demoted = 0
        for block in range(3):
            for _ in range(3):
                grads = _grads(gen)
                _push(fa, grads)
                _push(fb, grads)
                fa.fsa_step()
                fb.fsa_step()
                torch.cuda.synchronize()
                ref.step(grads, bsc_select=_adopt(fa, []))
                ema = R.dgt_ema(ema, torch.cat(ref.agg).abs().view(-1, 1024).mean(1), 0.3)
                for a, b in ((fa.w, fb.w), (fa.s0, fb.s0), (fa.s1, fb.s1), (fa.param.tensor, fb.param.tensor), (fa.bsc_u, fb.bsc_u),
                             (fa.bsc_v, fb.bsc_v), (fa.dgt_contrib, fb.dgt_contrib)):
                    assert torch.equal(a, b), "the tile order changed the arithmetic"
                W = [fa.layout.view(fa.w, i) for i in range(len(KEY_SIZES))]
                e = (R.displacement_err(W, W0, ref.w, stores=ref.t[0]), _bsc_state_err(fa, ref), R.rel(fa.dgt_contrib, ema))
                worst = [max(x, y) for x, y in zip(worst, e)]
                assert e[0] < TOL and e[1] < TOL and e[2] < 1e-5, (block, e)
            if block == 2:
                break
            c = fa.dgt_rerank()
            torch.cuda.synchronize()
            assert R.rel(c, ema) < 1e-5
            order = fa.tile_order.cpu().long()
            assert sorted(order.tolist()) == list(range(fa.tiles))
            cs = c.cpu()[order]
            assert bool((cs[1:] <= cs[:-1]).all()), "tile order not non-increasing in the contributions"
            want_order, n_imp, fmts = R.dgt_formats(base, c.cpu(), fa.dgt_k, adaptive, 0.05 if adaptive else 0.2)
            assert fa.dgt_num_important == n_imp
            assert torch.equal(order, want_order)
            assert fa.tile_fmt.cpu().tolist() == [CODE[x] for x in fmts]
            important = set(want_order[:n_imp].tolist())
            assert all(fmts[t] == base[t] for t in range(fa.tiles) if t in important or base[t] == "bsc")
            demoted += sum(1 for t in range(fa.tiles) if fmts[t] != base[t])
            _set_ref_fmts(ref, fmts)
            fb.tile_fmt.copy_(fa.tile_fmt)            # the twin: same formats, identity order
            assert bool((fb.tile_order.cpu() == torch.arange(fb.tiles)).all())
        assert demoted > 0, "nothing was demoted"
        assert not fa.check_protocol_errors() and not fb.check_protocol_errors()
        print("\n  DGT %s: %d demotions  w %.1e  u/v %.1e  contributions %.1e" % ("adaptive" if adaptive else "fixed   ", demoted, *worst))
    finally:
        del fa, fb
        cleanup()


# ============================================================================================================ d. the engine
ENGINE = {
    "bsc": dict(update="local", bsc_threshold=0.01, size_lower_bound=1000),
    "mpq_dgt": dict(update="local", wire_dtype="mpq", size_lower_bound=1000, dgt=True, dgt_rerank_every=2),
}


def _engine(case, graph, seed=0):
    from geomx_b200.parallel import Topology
    torch.manual_seed(1234 + seed)
    return mx.models.HipsCNNTrainStep(batch_size=32, optimizer=_opt("adam"), topo=Topology(1, 0, 1, 0), use_graph=graph, loopback=True,
                                      fused_zero_grad=False, **ENGINE[case])


@pytest.mark.parametrize("case,graph", [("bsc", False), ("bsc", True), ("mpq_dgt", False)])
def test_engine_bsc_dgt_matches_fp64(nat, clean_env, case, graph):
    """The bench's ``bsc`` and ``mpq_dgt`` configurations in loop-back (local Adam, ``size_lower_bound=1000``; DGT re-ranks every 2 steps):
    six steps on distinct batches, the reference advanced with the engine's own gradient sums and, for Bi-Sparse tiles, the engine's own
    selection (checked to be a top-K); after every step the local master weights and the parameters, ``bsc_u`` / ``bsc_v``, the optimizer's
    step count; the step's (launch, stream) list; every relevant mutation, replayed on the same gradients, lands outside the tolerance.
    Graph mode restores everything its warm-up steps advanced, the Bi-Sparse state and the DGT ranking included."""
    eng = _engine(case, graph)
    try:
        f = eng.fabric
        B = eng.B
        batches = _batches(B, 6, 99)
        P0 = [p.clone() for p in eng.P]
        spec = dict(R.CASE_SPECS["adam"])
        spec["clip_gradient"] = _clip_for(P0, *batches[0], B, spec["rescale_grad"])
        eng._local_spec = dict(eng._local_spec, clip_gradient=spec["clip_gradient"])
        assert [(n, s) for n, s, _ in eng._steps()] == A_LOCAL
        assert eng.update == "local" and eng.overlap
        if graph:
            eng.x.copy_(batches[0][0]); eng.label.copy_(batches[0][1])
            ts = [f.param.tensor, f.w, f.s0, f.s1, eng.Wl, eng.s0l, eng.s1l, eng.opt_state]
            ts += [t for t in (f.bsc_u, f.bsc_v, f.dgt_contrib, f.tile_order, f.tile_fmt) if t is not None]
            snap = [(t, t.clone()) for t in ts]
            eng.capture()
            torch.cuda.synchronize()
            for t, v in snap:
                t.copy_(v)
            f.set_opt_step(0)
            eng.steps_done = 0
        base = [int(x) for x in f.tile_fmt.cpu()]
        name = {0: "fp32", 1: "fp16", 2: "bsc", 3: "fp8"}
        key_fmts = lambda: [[name[x] for x in f.tile_fmt.cpu()[sl.offset // 1024: sl.offset // 1024 + sl.tiles].tolist()] for sl in eng.layout.slots]
        # the conv keys' channel is replicated (its pull is a local store); the dense keys' channel pulls the aggregate, fp16 / fp8 as halves.
        # Bi-Sparse keys put both channels on the LL kernel, which rounds the scaled aggregate; otherwise the direct protocol rounds the raw sum
        has_bsc = 2 in base
        pull_half = [has_bsc or i >= 4 for i in range(10)]
        mk = lambda mut=None: R.UpdateRef(spec, P0, push_scale=1.0 / B, fmts=key_fmts(), round_after_scale=has_bsc, pull_half=pull_half,
                                          bsc_k=max(f.bsc_k, 1), mutation=mut)
        ref = mk()
        grads, sels, fmts_hist, worst = [], [], [], [0.0, 0.0, 0.0]
        reranks = []
        orig = f.dgt_rerank
        f.dgt_rerank = lambda: (reranks.append(eng.steps_done), orig())[1]
        for k, (X, y) in enumerate(batches, 1):
            eng.x.copy_(X); eng.label.copy_(y)
            eng.run_device()                # a re-rank happens before the step: the formats read now are the step's
            torch.cuda.synchronize()
            fm = key_fmts()
            gs = [x.detach().cpu().clone() for x in eng.G]    # fused zero_grad is off below: the sums stay readable
            grads.append(gs)
            fmts_hist.append(fm)
            ref.fmts = fm
            chosen = {}
            adopt = _adopt(f, []) if has_bsc else None
            ref.step(gs, bsc_select=lambda i, t, vt: chosen.setdefault((i, t), adopt(i, t, vt)))
            sels.append(chosen)
            M = [eng.layout.view(eng.Wl, i) for i in range(10)]
            e = (R.displacement_err(M, P0, ref.w, stores=k), R.displacement_err(eng.P, P0, ref.w, stores=k), _bsc_state_err(f, ref) if has_bsc else 0.0)
            worst = [max(a, b) for a, b in zip(worst, e)]
            assert int(eng.opt_state[0]) == k
            assert e[0] < TOL and e[1] < TOL and e[2] < TOL, (case, k, e)
        assert not f.check_protocol_errors()
        if case == "mpq_dgt":
            assert reranks == [2, 4], reranks
            assert any("fp8" in sum(fm, []) for fm in fmts_hist), "no tile was demoted"
        base_fmts = fmts_hist[0]
        muts = {}
        cand = R.relevant_mutations(spec, push_scale=1.0 / B) + (["bsc_no_momentum", "bsc_residual_kept"] if has_bsc else ["dgt_no_demotion"])
        for m in cand:
            bad = mk(m)
            for k, gs in enumerate(grads):
                bad.fmts = base_fmts if m == "dgt_no_demotion" else fmts_hist[k]
                bad.step(gs, bsc_select=lambda i, t, vt, k=k: sels[k].get((i, t)) if m not in ("bsc_no_momentum", "bsc_residual_kept") else None)
            muts[m] = R.displacement_err(bad.w, P0, ref.w)
        print("\n  engine %-8s %s  master %.1e  params %.1e  u/v %.1e | mutations: %s" % (
            case, "graph" if graph else "eager", *worst, "  ".join("%s %.1e" % kv for kv in muts.items())))
        weak = {m: e for m, e in muts.items() if not e > 10 * TOL}
        assert not weak, (case, weak)
    finally:
        del eng
        cleanup()


@pytest.mark.parametrize("graph", [False, True])
def test_engine_dgt_rerank_schedule(nat, clean_env, graph):
    """Eager and graphed engines re-rank on one schedule: before every step whose number of steps already taken (a graph's two warm-up
    steps included) is a positive multiple of ``dgt_rerank_every``; capturing the graph also ranks once, after its warm-up."""
    every, N = 3, 10
    eng = _engine("mpq_dgt", graph)
    eng._dgt_every = every
    try:
        calls = []
        orig = eng.fabric.dgt_rerank
        eng.fabric.dgt_rerank = lambda: (calls.append(eng.steps_done), orig())[1]
        X, y = _batches(32, 1, 3)[0]
        for _ in range(N):
            eng.step(X, y)
        torch.cuda.synchronize()
        warm = 2 if graph else 0
        want = ([warm] if graph else []) + [s for s in range(warm + 1, warm + N) if s % every == 0]
        assert calls == want, (graph, calls, want)
        assert eng.steps_done == warm + N
    finally:
        del eng
        cleanup()
