"""Checkpoints of the training engine without a GPU: the re-sharding of the fabric's server state (``gather_tile_state`` /
``scatter_tile_state`` over simulated topologies) and the checks that ``HipsCNNTrainStep.load_states`` applies to a file before it writes
anything (``_ckpt_read`` on a stand-in engine)."""
import types

import numpy as np
import pytest

import geomx_b200 as mx
from geomx_b200.models.cnn import CHECKPOINT_VERSION, CNN_PARAM_NAMES, CNN_PARAM_SHAPES, HipsCNNTrainStep
from geomx_b200.parallel.arena import ArenaLayout
from geomx_b200.parallel.fabric import Topology, gather_tile_state, global_tile_owners, held_tiles, scatter_tile_state

LAYOUT = ArenaLayout.build(list(enumerate(CNN_PARAM_SHAPES)))
T = LAYOUT.total // 1024
CONV_TILES = np.zeros(T, dtype=bool)
for _sl in LAYOUT.slots[:4]:
    CONV_TILES[_sl.offset // 1024: _sl.offset // 1024 + _sl.tiles] = True

# (world, parties, num_gs, protocol, replicated tiles): one rank; the sharded layouts of both protocols; explicit global servers; the
# one-hop replicated conv channel; a single replicated channel of all keys
TOPOS = [(1, 1, 1, "bulk", "all"), (1, 1, 0, "ll", "all")]
for _w in (2, 4, 8):
    for _p in (1, 2):
        for _gs in (0, 1):
            for _proto in ("ll", "bulk"):
                TOPOS.append((_w, _p, _gs, _proto, None))
        TOPOS.append((_w, _p, 0, "ll", "conv"))
TOPOS.append((4, 2, 0, "ll", "all"))


def _topo(world, parties, gs, proto, rep):
    owners = global_tile_owners(Topology(world, 0, parties, gs), LAYOUT, proto)
    replicated = {None: None, "conv": CONV_TILES, "all": np.ones(T, dtype=bool)}[rep]
    return owners, replicated


def _tid(t):
    return "w%d-p%d-gs%d-%s-%s" % (t[0], t[1], t[2], t[3], t[4] or "sharded")


def _ranks_holding(full, world, owners, replicated, rng):
    """Per-rank arrays as the ranks of a topology keep them: ``full`` on the tiles each rank holds, noise elsewhere."""
    noise = {r: rng.standard_normal(full.shape).astype(full.dtype) if full.dtype.kind == "f"
             else rng.integers(-9, -1, full.shape).astype(full.dtype) for r in range(world)}
    return [scatter_tile_state(full, {r: noise[r]}, owners, replicated)[r] for r in range(world)]


@pytest.mark.parametrize("topo", TOPOS, ids=[_tid(t) for t in TOPOS])
def test_gather_scatter_round_trip(topo):
    """master / s0 / s1 (1024 values per tile) and the per-tile step words: gather from the ranks that hold each tile, scatter back into
    fresh ranks; every held tile is restored bit for bit and no other tile is touched."""
    world = topo[0]
    owners, replicated = _topo(*topo)
    assert owners.shape == (T,) and owners.min() >= 0 and owners.max() < world
    rng = np.random.default_rng(world * 10 + topo[1])
    state = {k: rng.standard_normal(LAYOUT.total).astype(np.float32) for k in ("w", "s0", "s1")}
    state["step"] = rng.integers(0, 1000, T).astype(np.int32)
    for name, full in state.items():
        ranks = _ranks_holding(full, world, owners, replicated, rng)
        got = gather_tile_state(ranks, owners, replicated)
        assert got.dtype == full.dtype and np.array_equal(got, full), name
        fresh = {r: np.full_like(full, -7) for r in range(world)}
        scatter_tile_state(got, fresh, owners, replicated)
        for r in range(world):
            held = np.repeat(held_tiles(owners, replicated, r), full.size // T)
            assert np.array_equal(fresh[r][held], full[held]), (name, r)
            assert (fresh[r][~held] == -7).all(), (name, r, "a tile the rank does not hold was written")
        # every tile is held by at least one rank
        assert np.logical_or.reduce([held_tiles(owners, replicated, r) for r in range(world)]).all()


RESHARD = [((1, 1, 1, "bulk", "all"), (8, 2, 0, "ll", "conv")), ((8, 2, 0, "ll", "conv"), (1, 1, 0, "ll", "all")),
           ((2, 2, 0, "ll", None), (4, 1, 1, "bulk", None)), ((4, 2, 0, "ll", None), (2, 1, 0, "ll", "conv")),
           ((8, 1, 1, "ll", None), (2, 2, 0, "bulk", None))]


@pytest.mark.parametrize("a,b", RESHARD, ids=["%s->%s" % (_tid(a), _tid(b)) for a, b in RESHARD])
def test_state_saved_at_one_topology_lands_on_the_owners_of_another(a, b):
    rng = np.random.default_rng(3)
    full = rng.standard_normal(LAYOUT.total).astype(np.float32)
    oa, ra = _topo(*a)
    saved = gather_tile_state(_ranks_holding(full, a[0], oa, ra, rng), oa, ra)
    ob, rb = _topo(*b)
    ranks = {r: np.zeros_like(full) for r in range(b[0])}
    scatter_tile_state(saved, ranks, ob, rb)
    for t in range(T):
        holders = [r for r in range(b[0]) if held_tiles(ob, rb, r)[t]]
        assert int(ob[t]) in holders
        for r in holders:
            assert np.array_equal(ranks[r][t * 1024:(t + 1) * 1024], full[t * 1024:(t + 1) * 1024]), (t, r)
    assert np.array_equal(gather_tile_state([ranks[r] for r in range(b[0])], ob, rb), full)


# ------------------------------------------------------------------------------------------------------------ file checks
def _engine(hfa=None, bsc=0.0, dgt=False, world=1, parties=1, lookahead=False, B=32):
    """A stand-in for the engine: the attributes ``_ckpt_read`` reads."""
    # one exchange of all keys (the one-rank step without channels): every key shares one optimizer step word
    fab = types.SimpleNamespace(tiles=T, FMT_BSC=2, FMT_F8=3, tile_step_words=lambda: np.array(["fsa"] * T, dtype=object))
    return types.SimpleNamespace(hfa=hfa, _bsc_threshold=bsc, _sched=None, _lr=0.01, lookahead=lookahead, B=B, fabric=fab, layout=LAYOUT,
                                 topo=types.SimpleNamespace(world=world, num_parties=parties), dgt=dgt,
                                 update="local" if hfa else "server", mode="dist_sync")


def _entries(eng, kind=1, world=None):
    """The entries of a checkpoint of ``eng`` (sync mode, server update unless HFA)."""
    world = eng.topo.world if world is None else world
    rng = np.random.default_rng(0)
    i32 = lambda *v: np.array(v, dtype=np.int32)
    fmts = np.zeros(T, dtype=np.uint8)
    if eng._bsc_threshold:
        fmts[LAYOUT.slots[4].offset // 1024: LAYOUT.slots[4].offset // 1024 + LAYOUT.slots[4].tiles] = 2
    d = {"meta:version": i32(CHECKPOINT_VERSION), "meta:opt_kind": i32(kind), "meta:update": i32(bool(eng.hfa)), "meta:mode": i32(0),
         "meta:hfa": i32(*(eng.hfa or (0, 0))), "meta:wire_formats": fmts, "meta:bsc_threshold": np.array([eng._bsc_threshold]),
         "meta:dgt": i32(eng.dgt), "meta:topology": i32(world, eng.topo.num_parties, 0), "meta:steps_done": np.array([7], dtype=np.int64),
         "meta:lr": np.array([0.01])}
    lead = (world,) if eng.hfa else ()
    for i, n in enumerate(CNN_PARAM_NAMES):
        sl = LAYOUT.slots[i]
        d[n] = rng.standard_normal(CNN_PARAM_SHAPES[i]).astype(np.float32)
        for p in ("master:", "s0:", "s1:"):
            d[p + n] = rng.standard_normal(lead + CNN_PARAM_SHAPES[i]).astype(np.float32)
        d["step:" + n] = np.full(world if eng.hfa else 1, 7, dtype=np.int32)
        if eng._bsc_threshold:
            d["bsc_u:" + n] = d["bsc_v:" + n] = np.zeros((world, sl.tiles * 1024), dtype=np.float32)
        if eng.dgt:
            d["dgt_contrib:" + n] = rng.random(sl.tiles).astype(np.float32)
            d["dgt_fmt:" + n] = fmts[sl.offset // 1024: sl.offset // 1024 + sl.tiles].copy()
    if eng.dgt:
        d["dgt:order"] = rng.permutation(T).astype(np.int32)
    return d


def _save(path, d):
    import torch
    mx.nd.save(str(path), {k: mx.nd.NDArray(torch.from_numpy(np.ascontiguousarray(v))) for k, v in d.items()})
    return str(path)


def _read(eng, path, own):
    """``_ckpt_read`` of the stand-in, whose own entries are ``own``: its meta block and the layout of the rest."""
    meta = {k: v for k, v in own.items() if k.startswith("meta:")}
    layout = {k: (v.shape, v.dtype) for k, v in own.items() if not k.startswith("batch:")}
    return HipsCNNTrainStep._ckpt_read(eng, path, meta, layout)


def test_valid_file_is_read(tmp_path):
    eng = _engine(dgt=True)
    own = _entries(eng)
    got = _read(eng, _save(tmp_path / "c.params", own), own)
    assert set(got) == set(own) and all(np.array_equal(got[k], own[k]) for k in own)


def _mutated(own, name, value):
    d = dict(own)
    if value is None:
        del d[name]
    else:
        d[name] = value
    return d


CASES = {
    "missing key": (lambda o: _mutated(o, "s1:4.weight", None), "s1:4.weight"),
    "missing live weight": (lambda o: _mutated(o, "6.bias", None), "6.bias"),
    "wrong shape": (lambda o: _mutated(o, "master:2.weight", o["master:2.weight"].reshape(32, 400)), "master:2.weight"),
    "wrong dtype": (lambda o: _mutated(o, "s0:0.bias", o["s0:0.bias"].astype(np.float64)), "s0:0.bias"),
    "wrong step dtype": (lambda o: _mutated(o, "step:5.weight", o["step:5.weight"].astype(np.int64)), "step:5.weight"),
    "unknown version": (lambda o: _mutated(o, "meta:version", np.array([CHECKPOINT_VERSION + 1], dtype=np.int32)), "meta:version"),
    "no version": (lambda o: _mutated(o, "meta:version", None), "meta:version"),
    "other optimizer": (lambda o: _mutated(o, "meta:opt_kind", np.array([0], dtype=np.int32)), "meta:opt_kind"),
    "other mode": (lambda o: _mutated(o, "meta:mode", np.array([1], dtype=np.int32)), "meta:mode"),
    "other wire formats": (lambda o: _mutated(o, "meta:wire_formats", np.ones(T, dtype=np.uint8)), "meta:wire_formats"),
    "DGT off": (lambda o: _mutated(o, "meta:dgt", np.array([0], dtype=np.int32)), "meta:dgt"),
    "order not a permutation": (lambda o: _mutated(o, "dgt:order", np.zeros(T, dtype=np.int32)), "dgt:order"),
    "format outside the base": (lambda o: _mutated(o, "dgt_fmt:4.weight", np.full_like(o["dgt_fmt:4.weight"], 2)), "dgt_fmt:4.weight"),
    "different counts in one exchange": (lambda o: _mutated(o, "step:6.bias", np.array([8], dtype=np.int32)), "step:6.bias"),
    "negative steps_done": (lambda o: _mutated(o, "meta:steps_done", np.array([-1], dtype=np.int64)), "meta:steps_done"),
}


@pytest.mark.parametrize("case", list(CASES))
def test_malformed_or_mismatched_file_is_refused(tmp_path, case):
    eng = _engine(dgt=True)
    own = _entries(eng)
    make, field = CASES[case]
    path = _save(tmp_path / "c.params", make(own))
    with pytest.raises(ValueError, match=field.replace(".", r"\.")):
        _read(eng, path, own)


@pytest.mark.parametrize("kind", ["hfa", "bsc"])
def test_worker_state_needs_the_same_ranks(tmp_path, kind):
    """HFA state belongs to each worker and Bi-Sparse residuals to each party owner: a file from 4 ranks does not load into 2."""
    eng = _engine(hfa=(2, 2) if kind == "hfa" else None, bsc=0.01 if kind == "bsc" else 0.0, world=2, parties=2)
    own = _entries(eng)
    assert _read(eng, _save(tmp_path / "ok.params", own), own)["meta:topology"].tolist() == [2, 2, 0]
    other = _entries(eng, world=4)
    # the per-rank rows no longer fit either; the topology is what the message names
    path = _save(tmp_path / "c.params", other)
    with pytest.raises(ValueError, match="meta:topology"):
        _read(eng, path, own)


def test_damaged_or_foreign_files_are_refused(tmp_path):
    eng = _engine()
    own = _entries(eng)
    good = open(_save(tmp_path / "c.params", own), "rb").read()
    for name, data in (("truncated", good[:len(good) // 2]), ("garbage", b"\x00" * 64), ("empty", b"")):
        p = tmp_path / name
        p.write_bytes(data)
        with pytest.raises(ValueError):
            _read(eng, str(p), own)
    import torch
    mx.nd.save(str(tmp_path / "list.params"), [mx.nd.NDArray(torch.zeros(3))])
    with pytest.raises(ValueError, match="unnamed"):
        _read(eng, str(tmp_path / "list.params"), own)


def test_primed_batches_are_taken_only_by_a_lookahead_engine_of_the_same_ranks_and_batch(tmp_path):
    """One primed batch per saving rank: a look-ahead engine with the same batch size, world size and parties takes them up (each rank
    its own row); any other engine warns that it does not train on them."""
    own = _entries(_engine(world=2, parties=1))
    d = dict(own, **{"batch:x": np.zeros((2, 32, 1, 28, 28), np.float32), "batch:label": np.zeros((2, 32), np.float32)})
    path = _save(tmp_path / "c.params", d)
    assert _read(_engine(lookahead=True, world=2), path, own)["batch:x"].shape == (2, 32, 1, 28, 28)
    for other in (dict(B=64), dict(world=4), dict(lookahead=False)):
        kw = dict(dict(lookahead=True, world=2), **other)
        eng = _engine(**kw)
        mine = _entries(eng)
        with pytest.warns(UserWarning, match="primed batches"):
            assert "batch:x" not in _read(eng, path, mine)
    bad = _save(tmp_path / "b.params", dict(d, **{"batch:label": np.zeros((2, 31), np.float32)}))
    with pytest.raises(ValueError, match="batch"):
        _read(_engine(lookahead=True, world=2), bad, own)
    one_row = _save(tmp_path / "r.params", dict(d, **{"batch:x": d["batch:x"][:1], "batch:label": d["batch:label"][:1]}))
    with pytest.raises(ValueError, match="batch"):
        _read(_engine(lookahead=True, world=2), one_row, own)
