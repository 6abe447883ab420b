"""Spec tests for the wire/identity protocol and codecs (SURVEY §7.2-1): Cantor cmd pairing, node-id arithmetic, key sharding, 2-bit bit
layout, Bi-Sparse contract, DGT channel function + 4-bit codec, TSEngine epsilon-greedy pick, half conversion, HFA algebra, meta codec."""
import math

import numpy as np
import pytest
import torch

from geomx_b200 import runtime
from geomx_b200.kvstore import compression as gc
from geomx_b200.parallel.arena import ArenaLayout, TILE

needs_c = pytest.mark.skipif(not runtime.available(), reason="native runtime not built")


@needs_c
def test_cantor_command_pairing():
    C = runtime.C()
    # reference kvstore_dist_server.h:82-104 -> default/f32=0, default/f64=2, 2bit/f32=3, default/f16=5, BSC/f32=6 (the valid_heads)
    assert [C.get_command_type(0, 0), C.get_command_type(0, 1), C.get_command_type(2, 0), C.get_command_type(0, 2), C.get_command_type(3, 0)] == [0, 2, 3, 5, 6]
    for req in range(4):
        for dt in (0, 1, 2, 3, 4, 5, 6, 12):
            assert C.depair_command_type(C.get_command_type(req, dt)) == (req, dt)


@needs_c
def test_node_id_arithmetic():
    C = runtime.C()
    assert [C.server_rank_to_id(r, 0) for r in range(3)] == [100, 102, 104]       # local plane: servers even >= 100
    assert [C.worker_rank_to_id(r, 0) for r in range(3)] == [101, 103, 105]       # workers odd > 100
    assert [C.server_rank_to_id(r, 1) for r in range(2)] == [8, 10]               # global plane: < 100
    assert [C.worker_rank_to_id(r, 1) for r in range(2)] == [9, 11]
    for plane in (0, 1):
        for r in range(5):
            assert C.id_to_rank(C.server_rank_to_id(r, plane), plane) == r and C.id_to_rank(C.worker_rank_to_id(r, plane), plane) == r


@needs_c
def test_meta_codec_roundtrip():
    C = runtime.C()
    out = C.pack_unpack_meta(5, "hello", -3, 7, True)
    assert out[:10] == (5, "hello", -3, 7, 3, 7, 9, 101, True, True)
    assert out[10] == [0.5, 2.0] and out[11] == 2 and out[12] == "10.0.0.1" and out[13] == 2
    assert C.pack_unpack_meta(1, "", 0, 0, False)[11] == 0


def test_key_sharding_rules():
    # small keys hashed (key*9973) % n, big keys partitioned per tile across all global servers (kvstore_dist_server.h:1770-1810)
    lay = ArenaLayout.build([(0, (400,)), (1, (16,)), (2, (5000,)), (3, (2, 3))])
    assert lay.total % TILE == 0 and [s.tiles for s in lay.slots] == [1, 1, 5, 1]
    own = lay.global_owner_index(num_gs=3, bigarray_bound=2000)
    assert own[0] == (0 * 9973) % 3 and own[1] == (1 * 9973) % 3 and own[7] == (3 * 9973) % 3
    assert list(own[2:7]) == [0, 1, 2, 0, 1]
    assert list(lay.tile_key()) == [0, 1, 2, 2, 2, 2, 2, 3]


def test_fabric_global_tile_ownership():
    """Who plays global server for a tile on the fabric: sharded over ALL ranks by default (balanced; the owner is the tile's party owner
    inside its own party), whole keys per rank for the flag protocol, the reference's hashing / partitioning when DMLC_NUM_GLOBAL_SERVER is given."""
    import numpy as np
    from geomx_b200.models.cnn import CNN_PARAM_SHAPES
    from geomx_b200.parallel.fabric import Topology, global_tile_owners
    lay = ArenaLayout.build(list(enumerate(CNN_PARAM_SHAPES)))
    T = lay.total // TILE
    for world, parties in ((8, 2), (8, 4), (4, 2), (2, 2), (2, 1), (1, 1)):
        topo = Topology(world, 0, parties, 0)
        assert topo.tile_sharded and topo.num_gs == world and sorted(topo.gs_ranks) == list(range(world))
        own = global_tile_owners(topo, lay, "ll")
        cnt = np.bincount(own, minlength=world)
        assert own.shape == (T,) and cnt.max() - cnt.min() <= 1                       # balanced to within one tile
        assert ((own % topo.party_size) == (np.arange(T) % topo.party_size)).all()    # global owner = the tile's party owner in its own party
        bulk = global_tile_owners(topo, lay, "bulk")
        for sl in lay.slots:                                                           # one owner per key
            assert len(set(bulk[sl.offset // TILE: sl.offset // TILE + sl.tiles].tolist())) == 1
        assert np.bincount(bulk, minlength=world).max() == max(s.tiles for s in lay.slots) or world == 1
    topo = Topology(8, 3, 2, 2)                                                        # two explicit global servers: ranks 0 and 4 (one per party)
    assert not topo.tile_sharded and topo.gs_ranks == [0, 4]
    own = global_tile_owners(topo, lay, "ll", bigarray_bound=1000000)
    assert set(own.tolist()) <= {0, 4}
    assert [int(own[s.offset // TILE]) for s in lay.slots] == [topo.gs_ranks[(i * 9973) % 2] for i in range(len(lay.slots))]


def test_2bit_bit_layout_and_residual():
    # posbits {0xc0,0x30,0x0c,0x03}: value j of a 16-value word lives in byte j>>2, bit pair 6-2*(j&3); 11=+thr 10=-thr 00=0
    g = torch.zeros(16); g[0] = 1.0; g[1] = -1.0; g[5] = 0.7; g[15] = -0.2
    r = torch.zeros(16)
    q = gc.quantize_2bit(g, r, 0.5)
    b = q.view(torch.uint8).tolist()
    assert b[0] == 0xC0 | 0x20 and b[1] == 0x30 and b[2] == 0 and b[3] == 0
    assert r[0] == pytest.approx(0.5) and r[1] == pytest.approx(-0.5) and r[5] == pytest.approx(0.2) and r[15] == pytest.approx(-0.2)
    d = gc.dequantize_2bit(q, 16, 0.5)
    assert d.tolist()[:2] == [0.5, -0.5] and d[5] == 0.5 and d[15] == 0
    assert gc.compressed_size_2bit(17) == 2 and gc.compressed_size_2bit(16) == 1


def test_compress_reference_self_check():
    """tests/_compress_ref.py, the GPU codec tests' reference: its 2-bit packer gives the bytes above, its e4m3 table is torch's for every
    finite code, its rounding is torch's (nearest, ties to even) on values between the codes, and its fp32 FMA rounds once."""
    import _compress_ref as CR
    g = np.zeros(16, np.float32); g[0] = 1.0; g[1] = -1.0; g[5] = 0.7; g[15] = -0.2
    words, r = CR.quantize_2bit(g, np.zeros(16, np.float32), 0.5)
    assert words.view(np.uint8).tolist()[:4] == [0xC0 | 0x20, 0x30, 0, 0]
    assert r.tolist() == np.array([0.5, -0.5, 0, 0, 0, np.float32(0.7) - np.float32(0.5)] + [0] * 9 + [-0.2], np.float32).tolist()
    assert CR.dequantize_2bit(words, 16, 0.5).tolist() == [0.5, -0.5, 0, 0, 0, 0.5] + [0.0] * 10
    for n in (1, 17, 1000):
        x = (torch.randn(n) * 0.6).numpy()
        rt = torch.zeros(n)
        q = gc.quantize_2bit(torch.from_numpy(x), rt, 0.1)
        w, rr = CR.quantize_2bit(x, np.zeros(n, np.float32), 0.1)
        assert np.array_equal(q.view(torch.int32).numpy().view(np.uint32), w) and np.array_equal(rt.numpy(), rr)
    table = CR.e4m3_table()
    codes = torch.arange(256, dtype=torch.uint8)
    finite = (codes & 0x7F) != 0x7F
    assert np.array_equal(table[finite.numpy()], codes[finite].view(torch.float8_e4m3fn).double().numpy())
    assert np.isnan(table[~finite.numpy()]).all()
    mags = table[:127]
    mids = ((mags[:-1] + mags[1:]) / 2).astype(np.float32)            # exact ties between neighbouring codes
    x = np.concatenate([mids, -mids, np.nextafter(mids, 0), np.nextafter(mids, 1000), np.float32([0, -0.0, 448, 460, 1e-9, 2.0 ** -10, 3 * 2.0 ** -11]),
                        (np.random.RandomState(0).randn(5000) * 50).astype(np.float32)]).astype(np.float32)
    assert np.array_equal(CR.to_e4m3(x), torch.from_numpy(x).to(torch.float8_e4m3fn).view(torch.uint8).numpy())
    assert CR.to_e4m3(np.float32([1e6, -1e6])).tolist() == [0x7E, 0xFE]     # saturates (torch's cast gives NaN there)
    a, b, c = np.float32([1 + 2.0 ** -23]), np.float32([1 - 2.0 ** -23]), np.float32([-1.0])
    assert CR.fma32(a, b, c)[0] == np.float32(-2.0 ** -46)                # one rounding; two roundings would give 0


@needs_c
def test_2bit_native_matches_python():
    C = runtime.C()
    comp = C.GradientCompression(); comp.set_params("2bit", 0.5)
    g = (torch.randn(1000) * 0.6)
    r1, r2 = torch.zeros(1000), np.zeros(1000, dtype=np.float32)
    q1 = gc.quantize_2bit(g, r1, 0.5)
    q2 = comp.quantize_2bit(g.numpy(), r2)
    assert np.array_equal(q1.view(torch.int32).numpy().view(np.uint32), q2) and np.allclose(r1.numpy(), r2)
    assert np.array_equal(comp.dequantize_2bit(q2, 1000), gc.dequantize_2bit(q1, 1000, 0.5).numpy())
    comp2 = C.GradientCompression(); comp2.decode_params(comp.encode_params())
    assert comp2.encode_params() == comp.encode_params()


def test_bsc_contract():
    torch.manual_seed(0)
    n, thr = 20000, 0.01
    k, sample, k_sample = gc.bsc_sizes(n, thr)
    assert k == 200 and sample == 1000 and k_sample == 10      # n*0.005*thr < 10 -> sample = 10/thr
    g = torch.randn(n); u = torch.zeros(n); v = torch.zeros(n)
    z = gc.bsc_compress(g, u, v, thr)
    assert z.numel() == 2 * k
    vals, idx = z[:k], z[k:]
    sent = idx >= 0
    assert int(sent.sum()) <= k
    ii = idx[sent].long()
    assert torch.all(ii[1:] > ii[:-1])                          # index order, first-k-above-boundary (not exact top-k)
    assert torch.all(u[ii] == 0) and torch.all(v[ii] == 0)      # error feedback reset exactly at sent indices
    assert torch.all(vals[~sent] == gc.BSC_PAD_VAL) and torch.all(idx[~sent] == gc.BSC_PAD_IDX)
    boundary = vals[sent].abs().min()
    unsent = torch.ones(n, dtype=torch.bool); unsent[ii] = False
    if int(sent.sum()) < k:                                     # everything above the boundary was sent
        assert torch.all(v[unsent].abs() < boundary + 1e-6)
    dense = gc.bsc_decompress(z, n)
    assert torch.allclose(dense[ii], vals[sent]) and int((dense != 0).sum()) == int(sent.sum())
    # pull side: capacity k * parties, non-zeros in index order
    z2 = gc.bsc_pull_compress(dense, thr, 2)
    assert z2.numel() == 2 * int(n * thr * 2) and torch.allclose(gc.bsc_decompress(z2, n), dense)


def test_bsc_sizes_and_refusals():
    """A threshold above 1 takes the smallest sampled |v| as the boundary (k_sample clamped to the sample, as the reference's heap does); more
    than 2^24 elements, whose indices float32 cannot hold, is refused; state the codec updates in place must be contiguous."""
    from geomx_b200.base import MXNetError
    assert gc.bsc_sizes(1000, 2.0) == (2000, 5, 5)
    g = torch.tensor([3.0, -1.0, 0.5, 2.0, -0.25]); u = torch.zeros(5); v = torch.zeros(5)
    z = gc.bsc_compress(g, u, v, 2.0)                    # sample 5, k_sample 5 -> boundary = smallest |v| = 0.25: everything is sent
    assert z[:5].tolist() == g.tolist() and z[5:10].tolist() == [-65530.0] * 5
    assert z[10:15].tolist() == [0, 1, 2, 3, 4] and z[15:].tolist() == [-1.0] * 5
    big = torch.zeros(1)
    big_n = (1 << 24) + 1
    with pytest.raises(MXNetError, match="2\\^24"):
        gc.bsc_compress(big.expand(big_n), big.expand(big_n), big.expand(big_n), 0.01)
    with pytest.raises(MXNetError, match="2\\^24"):
        gc.bsc_pull_compress(big.expand(big_n), 0.01, 1)
    g = torch.randn(64)
    st = torch.zeros(64, 2)[:, 0]
    for call in (lambda: gc.quantize_2bit(g, st, 0.5), lambda: gc.bsc_compress(g, st, torch.zeros(64), 0.5),
                 lambda: gc.bsc_compress(g, torch.zeros(64), st, 0.5), lambda: gc.fp8_block_quantize(g, st),
                 lambda: gc.dequantize_2bit(gc.quantize_2bit(g, torch.zeros(64), 0.5), 64, 0.5, out=st),
                 lambda: gc.bsc_decompress(torch.zeros(4), 64, out=st), lambda: gc.fp8_block_dequantize(*gc.fp8_block_quantize(g), 64, out=st)):
        with pytest.raises(MXNetError, match="contiguous"):
            call()
    assert torch.count_nonzero(st) == 0
    r16, r32 = torch.zeros(64), torch.zeros(64)            # an fp16 gradient is cast, as the CUDA path does
    assert torch.equal(gc.quantize_2bit(g.half(), r16, 0.5), gc.quantize_2bit(g.half().float(), r32, 0.5)) and torch.equal(r16, r32)


@needs_c
def test_bsc_native_matches_python():
    C = runtime.C()
    comp = C.GradientCompression(); comp.set_params("bsc", 0.01)
    torch.manual_seed(1)
    n = 20000
    g = torch.randn(n)
    u1, v1 = torch.zeros(n), torch.zeros(n)
    u2, v2 = np.zeros(n, np.float32), np.zeros(n, np.float32)
    for _ in range(2):
        z1 = gc.bsc_compress(g, u1, v1, 0.01)
        z2 = comp.bsc_compress(g.numpy(), u2, v2)
        assert np.allclose(z1.numpy(), z2) and np.allclose(v1.numpy(), v2)
    dense = C.GradientCompression.bsc_decompress(z2, n)
    assert np.allclose(dense, gc.bsc_decompress(z1, n).numpy())
    assert np.allclose(comp.bsc_pull_compress(dense, 2), gc.bsc_pull_compress(torch.from_numpy(dense), 0.01, 2).numpy())


@needs_c
def test_dgt_channels_and_4bit_codec():
    C = runtime.C()
    # top K fraction on the reliable channel 0, the rest spread over channels 1..C in rank order
    ch = [C.dgt_get_channel(r, 10, 0.5, 3) for r in range(10)]
    assert ch[:5] == [0] * 5 and ch[5:] == sorted(ch[5:]) and set(ch[5:]) <= {1, 2, 3} and max(ch) == 3
    assert [C.dgt_get_channel(r, 4, 1.0, 3) for r in range(4)] == [0, 0, 0, 0]
    x = np.linspace(-1, 2, 64).astype(np.float32)
    blob, mn, mx = C.dgt_encode4(x)
    assert len(blob) == 32 and mn == pytest.approx(-1) and mx == pytest.approx(2)
    y = C.dgt_decode4(blob, 64, mn, mx)
    assert np.max(np.abs(x - y)) <= (mx - mn) / 15 / 2 + 1e-6


@needs_c
def test_tsengine_epsilon_greedy():
    C = runtime.C()
    # all idle receivers known + greed cap 1.0 -> always the highest recorded throughput
    picks = set(C.ts_pick_receiver(101, [103, 105, 107], {103: 10, 105: 99, 107: 50}, 1.0, 20))
    assert picks == {105}
    # nothing known -> uniformly random among idle nodes
    picks = set(C.ts_pick_receiver(101, [103, 105, 107], {}, 0.9, 200))
    assert picks == {103, 105, 107}
    assert C.ts_pick_receiver(101, [], {}, 0.9) == [-1]


@needs_c
def test_half_conversion():
    C = runtime.C()
    for f in (0.0, 1.0, -2.5, 65504.0, 1e-5, 3.14159, -0.333):
        h, b, bits = C.half_roundtrip(f)
        assert h == pytest.approx(float(torch.tensor(f).half().float()), abs=0) and b == pytest.approx(float(torch.tensor(f).bfloat16().float()), abs=0)
        assert bits == int(torch.tensor(f).half().view(torch.int16)) & 0xFFFF


def test_hfa_algebra():
    # local server: stored=(party_avg - milestone)/P pushed; global sums deltas; on pull stored = milestone + sum; milestone = stored
    P, w0 = 2, 1.0
    party_avg = [3.0, 7.0]
    deltas = [(a - w0) / P for a in party_avg]
    new = w0 + sum(deltas)
    assert new == pytest.approx(w0 + (sum(party_avg) / P - w0))       # = global average of party averages


def test_fp8_block_codec_cpu():
    x = torch.randn(300) * 5
    res = torch.zeros(300)
    q, s = gc.fp8_block_quantize(x, res)
    assert q.numel() == 384 and s.numel() == 3
    y = gc.fp8_block_dequantize(q, s, 300)
    assert torch.allclose(y + res, x, atol=1e-5) and float((y - x).abs().max()) < 0.07 * float(x.abs().max())


def test_topology_solver_and_tree_comm():
    """gpu_topology.h: Kernighan-Lin bisection keeps strongly linked devices together; the reduction tree is a spanning binary-depth tree
    whose first-round edges are the heavy links; CommDeviceTree reduces/broadcasts exactly (CPU tensors stand in for devices)."""
    import numpy as np
    import torch
    import geomx_b200 as mx
    from geomx_b200 import runtime
    from geomx_b200.kvstore import comm_tree
    if not runtime.available():
        pytest.skip("native runtime not built")
    n = 8
    W = np.ones((n, n), dtype=np.float32); np.fill_diagonal(W, 0)
    for a, b in ((0, 1), (2, 3), (4, 5), (6, 7)):                # NVLink pairs
        W[a, b] = W[b, a] = 10
    for a, b in ((0, 2), (1, 3), (4, 6), (5, 7)):                # quads
        W[a, b] = W[b, a] = 4
    A, B = runtime.C().topology_bisect(W.reshape(-1).tolist(), n, list(range(n)), 0)
    assert sorted(A) == [0, 1, 2, 3] and sorted(B) == [4, 5, 6, 7]
    parent, rnd, depth = comm_tree.compute_tree(W.tolist(), 0)
    assert depth == 3 and parent[0] == -1 and sum(p == -1 for p in parent) == 1
    for d in range(n):                                            # spanning: every device reaches the root
        seen, x = set(), d
        while parent[x] != -1:
            assert x not in seen; seen.add(x); x = parent[x]
        assert x == 0
    first = sorted((d, parent[d]) for d in range(n) if rnd[d] == 0)
    assert all(W[d, p] == 10 for d, p in first) and len(first) == 4      # round 0 uses the four NVLink pairs
    # exact reduce / broadcast
    comm = comm_tree.CommDeviceTree()
    vals = [mx.nd.array(np.full((5, 3), float(i + 1), dtype=np.float32)) for i in range(n)]
    comm._devices = None
    import os
    os.environ["GEOMX_LINK_MATRIX"] = ";".join(",".join(str(x) for x in row) for row in W.tolist())
    try:
        comm.init(3, vals[0])
        out = comm.reduce(3, vals)
        assert torch.equal(out, torch.full((5, 3), float(sum(range(1, n + 1)))))
        comm.array_bound = 4                                      # force the sliced (reduce-scatter) path
        out = comm.reduce(3, vals)
        assert torch.equal(out, torch.full((5, 3), float(sum(range(1, n + 1)))))
        outs = [mx.nd.zeros((5, 3)) for _ in range(n)]
        comm.broadcast(3, out, outs)
        assert all(torch.equal(o._t, out) for o in outs)
    finally:
        os.environ.pop("GEOMX_LINK_MATRIX", None)


def test_tsengine_node_helpers():
    """ts_node.h: payload merges in fp32 / fp16 / bf16, origin-list codec, dtype recovered from the Cantor-paired data command."""
    import numpy as np
    from geomx_b200 import runtime
    if not runtime.available():
        pytest.skip("native runtime not built")
    C = runtime.C()
    a = np.arange(8, dtype=np.float32); b = np.ones(8, dtype=np.float32) * 0.5
    C.ts_merge_bytes(a, b, 0)
    assert np.array_equal(a, np.arange(8, dtype=np.float32) + 0.5)
    h = np.array([1.0, 2.5, -3.0, 1000.0], dtype=np.float16); g = np.array([0.5, 0.25, 3.0, 24.0], dtype=np.float16)
    C.ts_merge_bytes(h, g, 2)
    assert np.array_equal(h, (np.array([1.0, 2.5, -3.0, 1000.0], dtype=np.float32) + np.array([0.5, 0.25, 3.0, 24.0], dtype=np.float32)).astype(np.float16))
    import torch
    x = torch.tensor([1.0, 3.0, -2.0, 100.0], dtype=torch.bfloat16); y = torch.tensor([0.5, 1.0, 2.0, 1.0], dtype=torch.bfloat16)
    xv = x.view(torch.int16).numpy(); C.ts_merge_bytes(xv, y.view(torch.int16).numpy(), 12)
    assert torch.equal(torch.from_numpy(xv).view(torch.bfloat16), (torch.tensor([1.0, 3.0, -2.0, 100.0]) + torch.tensor([0.5, 1.0, 2.0, 1.0])).to(torch.bfloat16))
    origins = [(101, 7, 0), (103, 12, 0), (9, 3, 1)]
    assert C.ts_origins_roundtrip(origins) == origins and C.ts_origins_roundtrip([]) == []
    # Cantor pairing (request type, dtype): default/f32 = 0, default/f64 = 2, 2bit/f32 = 3, default/f16 = 5, BSC/f32 = 6
    assert [C.ts_dtype_of_cmd(c) for c in (0, 2, 3, 5, 6)] == [0, 1, 0, 2, 0]


def test_dgt_adaptive_k():
    """ADAPTIVE_K_FLAG / DMLC_K_MIN (parsed but unused by the reference): K as a share of the contribution mass, python (fabric) and native
    (TCP plane) implementations agree."""
    import torch
    from geomx_b200 import runtime
    from geomx_b200.parallel.fabric import dgt_num_important
    c = [10.0, 5.0, 2.0, 1.0, 1.0, 1.0, 0.0, 0.0, 0.0, 0.0]
    t = torch.tensor(c)
    cases = [((0.5, False, 0.2), 5), ((0.5, True, 0.1), 1), ((0.8, True, 0.1), 3), ((0.8, True, 0.5), 5), ((1.0, True, 0.1), 6)]
    for (k, ad, kmin), want in cases:
        assert dgt_num_important(t, k, ad, kmin) == want
        if runtime.available():
            frac = runtime.C().dgt_effective_k(c, k, ad, kmin)
            assert (round(frac * len(c)) == want) if ad else (frac == pytest.approx(k))
    assert dgt_num_important(torch.zeros(10), 0.8, True, 0.2) == 2
    if runtime.available():
        C = runtime.C()
        # with the effective fraction, ranks below the prefix go to the reliable channel, the rest to the low-priority ones
        frac = C.dgt_effective_k(c, 0.8, True, 0.1)
        assert [C.dgt_get_channel(r, 10, frac, 3) for r in range(4)] == [0, 0, 0, 1]
