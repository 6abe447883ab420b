"""The training step's kernel path as a pure function (``step_path`` in geomx_b200/models/cnn.py) of the batch size, the engine's arguments
and the step switches: paths A-G of ``tests/test_step_paths_gpu.py`` at each of its cases, look-ahead, every batch-size regime, the
exchange variants at one and at several ranks.  Every check compares the whole record, so a field that changes unasked fails too."""
import pytest

from geomx_b200.models.cnn import STEP_SWITCHES, StepPath, step_path

from _cnn_ref import CASE_IDS, CASES

# path -> the fields that set it apart; the rest are those of one rank with default switches (see classic())
PATHS = {
    "A": dict(direct_conv=True, dense="dz3", wgrad="comm", bwd="one_grid"),
    "B": dict(direct_conv=True, dense="dz3", wgrad="comm", bwd="two_launch"),
    "C": dict(direct_conv=True, dense="dz3", wgrad="comm", bwd="exchange_tail"),
    "D": dict(direct_conv=True, dense="gemm", wgrad=None, bwd="one_grid"),
    "E": dict(direct_conv=False, dense="a2", wgrad="comm", bwd="gemm"),
    "F": dict(direct_conv=False, dense="a2", wgrad="comm", bwd="gemm", pool_fusion=False),
    "G": dict(direct_conv=False, dense="gemm", wgrad=None, bwd="gemm"),
}


def classic(path, **fields):
    """The record of ``path`` on one rank (overlapped channels, the conv keys' exchange last), with ``fields`` overriding it."""
    rec = dict(PATHS[path])
    rec.update(pool_fusion=rec.get("pool_fusion", True), exchange="conv", local_tail=False, overlap=True, single=None,
               n_fwd=1 if rec["direct_conv"] else 2, lookahead=False,
               lookahead_join="join_comm" if rec["dense"] in ("a3", "dz3") else "join", direct_input=True)
    rec.update(fields)
    return StepPath(**rec)


@pytest.mark.parametrize("path,B,env", CASES, ids=CASE_IDS)
def test_paths_a_to_g(path, B, env):
    assert step_path(B, conv_tail_capable=True, env=env) == classic(path)


def test_switches_at_their_defaults():
    """Every step switch set to its default value chooses what an unset one does (one rank)."""
    defaults = {"GEOMX_STEP_OVERLAP": "1", "GEOMX_STEP_EXCHANGE": "ll", "GEOMX_FUSED_MLP": "1", "GEOMX_DIRECT_CONV": "1",
                "GEOMX_CNN_BWD_ONE_LAUNCH": "1", "GEOMX_NO_POOL_FUSION": "0", "GEOMX_FUSED_EXCHANGE": "0", "GEOMX_E2E_DIRECT_INPUT": "1"}
    assert set(defaults) == set(STEP_SWITCHES)
    for B in (1, 32, 48, 96):
        assert step_path(B, conv_tail_capable=True, env=defaults) == step_path(B, conv_tail_capable=True)


def test_lookahead_b32_takes_the_tail_from_a3():
    """The look-ahead launch ends with the next batch's forward kernel: the forward kernel stops at a3 (no head), the dense weight
    gradients stay on the side stream, the launch joins the comm stream before the next forward kernel (it reads W0), one input graph."""
    want = classic("A", dense="a3", wgrad="side", lookahead=True, direct_input=False)
    assert step_path(32, lookahead=True, conv_tail_capable=True) == want
    assert step_path(32, lookahead=True, conv_tail_capable=True, env={"GEOMX_FUSED_EXCHANGE": "1"}) == want._replace(bwd="exchange_tail")
    # where the forward kernel does not compute dense0, the side branch is all the next forward launches wait for
    assert step_path(31, lookahead=True) == classic("E", wgrad="side", lookahead=True, direct_input=False)
    assert step_path(48, lookahead=True) == classic("D", lookahead=True, direct_input=False)
    assert step_path(33, lookahead=True) == classic("G", lookahead=True, direct_input=False)


@pytest.mark.parametrize("B", range(34, 65, 2))
def test_even_batches_above_32_take_path_d(B):
    assert step_path(B, conv_tail_capable=True) == classic("D")


@pytest.mark.parametrize("B", range(1, 64, 2))
def test_odd_batches_take_the_gemm_convolutions(B):
    assert step_path(B, conv_tail_capable=True) == classic("E" if B <= 31 else "G")


@pytest.mark.parametrize("B", [33, 65, 66, 96, 128, 256])
def test_b33_and_above_64_take_path_g(B):
    assert step_path(B, conv_tail_capable=True) == classic("G")
    assert step_path(B, conv_tail_capable=True, env={"GEOMX_FUSED_EXCHANGE": "1"}) == classic("G")


def test_dist_async():
    """No channels: the one-sided exchange after the backward pass, the dense weight gradients on the side stream, no look-ahead."""
    want = classic("A", exchange="async", overlap=False, wgrad="side")
    assert step_path(32, mode="dist_async", conv_tail_capable=True) == want
    assert step_path(32, mode="dist_async", lookahead=True, conv_tail_capable=True) == want
    assert step_path(32, mode="dist_async", conv_tail_capable=True, env={"GEOMX_FUSED_EXCHANGE": "1"}) == want


def test_update_local():
    assert step_path(32, update="local", conv_tail_capable=True) == classic("A", local_tail=True)
    assert step_path(96, update="local") == classic("G", local_tail=True)


@pytest.mark.parametrize("world", [1, 4])
def test_hfa(world):
    """HFA: no exchange inside the step, the local optimizer on the worker's own gradients, no look-ahead, whatever the switches say."""
    want = classic("A", exchange="local_opt", overlap=False, wgrad="side")
    for env in ({}, {"GEOMX_STEP_OVERLAP": "1", "GEOMX_STEP_EXCHANGE": "sharded", "GEOMX_FUSED_EXCHANGE": "1"}):
        assert step_path(32, update="local", hfa=True, lookahead=True, world=world, direct_protocol=True, conv_tail_capable=True,
                         env=env) == want
    assert step_path(33, update="local", hfa=True) == classic("G", exchange="local_opt", overlap=False)


@pytest.mark.parametrize("exchange", ["ll", "sharded", "replicated"])
def test_no_overlap_at_one_rank(exchange):
    """GEOMX_STEP_OVERLAP=0 on one rank: the fused exchange of all keys (the single channel needs several ranks)."""
    env = {"GEOMX_STEP_OVERLAP": "0", "GEOMX_STEP_EXCHANGE": exchange}
    want = classic("A", exchange="fsa", overlap=False, wgrad="side")
    assert step_path(32, direct_protocol=True, conv_tail_capable=True, env=env) == want
    assert step_path(32, direct_protocol=True, conv_tail_capable=True, env=dict(env, GEOMX_FUSED_EXCHANGE="1")) == want


@pytest.mark.parametrize("exchange", ["ll", "sharded", "replicated"])
def test_no_overlap_at_several_ranks(exchange):
    """Several ranks default to one exchange after the backward pass; `sharded` / `replicated` run it as the single direct-protocol
    channel of all keys, which needs the direct-protocol buffers."""
    single = exchange != "ll"
    want = classic("A", exchange="all" if single else "fsa", overlap=False, single="all" if single else None, wgrad="side")
    for env in ({"GEOMX_STEP_EXCHANGE": exchange}, {"GEOMX_STEP_OVERLAP": "0", "GEOMX_STEP_EXCHANGE": exchange}):
        assert step_path(32, world=4, direct_protocol=True, env=env) == want
        assert step_path(32, world=4, direct_protocol=False, env=env) == want._replace(exchange="fsa", single=None)


def test_overlap_at_several_ranks_needs_the_direct_protocol():
    env = {"GEOMX_STEP_OVERLAP": "1"}
    assert step_path(32, world=4, direct_protocol=True, conv_tail_capable=True, env=env) == classic("A")
    assert step_path(32, world=4, direct_protocol=False, env=env) == classic("A", exchange="fsa", overlap=False, wgrad="side")


def test_fused_exchange_needs_a_capable_channel():
    """GEOMX_FUSED_EXCHANGE=1 asks for the conv keys' exchange in the backward grid's tail; a channel that cannot run there (Bi-Sparse
    tiles, DGT, no direct-protocol buffers) keeps its own launch, and so do the paths without the one-grid backward."""
    env = {"GEOMX_FUSED_EXCHANGE": "1"}
    assert step_path(32, conv_tail_capable=False, env=env) == classic("A")
    assert step_path(32, update="local", conv_tail_capable=False, env=env) == classic("A", local_tail=True)
    assert step_path(32, conv_tail_capable=True, env=dict(env, GEOMX_CNN_BWD_ONE_LAUNCH="0")) == classic("B")
    assert step_path(32, conv_tail_capable=True, env=dict(env, GEOMX_DIRECT_CONV="0")) == classic("E")
