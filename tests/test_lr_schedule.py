"""Learning-rate schedules on the device, host side: ``LRScheduler.device_spec()`` (the one description of a schedule that the update kernels
evaluate), what ``Optimizer.spec()`` carries, the ctypes packing and the engine's per-key multipliers.  That the update kernels evaluating
the schedule compile without spills is a row of ``test_kernel_budgets.py``; the device values are checked in ``test_lr_schedule_gpu.py``."""
import ctypes

import pytest

import geomx_b200 as mx
from geomx_b200 import lr_scheduler as S
from geomx_b200.models.cnn import _key_mults
from geomx_b200.ops import _native_api as api

BASE = dict(warmup_steps=0, warmup_begin_lr=0.0, warmup_mode="linear", step=0, factor=1.0, stop_factor_lr=0.0, milestones=[], max_update=0,
            final_lr=0.0, pwr=1.0)


@pytest.mark.parametrize("mode", ["linear", "constant"])
def test_device_spec_fields(mode):
    wu = dict(warmup_steps=7, warmup_begin_lr=0.001, warmup_mode=mode)
    cases = [
        (S.FactorScheduler(step=30, factor=0.5, stop_factor_lr=1e-4, base_lr=0.1, **wu),
         dict(kind="factor", step=30, factor=0.5, stop_factor_lr=1e-4)),
        (S.MultiFactorScheduler(step=[10, 40, 90], factor=0.3, base_lr=0.1, **wu), dict(kind="multifactor", milestones=[10, 40, 90], factor=0.3)),
        (S.PolyScheduler(max_update=300, base_lr=0.1, pwr=1.5, final_lr=0.002, **wu), dict(kind="poly", max_update=300, final_lr=0.002, pwr=1.5)),
        (S.CosineScheduler(max_update=400, base_lr=0.1, final_lr=0.001, **wu), dict(kind="cosine", max_update=400, final_lr=0.001)),
    ]
    for sched, fields in cases:
        assert sched.device_spec() == dict(BASE, **wu, **fields), type(sched).__name__


def test_device_spec_accepts_plain_subclass():
    class MyCosine(S.CosineScheduler):
        pass
    assert MyCosine(max_update=10).device_spec()["kind"] == "cosine"


def test_device_spec_refusals():
    class Step(S.LRScheduler):
        def decayed(self, num_update):
            return self.base_lr
    class Wobbly(S.FactorScheduler):
        def decayed(self, num_update):
            return super().decayed(num_update) * 1.01
    class Shaped(S.CosineScheduler):
        def shape(self, progress):
            return 1.0 - progress
    with pytest.raises(ValueError, match="Step"):
        Step().device_spec()
    with pytest.raises(ValueError, match="Wobbly.*decayed"):
        Wobbly(step=10).device_spec()
    with pytest.raises(ValueError, match="Shaped.*shape"):
        Shaped(max_update=10).device_spec()
    class Stretched(S.PolyScheduler):
        @property
        def max_steps(self):
            return 2 * self.max_update
    with pytest.raises(ValueError, match="Stretched.*max_steps"):
        Stretched(max_update=10).device_spec()
    S.MultiFactorScheduler(step=list(range(1, 17))).device_spec()
    with pytest.raises(ValueError, match="MultiFactorScheduler.*17 milestones"):
        S.MultiFactorScheduler(step=list(range(1, 18))).device_spec()


def test_spec_carries_schedule_only_with_scheduler():
    plain = mx.optimizer.Adam(learning_rate=0.01)
    assert "lr_schedule" not in plain.spec() and plain.spec_is_static()
    sched = S.CosineScheduler(max_update=100, warmup_steps=5)
    opt = mx.optimizer.SGD(learning_rate=0.1, momentum=0.9, lr_scheduler=sched)
    assert opt.spec()["lr_schedule"] == sched.device_spec()
    assert opt.spec()["lr"] == 0.1 and not opt.spec_is_static()

    class Custom(S.LRScheduler):
        def decayed(self, num_update):
            return self.base_lr
    # spec() itself never raises: the KVStores and the Trainer call it for every optimizer and keep their Python path for this one
    custom = mx.optimizer.Adam(learning_rate=0.01, lr_scheduler=Custom())
    assert "lr_schedule" not in custom.spec() and not custom.spec_is_static()


def test_pack_schedule():
    assert api.pack_schedule(None).kind == 0
    d = S.MultiFactorScheduler(step=[3, 8], factor=0.25, base_lr=0.2, warmup_steps=2, warmup_begin_lr=0.05, warmup_mode="constant").device_spec()
    s = api.pack_schedule(d)
    assert (s.kind, s.warmup_steps, s.warmup_linear, s.num_milestones, list(s.milestones[:3])) == (2, 2, 0, 2, [3, 8, 0])
    assert s.factor == pytest.approx(0.25) and s.warmup_begin_lr == pytest.approx(0.05)
    c = api.pack_schedule(S.PolyScheduler(max_update=50, pwr=3, final_lr=0.01).device_spec())
    assert (c.kind, c.max_update, c.pwr, c.warmup_linear) == (3, 50, 3.0, 1)
    # LrSchedule is the last member of the fabric's OptHyper mirror
    from geomx_b200.parallel.fabric import _OptHyperF
    assert _OptHyperF._fields_[-1] == ("sched", api.LrSchedule)
    assert ctypes.sizeof(api.LrSchedule) == 4 * (11 + api.SCHED_MAX_MILESTONES)


def test_engine_key_mults():
    opt = mx.optimizer.SGD(learning_rate=0.1, wd=0.01, param_idx2name={i: "w%d_%s" % (i, "weight" if i % 2 == 0 else "bias") for i in range(10)})
    opt.set_lr_mult({0: 0.5, "w2_weight": 2.0})
    m = _key_mults(opt, None)
    assert m[0] == (0.5, 1.0) and m[2] == (2.0, 1.0)
    assert all(m[i] == (1.0, 0.0) for i in range(1, 10, 2))      # set_wd_mult: no weight decay on the biases
    net = mx.models.build_cnn()
    params = list(net.collect_params().values())
    params[0].lr_mult = 0.5
    for p in params[1::2]:
        p.wd_mult = 0.0
    m = _key_mults(opt, net)                                     # the net's Parameters win, as gluon.Trainer's param_dict does
    assert m[0] == (0.5, 1.0) and m[2] == (1.0, 1.0)
    assert all(m[i] == (1.0, 0.0) for i in range(1, 10, 2))
