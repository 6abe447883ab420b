"""Learning-rate schedules (``mx.lr_scheduler``).

Same classes, constructor arguments and values as the reference's ``python/mxnet/lr_scheduler.py`` (Factor / MultiFactor / Poly / Cosine with an
optional linear or constant warm-up), but every schedule here is a **pure function** ``lr = f(num_update)`` of the update count and the
scheduler's ``base_lr``: nothing is accumulated between calls, so a schedule can be evaluated for any step in any order (the server-side
optimizer, a resumed run and a plotting script all get the same value), and ``base_lr`` always means "the learning rate before decay".
"""
from __future__ import annotations

import bisect
import math

__all__ = ["LRScheduler", "FactorScheduler", "MultiFactorScheduler", "PolyScheduler", "CosineScheduler"]


class LRScheduler:
    """Base: handles the warm-up phase, subclasses implement :meth:`decayed` for the steps after it.

    ``warmup_mode``: ``'linear'`` ramps from ``warmup_begin_lr`` to ``base_lr`` over ``warmup_steps`` updates, ``'constant'`` holds
    ``warmup_begin_lr``."""

    def __init__(self, base_lr=0.01, warmup_steps=0, warmup_begin_lr=0, warmup_mode="linear"):
        if warmup_mode not in ("linear", "constant"):
            raise ValueError("warmup_mode must be 'linear' or 'constant', got %r" % (warmup_mode,))
        if warmup_steps < 0 or warmup_begin_lr > base_lr:
            raise ValueError("warm-up must start at or below base_lr and last a non-negative number of steps")
        self.base_lr = base_lr
        self.warmup_steps = int(warmup_steps)
        self.warmup_begin_lr = warmup_begin_lr
        self.warmup_mode = warmup_mode

    @property
    def warmup_final_lr(self):
        return self.base_lr

    def get_warmup_lr(self, num_update):
        if self.warmup_mode == "constant" or self.warmup_steps == 0:
            return self.warmup_begin_lr
        frac = min(max(float(num_update) / self.warmup_steps, 0.0), 1.0)
        return self.warmup_begin_lr + frac * (self.base_lr - self.warmup_begin_lr)

    def decayed(self, num_update):
        """Learning rate at ``num_update >= warmup_steps``."""
        raise NotImplementedError

    def __call__(self, num_update):
        return self.get_warmup_lr(num_update) if num_update < self.warmup_steps else self.decayed(num_update)

    def device_spec(self):
        """The schedule as a plain dict of fixed fields, for optimizers that evaluate it on the device from their step counter
        (``sched_lr`` in ``csrc/kernels/optim.cuh``): ``kind`` ('factor', 'multifactor', 'poly' or 'cosine'), the warm-up fields and the
        fields of that kind.  ``base_lr`` is not part of it: the optimizer passes it to the kernels as their ``lr``.

        Raises ``ValueError`` for a scheduler whose values cannot be derived from these fields: a class other than the four above, a
        subclass that overrides ``__call__`` / ``get_warmup_lr`` / ``decayed`` / ``shape`` / ``max_steps``, or a ``MultiFactorScheduler``
        with more than :data:`DEVICE_MAX_MILESTONES` milestones (the size of the device struct's table)."""
        name = type(self).__name__
        base = next((c for c in type(self).__mro__ if c in _DEVICE_KINDS), None)
        if base is None:
            raise ValueError("%s cannot run on the device: only Factor / MultiFactor / Poly / Cosine schedules can" % name)
        for attr in ("__call__", "get_warmup_lr", "decayed", "shape", "max_steps"):
            if getattr(type(self), attr, None) is not getattr(base, attr, None):
                raise ValueError("%s overrides %s: its values are no longer those of %s, so it cannot run on the device"
                                 % (name, attr, base.__name__))
        d = dict(kind=_DEVICE_KINDS[base], warmup_steps=int(self.warmup_steps), warmup_begin_lr=float(self.warmup_begin_lr),
                 warmup_mode=self.warmup_mode, step=0, factor=1.0, stop_factor_lr=0.0, milestones=[], max_update=0, final_lr=0.0, pwr=1.0)
        if base is FactorScheduler:
            d.update(step=int(self.step), factor=float(self.factor), stop_factor_lr=float(self.stop_factor_lr))
        elif base is MultiFactorScheduler:
            if len(self.step) > DEVICE_MAX_MILESTONES:
                raise ValueError("%s has %d milestones; the device schedule holds at most %d" % (name, len(self.step), DEVICE_MAX_MILESTONES))
            d.update(milestones=[int(s) for s in self.step], factor=float(self.factor))
        else:
            d.update(max_update=int(self.max_update), final_lr=float(self.final_lr))
            if base is PolyScheduler:
                d.update(pwr=float(self.power))
        return d


class FactorScheduler(LRScheduler):
    """``base_lr * factor**k`` with one more factor every ``step`` updates (``k = (num_update - 1) // step``), never below ``stop_factor_lr``."""

    def __init__(self, step, factor=1, stop_factor_lr=1e-8, base_lr=0.01, **kw):
        super().__init__(base_lr, **kw)
        if step < 1:
            raise ValueError("step must be at least 1 update")
        if factor > 1.0:
            raise ValueError("factor must not exceed 1: the schedule only decays")
        self.step, self.factor, self.stop_factor_lr = int(step), factor, stop_factor_lr

    def decayed(self, num_update):
        k = max(0, (int(num_update) - 1) // self.step)
        return max(self.base_lr * self.factor ** k, self.stop_factor_lr) if k else self.base_lr


class MultiFactorScheduler(LRScheduler):
    """One more ``factor`` after each milestone in ``step`` (a strictly increasing list) has been passed."""

    def __init__(self, step, factor=1, base_lr=0.01, **kw):
        super().__init__(base_lr, **kw)
        milestones = [int(s) for s in step]
        if not milestones or milestones[0] < 1 or any(b <= a for a, b in zip(milestones, milestones[1:])):
            raise ValueError("step must be an increasing list of positive update counts")
        if factor > 1.0:
            raise ValueError("factor must not exceed 1: the schedule only decays")
        self.step, self.factor = milestones, factor

    def decayed(self, num_update):
        passed = bisect.bisect_left(self.step, int(num_update))      # milestones strictly below num_update
        return self.base_lr * self.factor ** passed


class _Annealing(LRScheduler):
    """Shared shape of Poly / Cosine: anneal from ``base_lr`` to ``final_lr`` between the end of warm-up and ``max_update``."""

    def __init__(self, max_update, base_lr=0.01, final_lr=0, **kw):
        super().__init__(base_lr, **kw)
        if max_update < 1 or max_update <= self.warmup_steps:
            raise ValueError("max_update must be positive and larger than warmup_steps")
        self.max_update, self.final_lr = int(max_update), final_lr

    @property
    def max_steps(self):
        return self.max_update - self.warmup_steps

    def shape(self, progress):
        """Remaining fraction of (base_lr - final_lr) at ``progress`` in [0, 1]."""
        raise NotImplementedError

    def decayed(self, num_update):
        progress = min(float(num_update - self.warmup_steps) / self.max_steps, 1.0)
        return self.final_lr + (self.base_lr - self.final_lr) * self.shape(progress)


class PolyScheduler(_Annealing):
    """``final_lr + (base_lr - final_lr) * (1 - progress) ** pwr``."""

    def __init__(self, max_update, base_lr=0.01, pwr=2, final_lr=0, **kw):
        super().__init__(max_update, base_lr, final_lr, **kw)
        self.power = pwr

    def shape(self, progress):
        return (1.0 - progress) ** self.power


class CosineScheduler(_Annealing):
    """Half a cosine period from ``base_lr`` down to ``final_lr``."""

    def shape(self, progress):
        return 0.5 * (1.0 + math.cos(math.pi * progress))


# LRScheduler.device_spec: the classes the device evaluates, and the milestone table of its struct (LrSchedule::milestones)
DEVICE_MAX_MILESTONES = 16
_DEVICE_KINDS = {FactorScheduler: "factor", MultiFactorScheduler: "multifactor", PolyScheduler: "poly", CosineScheduler: "cosine"}
