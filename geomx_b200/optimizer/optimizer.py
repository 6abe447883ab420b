"""Optimizers and the ``Updater`` used by KVStore / Trainer.

Parity: ``python/mxnet/optimizer/optimizer.py`` — ``Optimizer`` base (registry, lr/wd
multipliers, ``rescale_grad``, ``clip_gradient``, ``multi_precision`` master weights,
``_index_update_count`` / ``num_update``), SGD :452, Signum, FTML, LBSGD(≈SGD w/ warmup), DCASGD :872,
NAG, SGLD, Adam :1017, AdaGrad, RMSProp, AdaDelta, Ftrl, Adamax, Nadam, Test, and ``Updater``
:1511 (``get_states`` / ``set_states`` pickle layout).

H100 design: every optimizer also exposes ``spec()`` — a *declarative* description
(name + hyper-parameters) that the native fused kernels (``csrc/kernels/optim.cu``) and the
native parameter-server (``csrc/hips/server_optim.h``) execute without Python; the dense
update of SGD / SGD-momentum / Adam / DCASGD on CUDA tensors goes through those kernels; NAG, Signum, RMSProp (not centered),
AdaGrad, AdaDelta and Ftrl have a spec too, which the training engine, the fabric KVStore and the Trainer's fused update run.
Arbitrary user optimizers still work everywhere through the Python ``update`` (on servers via
the host-callback path, like the reference's ``Executor`` hand-off).
"""
from __future__ import annotations

import math
import pickle

import numpy as np
import torch

from ..ndarray import NDArray

__all__ = ["Optimizer", "SGD", "Signum", "FTML", "LBSGD", "DCASGD", "NAG", "SGLD", "ccSGD", "Adam", "AdaGrad",
           "RMSProp", "AdaDelta", "Ftrl", "Adamax", "Nadam", "Test", "Updater", "get_updater", "create",
           "register"]


def _on_clip(c):
    """The clip the reference's RMSProp / Ftrl / Signum apply: they pass ``clip_gradient`` / ``clip_weights`` to the operator only when it
    is truthy, and the operator clips only when it is >= 0, so None, 0 and negative values all mean "off"."""
    return c if c and c >= 0 else None


def _t(x):
    """NDArray | Tensor -> raw tensor (detached view for in-place updates)."""
    t = x._t if isinstance(x, NDArray) else x
    return t.detach() if t.requires_grad else t


class Optimizer:
    opt_registry = {}

    @staticmethod
    def register(klass):
        Optimizer.opt_registry[klass.__name__.lower()] = klass
        return klass

    @staticmethod
    def create_optimizer(name, **kwargs):
        if isinstance(name, Optimizer):
            return name
        k = name.lower()
        if k not in Optimizer.opt_registry:
            raise ValueError("Cannot find optimizer %s" % name)
        return Optimizer.opt_registry[k](**kwargs)

    def __init__(self, rescale_grad=1.0, param_idx2name=None, wd=0.0, clip_gradient=None, learning_rate=0.01,
                 lr_scheduler=None, sym=None, begin_num_update=0, multi_precision=False, param_dict=None):
        self.rescale_grad = rescale_grad
        self.lr = learning_rate
        self.lr_scheduler = lr_scheduler
        if lr_scheduler is not None:
            self.lr_scheduler.base_lr = learning_rate
        self.wd = wd
        self.lr_mult, self.wd_mult = {}, {}
        self.begin_num_update = begin_num_update
        self.num_update = begin_num_update
        self._index_update_count = {}
        self.clip_gradient = clip_gradient
        self.multi_precision = multi_precision
        self.aggregate_num = 0
        self.idx2name = dict(param_idx2name or {})
        self.param_dict = param_dict if param_dict else {}
        self.set_lr_mult({}); self.set_wd_mult({})

    # -- declarative spec for native executors -------------------------------------------------
    native_name = None

    def spec(self):
        """dict(name=..., hyper-parameters...) if a native fused kernel implements this optimizer, else None."""
        return None

    def _base_spec(self, **kw):
        d = dict(name=self.native_name, lr=float(self.lr), wd=float(self.wd), rescale_grad=float(self.rescale_grad),
                 clip_gradient=float(self.clip_gradient) if self.clip_gradient is not None else -1.0,
                 multi_precision=bool(self.multi_precision))
        if self.lr_scheduler is not None:
            # the schedule as the device evaluates it.  A schedule the device cannot evaluate leaves the key out (spec() itself must not
            # raise: the KVStores and the Trainer call it for every optimizer); whoever needs the schedule on the device calls
            # lr_scheduler.device_spec() for the reason.  spec_is_static() still says False, so the KVStores keep scheduled optimizers in Python.
            try:
                d["lr_schedule"] = self.lr_scheduler.device_spec()
            except (ValueError, AttributeError):
                pass
        d.update(kw)
        return d

    # -- state ------------------------------------------------------------------------------
    def create_state(self, index, weight):
        return None

    def create_state_multi_precision(self, index, weight):
        w = _t(weight)
        if self.multi_precision and w.dtype in (torch.float16, torch.bfloat16):
            master = NDArray(w.float().clone())
            return (master, self.create_state(index, master))
        return self.create_state(index, weight)

    def update(self, index, weight, grad, state):
        raise NotImplementedError()

    def update_multi_precision(self, index, weight, grad, state):
        w = _t(weight)
        if self.multi_precision and w.dtype in (torch.float16, torch.bfloat16):
            master, st = state
            g32 = NDArray(_t(grad).float())
            self.update(index, master, g32, st)
            w.copy_(_t(master))
        else:
            self.update(index, weight, grad, state)

    # -- lr / wd ------------------------------------------------------------------------------
    def set_learning_rate(self, lr):
        if self.lr_scheduler is not None:
            raise UserWarning("LRScheduler of the optimizer has already been defined.")
        self.lr = lr

    @property
    def learning_rate(self):
        return self.lr_scheduler(self.num_update) if self.lr_scheduler is not None else self.lr

    def set_lr_scale(self, args_lrscale):
        """[DEPRECATED] use ``set_lr_mult``."""
        raise DeprecationWarning("set_lr_scale is deprecated, use set_lr_mult instead")

    def set_lr_mult(self, args_lr_mult):
        self.lr_mult = dict(args_lr_mult)

    def set_wd_mult(self, args_wd_mult):
        self.wd_mult = {}
        for n in self.idx2name.values():
            if not (n.endswith("_weight") or n.endswith("_gamma") or n.endswith(".weight") or n.endswith(".gamma")):
                self.wd_mult[n] = 0.0
        self.wd_mult.update(args_wd_mult)

    def _update_count(self, index):
        if not isinstance(index, (list, tuple)):
            index = [index]
        for idx in index:
            if idx not in self._index_update_count:
                self._index_update_count[idx] = self.begin_num_update
            self._index_update_count[idx] += 1
            self.num_update = max(self._index_update_count[idx], self.num_update)

    def _get_lr(self, index):
        lr = self.lr_scheduler(self.num_update) if self.lr_scheduler is not None else self.lr
        if index in self.param_dict:
            lr *= self.param_dict[index].lr_mult
        elif index in self.lr_mult:
            lr *= self.lr_mult[index]
        elif index in self.idx2name:
            lr *= self.lr_mult.get(self.idx2name[index], 1.0)
        return lr

    def _get_wd(self, index):
        wd = self.wd
        if index in self.param_dict:
            wd *= self.param_dict[index].wd_mult
        elif index in self.wd_mult:
            wd *= self.wd_mult[index]
        elif index in self.idx2name:
            wd *= self.wd_mult.get(self.idx2name[index], 1.0)
        return wd

    def _prep_grad(self, grad, weight=None, wd=0.0, wd_before_clip=False):
        """rescale -> clip -> + wd*w (sgd_update & friends), or rescale -> + wd*w -> clip when ``wd_before_clip`` (adam_update clips the
        regularised gradient: src/operator/optimizer_op-inl.h:840-873)."""
        g = _t(grad)
        if g.dtype != torch.float32 and weight is not None and _t(weight).dtype == torch.float32:
            g = g.float()
        g = g * self.rescale_grad
        if wd_before_clip and wd and weight is not None:
            g = g + wd * _t(weight)
        if self.clip_gradient is not None:
            g = g.clamp(-self.clip_gradient, self.clip_gradient)
        if not wd_before_clip and wd and weight is not None:
            g = g + wd * _t(weight)
        return g

    def spec_is_static(self):
        """True when ``spec()`` (scalar lr / wd) describes this optimizer completely: no lr_scheduler and no per-parameter lr / wd multiplier
        different from 1.  Servers only execute the native spec in that case; otherwise the pickled optimizer itself is shipped, as the
        reference always does (python/mxnet/kvstore.py:452-499), so the scheduler and the multipliers run server-side."""
        if self.lr_scheduler is not None:
            return False
        mults = list(self.lr_mult.values()) + [getattr(p, "lr_mult", 1.0) for p in self.param_dict.values()]
        if self.wd != 0.0:      # weight-decay multipliers (wd_mult = 0 on biases / gamma / beta) only matter when there is weight decay
            mults += list(self.wd_mult.values()) + [getattr(p, "wd_mult", 1.0) for p in self.param_dict.values()]
        return all(float(m) == 1.0 for m in mults)

    def __getstate__(self):
        d = self.__dict__.copy()
        d["param_dict"] = {}  # Parameters are not shipped to servers (reference does the same)
        return d

    def __setstate__(self, st):
        self.__dict__.update(st)


register = Optimizer.register
create = Optimizer.create_optimizer


@register
class SGD(Optimizer):
    native_name = "sgd"

    def __init__(self, momentum=0.0, lazy_update=True, **kwargs):
        super().__init__(**kwargs)
        self.momentum, self.lazy_update = momentum, lazy_update

    def spec(self):
        return self._base_spec(momentum=float(self.momentum))

    def create_state(self, index, weight):
        return NDArray(torch.zeros_like(_t(weight))) if self.momentum != 0.0 else None

    def update(self, index, weight, grad, state):
        self._update_count(index)
        lr, wd = self._get_lr(index), self._get_wd(index)
        w = _t(weight); g = self._prep_grad(grad, weight, wd)
        if state is not None:
            m = _t(state); m.mul_(self.momentum).sub_(g, alpha=lr); w.add_(m)
        else:
            w.sub_(g.to(w.dtype), alpha=lr)


@register
class ccSGD(SGD):
    pass


@register
class LBSGD(SGD):
    def __init__(self, momentum=0.0, multi_precision=False, warmup_strategy="linear", warmup_epochs=5,
                 batch_scale=1, updates_per_epoch=32, begin_epoch=0, num_epochs=60, **kwargs):
        super().__init__(momentum=momentum, multi_precision=multi_precision, **kwargs)
        self.warmup_strategy, self.warmup_epochs, self.batch_scale = warmup_strategy, warmup_epochs, batch_scale
        self.updates_per_epoch, self.init_updates, self.num_epochs = updates_per_epoch, begin_epoch * updates_per_epoch, num_epochs

    def spec(self):
        return None


@register
class Signum(Optimizer):
    """``optimizer.py:558-622``: with momentum, signum_update; without, signsgd_update ``w = (1 - lr*wd)*w - lr*sign(grad)`` (decoupled wd,
    no clip, no wd_lh)."""
    native_name = "signum"

    def __init__(self, learning_rate=0.01, momentum=0.9, wd_lh=0.0, **kwargs):
        super().__init__(learning_rate=learning_rate, **kwargs)
        self.momentum, self.wd_lh = momentum, wd_lh

    def spec(self):
        if self.momentum < 0:     # the reference runs signum_update with momentum 0 then: no native kind does that
            return None
        return self._base_spec(momentum=float(self.momentum), wd_lh=float(self.wd_lh))

    def create_state(self, index, weight):
        return NDArray(torch.zeros_like(_t(weight))) if self.momentum != 0.0 else None

    def update(self, index, weight, grad, state):
        self._update_count(index)
        lr, wd = self._get_lr(index), self._get_wd(index)
        w = _t(weight)
        if state is not None:
            # SignumKernel: mom = mu*mom - (1-mu)*wd*w - (1-mu)*clip(rescale*g); w = (1 - lr*wd_lh)*w + lr*sign(mom)
            mu, clip = (self.momentum if self.momentum > 0 else 0.0), _on_clip(self.clip_gradient)
            g = _t(grad).to(w.dtype) * self.rescale_grad
            if clip is not None:
                g = g.clamp(-clip, clip)
            m = _t(state); m.mul_(mu).sub_(g + wd * w, alpha=(1 - mu))
            w.mul_(1 - lr * self.wd_lh).add_(torch.sign(m), alpha=lr)
        else:
            w.mul_(1 - lr * wd).sub_(torch.sign(_t(grad)).to(w.dtype), alpha=lr)


@register
class FTML(Optimizer):
    def __init__(self, beta1=0.6, beta2=0.999, epsilon=1e-8, **kwargs):
        super().__init__(**kwargs); self.beta1, self.beta2, self.epsilon = beta1, beta2, epsilon

    def create_state(self, index, weight):
        z = lambda: NDArray(torch.zeros_like(_t(weight)))
        return (z(), z(), z())  # d, v, z

    def update(self, index, weight, grad, state):
        self._update_count(index)
        lr, wd = self._get_lr(index), self._get_wd(index); t = self._index_update_count[index]
        w = _t(weight); g = self._prep_grad(grad, weight, wd)
        d, v, z = map(_t, state)
        v.mul_(self.beta2).addcmul_(g, g, value=1 - self.beta2)
        d_t = (1 - self.beta1 ** t) / lr * (torch.sqrt(v / (1 - self.beta2 ** t)) + self.epsilon)
        sigma = d_t - self.beta1 * d
        z.mul_(self.beta1).add_(g, alpha=1 - self.beta1).sub_(sigma * w)
        d.copy_(d_t); w.copy_(-z / d_t)


@register
class DCASGD(Optimizer):
    """Delay-compensated ASGD (``optimizer.py:872-925``): one ``previous_weight`` per key."""
    native_name = "dcasgd"

    def __init__(self, momentum=0.0, lamda=0.04, **kwargs):
        super().__init__(**kwargs)
        self.momentum, self.weight_previous, self.lamda = momentum, {}, lamda

    def spec(self):
        return self._base_spec(momentum=float(self.momentum), lamda=float(self.lamda))

    def create_state(self, index, weight):
        w = _t(weight)
        mom = None if self.momentum == 0.0 else NDArray(torch.zeros_like(w))
        return (mom, NDArray(w.clone()))

    def update(self, index, weight, grad, state):
        self._update_count(index)
        lr, wd = self._get_lr(index), self._get_wd(index)
        w = _t(weight)
        g = _t(grad) * self.rescale_grad
        if self.clip_gradient is not None:
            g = g.clamp(-self.clip_gradient, self.clip_gradient)
        mom, prev = state
        prev = _t(prev)
        upd = g + wd * w + self.lamda * g * g * (w - prev)
        if mom is not None:
            m = _t(mom); m.mul_(self.momentum).sub_(upd, alpha=lr); step = m
        else:
            step = -lr * upd
        prev.copy_(w)
        w.add_(step)


@register
class NAG(Optimizer):
    """``optimizer.py:928-978``: rescale, clip, ``+ wd*w``; ``mom = mu*mom + g``, ``w -= lr*(g + mu*mom)``."""
    native_name = "nag"

    def __init__(self, momentum=0.0, **kwargs):
        super().__init__(**kwargs); self.momentum = momentum

    def spec(self):
        return self._base_spec(momentum=float(self.momentum))

    def create_state(self, index, weight):
        return NDArray(torch.zeros_like(_t(weight))) if self.momentum != 0.0 else None

    def update(self, index, weight, grad, state):
        self._update_count(index)
        lr, wd = self._get_lr(index), self._get_wd(index)
        w = _t(weight); g = self._prep_grad(grad, weight, wd)
        if state is not None:
            m = _t(state); m.mul_(self.momentum).add_(g)
            w.sub_(g + self.momentum * m, alpha=lr)
        else:
            w.sub_(g, alpha=lr)


@register
class SGLD(Optimizer):
    def update(self, index, weight, grad, state):
        self._update_count(index)
        lr, wd = self._get_lr(index), self._get_wd(index)
        w = _t(weight); g = self._prep_grad(grad, weight, wd)
        w.sub_(g, alpha=lr / 2).add_(torch.randn_like(w) * math.sqrt(lr))


@register
class Adam(Optimizer):
    """``optimizer.py:1017``: lr_t = lr*sqrt(1-b2^t)/(1-b1^t); w -= lr_t * m / (sqrt(v)+eps)."""
    native_name = "adam"

    def __init__(self, learning_rate=0.001, beta1=0.9, beta2=0.999, epsilon=1e-8, lazy_update=True, **kwargs):
        super().__init__(learning_rate=learning_rate, **kwargs)
        self.beta1, self.beta2, self.epsilon, self.lazy_update = beta1, beta2, epsilon, lazy_update

    def spec(self):
        return self._base_spec(beta1=float(self.beta1), beta2=float(self.beta2), epsilon=float(self.epsilon))

    def create_state(self, index, weight):
        w = _t(weight)
        return (NDArray(torch.zeros_like(w)), NDArray(torch.zeros_like(w)))

    def update(self, index, weight, grad, state):
        self._update_count(index)
        lr, wd = self._get_lr(index), self._get_wd(index)
        t = self._index_update_count[index]
        lr = lr * math.sqrt(1.0 - self.beta2 ** t) / (1.0 - self.beta1 ** t)
        w = _t(weight); m, v = map(_t, state)
        if w.is_cuda and w.dtype == torch.float32 and _t(grad).dtype == torch.float32:
            from ..ops import native
            if native.available():
                native.adam_update(w, _t(grad), m, v, lr, self.beta1, self.beta2, self.epsilon, wd,
                                   self.rescale_grad, -1.0 if self.clip_gradient is None else self.clip_gradient)
                return
        g = self._prep_grad(grad, weight, wd, wd_before_clip=True)
        m.mul_(self.beta1).add_(g, alpha=1 - self.beta1)
        v.mul_(self.beta2).addcmul_(g, g, value=1 - self.beta2)
        w.addcdiv_(m, v.sqrt().add_(self.epsilon), value=-lr)


@register
class AdaGrad(Optimizer):
    """``optimizer.py:1099-1155`` (dense): rescale, clip; ``history += g^2``; ``w += (g / sqrt(history + eps) + wd*w) * -lr``."""
    native_name = "adagrad"

    def __init__(self, eps=1e-7, **kwargs):
        super().__init__(**kwargs); self.float_stable_eps = eps

    def spec(self):
        return self._base_spec(epsilon=float(self.float_stable_eps))

    def create_state(self, index, weight):
        return NDArray(torch.zeros_like(_t(weight)))

    def update(self, index, weight, grad, state):
        self._update_count(index)
        lr, wd = self._get_lr(index), self._get_wd(index)
        w = _t(weight); g = self._prep_grad(grad); h = _t(state)
        h.addcmul_(g, g)
        w.sub_(lr * (g / torch.sqrt(h + self.float_stable_eps) + wd * w))


@register
class RMSProp(Optimizer):
    """``optimizer.py:1158-1233``, rmsprop_update / rmspropalex_update: ``g = rescale*g + wd*w``, then clip; ``eps`` inside the square
    root; ``clip_weights`` clamps the new weight.  Only the plain form (``centered=False``) has a native spec."""
    native_name = "rmsprop"

    def __init__(self, learning_rate=0.001, gamma1=0.9, gamma2=0.9, epsilon=1e-8, centered=False,
                 clip_weights=None, **kwargs):
        super().__init__(learning_rate=learning_rate, **kwargs)
        self.gamma1, self.gamma2, self.centered, self.epsilon, self.clip_weights = gamma1, gamma2, centered, epsilon, clip_weights

    def spec(self):
        if self.centered:
            return None
        cw = _on_clip(self.clip_weights)
        return self._base_spec(gamma1=float(self.gamma1), epsilon=float(self.epsilon), clip_weights=-1.0 if cw is None else float(cw))

    def create_state(self, index, weight):
        z = lambda: NDArray(torch.zeros_like(_t(weight)))
        return (z(), z(), z()) if self.centered else (z(),)

    def update(self, index, weight, grad, state):
        self._update_count(index)
        lr, wd = self._get_lr(index), self._get_wd(index)
        w = _t(weight)
        g = _t(grad).to(w.dtype) * self.rescale_grad + wd * w
        clip = _on_clip(self.clip_gradient)
        if clip is not None:
            g = g.clamp(-clip, clip)
        if not self.centered:
            n = _t(state[0]); n.mul_(self.gamma1).addcmul_(g, g, value=1 - self.gamma1)
            w.sub_(lr * g / torch.sqrt(n + self.epsilon))
        else:
            n, gm, delta = map(_t, state)
            n.mul_(self.gamma1).addcmul_(g, g, value=1 - self.gamma1)
            gm.mul_(self.gamma1).add_(g, alpha=1 - self.gamma1)
            delta.mul_(self.gamma2).sub_(lr * g / torch.sqrt(n - gm * gm + self.epsilon))
            w.add_(delta)
        cw = _on_clip(self.clip_weights)
        if cw is not None:
            w.clamp_(-cw, cw)


@register
class AdaDelta(Optimizer):
    """``optimizer.py:1236-1289``: no learning rate (nor its schedule or lr_mult); rescale, clip; wd outside: ``w -= delta + wd*w``."""
    native_name = "adadelta"

    def __init__(self, rho=0.90, epsilon=1e-5, **kwargs):
        super().__init__(**kwargs); self.rho, self.epsilon = rho, epsilon

    def spec(self):
        return self._base_spec(rho=float(self.rho), epsilon=float(self.epsilon))

    def create_state(self, index, weight):
        z = lambda: NDArray(torch.zeros_like(_t(weight)))
        return (z(), z())

    def update(self, index, weight, grad, state):
        self._update_count(index)
        wd = self._get_wd(index)
        w = _t(weight); g = self._prep_grad(grad)
        acc_g, acc_d = map(_t, state)
        acc_g.mul_(self.rho).addcmul_(g, g, value=1 - self.rho)
        cur = torch.sqrt(acc_d + self.epsilon) / torch.sqrt(acc_g + self.epsilon) * g
        acc_d.mul_(self.rho).addcmul_(cur, cur, value=1 - self.rho)
        w.sub_(cur + wd * w)


@register
class Ftrl(Optimizer):
    """``optimizer.py:1294-1366``, ftrl_update: the weight is recomputed from ``z`` and ``n`` on every update."""
    native_name = "ftrl"

    def __init__(self, lamda1=0.01, learning_rate=0.1, beta=1, **kwargs):
        super().__init__(learning_rate=learning_rate, **kwargs); self.lamda1, self.beta = lamda1, beta

    def spec(self):
        return self._base_spec(lamda1=float(self.lamda1), beta=float(self.beta))

    def create_state(self, index, weight):
        z = lambda: NDArray(torch.zeros_like(_t(weight)))
        return (z(), z())  # z, n

    def update(self, index, weight, grad, state):
        self._update_count(index)
        lr, wd = self._get_lr(index), self._get_wd(index)
        w = _t(weight)
        g = _t(grad).to(w.dtype) * self.rescale_grad
        clip = _on_clip(self.clip_gradient)
        if clip is not None:
            g = g.clamp(-clip, clip)
        z, n = map(_t, state)
        z.add_(g - (torch.sqrt(n + g * g) - torch.sqrt(n)) * w / lr)
        n.addcmul_(g, g)
        w.copy_((torch.sign(z) * self.lamda1 - z) / ((self.beta + torch.sqrt(n)) / lr + wd) * (z.abs() > self.lamda1))


@register
class Adamax(Optimizer):
    def __init__(self, learning_rate=0.002, beta1=0.9, beta2=0.999, **kwargs):
        super().__init__(learning_rate=learning_rate, **kwargs); self.beta1, self.beta2 = beta1, beta2

    def create_state(self, index, weight):
        z = lambda: NDArray(torch.zeros_like(_t(weight)))
        return (z(), z())

    def update(self, index, weight, grad, state):
        self._update_count(index)
        lr, wd = self._get_lr(index), self._get_wd(index); t = self._index_update_count[index]
        lr /= (1.0 - self.beta1 ** t)
        w = _t(weight); g = self._prep_grad(grad, weight, wd)
        m, u = map(_t, state)
        m.mul_(self.beta1).add_(g, alpha=1 - self.beta1)
        torch.maximum(u * self.beta2, g.abs(), out=u)
        w.sub_(lr * m / u)


@register
class Nadam(Optimizer):
    def __init__(self, learning_rate=0.001, beta1=0.9, beta2=0.999, epsilon=1e-8, schedule_decay=0.004, **kwargs):
        super().__init__(learning_rate=learning_rate, **kwargs)
        self.beta1, self.beta2, self.epsilon, self.schedule_decay, self.m_schedule = beta1, beta2, epsilon, schedule_decay, 1.0

    def create_state(self, index, weight):
        z = lambda: NDArray(torch.zeros_like(_t(weight)))
        return (z(), z())

    def update(self, index, weight, grad, state):
        self._update_count(index)
        lr, wd = self._get_lr(index), self._get_wd(index); t = self._index_update_count[index]
        w = _t(weight); g = self._prep_grad(grad, weight, wd)
        mom_t = self.beta1 * (1.0 - 0.5 * (0.96 ** (t * self.schedule_decay)))
        mom_t1 = self.beta1 * (1.0 - 0.5 * (0.96 ** ((t + 1) * self.schedule_decay)))
        self.m_schedule *= mom_t; m_sched_next = self.m_schedule * mom_t1
        m, v = map(_t, state)
        m.mul_(self.beta1).add_(g, alpha=1 - self.beta1)
        v.mul_(self.beta2).addcmul_(g, g, value=1 - self.beta2)
        g_p = g / (1.0 - self.m_schedule); m_p = m / (1.0 - m_sched_next); v_p = v / (1.0 - self.beta2 ** t)
        m_bar = (1.0 - mom_t) * g_p + mom_t1 * m_p
        w.sub_(lr * m_bar / (torch.sqrt(v_p) + self.epsilon))


@register
class Test(Optimizer):
    def create_state(self, index, weight):
        return NDArray(torch.zeros_like(_t(weight)))

    def update(self, index, weight, grad, state):
        w = _t(weight); w.add_(_t(grad) * self.rescale_grad); _t(state).copy_(w)


class Updater:
    """Stateful closure ``updater(index, grad, weight)`` (``optimizer.py:1511-1562``)."""

    def __init__(self, optimizer):
        self.optimizer = optimizer
        self.states, self.states_synced = {}, {}
        self.aggregate_updates = False

    def __call__(self, index, grad, weight):
        if not isinstance(index, (list, tuple)):
            index, grad, weight = [index], [grad], [weight]
        for i, g, w in zip(index, grad, weight):
            if i not in self.states:
                self.states[i] = self.optimizer.create_state_multi_precision(i, w)
                self.states_synced[i] = True
            elif not self.states_synced[i]:
                self.states[i] = self.sync_state_context(self.states[i], w.context if isinstance(w, NDArray) else None)
                self.states_synced[i] = True
            self.optimizer.update_multi_precision(i, w, g, self.states[i])

    def sync_state_context(self, state, context):
        if isinstance(state, NDArray):
            return state.as_in_context(context) if context is not None else state
        if isinstance(state, (tuple, list)):
            return type(state)(self.sync_state_context(s, context) for s in state)
        return state

    @staticmethod
    def _to_host(state):
        if isinstance(state, NDArray):
            return ("__nd__", state.asnumpy())
        if isinstance(state, (tuple, list)):
            return type(state)(Updater._to_host(s) for s in state)
        return state

    @staticmethod
    def _from_host(state):
        if isinstance(state, tuple) and len(state) == 2 and isinstance(state[0], str) and state[0] == "__nd__":
            return NDArray(torch.from_numpy(np.array(state[1])))
        if isinstance(state, (tuple, list)):
            return type(state)(Updater._from_host(s) for s in state)
        return state

    def set_states(self, states):
        states = pickle.loads(states)
        if isinstance(states, tuple) and len(states) == 2:
            self.states, self.optimizer = states
        else:
            self.states = states
        self.states = {k: Updater._from_host(v) for k, v in self.states.items()}
        self.states_synced = dict.fromkeys(self.states.keys(), False)

    def get_states(self, dump_optimizer=False):
        host = {k: Updater._to_host(v) for k, v in self.states.items()}
        return pickle.dumps((host, self.optimizer) if dump_optimizer else host)


def get_updater(optimizer):
    return Updater(optimizer)
