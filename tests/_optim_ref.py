"""fp64 reference of the element-wise optimizers beyond SGD / Adam / DCASGD that the update kernels run, and named mutations of them.

Written from the reference's definitions (``optimizer.py`` NAG / AdaGrad / AdaDelta, ``optimizer_op-inl.h`` SignumKernel / SignSGDKernel /
RMSPropUpdate / FtrlUpdate), not from the kernels; every state starts at 0:

* NAG       rescale, clip, ``g += wd*w``; ``mom = mu*mom + g``; ``w -= lr*(g + mu*mom)`` (no momentum: ``w -= lr*g``).
* Signum    ``mom = mu*mom - (1-mu)*(clip(rescale*g) + wd*w)``; ``w = (1 - lr*wd_lh)*w + lr*sign(mom)``.  Without momentum signsgd:
            ``w = (1 - lr*wd)*w - lr*sign(g)``.
* RMSProp   ``g = clip(rescale*g + wd*w)``; ``n = (1-gamma1)*g^2 + gamma1*n``; ``w = clip_w(w - lr*g/sqrt(n + eps))``.
* AdaGrad   rescale, clip; ``h += g^2``; ``w -= lr*(g/sqrt(h + eps) + wd*w)``.
* AdaDelta  rescale, clip; ``acc_g = rho*acc_g + (1-rho)*g^2``; ``d = sqrt(acc_d + eps)/sqrt(acc_g + eps)*g``;
            ``acc_d = rho*acc_d + (1-rho)*d^2``; ``w -= d + wd*w`` (no lr).
* Ftrl      rescale, clip; ``z += g - (sqrt(n + g^2) - sqrt(n))*w/lr``; ``n += g^2``;
            ``w = (sign(z)*lamda1 - z)/((beta + sqrt(n))/lr + wd)`` where ``|z| > lamda1``, else 0.

RMSProp, Signum and Ftrl treat ``clip_gradient = 0`` as "no clipping" (the reference passes the clip only when it is truthy).

The module extends ``_update_ref.py``: :func:`hyper`, :func:`update`, :func:`relevant_mutations` and :class:`UpdateRef` take every kind,
the kinds of ``_update_ref.py`` through its own functions; its tolerance and comparison helpers are re-exported.
"""
import numpy as np
import torch

import _update_ref as base
from _update_ref import DISP_TOL, cnn_like_grads, displacement_err, rel  # noqa: F401

# the kinds of this module, and those of them that treat clip_gradient = 0 as "off"
NEW_KINDS = ("nag", "signum", "rmsprop", "adagrad", "adadelta", "ftrl")
CLIP_ZERO_OFF = ("signum", "rmsprop", "ftrl")

KIND_MUTATIONS = {
    "rmsprop_clip_before_wd": "RMSProp clips the gradient before adding wd*w",
    "rmsprop_eps_outside": "RMSProp adds eps outside the square root",
    "nag_no_lookahead": "NAG steps by the gradient alone, without the look-ahead term mu*mom",
    "signum_wd_in_sign": "signsgd takes the sign of (rescale*g + wd*w) instead of decaying the weight by lr*wd",
    "adadelta_lr": "AdaDelta scales its step by the learning rate",
    "adagrad_wd_inside": "AdaGrad adds wd*w to the gradient before the history",
    "ftrl_no_mask": "Ftrl does not zero the weights where |z| <= lamda1",
    "slots_swapped": "each state slot is stored into the other one",
}


def hyper(spec, fp32=True):
    """``_update_ref.hyper`` plus the hyper-parameters of the kinds of :data:`NEW_KINDS` (clip 0 -> off for :data:`CLIP_ZERO_OFF`)."""
    if spec["name"] not in NEW_KINDS:
        return base.hyper(spec, fp32)
    f = (lambda x: float(np.float32(x))) if fp32 else float
    if spec["name"] in CLIP_ZERO_OFF and not spec.get("clip_gradient", -1.0):
        spec = dict(spec, clip_gradient=-1.0)
    h = base.hyper(spec, fp32)
    h.update(wd_lh=f(spec.get("wd_lh", 0.0)), clip_weights=f(spec.get("clip_weights", -1.0)), gamma1=f(spec.get("gamma1", 0.9)),
             rho=f(spec.get("rho", 0.9)), beta=f(spec.get("beta", 1.0)), lamda1=f(spec.get("lamda1", 0.01)))
    return h


def relevant_mutations(spec, push_scale=1.0, mults=None):
    """The mutations (of ``_update_ref.MUTATIONS`` and :data:`KIND_MUTATIONS`) that change the result of ``spec``."""
    if spec["name"] not in NEW_KINDS:
        return base.relevant_mutations(spec, push_scale, mults)
    h = hyper(spec)
    k, mu = h["kind"], h["momentum"]
    out = ["grad_not_cleared"]
    if push_scale != 1.0 and not (k == "signum" and mu == 0.0):      # signsgd: sign(g) does not see the scale
        out.append("no_push_scale")
    if mults is not None and any(tuple(m) != (1.0, 1.0) for m in mults):
        out.append("mults_ignored")
    if k in ("nag", "signum") and mu != 0.0:
        out.append("momentum_lost")
    if k == "nag" and mu != 0.0:
        out.append("nag_no_lookahead")
    if k == "signum" and mu == 0.0 and h["wd"]:
        out.append("signum_wd_in_sign")
    if k == "rmsprop":
        out.append("rmsprop_eps_outside")
        if h["wd"] and h["clip"] >= 0:
            out.append("rmsprop_clip_before_wd")
    if k == "adagrad" and h["wd"]:
        out.append("adagrad_wd_inside")
    if k == "adadelta":
        out.append("adadelta_lr")
    if k == "ftrl":
        out += ["ftrl_no_mask", "slots_swapped"]
    return out


def update(h, w, g, s0, s1, t, lr_mult=1.0, wd_mult=1.0, mutation=None):
    """One update of fp64 tensors, in place (``_update_ref.update`` for its kinds).  Signum returns a mask of the elements whose new
    momentum lies within fp32 rounding of zero, where an fp32 kernel may take the other sign; every other kind returns None."""
    if h["kind"] not in NEW_KINDS:
        return base.update(h, w, g, s0, s1, t, lr_mult, wd_mult, mutation)
    lr, wd = h["lr"] * lr_mult, h["wd"] * wd_mult
    clip = h["clip"]
    cl = (lambda x: x.clamp(-clip, clip)) if clip >= 0 else (lambda x: x)
    amb = _update_new(h, w, g, s0, s1, lr, wd, cl, mutation)
    if mutation == "slots_swapped":
        s0_new = s0.clone()
        s0.copy_(s1)
        s1.copy_(s0_new)
    return amb


def _update_new(h, w, g, s0, s1, lr, wd, cl, mutation):
    kind, mu = h["kind"], h["momentum"]
    if kind == "nag":
        g = cl(g * h["rescale"]) + wd * w
        if mu != 0.0:
            if mutation == "momentum_lost":
                s0.zero_()
            s0.mul_(mu).add_(g)
            w.sub_(lr * (g if mutation == "nag_no_lookahead" else g + mu * s0))
        else:
            w.sub_(lr * g)
    elif kind == "signum":
        if mu != 0.0:
            if mutation == "momentum_lost":
                s0.zero_()
            term = cl(g * h["rescale"]) + wd * w
            bound = 16 * 2.0 ** -24 * (mu * s0.abs() + (1.0 - mu) * (cl(g * h["rescale"]).abs() + (wd * w).abs()))
            s0.mul_(mu).sub_((1.0 - mu) * term)
            w.mul_(1.0 - lr * h["wd_lh"]).add_(lr * torch.sign(s0))
            return s0.abs() < bound
        if mutation == "signum_wd_in_sign":
            w.sub_(lr * torch.sign(g * h["rescale"] + wd * w))
        else:
            w.mul_(1.0 - lr * wd).sub_(lr * torch.sign(g))
    elif kind == "rmsprop":
        g = g * h["rescale"]
        g = cl(g) + wd * w if mutation == "rmsprop_clip_before_wd" else cl(g + wd * w)
        s0.mul_(h["gamma1"]).add_((1.0 - h["gamma1"]) * g * g)
        den = s0.sqrt() + h["eps"] if mutation == "rmsprop_eps_outside" else (s0 + h["eps"]).sqrt()
        w.sub_(lr * g / den)
        if h["clip_weights"] >= 0:
            w.clamp_(-h["clip_weights"], h["clip_weights"])
    elif kind == "adagrad":
        g = cl(g * h["rescale"])
        if mutation == "adagrad_wd_inside":
            g = g + wd * w
            s0.add_(g * g)
            w.sub_(lr * g / (s0 + h["eps"]).sqrt())
        else:
            s0.add_(g * g)
            w.sub_(lr * (g / (s0 + h["eps"]).sqrt() + wd * w))
    elif kind == "adadelta":
        g = cl(g * h["rescale"])
        rho, eps = h["rho"], h["eps"]
        s0.mul_(rho).add_((1.0 - rho) * g * g)
        d = (s1 + eps).sqrt() / (s0 + eps).sqrt() * g
        s1.mul_(rho).add_((1.0 - rho) * d * d)
        w.sub_((lr * d if mutation == "adadelta_lr" else d) + wd * w)
    elif kind == "ftrl":
        g = cl(g * h["rescale"])
        s0.add_(g - ((s1 + g * g).sqrt() - s1.sqrt()) * w / lr)
        s1.add_(g * g)
        new = (torch.sign(s0) * h["lamda1"] - s0) / ((h["beta"] + s1.sqrt()) / lr + wd)
        w.copy_(new if mutation == "ftrl_no_mask" else torch.where(s0.abs() > h["lamda1"], new, torch.zeros_like(new)))
    else:
        raise ValueError(kind)
    return None


class UpdateRef(base.UpdateRef):
    """``_update_ref.UpdateRef`` for every kind.  ``sign_ambiguous[i]``: the elements of key i where Signum's sign was within rounding
    in some round (see :func:`update`)."""

    def __init__(self, spec, weights, mutation=None, **kw):
        assert mutation is None or mutation in base.MUTATIONS or mutation in KIND_MUTATIONS, mutation
        super().__init__(spec, weights, mutation=None if mutation in KIND_MUTATIONS else mutation, **kw)
        self.mutation = mutation
        self.h = None if spec is None else hyper(spec)
        self.sign_ambiguous = [torch.zeros(w.shape, dtype=torch.bool) for w in self.w]

    def step(self, grads, active=None, bsc_select=None):
        """One round, as ``_update_ref.UpdateRef.step`` (wire rounding, Bi-Sparse stage, multipliers) with this module's update."""
        if self.h is None or self.h["kind"] not in NEW_KINDS:
            return super().step(grads, active, bsc_select)
        keys = range(len(self.w)) if active is None else active
        for i in keys:
            g = torch.as_tensor(grads[i]).detach().cpu()
            if self.mutation == "grad_not_cleared":
                self._acc[i] += g.double()
                g = self._acc[i].float()
            fmt = self.fmts[i]
            if isinstance(fmt, str) and fmt != "bsc" and not self.pull_half[i]:
                if self.round_after_scale:
                    g = base.wire(g.float() * np.float32(self.push_scale), fmt).double()
                else:
                    g = base.wire(g, fmt).double() * self.push_scale
                self.agg[i].zero_()
                self.agg[i][:g.numel()] = g.reshape(-1)
            else:
                self.agg[i] = self._aggregate(i, g, bsc_select)
                g = self.agg[i][:self.w[i].numel()]
            self.t[i] += 1
            lm, wm = self.mults[i]
            amb = update(self.h, self.w[i], g.reshape(self.w[i].shape), self.s0[i], self.s1[i], self.t[i], lm, wm, self.mutation)
            if amb is not None:
                self.sign_ambiguous[i] |= amb
