"""fp64 reference of the optimizer updates that the exchange and optimizer kernels apply, and named mutations of it.

Written from the reference's definitions (``src/operator/optimizer_op-inl.h`` sgd / adam updates, ``optimizer.py`` DCASGD), not from the
kernels:

* SGD     rescale, clip, ``+ wd*w``; momentum stored as ``mom = mu*mom - lr*g``, ``w += mom``.
* Adam    rescale, ``+ wd*w``, clip (adam_update clips the regularised gradient); ``lr_t = lr*sqrt(1-b2^t)/(1-b1^t)``.
* DCASGD  rescale, clip, ``upd = g + wd*w + lamda*g^2*(w - prev)``; optional momentum; ``prev`` starts as the initial weight.

``lr`` / ``wd`` carry the key's ``lr_mult`` / ``wd_mult``.  The gradient a kernel's optimizer sees is the pushed sum times ``push_scale``
(the script-level ``grad / num_samples``), rounded to the key's wire format on the way.  ``UpdateRef`` keeps one step count per key, as the
reference's ``_index_update_count`` does.

A mutation (``UpdateRef(..., mutation=name)``) computes what a plausible bug in a kernel would produce; the tests use them to show that their
tolerances can tell each bug from the correct update.
"""
import math

import numpy as np
import torch

F64 = torch.float64
INV448 = float(np.float32(1.0 / 448.0))        # the kernels' fp32 constant 1.f / 448.f

MUTATIONS = {
    "t_frozen": "Adam's bias-correction step count stays at 1",
    "t_double": "the step count advances twice per update",
    "no_push_scale": "the push scale (1 / batch) is not applied",
    "adam_clip_before_wd": "Adam clips the gradient before adding wd*w",
    "sgd_wd_before_clip": "SGD adds wd*w before clipping",
    "momentum_lost": "the momentum is not persisted between updates",
    "dcasgd_prev_zero": "DCASGD's previous weight starts at 0",
    "mults_ignored": "per-key lr / wd multipliers are ignored",
    "grad_not_cleared": "the gradient arena is not cleared between steps",
}

# Norm-relative tolerance of a key's displacement P_k - P_0 (fp32 arenas, fp32 kernels) in the GPU tests, after the fp32 rounding of each
# weight store is discounted (displacement_err).  What it rests on: on an H100 the engine cases measure 1-3e-6, the fabric cases up to 3e-6;
# before that discount keys with a near-zero displacement reached 1.1-1.8e-5.  2e-5 leaves headroom above fp32 rounding and stays >1000x
# below the smallest mutation.
DISP_TOL = 2e-5

# The optimizer settings of the GPU tests' engine cases (and of the mutation check on CPU): clip cuts part of the CNN's mean gradients,
# weight decay and momentum are active, DCASGD's lamda is large enough that its delay term matters.
CASE_SPECS = {
    "adam": dict(name="adam", lr=0.01, wd=0.05, rescale_grad=1.0, clip_gradient=0.01, beta1=0.9, beta2=0.999, epsilon=1e-8),
    "sgd": dict(name="sgd", lr=0.1, wd=0.01, rescale_grad=2.0, clip_gradient=0.01, momentum=0.9),
    "dcasgd": dict(name="dcasgd", lr=0.1, wd=0.01, rescale_grad=1.0, clip_gradient=-1.0, momentum=0.9, lamda=40.0),
}


def relevant_mutations(spec, push_scale=1.0, mults=None):
    """The mutations that change the result of ``spec`` with this push scale and these multipliers."""
    h = hyper(spec)
    out = ["grad_not_cleared"]
    if push_scale != 1.0:
        out.append("no_push_scale")
    if mults is not None and any(tuple(m) != (1.0, 1.0) for m in mults):
        out.append("mults_ignored")
    if h["kind"] == "adam":
        out += ["t_frozen", "t_double"]
        if h["wd"] and h["clip"] >= 0:
            out.append("adam_clip_before_wd")
    if h["kind"] == "sgd" and h["wd"] and h["clip"] >= 0:
        out.append("sgd_wd_before_clip")
    if h["kind"] in ("sgd", "dcasgd") and h["momentum"] != 0.0:
        out.append("momentum_lost")
    if h["kind"] == "dcasgd" and h["lamda"] != 0.0:
        out.append("dcasgd_prev_zero")
    return out


def hyper(spec, fp32=True):
    """Plain dict of the hyper-parameters of an ``Optimizer.spec()`` (clip < 0: off), by default each rounded to fp32 as the kernels receive
    it (e.g. ``1 - fp32(0.999)`` is 1.3e-5 away from 0.001)."""
    f = (lambda x: float(np.float32(x))) if fp32 else float
    clip = spec.get("clip_gradient", -1.0)
    return dict(kind=spec["name"], lr=f(spec["lr"]), wd=f(spec["wd"]), rescale=f(spec["rescale_grad"]),
                clip=-1.0 if clip is None else f(clip), momentum=f(spec.get("momentum", 0.0)), beta1=f(spec.get("beta1", 0.9)),
                beta2=f(spec.get("beta2", 0.999)), eps=f(spec.get("epsilon", 1e-8)), lamda=f(spec.get("lamda", 0.04)))


def adam_lr(h, t):
    return h["lr"] * math.sqrt(1.0 - h["beta2"] ** t) / (1.0 - h["beta1"] ** t)


def update(h, w, g, s0, s1, t, lr_mult=1.0, wd_mult=1.0, mutation=None):
    """One update of fp64 tensors, in place: ``w`` weight, ``g`` gradient (already scaled by the push scale), ``s0`` / ``s1`` the state
    slots (SGD: s0 = momentum; Adam: s0 = m, s1 = v; DCASGD: s0 = momentum, s1 = previous weight).  ``t`` = this update's step count."""
    lr, wd = h["lr"] * lr_mult, h["wd"] * wd_mult
    clip = h["clip"]
    cl = (lambda x: x.clamp(-clip, clip)) if clip >= 0 else (lambda x: x)
    kind = h["kind"]
    if kind == "adam":
        lr_t = lr * math.sqrt(1.0 - h["beta2"] ** t) / (1.0 - h["beta1"] ** t)
        g = g * h["rescale"]
        g = cl(g) + wd * w if mutation == "adam_clip_before_wd" else cl(g + wd * w)
        s0.mul_(h["beta1"]).add_((1.0 - h["beta1"]) * g)
        s1.mul_(h["beta2"]).add_((1.0 - h["beta2"]) * g * g)
        w.sub_(lr_t * s0 / (s1.sqrt() + h["eps"]))
        return
    g = g * h["rescale"]
    if kind == "sgd":
        upd = cl(g + wd * w) if mutation == "sgd_wd_before_clip" else cl(g) + wd * w
    elif kind == "dcasgd":
        g = cl(g)
        upd = g + wd * w + h["lamda"] * g * g * (w - s1)
        s1.copy_(w)
    else:
        raise ValueError(kind)
    if h["momentum"] != 0.0:
        if mutation == "momentum_lost":
            s0.zero_()
        s0.mul_(h["momentum"]).sub_(lr * upd)
        w.add_(s0)
    else:
        w.sub_(lr * upd)


# ------------------------------------------------------------------------------------------------------------------------- wire formats
def fp16_wire(x):
    """What a half-precision hop delivers: round to fp16 (from fp32), back to fp32."""
    return x.float().half().float()


def fp8_wire(x):
    """Block-scaled e4m3 hop: one fp32 scale per 128 consecutive values, ``scale = max(amax, 1e-30) * fp32(1/448)``; the value sent is
    ``v * fp32(1/scale)`` in fp32, saturated to +-448 and rounded to e4m3; the receiver multiplies by the scale in fp32.  ``x`` is a flat
    tensor whose blocks start at index 0 (keys start on 1024-float tiles); a short last block is padded with zeros, as the arena is."""
    x = x.float().reshape(-1)
    n = x.numel()
    pad = (-n) % 128
    xb = torch.cat([x, torch.zeros(pad, dtype=torch.float32, device=x.device)]).view(-1, 128)
    amax = xb.abs().amax(1, keepdim=True)
    scale = amax.clamp_min(1e-30) * torch.tensor(INV448, dtype=torch.float32)
    inv = torch.tensor(1.0, dtype=torch.float32) / scale
    q = (xb * inv).clamp(-448.0, 448.0).to(torch.float8_e4m3fn)
    return (q.float() * scale).reshape(-1)[:n]


def wire(x, fmt):
    if fmt in (None, "fp32"):
        return x.float()
    if fmt == "fp16":
        return fp16_wire(x)
    if fmt == "fp8":
        return fp8_wire(x.reshape(-1)).reshape(x.shape)
    raise ValueError(fmt)


def param_wire(w, fmt):
    """Parameters of fp16 and fp8 keys return as halves; fp32 keys exactly."""
    return w.float().half().double() if fmt in ("fp16", "fp8") else w


# ------------------------------------------------------------------------------------------------------------------------- multi-key state
class UpdateRef:
    """fp64 server state of a list of keys.

    ``weights``: initial weights, one tensor per key.  ``mults``: per-key ``(lr_mult, wd_mult)``.  ``push_scale``: factor on the pushed
    gradient.  ``fmts``: per-key wire format (``'fp32'`` / ``'fp16'`` / ``'fp8'``).  ``round_after_scale``: the wire rounding applies to the
    scaled aggregate (the three-hop LL exchange rounds on its second hop, after the party sum was scaled) instead of to the raw gradient (the
    direct protocol's first hop).  ``mutation``: one of :data:`MUTATIONS` or None."""

    def __init__(self, spec, weights, mults=None, push_scale=1.0, fmts=None, round_after_scale=False, mutation=None):
        assert mutation is None or mutation in MUTATIONS, mutation
        self.h = hyper(spec)
        self.mutation = mutation
        self.w = [torch.as_tensor(w).detach().double().cpu().clone() for w in weights]
        K = len(self.w)
        self.mults = list(mults) if mults is not None else [(1.0, 1.0)] * K
        if mutation == "mults_ignored":
            self.mults = [(1.0, 1.0)] * K
        self.push_scale = 1.0 if mutation == "no_push_scale" else float(push_scale)
        self.fmts = list(fmts) if fmts is not None else ["fp32"] * K
        self.round_after_scale = round_after_scale
        self.s0 = [torch.zeros_like(w) for w in self.w]
        if self.h["kind"] == "dcasgd" and mutation != "dcasgd_prev_zero":
            self.s1 = [w.clone() for w in self.w]
        else:
            self.s1 = [torch.zeros_like(w) for w in self.w]
        self.t = [0] * K
        self._acc = [torch.zeros_like(w) for w in self.w]

    def step(self, grads, active=None):
        """One round: ``grads[i]`` is the pushed sum of key i (fp32, as it lies in the gradient arena).  ``active``: the keys updated this
        round (default all); the others keep weights, state and step count."""
        keys = range(len(self.w)) if active is None else active
        for i in keys:
            g = torch.as_tensor(grads[i]).detach().cpu()
            if self.mutation == "grad_not_cleared":
                self._acc[i] += g.double()
                g = self._acc[i].float()
            fmt = self.fmts[i]
            if self.round_after_scale:
                g = wire(g.float() * np.float32(self.push_scale), fmt).double()
            else:
                g = wire(g, fmt).double() * self.push_scale
            self.t[i] += 2 if self.mutation == "t_double" else 1
            t = 1 if self.mutation == "t_frozen" else self.t[i]
            lm, wm = self.mults[i]
            update(self.h, self.w[i], g.reshape(self.w[i].shape), self.s0[i], self.s1[i], t, lm, wm, self.mutation)

    def params(self):
        """The parameters as the pull delivers them (halves for fp16 / fp8 keys)."""
        return [param_wire(w, f) for w, f in zip(self.w, self.fmts)]


def rel(a, b):
    """Norm-relative difference of ``a`` from ``b`` (fp64)."""
    a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double().cpu()
    return float((a - b).norm() / (b.norm() + 1e-300))


def displacement_err(P, P0, ref_w, stores=0):
    """Worst norm-relative error, over keys, of the displacement ``P - P0`` against the reference's ``ref_w - P0``.

    ``stores``: how many times the kernel rounded the weight to fp32.  Each store may move it by half an fp32 ulp (<= 2^-24 |w|), which is
    not an error of the update; that much of the difference is discounted.  It matters for keys whose displacement is tiny next to the weight
    (a single bias whose gradient happened to be zero)."""
    out = 0.0
    for p, p0, r in zip(P, P0, ref_w):
        p0 = torch.as_tensor(p0).double().cpu()
        r = r.double().reshape(p0.shape)
        d_ref = r - p0
        diff = float((torch.as_tensor(p).double().cpu().reshape(p0.shape) - r).norm())
        diff = max(0.0, diff - stores * 2.0 ** -24 * float(r.norm()))
        if float(d_ref.norm()) == 0.0:
            out = max(out, diff)
            continue
        out = max(out, diff / float(d_ref.norm()))
    return out


def cnn_like_grads(gen, shapes, steps, batch=32):
    """Synthetic per-step gradient SUMS over a batch with the demo CNN's magnitudes: per-element mean gradient ~1e-3 .. 1e-2 (heavier on
    biases), a per-step drift and sign changes, some exact zeros (dead units), times the batch size."""
    out = []
    base = [torch.randn(s, generator=gen, dtype=F64) * (0.02 if len(s) == 1 else 0.004) for s in shapes]
    for k in range(steps):
        gs = []
        for b in base:
            g = b * (1.0 + 0.3 * k) + torch.randn(b.shape, generator=gen, dtype=F64) * b.abs().mean()
            g = torch.where(torch.rand(b.shape, generator=gen, dtype=F64) < 0.05, torch.zeros_like(g), g)
            gs.append((g * batch).float())
        out.append(gs)
    return out
