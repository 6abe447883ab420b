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

Bi-Sparse tiles (``fmt 'bsc'``), from the contract of ``HipsFabric.set_wire_formats`` and the reference's BSCompress / BSCPullCompress /
BSCDecompress: per 1024-float tile (padding included) the party owner keeps ``u`` and ``v``; with the scaled party aggregate ``g`` it computes
``u = 0.9u + g; v += u``, sends the ``K = max(1, floor(1024 * threshold))`` entries of largest ``|v|`` (ties at the K-th magnitude to the
lowest index) as (value, index) pairs and clears ``u`` and ``v`` there.  The global owner scatters the pairs into a zeroed tile.  Without a
server optimizer the aggregate goes back the same way: the parameter tile is zeroed and the non-zeros scattered into it.

DGT re-ranking (``HipsFabric.dgt_rerank``): the tiles are ordered by their contribution (descending, stable), the first
:func:`num_important` keep their base format and the other fp32 / fp16 tiles travel as fp8; Bi-Sparse tiles keep their format.
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

# Mutations of the Bi-Sparse stage and of the DGT re-ranking (kept apart from MUTATIONS: they only apply to arenas that have such tiles)
STAGE_MUTATIONS = {
    "bsc_no_momentum": "the Bi-Sparse u is not carried between rounds (u = g)",
    "bsc_residual_kept": "the sent entries of u and v are not cleared",
    "bsc_ties_high_index": "ties at the K-th magnitude go to the highest index",
    "bsc_scale_after_select": "the push scale is applied to the sent values instead of before the stage (u and v hold unscaled sums)",
    "dgt_no_demotion": "re-ranking leaves unimportant fp32 / fp16 tiles at their base format",
}

TILE = 1024
BSC_MOMENTUM = float(np.float32(0.9))           # the kernel's fp32 constant 0.9f

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


# ------------------------------------------------------------------------------------------------------------------------- Bi-Sparse
def bsc_k(threshold):
    """Packets per tile and party: ``max(1, floor(1024 * threshold))``."""
    return max(1, int(TILE * float(threshold)))


def bsc_topk(mag, K, high_index=False):
    """Sorted indices of the ``K`` largest entries of ``mag`` (one tile), ties at the K-th magnitude to the lowest index (``high_index``: to
    the highest, a mutation)."""
    if high_index:
        return (mag.numel() - 1 - torch.argsort(mag.flip(0), descending=True, stable=True)[:K]).sort().values
    return torch.argsort(mag, descending=True, stable=True)[:K].sort().values


def bsc_round(u, v, acc, K, mutation=None, scale=1.0, select=None):
    """One round of the Bi-Sparse stage on flat, tile-padded fp64 tensors ``u`` / ``v`` (updated in place) with the party aggregate ``acc``.
    ``scale`` multiplies the sent values (1 unless the push scale is applied after the selection, a mutation).  ``select(t, v_tile)``, if
    given, returns the indices to send in tile ``t`` (or None for the reference's own choice): how a test adopts a kernel's selection.
    Returns the decompressed aggregate (sent values scattered into zeros) and the per-tile selections."""
    if mutation == "bsc_no_momentum":
        u.copy_(acc)
    else:
        u.mul_(BSC_MOMENTUM).add_(acc)
    v.add_(u)
    out = torch.zeros_like(v)
    sels = []
    for t in range(v.numel() // TILE):
        a = t * TILE
        vt = v[a:a + TILE]
        sel = select(t, vt) if select is not None else None
        if sel is None:
            sel = bsc_topk(vt.abs(), K, high_index=mutation == "bsc_ties_high_index")
        idx = torch.as_tensor(sel, dtype=torch.long) + a
        out[idx] = v[idx] * scale
        if mutation != "bsc_residual_kept":
            u[idx] = 0.0
            v[idx] = 0.0
        sels.append(torch.as_tensor(sel, dtype=torch.long))
    return out, sels


def selection_slack(v_tile, sel, K):
    """How far a selection ``sel`` (indices into one tile) is from a valid top-``K`` of ``|v_tile|``: 0 for an exact top-K, else the largest
    relative amount by which a selected magnitude falls below, or an unselected one rises above, the K-th largest magnitude.  ``inf`` when
    more than K entries were selected."""
    sel = torch.as_tensor(sel, dtype=torch.long)
    if sel.numel() > K:
        return float("inf")
    mag = v_tile.abs().double()
    kth = float(mag.sort(descending=True).values[K - 1])
    chosen = torch.zeros(mag.numel(), dtype=torch.bool)
    chosen[sel] = True
    if kth == 0.0:                   # fewer than K non-zeros: all of them must go
        return 0.0 if bool(chosen[mag > 0].all()) else float("inf")
    if sel.numel() < K:
        return float("inf")
    low = float(mag[chosen].min()) if sel.numel() else kth
    high = float(mag[~chosen].max()) if (~chosen).any() else 0.0
    return max(0.0, (kth - low) / kth, (high - kth) / kth)


# ------------------------------------------------------------------------------------------------------------------------- DGT re-ranking
def num_important(sorted_contrib, k, adaptive=False, k_min=0.2):
    """Size of the important set from the contributions in descending order: fixed, ``max(1, round(k * n))`` tiles; adaptive, the shortest
    prefix that carries ``k`` of the total contribution, at least ``round(k_min * n)`` tiles (``max(1, round(k_min * n))`` when the total
    is 0)."""
    c = [float(x) for x in sorted_contrib]
    n = len(c)
    if n == 0:
        return 0
    if not adaptive:
        return max(1, int(round(k * n)))
    total = sum(c)
    if total <= 0.0:
        return max(1, int(round(k_min * n)))
    acc, need = 0.0, n
    for i, x in enumerate(c):
        acc += x
        if acc / total >= k - 1e-12:
            need = i + 1
            break
    return max(1, min(n, max(need, int(round(k_min * n)))))


def dgt_formats(base, contrib, k, adaptive=False, k_min=0.2, mutation=None):
    """Re-ranking of per-tile formats ``base`` (list of 'fp32' / 'fp16' / 'fp8' / 'bsc') by the contributions ``contrib`` (one per tile):
    returns (order, number of important tiles, new per-tile formats)."""
    c = torch.as_tensor(contrib).double().cpu()
    order = torch.argsort(c, descending=True, stable=True)
    n_imp = num_important(c[order], k, adaptive, k_min)
    fmts = list(base)
    if mutation != "dgt_no_demotion":
        for t in order[n_imp:].tolist():
            if fmts[t] in ("fp32", "fp16"):
                fmts[t] = "fp8"
    return order, n_imp, fmts


def dgt_ema(old, mean, alpha):
    """The per-tile contribution EMA: the first value as is, then ``alpha * old + (1 - alpha) * mean``."""
    return torch.where(old == 0, mean, alpha * old + (1.0 - alpha) * mean)


# ------------------------------------------------------------------------------------------------------------------------- multi-key state
class UpdateRef:
    """fp64 server state of a list of keys.

    ``spec``: ``Optimizer.spec()`` dict, or None for no server optimizer (the master weight of a round is its aggregate).  ``weights``:
    initial weights, one tensor per key.  ``mults``: per-key ``(lr_mult, wd_mult)``.  ``push_scale``: factor on the pushed gradient.
    ``fmts``: per-key wire format (``'fp32'`` / ``'fp16'`` / ``'fp8'`` / ``'bsc'``), or for a key whose tiles differ (after a DGT
    demotion) a list with one format per 1024-float tile; ``fmts`` may be changed between rounds.  ``round_after_scale``: the wire
    rounding applies to the scaled aggregate (the three-hop LL exchange rounds on its second hop, after the party sum was scaled) instead of
    to the raw gradient (the direct protocol's first hop); Bi-Sparse tiles always see the scaled aggregate.  ``pull_half``: per key, whether
    the aggregate itself crosses the pull (no server optimizer, sharded or LL pull), so that fp16 / fp8 tiles of it arrive as halves.
    ``bsc_k``: packets per Bi-Sparse tile.  ``mutation``: one of :data:`MUTATIONS` / :data:`STAGE_MUTATIONS` or None.

    After ``step``, ``agg[i]`` holds the aggregate of key i (tile-padded fp64) that the optimizer (or the pull) received, and ``u[i]`` /
    ``v[i]`` the Bi-Sparse state (tile-padded, zero outside Bi-Sparse tiles)."""

    def __init__(self, spec, weights, mults=None, push_scale=1.0, fmts=None, round_after_scale=False, mutation=None, pull_half=None,
                 bsc_k=10):
        assert mutation is None or mutation in MUTATIONS or mutation in STAGE_MUTATIONS, mutation
        self.h = None if spec is None else hyper(spec)
        self.mutation = mutation
        self.w = [torch.as_tensor(w).detach().double().cpu().clone() for w in weights]
        K = len(self.w)
        self.mults = list(mults) if mults is not None else [(1.0, 1.0)] * K
        if mutation == "mults_ignored":
            self.mults = [(1.0, 1.0)] * K
        self.push_scale = 1.0 if mutation == "no_push_scale" else float(push_scale)
        self.fmts = list(fmts) if fmts is not None else ["fp32"] * K
        self.round_after_scale = round_after_scale
        self.pull_half = list(pull_half) if pull_half is not None else [False] * K
        self.bsc_k = int(bsc_k)
        self.s0 = [torch.zeros_like(w) for w in self.w]
        if self.h is not None and self.h["kind"] == "dcasgd" and mutation != "dcasgd_prev_zero":
            self.s1 = [w.clone() for w in self.w]
        else:
            self.s1 = [torch.zeros_like(w) for w in self.w]
        self.t = [0] * K
        self._acc = [torch.zeros_like(w) for w in self.w]
        pad = [-(-w.numel() // TILE) * TILE for w in self.w]
        self.u = [torch.zeros(p, dtype=F64) for p in pad]
        self.v = [torch.zeros(p, dtype=F64) for p in pad]
        self.agg = [torch.zeros(p, dtype=F64) for p in pad]

    def tile_fmts(self, i):
        """Per-tile wire formats of key i."""
        f = self.fmts[i]
        return [f] * (self.u[i].numel() // TILE) if isinstance(f, str) else list(f)

    def _aggregate(self, i, g, select):
        """The aggregate of key i that leaves the exchange (tile-padded fp64) from its pushed sum ``g``."""
        fmts = self.tile_fmts(i)
        n, ps = g.numel(), self.push_scale
        gp = torch.zeros(self.u[i].numel(), dtype=torch.float32)
        gp[:n] = g.float().reshape(-1)
        scaled = gp * np.float32(ps)                     # the kernels scale in fp32
        out = torch.zeros(gp.numel(), dtype=F64)
        for t, fmt in enumerate(fmts):
            if fmt == "bsc":
                continue
            a = slice(t * TILE, (t + 1) * TILE)
            x = wire(scaled[a], fmt).double() if self.round_after_scale else wire(gp[a], fmt).double() * ps
            if self.pull_half[i] and fmt in ("fp16", "fp8"):
                x = x.float().half().double()
            out[a] = x
        bsc = [t for t, fmt in enumerate(fmts) if fmt == "bsc"]
        if bsc:
            idx = torch.cat([torch.arange(t * TILE, (t + 1) * TILE) for t in bsc])
            after = self.mutation == "bsc_scale_after_select"
            u, v = self.u[i][idx], self.v[i][idx]
            sub = None if select is None else (lambda j, vt: select(i, bsc[j], vt))
            agg, _ = bsc_round(u, v, (gp if after else scaled)[idx].double(), self.bsc_k, self.mutation, scale=ps if after else 1.0, select=sub)
            self.u[i][idx], self.v[i][idx] = u, v
            out[idx] = agg
        return out

    def step(self, grads, active=None, bsc_select=None):
        """One round: ``grads[i]`` is the pushed sum of key i (fp32, as it lies in the gradient arena).  ``active``: the keys updated this
        round (default all); the others keep weights, state, Bi-Sparse state and step count.  ``bsc_select(key, tile, v_tile)``: see
        :func:`bsc_round` (``tile`` counts within the key)."""
        keys = range(len(self.w)) if active is None else active
        for i in keys:
            g = torch.as_tensor(grads[i]).detach().cpu()
            if self.mutation == "grad_not_cleared":
                self._acc[i] += g.double()
                g = self._acc[i].float()
            fmt = self.fmts[i]
            if isinstance(fmt, str) and fmt != "bsc" and not self.pull_half[i]:
                if self.round_after_scale:
                    g = wire(g.float() * np.float32(self.push_scale), fmt).double()
                else:
                    g = wire(g, fmt).double() * self.push_scale
                self.agg[i].zero_()
                self.agg[i][:g.numel()] = g.reshape(-1)
            else:
                self.agg[i] = self._aggregate(i, g, bsc_select)
                g = self.agg[i][:self.w[i].numel()]
            self.t[i] += 2 if self.mutation == "t_double" else 1
            t = 1 if self.mutation == "t_frozen" else self.t[i]
            if self.h is None:
                self.w[i].copy_(g.reshape(self.w[i].shape))
                continue
            lm, wm = self.mults[i]
            update(self.h, self.w[i], g.reshape(self.w[i].shape), self.s0[i], self.s1[i], t, lm, wm, self.mutation)

    def params(self):
        """The parameters as the pull delivers them: halves for fp16 / fp8 tiles; without a server optimizer the Bi-Sparse tiles return
        their non-zeros scattered into zeros (+0.0)."""
        out = []
        for i, w in enumerate(self.w):
            fm = self.tile_fmts(i)
            p = torch.zeros(self.u[i].numel(), dtype=F64)
            p[:w.numel()] = w.reshape(-1)
            for t, f in enumerate(fm):
                a = slice(t * TILE, (t + 1) * TILE)
                if f in ("fp16", "fp8"):
                    p[a] = p[a].float().half().double()
                elif f == "bsc" and self.h is None:
                    p[a] = torch.where(p[a] != 0, p[a], torch.zeros_like(p[a]))
            out.append(p[:w.numel()].reshape(w.shape))
        return out


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
