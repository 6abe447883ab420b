// The optimizer rules of the library, one definition each: the arena / multi-tensor / single-tensor kernels of optim.cu and every server
// update of the HiPS fabric kernels (hips_ll.cuh, hips_fabric.cu, cnn_direct.cu) apply them.  The learning-rate schedule is evaluated
// here too, from the device-side step count, so a scheduled update stays CUDA-graph replayable.
#pragma once
#include "common.cuh"

namespace gx {

enum OptKind { OPT_NONE = -1, OPT_SGD = 0, OPT_ADAM = 1, OPT_DCASGD = 2 };

// The learning-rate schedules of lr_scheduler.py, as LRScheduler.device_spec() describes them; ops/_native_api.py packs that dict.
enum SchedKind { SCHED_NONE = 0, SCHED_FACTOR = 1, SCHED_MULTIFACTOR = 2, SCHED_POLY = 3, SCHED_COSINE = 4 };
constexpr int SCHED_MAX_MILESTONES = 16;

struct LrSchedule {
  int kind;                                 // SchedKind; SCHED_NONE: the constant OptHyper::lr
  int warmup_steps, warmup_linear;          // warm-up while t < warmup_steps: linear ramp from warmup_begin_lr (warmup_linear) or constant
  float warmup_begin_lr;
  int step;                                 // factor: one more factor every `step` updates
  float factor, stop_factor_lr;             // factor / multifactor
  int num_milestones, milestones[SCHED_MAX_MILESTONES];   // multifactor, increasing
  int max_update;                           // poly / cosine
  float final_lr, pwr;
};

// Field order is part of the ABI: parallel/fabric.py's _OptHyperF mirrors it inside FabricParams.
struct OptHyper {
  float lr, wd, rescale, clip;      // clip < 0 -> off; lr: the base lr of a schedule
  float momentum;                   // sgd / dcasgd
  float beta1, beta2, eps;          // adam
  float lamda;                      // dcasgd
  int kind;                         // OptKind; OPT_NONE (fabric only): store the aggregated gradient (Bi-Sparse / local-optimizer modes)
  LrSchedule sched;
};

// one element of each optimizer (s0/s1 = state slots: sgd: s0=mom; adam: s0=m, s1=v; dcasgd: s0=mom, s1=prev_weight)
template <int KIND>
__device__ __forceinline__ void opt_elem(float& w, float g, float& s0, float& s1, const OptHyper& h, float lr, float wd) {
  if (KIND == OPT_SGD) {
    g *= h.rescale;
    if (h.clip >= 0.f) g = fminf(fmaxf(g, -h.clip), h.clip);
    g = fmaf(wd, w, g);
    if (h.momentum != 0.f) { s0 = h.momentum * s0 - lr * g; w += s0; }
    else w -= lr * g;
  } else if (KIND == OPT_ADAM) {
    // adam_update clips the REGULARISED gradient: rescale, + wd*w, then clip (src/operator/optimizer_op-inl.h:840-873)
    g = fmaf(wd, w, g * h.rescale);
    if (h.clip >= 0.f) g = fminf(fmaxf(g, -h.clip), h.clip);
    s0 = h.beta1 * s0 + (1.f - h.beta1) * g;
    s1 = h.beta2 * s1 + (1.f - h.beta2) * g * g;
    w -= lr * s0 / (sqrtf(s1) + h.eps);
  } else {
    g *= h.rescale;
    if (h.clip >= 0.f) g = fminf(fmaxf(g, -h.clip), h.clip);
    const float upd = g + wd * w + h.lamda * g * g * (w - s1);
    const float prev = w;
    if (h.momentum != 0.f) { s0 = h.momentum * s0 - lr * upd; w += s0; }
    else w -= lr * upd;
    s1 = prev;
  }
}

// the same, with the kind chosen at run time by h.kind
__device__ __forceinline__ void opt_apply(float& w, float g, float& s0, float& s1, const OptHyper& h, float lr, float wd) {
  if (h.kind == OPT_ADAM) opt_elem<OPT_ADAM>(w, g, s0, s1, h, lr, wd);
  else if (h.kind == OPT_SGD) opt_elem<OPT_SGD>(w, g, s0, s1, h, lr, wd);
  else if (h.kind == OPT_DCASGD) opt_elem<OPT_DCASGD>(w, g, s0, s1, h, lr, wd);
  else w = g;  // no optimizer on the server: store the aggregate (reference ApplyUpdates without updater_, :547-550)
}

// four consecutive elements (one float4 of each operand)
__device__ __forceinline__ void opt_apply4(float4& W, float4 G, float4& A, float4& B, const OptHyper& h, float lr, float wd) {
  opt_apply(W.x, G.x, A.x, B.x, h, lr, wd);
  opt_apply(W.y, G.y, A.y, B.y, h, lr, wd);
  opt_apply(W.z, G.z, A.z, B.z, h, lr, wd);
  opt_apply(W.w, G.w, A.w, B.w, h, lr, wd);
}

// learning rate of update t (1-based) before Adam's bias correction: the fp32 mirror of LRScheduler.__call__(t) with base_lr = h.lr.
// Every branch is decided in integers, so no boundary (end of warm-up, a factor step, a milestone, max_update) can move by a step.  One
// powf serves every kind that needs one (factor^k, factor^passed, q^pwr); the cosine uses sinpif.
__device__ __forceinline__ float sched_lr(const OptHyper& h, int t) {
  const LrSchedule& s = h.sched;
  if (s.kind == SCHED_NONE) return h.lr;
  if (t < s.warmup_steps) return s.warmup_linear ? s.warmup_begin_lr + ((float)t / (float)s.warmup_steps) * (h.lr - s.warmup_begin_lr)
                                                 : s.warmup_begin_lr;
  int k = 0;   // factor: factors applied; multifactor: milestones strictly below t
  if (s.kind == SCHED_FACTOR) {
    k = max(0, (t - 1) / s.step);
  } else if (s.kind == SCHED_MULTIFACTOR) {
    for (int i = 0; i < s.num_milestones; ++i) k += s.milestones[i] < t;
  }
  // poly / cosine: q = 1 - progress = (max_update - t) / (max_update - warmup_steps), 0 from max_update on
  const float q = (float)max(s.max_update - t, 0) / (float)(s.max_update - s.warmup_steps);
  float shape;
  if (s.kind == SCHED_COSINE) {
    const float sn = sinpif(0.5f * q);  // 0.5 * (1 + cos(pi * progress)) = sin^2(pi * q / 2): no cancellation near the end
    shape = sn * sn;
  } else {
    const bool decay = s.kind == SCHED_FACTOR || s.kind == SCHED_MULTIFACTOR;
    shape = powf(decay ? s.factor : q, decay ? (float)k : s.pwr);
  }
  if (s.kind == SCHED_FACTOR) return k == 0 ? h.lr : fmaxf(h.lr * shape, s.stop_factor_lr);
  if (s.kind == SCHED_MULTIFACTOR) return h.lr * shape;
  return s.final_lr + (h.lr - s.final_lr) * shape;
}

// step size of update t (1-based): the lr (scheduled when SCHED), with Adam's bias correction folded in for Adam.  Every update kernel is
// instantiated twice and its launcher picks the instance from h.sched.kind: the constant-lr instance (SCHED = false) compiles to the code it
// had before schedules existed, the scheduled one evaluates sched_lr.
template <bool SCHED>
__device__ __forceinline__ float step_lr(const OptHyper& h, int t) {
  const float lr = SCHED ? sched_lr(h, t) : h.lr;
  if (h.kind != OPT_ADAM) return lr;
  return lr * sqrtf(1.f - powf(h.beta2, (float)t)) / (1.f - powf(h.beta1, (float)t));
}

}  // namespace gx
