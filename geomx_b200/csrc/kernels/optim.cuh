// The optimizer rules of the library, one definition each: the arena / multi-tensor / single-tensor kernels of optim.cu and every server
// update of the HiPS fabric kernels (hips_ll.cuh, hips_fabric.cu, cnn_direct.cu) apply them.  The learning-rate schedule is evaluated
// here too, from the device-side step count, so a scheduled update stays CUDA-graph replayable.
#pragma once
#include "common.cuh"

namespace gx {

enum OptKind {
  OPT_NONE = -1, OPT_SGD = 0, OPT_ADAM = 1, OPT_DCASGD = 2,
  OPT_NAG = 3, OPT_SIGNUM = 4, OPT_RMSPROP = 5, OPT_ADAGRAD = 6, OPT_ADADELTA = 7, OPT_FTRL = 8
};

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

// Field order is part of the ABI: ops/_native_api.py's OptHyper mirrors it (also inside parallel/fabric.py's FabricParams); the
// static_asserts below pin the offsets that the Python side asserts too.
struct OptHyper {
  float lr, wd, rescale, clip;      // clip < 0 -> off; lr: the base lr of a schedule
  float momentum;                   // sgd / dcasgd / nag / signum
  float beta1, beta2, eps;          // adam; eps also rmsprop / adagrad / adadelta
  float lamda;                      // dcasgd
  float wd_lh;                      // signum: decoupled weight decay
  float clip_weights;               // rmsprop: clamp of the new weight, < 0 -> off
  float gamma1;                     // rmsprop: decay of the squared-gradient average
  float rho;                        // adadelta
  float beta, lamda1;               // ftrl
  int kind;                         // OptKind; OPT_NONE (fabric only): store the aggregated gradient (Bi-Sparse / local-optimizer modes)
  LrSchedule sched;
};
static_assert(sizeof(LrSchedule) == 108, "LrSchedule layout (ops/_native_api.py)");
static_assert(offsetof(OptHyper, wd_lh) == 36 && offsetof(OptHyper, lamda1) == 56 && offsetof(OptHyper, kind) == 60 &&
              offsetof(OptHyper, sched) == 64 && sizeof(OptHyper) == 172, "OptHyper layout (ops/_native_api.py)");

__device__ __forceinline__ float clip_to(float x, float c) { return c >= 0.f ? fminf(fmaxf(x, -c), c) : x; }
__device__ __forceinline__ float sign_of(float x) { return (float)((x > 0.f) - (x < 0.f)); }

// One element of each optimizer, written from the reference's update operators (src/operator/optimizer_op-inl.h) and optimizer.py.
// State slots s0 / s1: sgd, nag, signum: s0 = mom; adam: s0 = m, s1 = v; dcasgd: s0 = mom, s1 = previous weight; rmsprop: s0 = n;
// adagrad: s0 = history; adadelta: s0 = acc_g, s1 = acc_delta; ftrl: s0 = z, s1 = n.  Every state starts at 0 except dcasgd's s1.
template <int KIND>
__device__ __forceinline__ void opt_elem(float& w, float g, float& s0, float& s1, const OptHyper& h, float lr, float wd) {
  if (KIND == OPT_NAG) {
    // optimizer.py NAG: rescale, clip, then mom = mu*mom + (g + wd*w); w -= lr * (g + wd*w + mu*mom)
    g = fmaf(wd, w, clip_to(g * h.rescale, h.clip));
    if (h.momentum != 0.f) { s0 = fmaf(h.momentum, s0, g); g = fmaf(h.momentum, s0, g); }
    w -= lr * g;
  } else if (KIND == OPT_SIGNUM) {
    if (h.momentum != 0.f) {
      // SignumKernel: mom = mu*mom - (1-mu)*wd*w - (1-mu)*clip(rescale*g); w = (1 - lr*wd_lh)*w + lr*sign(mom)
      s0 = h.momentum * s0 - (1.f - h.momentum) * fmaf(wd, w, clip_to(g * h.rescale, h.clip));
      w = (1.f - lr * h.wd_lh) * w + lr * sign_of(s0);
    } else {
      // SignSGDKernel: decoupled wd, no clip, no wd_lh
      w = (1.f - lr * wd) * w - lr * sign_of(g);
    }
  } else if (KIND == OPT_RMSPROP) {
    // RMSPropUpdate: rescale, + wd*w, THEN clip; eps inside the sqrt; clip_weights clamps the new weight
    g = clip_to(fmaf(wd, w, g * h.rescale), h.clip);
    s0 = (1.f - h.gamma1) * g * g + h.gamma1 * s0;
    w = clip_to(w - lr * (g / sqrtf(s0 + h.eps)), h.clip_weights);
  } else if (KIND == OPT_ADAGRAD) {
    // optimizer.py AdaGrad (dense): rescale, clip; history += g^2; w += (g / sqrt(history + eps) + wd*w) * -lr
    g = clip_to(g * h.rescale, h.clip);
    s0 = fmaf(g, g, s0);
    w -= lr * (g / sqrtf(s0 + h.eps) + wd * w);
  } else if (KIND == OPT_ADADELTA) {
    // optimizer.py AdaDelta: no learning rate; wd outside the adaptive step
    g = clip_to(g * h.rescale, h.clip);
    s0 = h.rho * s0 + (1.f - h.rho) * g * g;
    const float d = sqrtf(s1 + h.eps) / sqrtf(s0 + h.eps) * g;
    s1 = h.rho * s1 + (1.f - h.rho) * d * d;
    w -= d + wd * w;
  } else if (KIND == OPT_FTRL) {
    // FtrlUpdate: z += g - (sqrt(n + g^2) - sqrt(n)) * w / lr; n += g^2; w = (sign(z)*lamda1 - z) / ((beta + sqrt(n)) / lr + wd) masked by
    // |z| > lamda1.  sqrt(n + g^2) - sqrt(n) is computed as g^2 / (sqrt(n + g^2) + sqrt(n)), the same value without the cancellation that
    // the literal difference suffers in fp32 once n >> g^2 (it would lose every digit of the increment after a few hundred updates).
    g = clip_to(g * h.rescale, h.clip);
    const float g2 = g * g, sn = sqrtf(s1), sn1 = sqrtf(s1 + g2);
    const float sigma = sn1 + sn > 0.f ? g2 / (sn1 + sn) : 0.f;
    s0 += g - sigma * w / lr;
    s1 += g2;
    w = fabsf(s0) > h.lamda1 ? (sign_of(s0) * h.lamda1 - s0) / ((h.beta + sn1) / lr + wd) : 0.f;
  } else if (KIND == OPT_SGD) {
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

// the run-time dispatch over SGD / Adam / DCASGD, one element
__device__ __forceinline__ void opt_apply(float& w, float g, float& s0, float& s1, const OptHyper& h, float lr, float wd) {
  if (h.kind == OPT_ADAM) opt_elem<OPT_ADAM>(w, g, s0, s1, h, lr, wd);
  else if (h.kind == OPT_SGD) opt_elem<OPT_SGD>(w, g, s0, s1, h, lr, wd);
  else if (h.kind == OPT_DCASGD) opt_elem<OPT_DCASGD>(w, g, s0, s1, h, lr, wd);
  else w = g;  // no optimizer on the server: store the aggregate (reference ApplyUpdates without updater_, :547-550)
}

template <int KIND>
__device__ __forceinline__ void opt_elem4(float4& W, float4 G, float4& A, float4& B, const OptHyper& h, float lr, float wd) {
  opt_elem<KIND>(W.x, G.x, A.x, B.x, h, lr, wd);
  opt_elem<KIND>(W.y, G.y, A.y, B.y, h, lr, wd);
  opt_elem<KIND>(W.z, G.z, A.z, B.z, h, lr, wd);
  opt_elem<KIND>(W.w, G.w, A.w, B.w, h, lr, wd);
}

// The server update of the fabric kernels: four consecutive elements (one float4 of each operand), the kind chosen at run time by h.kind.
// EXT: the instance also runs the kinds after DCASGD (NAG .. Ftrl).  The fabric kernels are instantiated with and without them and their
// launchers pick EXT only for those kinds (GX_FAB_INSTANCE, hips_ll.cuh): the SGD / Adam / DCASGD instances compile to the code they had
// before the later kinds existed, which keeps the training step's exchange kernels as short as they were.
template <bool EXT>
__device__ __forceinline__ void opt_apply4(float4& W, float4 G, float4& A, float4& B, const OptHyper& h, float lr, float wd) {
  if (!EXT) {
    opt_apply(W.x, G.x, A.x, B.x, h, lr, wd);
    opt_apply(W.y, G.y, A.y, B.y, h, lr, wd);
    opt_apply(W.z, G.z, A.z, B.z, h, lr, wd);
    opt_apply(W.w, G.w, A.w, B.w, h, lr, wd);
  } else if (h.kind == OPT_NAG) opt_elem4<OPT_NAG>(W, G, A, B, h, lr, wd);
  else if (h.kind == OPT_SIGNUM) opt_elem4<OPT_SIGNUM>(W, G, A, B, h, lr, wd);
  else if (h.kind == OPT_RMSPROP) opt_elem4<OPT_RMSPROP>(W, G, A, B, h, lr, wd);
  else if (h.kind == OPT_ADAGRAD) opt_elem4<OPT_ADAGRAD>(W, G, A, B, h, lr, wd);
  else if (h.kind == OPT_ADADELTA) opt_elem4<OPT_ADADELTA>(W, G, A, B, h, lr, wd);
  else if (h.kind == OPT_FTRL) opt_elem4<OPT_FTRL>(W, G, A, B, h, lr, wd);
  else opt_apply4<false>(W, G, A, B, h, lr, wd);
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
