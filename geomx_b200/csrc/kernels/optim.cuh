// The optimizer rules of the library, one definition each: the arena / multi-tensor / single-tensor kernels of optim.cu and every server
// update of the HiPS fabric kernels (hips_ll.cuh, hips_fabric.cu, cnn_direct.cu) apply them.
#pragma once
#include "common.cuh"

namespace gx {

enum OptKind { OPT_NONE = -1, OPT_SGD = 0, OPT_ADAM = 1, OPT_DCASGD = 2 };

// Field order is part of the ABI: parallel/fabric.py's _OptHyperF mirrors it inside FabricParams.
struct OptHyper {
  float lr, wd, rescale, clip;      // clip < 0 -> off
  float momentum;                   // sgd / dcasgd
  float beta1, beta2, eps;          // adam
  float lamda;                      // dcasgd
  int kind;                         // OptKind; OPT_NONE (fabric only): store the aggregated gradient (Bi-Sparse / local-optimizer modes)
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

// step size of update t (1-based): Adam's bias correction folded into lr, h.lr for the other kinds
__device__ __forceinline__ float adam_lr(const OptHyper& h, int t) {
  if (h.kind != OPT_ADAM) return h.lr;
  return h.lr * sqrtf(1.f - powf(h.beta2, (float)t)) / (1.f - powf(h.beta1, (float)t));
}

}  // namespace gx
