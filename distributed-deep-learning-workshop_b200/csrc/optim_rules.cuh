// Per-element update rules of the fused flat-buffer optimizers: update_kernel<Rule> (csrc/optim.cu) runs one over
// every element, and allreduce_sgd_nvls_kernel (csrc/allreduce.cu) applies SgdRule to the all-reduced gradient.
//
// A rule's constructor reads the device hyper array once (slots in ops_api.h), including values derived from it; its
// operator()(w, g, s) updates one weight w from its unscaled gradient g and its kStates state values s[0..kStates), in
// the order the optimizer's state buffers are passed.  The output bits depend on each fmaf and its operand order.
#pragma once
#include "ops_api.h"

namespace b200 {

template <bool NESTEROV>
struct SgdRule {
  static constexpr int kStates = 1;   // momentum
  float lr, mu, wd, gs;
  __device__ explicit SgdRule(const float* __restrict__ h)
      : lr(h[kHypLr]), mu(h[kHypMom]), wd(h[kHypWd]), gs(h[kHypGScale]) {}
  // gs given by the caller (the fused all-reduce passes its 1 / world scale)
  __device__ SgdRule(const float* __restrict__ h, float gs) : lr(h[kHypLr]), mu(h[kHypMom]), wd(h[kHypWd]), gs(gs) {}
  __device__ __forceinline__ void operator()(float& w, float g, float* s) const {
    const float d = fmaf(wd, w, g * gs);
    s[0] = fmaf(mu, s[0], d);
    const float upd = NESTEROV ? fmaf(mu, s[0], d) : s[0];
    w = fmaf(-lr, upd, w);
  }
};

// DECOUPLED (AdamW): p *= 1 - lr * wd before the Adam step, and the gradient carries no L2 term.
template <bool DECOUPLED>
struct AdamRule {
  static constexpr int kStates = 2;   // m, v
  float lr, b1, b2, eps, wd, gs, step, inv_sqrt_bc2, decay;
  __device__ explicit AdamRule(const float* __restrict__ h)
      : lr(h[kHypLr]), b1(h[kHypMom]), b2(h[kHypBeta2]), eps(h[kHypEps]), wd(h[kHypWd]), gs(h[kHypGScale]),
        step(lr / h[kHypBc1]), inv_sqrt_bc2(rsqrtf(h[kHypBc2])), decay(1.f - lr * wd) {}
  __device__ __forceinline__ void operator()(float& w, float g, float* s) const {
    float d;
    if constexpr (DECOUPLED) {
      w *= decay;
      d = g * gs;
    } else {
      d = fmaf(wd, w, g * gs);
    }
    s[0] = fmaf(b1, s[0], (1.f - b1) * d);
    s[1] = fmaf(b2, s[1], (1.f - b2) * d * d);
    const float denom = sqrtf(s[1]) * inv_sqrt_bc2 + eps;
    w = w - step * s[0] / denom;
  }
};

struct AdadeltaRule {
  static constexpr int kStates = 2;   // mean square of the gradient, of the update
  float lr, rho, eps, wd, gs;
  __device__ explicit AdadeltaRule(const float* __restrict__ h)
      : lr(h[kHypLr]), rho(h[kHypBeta2]), eps(h[kHypEps]), wd(h[kHypWd]), gs(h[kHypGScale]) {}
  __device__ __forceinline__ void operator()(float& w, float g, float* s) const {
    const float d = fmaf(wd, w, g * gs);
    s[0] = fmaf(rho, s[0], (1.f - rho) * d * d);
    const float delta = sqrtf(s[1] + eps) / sqrtf(s[0] + eps) * d;
    s[1] = fmaf(rho, s[1], (1.f - rho) * delta * delta);
    w = fmaf(-lr, delta, w);
  }
};

// torch.optim.RMSprop: v = rho v + (1 - rho) d^2; CENTERED: a = rho a + (1 - rho) d, denom = sqrt(v - a^2) + eps
// (v - a^2 >= 0 in exact arithmetic; clamped at 0 so that rounding cannot make it NaN); MOMENTUM: buf = mu buf + d / denom,
// p -= lr buf; otherwise p -= lr d / denom.
template <bool CENTERED, bool MOMENTUM>
struct RmspropRule {
  static constexpr int kMom = 1, kAvg = MOMENTUM ? 2 : 1;
  static constexpr int kStates = 1 + MOMENTUM + CENTERED;   // v, then buf with MOMENTUM, then a when CENTERED
  float lr, mu, rho, eps, wd, gs;
  __device__ explicit RmspropRule(const float* __restrict__ h)
      : lr(h[kHypLr]), mu(h[kHypMom]), rho(h[kHypBeta2]), eps(h[kHypEps]), wd(h[kHypWd]), gs(h[kHypGScale]) {}
  __device__ __forceinline__ void operator()(float& w, float g, float* s) const {
    const float d = fmaf(wd, w, g * gs);
    s[0] = fmaf(rho, s[0], (1.f - rho) * d * d);
    float var = s[0];
    if constexpr (CENTERED) {
      s[kAvg] = fmaf(rho, s[kAvg], (1.f - rho) * d);
      var = fmaxf(fmaf(-s[kAvg], s[kAvg], s[0]), 0.f);
    }
    const float q = d / (sqrtf(var) + eps);
    if constexpr (MOMENTUM) {
      s[kMom] = fmaf(mu, s[kMom], q);
      w = fmaf(-lr, s[kMom], w);
    } else {
      w = fmaf(-lr, q, w);
    }
  }
};

// torch.optim.Adagrad (lr_decay 0): acc += d^2, p -= lr d / (sqrt(acc) + eps).
struct AdagradRule {
  static constexpr int kStates = 1;   // acc
  float lr, eps, wd, gs;
  __device__ explicit AdagradRule(const float* __restrict__ h)
      : lr(h[kHypLr]), eps(h[kHypEps]), wd(h[kHypWd]), gs(h[kHypGScale]) {}
  __device__ __forceinline__ void operator()(float& w, float g, float* s) const {
    const float d = fmaf(wd, w, g * gs);
    s[0] = fmaf(d, d, s[0]);
    w = fmaf(-lr, d / (sqrtf(s[0]) + eps), w);
  }
};

// torch.optim.Adamax: m = b1 m + (1 - b1) d, u = max(b2 u, |d| + eps), p -= (lr / bc1) m / u.
struct AdamaxRule {
  static constexpr int kStates = 2;   // m, u
  float lr, b1, b2, eps, wd, gs, step;
  __device__ explicit AdamaxRule(const float* __restrict__ h)
      : lr(h[kHypLr]), b1(h[kHypMom]), b2(h[kHypBeta2]), eps(h[kHypEps]), wd(h[kHypWd]), gs(h[kHypGScale]),
        step(lr / h[kHypBc1]) {}
  __device__ __forceinline__ void operator()(float& w, float g, float* s) const {
    const float d = fmaf(wd, w, g * gs);
    s[0] = fmaf(b1, s[0], (1.f - b1) * d);
    s[1] = fmaxf(b2 * s[1], fabsf(d) + eps);
    w = w - step * s[0] / s[1];
  }
};

}  // namespace b200
