// optim_rules.cuh -- per-entry update rules of the flat optimiser kernels (optim.cu, finetune.cu).
//
// load() reads the step's scalars from the device `hyper` array; apply() takes a live entry's parameter pv and its
// clipped, weight-decayed gradient d, updates the rule's per-entry state (s0, s1) and returns the new parameter.
// Each restates its torch.optim.*.step (torch 2.x, single-tensor path) for one fp32 entry.
#pragma once
#include "common.cuh"

namespace gccb {

// torch.optim.Adam (train.py:667-672).  hyper: [0] lr, [1] 1 - beta1^t, [2] sqrt(1 - beta2^t).
// s0 = exp_avg, s1 = exp_avg_sq.
struct AdamRule {
  float beta1, beta2, eps;
  float lr, bc1, sbc2;
  __device__ __forceinline__ void load(const float* __restrict__ hyper) {
    lr = hyper[0];
    bc1 = hyper[1];
    sbc2 = hyper[2];
  }
  __device__ __forceinline__ float apply(int64_t i, float pv, float d, float* __restrict__ m,
                                         float* __restrict__ v) const {
    float mv = beta1 * m[i] + (1.0f - beta1) * d;
    float vv = beta2 * v[i] + (1.0f - beta2) * d * d;
    m[i] = mv;
    v[i] = vv;
    float denom = sqrtf(vv) / sbc2 + eps;
    return pv - (lr / bc1) * (mv / denom);
  }
};

// torch.optim.SGD with dampening 0 and no Nesterov (train.py:660-665).  hyper: [0] lr.  s0 = momentum_buffer,
// untouched (and may be null) when momentum == 0.
struct SgdRule {
  float momentum;
  float lr;
  __device__ __forceinline__ void load(const float* __restrict__ hyper) { lr = hyper[0]; }
  __device__ __forceinline__ float apply(int64_t i, float pv, float d, float* __restrict__ buf,
                                         float* __restrict__) const {
    if (momentum != 0.f) {
      // torch starts the buffer as a copy of d on the first step.  With dampening 0, a buffer that starts
      // at zero gives momentum * 0 + d = d, the same value, so the kernel needs no first-step branch.
      d = momentum * buf[i] + d;
      buf[i] = d;
    }
    return pv - lr * d;
  }
};

// torch.optim.Adagrad with initial_accumulator_value 0 (train.py:674-678).  hyper: [0] clr =
// lr / (1 + (t - 1) * lr_decay), computed in double on the host.  s0 = sum.
struct AdagradRule {
  float eps;
  float clr;
  __device__ __forceinline__ void load(const float* __restrict__ hyper) { clr = hyper[0]; }
  __device__ __forceinline__ float apply(int64_t i, float pv, float d, float* __restrict__ sum,
                                         float* __restrict__) const {
    float s = sum[i] + d * d;
    sum[i] = s;
    return pv - clr * (d / (sqrtf(s) + eps));
  }
};

// The step every optimiser takes on one live entry once its gradient gv is clipped: torch.optim's L2 weight decay
// (grad + weight_decay * p) folded into the gradient, then the rule's update.  Returns the new parameter.
template <class Rule>
__device__ __forceinline__ float decay_and_update(const Rule& rule, int64_t i, float pv, float gv, float wd,
                                                  float* __restrict__ s0, float* __restrict__ s1) {
  return rule.apply(i, pv, fmaf(wd, pv, gv), s0, s1);
}

}  // namespace gccb
