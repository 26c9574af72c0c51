// Per-unit arithmetic of compute_ppo_critic_loss (rlinf/algorithms/losses.py:315-380) and its explained-variance
// terms (rlinf/utils/metric_utils.py:232-258), in the reference's fp32 op order, shared by the embodied PPO loss
// (ppo_loss.cu) and the token-level critic loss of the reasoning workers (token_critic_loss.cu).
#pragma once
#include <cuda_runtime.h>

namespace rb {

// huber_loss(e, delta): 0.5 e^2 inside |e| < delta, delta (|e| - delta / 2) outside
__device__ __forceinline__ float huber(float e, float delta, float half_delta) {
  const float a = fabsf(e);
  return a < delta ? __fmul_rn(0.5f, __fmul_rn(e, e)) : __fmul_rn(delta, __fsub_rn(a, half_delta));
}
// d huber / d e as autograd computes it (sign(e) * delta outside, 0 at e == 0)
__device__ __forceinline__ float huber_grad(float e, float delta) {
  const float a = fabsf(e);
  return a < delta ? e : (e > 0.0f ? delta : (e < 0.0f ? -delta : 0.0f));
}

struct CriticOut {
  float dv;      // values - prev_values
  float vpc;     // value_pred_clipped = prev_values + clamp(dv, -value_clip, value_clip)
  float e1;      // returns - values: the unclipped error, also the EV error term
  float e2;      // returns - value_pred_clipped
  float lo, lc;  // huber of e1 / e2
  float vl;      // max(lo, lc)
};

__device__ __forceinline__ CriticOut critic_terms(float v, float pv, float rt, float value_clip, float delta,
                                                  float half_delta) {
  CriticOut o;
  o.dv = __fsub_rn(v, pv);
  const float dvc = fminf(fmaxf(o.dv, -value_clip), value_clip);
  o.vpc = __fadd_rn(pv, dvc);
  o.e1 = __fsub_rn(rt, v);
  o.e2 = __fsub_rn(rt, o.vpc);
  o.lo = huber(o.e1, delta, half_delta);
  o.lc = huber(o.e2, delta, half_delta);
  o.vl = fmaxf(o.lo, o.lc);
  return o;
}

// value_clip_indicator: (value_pred_clipped - prev_values).abs() > value_clip
__device__ __forceinline__ bool critic_clip_hit(const CriticOut& o, float pv, float value_clip) {
  return fabsf(__fsub_rn(o.vpc, pv)) > value_clip;
}

// d max(lo, lc) / d values: torch.max splits a tie evenly, clamp passes the gradient inside [-clip, clip]
__device__ __forceinline__ float critic_dvl(const CriticOut& o, float value_clip, float delta) {
  const float g1 = o.lo > o.lc ? 1.0f : (o.lo == o.lc ? 0.5f : 0.0f);
  const float g2 = o.lc > o.lo ? 1.0f : (o.lo == o.lc ? 0.5f : 0.0f);
  const bool pass_c = (o.dv >= -value_clip) && (o.dv <= value_clip);
  return -(g1 * huber_grad(o.e1, delta)) - (pass_c ? g2 * huber_grad(o.e2, delta) : 0.0f);
}

}  // namespace rb
