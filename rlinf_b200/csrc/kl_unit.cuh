// kl_penalty(a, b, kind) of rlinf/algorithms/utils.py:26-64 for one element, shared by the kl_penalty kernel
// (misc.cu), the reinforce++ returns (adv_extra.cu) and the token-level reasoning loss (token_loss.cu).
#pragma once

namespace rb {

// mode 0: k1 / kl (a - b), 1: abs, 2: k2 / mse (0.5 (a - b)^2), 3: k3 / low_var_kl (clamps +-20 / +-10).
// Returns the penalty; g = d penalty / d a.  Every kind is a function of a - b, so d penalty / d b = -g.
__device__ __forceinline__ float kl_penalty_unit(float a, float b, int mode, float& g) {
  float v;
  if (mode == 0) {
    v = __fsub_rn(a, b);
    g = 1.0f;
  } else if (mode == 1) {
    const float d = __fsub_rn(a, b);
    v = fabsf(d);
    g = d > 0.f ? 1.0f : (d < 0.f ? -1.0f : 0.0f);
  } else if (mode == 2) {
    const float d = __fsub_rn(a, b);
    v = __fmul_rn(0.5f, __fmul_rn(d, d));
    g = d;
  } else {
    const float raw = __fsub_rn(b, a);
    const float kl = fminf(fmaxf(raw, -20.0f), 20.0f);
    const float ratio = expf(kl);
    const float kld = __fsub_rn(__fsub_rn(ratio, kl), 1.0f);
    v = fminf(fmaxf(kld, -10.0f), 10.0f);
    const bool pass = (raw >= -20.0f && raw <= 20.0f) && (kld >= -10.0f && kld <= 10.0f);
    g = pass ? -(ratio - 1.0f) : 0.0f;  // d kld / d a = (ratio - 1) * d kl / d a, d kl / d a = -1
  }
  return v;
}

// True where a k3 clamp blocks the gradient: torch.clamp's backward writes 0 there whatever the upstream gradient,
// NaN included, so a caller that scales g by a non-finite upstream gradient must test this first.
__device__ __forceinline__ bool kl_penalty_blocked(float a, float b, int mode) {
  if (mode != 3) return false;
  const float raw = __fsub_rn(b, a);
  const float kl = fminf(fmaxf(raw, -20.0f), 20.0f);
  const float kld = __fsub_rn(__fsub_rn(expf(kl), kl), 1.0f);
  return !((raw >= -20.0f && raw <= 20.0f) && (kld >= -10.0f && kld <= 10.0f));
}

}  // namespace rb
