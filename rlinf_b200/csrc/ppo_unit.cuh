// Per-unit PPO-clip arithmetic of compute_ppo_actor_loss (rlinf/algorithms/losses.py:244-263), shared by the embodied
// loss kernels (ppo_loss.cu) and the token-level reasoning loss (token_loss.cu).
// Elementwise arithmetic mirrors the reference's fp32 op order, so discrete metrics such as clip_fraction agree; the
// gradient follows autograd's rules (torch.max / torch.min split ties in half, clamp passes the gradient at its bounds).
#pragma once

namespace rb {

// One ratio element: returns the aggregated-loss term and the metric terms; dL_dlp = dLoss_e/dlogprob before the
// aggregation coefficient (0 where the mask or a log-ratio clamp blocks it).
struct RatioOut {
  float loss_e, ratio, clipped, dual_ratio, lr_kl, clip_hit, dL_dlp;
};

// H carries clip_lo_bound / clip_hi_bound (fl32(1 - low), fl32(1 + high)), dual_c (<= 0: no dual clip) and the
// log-ratio clamps has_lr_min / lr_min / has_lr_max / lr_max.
template <class H>
__device__ __forceinline__ RatioOut ratio_terms(float lp, float old_lp, float adv, bool m, const H& h) {
  RatioOut o;
  const float lr_raw = __fsub_rn(lp, old_lp);
  float lr = lr_raw;
  bool pass = true;
  if (h.has_lr_min) {
    pass = pass && (lr >= h.lr_min);
    lr = fmaxf(lr, h.lr_min);
  }
  if (h.has_lr_max) {
    pass = pass && (lr <= h.lr_max);
    lr = fminf(lr, h.lr_max);
  }
  const float ratio = m ? expf(lr) : 0.0f;
  o.lr_kl = m ? lr : 0.0f;
  const float clipped = fminf(fmaxf(ratio, h.clip_lo_bound), h.clip_hi_bound);
  const float nadv = -adv;
  const float l1 = __fmul_rn(nadv, ratio), l2 = __fmul_rn(nadv, clipped);
  o.clip_hit = (l1 < l2) ? 1.0f : 0.0f;
  float le = fmaxf(l1, l2);
  // d max(l1,l2)/d ratio  (torch.maximum: ties split 1/2 - 1/2; clamp passes grad inside [lo,hi] inclusive)
  const bool in_range = (ratio >= h.clip_lo_bound) && (ratio <= h.clip_hi_bound);
  const float g1 = l1 > l2 ? 1.0f : (l1 == l2 ? 0.5f : 0.0f);
  const float g2 = l2 > l1 ? 1.0f : (l1 == l2 ? 0.5f : 0.0f);
  float dle = nadv * (g1 + (in_range ? g2 : 0.0f));
  bool dual_hit = false;
  if (h.dual_c > 0.0f) {
    const float sg = adv > 0.0f ? 1.0f : (adv < 0.0f ? -1.0f : 0.0f);
    const float l3 = __fmul_rn(__fmul_rn(sg, h.dual_c), adv);
    dual_hit = l3 < le;
    const float f = le < l3 ? 1.0f : (le == l3 ? 0.5f : 0.0f);  // torch.minimum backward
    le = fminf(le, l3);
    dle *= f;
  }
  o.loss_e = le;
  o.ratio = ratio;
  o.clipped = clipped;
  o.dual_ratio = (dual_hit && m) ? ratio : 0.0f;
  o.dL_dlp = (m && pass) ? dle * ratio : 0.0f;
  return o;
}

}  // namespace rb
