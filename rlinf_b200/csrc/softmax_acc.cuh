// Running softmax statistics of one row, shared by the logits kernels (logits.cu) and the fused LM-head kernels
// (lmhead.cu): (max m, s = sum exp(z - m), t = sum exp(z - m) * (z - m)), everything relative to the max, so the entropy
// log s - t / s has no cancellation for near-deterministic rows.  Entries outside the vocabulary window carry -inf.
#pragma once
#include <math.h>
#include <stdint.h>

namespace rb {
namespace smx {

struct Acc {
  float m, s, t;
};
__device__ __forceinline__ void acc_init(Acc& a) {
  a.m = -INFINITY;
  a.s = 0.f;
  a.t = 0.f;
}
// move the reference point of (s, t) from a.m to m (m >= a.m)
__device__ __forceinline__ void acc_rebase(Acc& a, float m) {
  if (a.m == -INFINITY) {  // empty: nothing to move
    a.m = m;
    return;
  }
  const float d = a.m - m;  // <= 0
  const float f = __expf(d);
  a.t = f * (a.t + a.s * d);
  a.s = f * a.s;
  a.m = m;
}
__device__ __forceinline__ void acc_merge(Acc& a, Acc b) {
  const float m = fmaxf(a.m, b.m);
  if (m == -INFINITY) return;  // both empty
  acc_rebase(a, m);
  acc_rebase(b, m);
  a.s += b.s;
  a.t += b.t;
}
// add 4 values (already scaled); entries outside the window carry -inf
__device__ __forceinline__ void acc_add4(Acc& a, float z0, float z1, float z2, float z3) {
  const float mx = fmaxf(fmaxf(z0, z1), fmaxf(z2, z3));
  if (mx == -INFINITY) return;
  if (mx > a.m) acc_rebase(a, mx);
  const float d0 = z0 - a.m, d1 = z1 - a.m, d2 = z2 - a.m, d3 = z3 - a.m;
  const float e0 = __expf(d0), e1 = __expf(d1), e2 = __expf(d2), e3 = __expf(d3);
  a.s += (e0 + e1) + (e2 + e3);
  // exp underflow / -inf entries: e = 0 and 0 * -inf would be NaN -> select (the reference's where(p > 0, ., 0))
  a.t += ((e0 > 0.f ? e0 * d0 : 0.f) + (e1 > 0.f ? e1 * d1 : 0.f)) + ((e2 > 0.f ? e2 * d2 : 0.f) + (e3 > 0.f ? e3 * d3 : 0.f));
}
__device__ __forceinline__ Acc warp_merge(Acc a) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    Acc b;
    b.m = __shfl_xor_sync(0xffffffffu, a.m, o);
    b.s = __shfl_xor_sync(0xffffffffu, a.s, o);
    b.t = __shfl_xor_sync(0xffffffffu, a.t, o);
    acc_merge(a, b);
  }
  return a;
}

// Row finish of row r: logprob = z_target - lse (-inf when the target lies outside the window), entropy = log s - t / s
// and lse (entropy, lse nullable)
__device__ __forceinline__ void finish_row(const Acc& acc, float z_t, bool t_in, int64_t r, float* logprob,
                                           float* entropy, float* lse) {
  const float ls = logf(acc.s);
  const float lse_r = acc.m + ls;
  logprob[r] = t_in ? (z_t - acc.m) - ls : -INFINITY;
  if (entropy) entropy[r] = ls - acc.t / acc.s;
  if (lse) lse[r] = lse_r;
}

// Gradient w.r.t. one logit x (z = x * inv_T) given the row's lse, entropy H and upstream gradients g_lp / g_H:
//   inv_T * (g_lp * (1[i = target] - p_i) - g_H * p_i * (log p_i + H))
__device__ __forceinline__ float dz_of(float x, float inv_t, float lse, float glp, float gh, float H, bool is_target) {
  const float z = x * inv_t;
  const float lp = z - lse;
  const float p = __expf(lp);
  float g = -glp * p;
  if (gh != 0.f && p > 0.f) g -= gh * p * (lp + H);
  if (is_target) g += glp;
  return g * inv_t;
}

}  // namespace smx
}  // namespace rb
