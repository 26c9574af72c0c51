// Token-level PPO critic loss of the reasoning workers, forward and backward on the device with no host sync: the
// loss block of MegatronCritic's loss_func (rlinf/workers/critic/megatron_critic_worker.py:92-123) -
// compute_ppo_critic_loss (rlinf/algorithms/losses.py:315-380) with its explained-variance statistics
// (rlinf/utils/metric_utils.py:232-258) - plus autograd's backward for a unit upstream gradient.
//
// Kept from the reference: the aggregation is always masked_mean (compute_ppo_critic_loss ignores the worker's
// loss_agg_func), so an all-masked batch gives the masked sum 0; critic/value_clip_ratio is the unmasked mean over all
// bsz * L cells; the explained-variance sums cover masked cells only.
//
// Four launches, no floating-point atomics, nothing that depends on the SM count:
//   1-2. the token loss's count_kernel and totals_kernel (token_counts.cuh): mask counts per row and in total.
//   3.   critic_main_kernel, one CTA per (segment, row): d values (it needs the total of step 2) and fp64 partial
//        sums per (segment, row), written to fixed slots.
//   4.   critic_finalize_kernel (one CTA): adds the partials in a fixed order and writes the loss and the metrics.
#include "common.cuh"
#include "critic_unit.cuh"
#include "token_counts.cuh"

namespace {

constexpr int kThreads = rb::kTokenThreads;
constexpr int kPerThread = rb::kTokenPerThread;
constexpr int kSeg = rb::kTokenSeg;

enum Slot { C_VL = 0, C_CLIP, C_R, C_R2, C_E, C_E2, kNC };
static_assert(kNC <= rb::kTokenSlots, "the critic's partials fit the token loss's workspace slots");

struct Hyper {
  float value_clip, huber_delta, half_huber_delta;
};

__global__ void __launch_bounds__(kThreads) critic_main_kernel(rb200_token_critic_loss_args a, Hyper h,
                                                               const long long* __restrict__ total,
                                                               double* __restrict__ partials) {
  __shared__ double red[kNC * 32];
  const int64_t row = blockIdx.y, seg = blockIdx.x;
  const long long tot = *total;
  const float coef = (float)(1.0 / (double)(tot > 0 ? tot : 1));  // masked_mean's d mean / d element

  double acc[kNC];
#pragma unroll
  for (int k = 0; k < kNC; ++k) acc[k] = 0.0;

#pragma unroll
  for (int k = 0; k < kPerThread; ++k) {
    const int64_t j = seg * kSeg + k * kThreads + threadIdx.x;
    if (j >= a.L) break;
    const bool m = a.loss_mask[row * a.loss_mask_stride + j] != 0;
    const float mf = m ? 1.0f : 0.0f;
    const float v = a.values[row * a.values_stride + j];
    const float pv = a.prev_values[row * a.prev_values_stride + j];
    const float rt = a.returns[row * a.returns_stride + j];
    const rb::CriticOut o = rb::critic_terms(v, pv, rt, h.value_clip, h.huber_delta, h.half_huber_delta);
    acc[C_VL] += (double)__fmul_rn(o.vl, mf);
    acc[C_CLIP] += rb::critic_clip_hit(o, pv, h.value_clip) ? 1.0 : 0.0;
    if (m) {
      acc[C_R] += (double)rt;
      acc[C_R2] += (double)__fmul_rn(rt, rt);
      acc[C_E] += (double)o.e1;
      acc[C_E2] += (double)__fmul_rn(o.e1, o.e1);
    }
    if (a.d_values) a.d_values[row * a.L + j] = m ? coef * rb::critic_dvl(o, h.value_clip, h.huber_delta) : 0.0f;
  }

  rb::block_sum<kNC>(acc, red);
  if (threadIdx.x == 0) {
    double* p = partials + (row * gridDim.x + seg) * rb::kTokenSlots;
#pragma unroll
    for (int k = 0; k < kNC; ++k) p[k] = acc[k];
  }
}

__global__ void __launch_bounds__(kThreads) critic_finalize_kernel(rb200_token_critic_loss_args a, int nseg,
                                                                   const long long* __restrict__ total,
                                                                   const double* __restrict__ partials) {
  __shared__ double red[kNC * 32];
  double acc[kNC];
#pragma unroll
  for (int k = 0; k < kNC; ++k) acc[k] = 0.0;
  for (int64_t i = threadIdx.x; i < a.bsz; i += blockDim.x) {
    for (int s = 0; s < nseg; ++s) {
      const double* p = partials + (i * nseg + s) * rb::kTokenSlots;
#pragma unroll
      for (int k = 0; k < kNC; ++k) acc[k] += p[k];
    }
  }
  rb::block_sum<kNC>(acc, red);
  if (threadIdx.x != 0) return;
  const long long tot = *total;
  const double loss = acc[C_VL] / (tot > 0 ? (double)tot : 1.0);  // masked_mean, or the plain (zero) sum
  float* M = a.metrics;
  M[RB200_CM_VALUE_LOSS] = (float)loss;
  M[RB200_CM_VALUE_CLIP_RATIO] = (float)(acc[C_CLIP] / ((double)a.bsz * (double)a.L));
  M[RB200_CM_EV_COUNT] = (float)tot;
  M[RB200_CM_EV_RET_SUM] = (float)acc[C_R];
  M[RB200_CM_EV_RET_SQ_SUM] = (float)acc[C_R2];
  M[RB200_CM_EV_ERR_SUM] = (float)acc[C_E];
  M[RB200_CM_EV_ERR_SQ_SUM] = (float)acc[C_E2];
  M[RB200_CM_FINAL_VALUE_LOSS] = (float)loss;
  a.loss[0] = (float)loss;
}

}  // namespace

extern "C" int rb200_token_critic_loss(const rb200_token_critic_loss_args* args, rb200_stream_t stream) {
  if (!args) return RB200_E_NULL;
  const rb200_token_critic_loss_args& a = *args;
  if (!a.values || !a.returns || !a.prev_values || !a.loss_mask || !a.loss || !a.metrics || !a.workspace)
    return RB200_E_NULL;
  const int64_t need = rb200_token_loss_workspace_bytes(a.bsz, a.L);
  if (need < 0) return RB200_E_SHAPE;
  if (a.workspace_bytes < need) return RB200_E_ARG;
  if ((reinterpret_cast<uintptr_t>(a.workspace) & 15) != 0) return RB200_E_ALIGN;
  if (a.values_stride < a.L || a.returns_stride < a.L || a.prev_values_stride < a.L || a.loss_mask_stride < a.L)
    return RB200_E_SHAPE;
  Hyper h;
  h.value_clip = (float)a.value_clip;
  h.huber_delta = (float)a.huber_delta;
  h.half_huber_delta = (float)(0.5 * a.huber_delta);

  cudaStream_t st = rb::as_stream(stream);
  const rb::TokenCounts c = rb::token_mask_counts(a.loss_mask, a.loss_mask_stride, a.bsz, a.L, a.workspace, st);
  critic_main_kernel<<<dim3((unsigned)c.nseg, (unsigned)a.bsz), kThreads, 0, st>>>(a, h, c.total, c.partials);
  rb::count_launch();
  critic_finalize_kernel<<<1, kThreads, 0, st>>>(a, (int)c.nseg, c.total, c.partials);
  rb::count_launch();
  RB_RETURN_LAUNCH();
}
