// K2: fused (gather +) PPO actor[-critic] loss, forward AND backward in one pass over the micro-batch.
// Reference: policy_loss (rlinf/algorithms/registry.py:77-92) -> preprocess_loss_inputs
// (algorithms/utils.py:280-376) -> compute_ppo_actor_loss (losses.py:170-312) +
// compute_ppo_critic_loss (losses.py:315-380) [+ entropy term and 1/grad_accum,
// workers/actor/embodied_fsdp_actor_worker.py:678-695] -> autograd backward.
// The reference runs ~40 eager elementwise/reduction ops plus their autograd graph, and one host sync
// per metric (.item()); here: one optional 1-byte/unit pre-pass (mask count) and ONE fused kernel that reads
// every input once, writes the gradients, and whose last CTA to finish forms loss + metrics and clears the
// reduction workspace for the next call (no memset node, no finalise node: round 1 spent three graph nodes on a
// 32 MB problem).
//
// Algorithmic HBM bytes per sample (action_level, C=1, A=8): idx 8 + logp 32 + old_logp 32 + adv/ret/V/prevV 16
// (+mask 1) read, dlogp 32 + dV 4 written = 124 (125) B.
//
// Elementwise arithmetic mirrors the reference's fp32 op order (so discrete metrics such as
// clip_fraction agree); the reductions accumulate in fp64.
#include "common.cuh"
#include "critic_unit.cuh"
#include "ppo_unit.cuh"

namespace {

enum SumSlot {
  S_CNT = 0,   // sum of mask over units (pre-pass)
  S_L,         // sum of aggregated policy-loss terms
  S_LABS,
  S_RATIO,
  S_RABS,
  S_CLIPPED,
  S_DUAL,
  S_KL,
  S_CLIPFRAC,
  S_VL,
  S_VCLIP,
  S_EV_N,
  S_EV_R,
  S_EV_R2,
  S_EV_E,
  S_EV_E2,
  S_ENT,
  S_NUM
};
static_assert(S_NUM <= 32, "workspace is 32 doubles");

struct Hyper {
  float clip_lo_bound, clip_hi_bound;  // fl32(1 - low), fl32(1 + high)
  float dual_c;                        // <=0: off
  int has_lr_min, has_lr_max;
  float lr_min, lr_max;
  float value_clip, huber_delta, half_huber_delta;
  float max_episode_steps;  // 0: masked_mean aggregation
  int critic_warmup;
  float entropy_bonus, loss_scale;
  float adv_eps;
};

__global__ void __launch_bounds__(256) mask_count_kernel(const uint8_t* __restrict__ mask,
                                                         const int64_t* __restrict__ idx, int64_t bsz, int U,
                                                         double* __restrict__ sums) {
  __shared__ double red[32];
  double v[1] = {0.0};
  const int64_t n_units = bsz * U;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t u = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; u < n_units; u += stride) {
    const int64_t i = u / U;
    const int c = (int)(u - i * U);
    const int64_t row = idx ? idx[i] : i;
    v[0] += mask[row * U + c] ? 1.0 : 0.0;
  }
  rb::block_sum<1>(v, red);
  if (threadIdx.x == 0 && v[0] != 0.0) atomicAdd(&sums[S_CNT], v[0]);
}

using rb::RatioOut;
using rb::ratio_terms;

__device__ void ppo_finalize(const rb200_ppo_args& a, const Hyper& h, int U, int g, int token_mode, const double* sums);

template <bool TOKEN>
__global__ void __launch_bounds__(256, 3) ppo_main_kernel(rb200_ppo_args a, Hyper h, int U, int g,
                                                       double* __restrict__ sums) {
  __shared__ double red[S_NUM * 32];
  __shared__ int is_last_sh;
  // per-thread partial sums in fp32 (a thread sees only a handful of units), widened to fp64 for the block/grid sums
  float acc[S_NUM];
#pragma unroll
  for (int k = 0; k < S_NUM; ++k) acc[k] = 0.0f;

  const int64_t n_units = a.bsz * U;
  const bool has_mask = a.loss_mask != nullptr;
  const bool ratio_agg = has_mask && a.loss_mask_sum != nullptr && h.max_episode_steps > 0.0f;
  const double n_elems = (double)n_units * (TOKEN ? g : 1);
  // aggregation coefficients (d loss / d term)
  const double mask_cnt = has_mask ? sums[S_CNT] : 0.0;
  float coef_actor, coef_unit;
  if (ratio_agg) {
    coef_actor = (float)(1.0 / n_elems);
    coef_unit = (float)(1.0 / (double)n_units);
  } else if (has_mask) {
    const double d = mask_cnt > 0.0 ? mask_cnt : 1.0;  // all-masked: masked_mean returns the plain sum (=0)
    coef_actor = (float)(1.0 / d);
    coef_unit = coef_actor;
  } else {
    coef_actor = (float)(1.0 / n_elems);
    coef_unit = (float)(1.0 / (double)n_units);
  }
  // deferred advantage normalisation (safe_normalize fused into the consumer)
  bool norm_adv = false;
  float adv_mean = 0.0f, adv_den = 1.0f;
  if (a.adv_stats != nullptr && a.adv_stats[0] > 0.0) {
    const double cnt = a.adv_stats[0];
    const double mean_d = a.adv_stats[1] / cnt;
    const double var_d = (a.adv_stats[2] - a.adv_stats[1] * mean_d) / (cnt - 1.0);
    adv_mean = (float)mean_d;
    adv_den = __fadd_rn((float)sqrt(var_d > 0.0 || !(var_d == var_d) ? var_d : 0.0), h.adv_eps);
    norm_adv = true;
  }
  const float scale = h.loss_scale;
  const bool vec4 = ((g & 3) == 0) &&
                    (((reinterpret_cast<uintptr_t>(a.logprobs) | reinterpret_cast<uintptr_t>(a.old_logprobs) |
                       reinterpret_cast<uintptr_t>(a.d_logprobs)) & 15) == 0);

  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t u = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; u < n_units; u += stride) {
    const int64_t i = u / U;
    const int c = (int)(u - i * U);
    const int64_t row = a.idx ? a.idx[i] : i;
    const int64_t so = row * U + c;
    const bool m = has_mask ? (a.loss_mask[so] != 0) : true;
    const float mf = m ? 1.0f : 0.0f;
    float adv = a.advantages[so];
    if (norm_adv) adv = __fdiv_rn(__fsub_rn(adv, adv_mean), adv_den);
    float w = 1.0f;
    if (ratio_agg) {
      const int64_t ms_row = a.mask_sum_row_mod > 0 ? (row % a.mask_sum_row_mod) : row;
      w = __fdiv_rn((float)a.loss_mask_sum[ms_row * U + c], h.max_episode_steps);
    }
    const float* lp_cur = a.logprobs + u * g;
    const float* lp_old = a.old_logprobs + so * g;
    float* dlp = a.d_logprobs ? a.d_logprobs + u * g : nullptr;

    if (TOKEN) {
      for (int k = 0; k < g; ++k) {
        const RatioOut o = ratio_terms(lp_cur[k], lp_old[k], adv, m, h);
        const float term = ratio_agg ? __fmul_rn(__fdiv_rn(o.loss_e, w), mf) : __fmul_rn(o.loss_e, mf);
        const float term_abs = ratio_agg ? __fmul_rn(__fdiv_rn(fabsf(o.loss_e), w), mf) : __fmul_rn(fabsf(o.loss_e), mf);
        acc[S_L] += term;
        acc[S_LABS] += term_abs;
        acc[S_RATIO] += (o.ratio * mf);
        acc[S_RABS] += (fabsf(__fsub_rn(o.ratio, 1.0f)) * mf);
        acc[S_CLIPPED] += (o.clipped * mf);
        acc[S_DUAL] += (o.dual_ratio * mf);
        acc[S_KL] += o.lr_kl;
        acc[S_CLIPFRAC] += (o.clip_hit * mf);
        if (dlp) {
          const float cw = ratio_agg ? coef_actor / w : coef_actor;
          dlp[k] = h.critic_warmup ? 0.0f : scale * cw * o.dL_dlp;
        }
      }
    } else {
      float lp = 0.0f, old = 0.0f;
      if (vec4) {  // 16-byte loads, same left-to-right summation order
        for (int k = 0; k < g; k += 4) {
          const float4 c4 = *reinterpret_cast<const float4*>(lp_cur + k);
          const float4 o4 = __ldg(reinterpret_cast<const float4*>(lp_old + k));
          lp = __fadd_rn(__fadd_rn(__fadd_rn(__fadd_rn(lp, c4.x), c4.y), c4.z), c4.w);
          old = __fadd_rn(__fadd_rn(__fadd_rn(__fadd_rn(old, o4.x), o4.y), o4.z), o4.w);
        }
      } else {
        for (int k = 0; k < g; ++k) {
          lp = __fadd_rn(lp, lp_cur[k]);
          old = __fadd_rn(old, lp_old[k]);
        }
      }
      const RatioOut o = ratio_terms(lp, old, adv, m, h);
      const float term = ratio_agg ? __fmul_rn(__fdiv_rn(o.loss_e, w), mf) : __fmul_rn(o.loss_e, mf);
      const float term_abs = ratio_agg ? __fmul_rn(__fdiv_rn(fabsf(o.loss_e), w), mf) : __fmul_rn(fabsf(o.loss_e), mf);
      acc[S_L] += term;
      acc[S_LABS] += term_abs;
      acc[S_RATIO] += (o.ratio * mf);
      acc[S_RABS] += (fabsf(__fsub_rn(o.ratio, 1.0f)) * mf);
      acc[S_CLIPPED] += (o.clipped * mf);
      acc[S_DUAL] += (o.dual_ratio * mf);
      acc[S_KL] += o.lr_kl;
      acc[S_CLIPFRAC] += (o.clip_hit * mf);
      if (dlp) {
        const float cw = ratio_agg ? coef_actor / w : coef_actor;
        const float gval = h.critic_warmup ? 0.0f : scale * cw * o.dL_dlp;
        if (vec4) {
          const float4 g4 = make_float4(gval, gval, gval, gval);
          for (int k = 0; k < g; k += 4) *reinterpret_cast<float4*>(dlp + k) = g4;
        } else {
          for (int k = 0; k < g; ++k) dlp[k] = gval;
        }
      }
    }

    if (a.with_critic) {
      const float v = a.values[u], pv = a.prev_values[so], rt = a.returns[so];
      const rb::CriticOut o = rb::critic_terms(v, pv, rt, h.value_clip, h.huber_delta, h.half_huber_delta);
      const float vl = o.vl;
      const float term = has_mask ? (ratio_agg ? __fmul_rn(__fdiv_rn(vl, w), mf) : __fmul_rn(vl, mf)) : vl;
      acc[S_VL] += term;
      acc[S_VCLIP] += rb::critic_clip_hit(o, pv, h.value_clip) ? 1.0f : 0.0f;
      if (m) {
        acc[S_EV_N] += 1.0f;
        acc[S_EV_R] += rt;
        acc[S_EV_R2] += __fmul_rn(rt, rt);
        acc[S_EV_E] += o.e1;
        acc[S_EV_E2] += __fmul_rn(o.e1, o.e1);
      }
      if (a.d_values) {
        const float dvl = rb::critic_dvl(o, h.value_clip, h.huber_delta);
        const float cw = has_mask ? (ratio_agg ? coef_unit / w : coef_unit) * mf : coef_unit;
        a.d_values[u] = scale * cw * dvl;
      }
    }

    if (a.entropy) {
      const float* en = a.entropy + u * g;
      float es = 0.0f;
      for (int k = 0; k < g; ++k) es = __fadd_rn(es, en[k]);
      acc[S_ENT] += (has_mask ? __fmul_rn(es, mf) : es);
      if (a.d_entropy) {
        const float cw = (has_mask ? coef_unit * mf : (float)(1.0 / (double)n_units));
        const float gval = (h.entropy_bonus > 0.0f && !h.critic_warmup) ? -scale * h.entropy_bonus * cw : 0.0f;
        float* de = a.d_entropy + u * g;
        for (int k = 0; k < g; ++k) de[k] = gval;
      }
    }
  }

  double accd[S_NUM];
#pragma unroll
  for (int k = 0; k < S_NUM; ++k) accd[k] = (double)acc[k];
  rb::block_sum<S_NUM>(accd, red);
  if (threadIdx.x == 0) {
#pragma unroll
    for (int k = 1; k < S_NUM; ++k)  // slot 0 (mask count) belongs to the pre-pass
      if (accd[k] != 0.0) atomicAdd(&sums[k], accd[k]);
    // last CTA to arrive finalises (threadFenceReduction pattern); slot 31 of the workspace is the arrival counter
    __threadfence();
    const unsigned long long prev = atomicAdd(reinterpret_cast<unsigned long long*>(sums + 31), 1ull);
    is_last_sh = (prev == (unsigned long long)gridDim.x - 1ull) ? 1 : 0;
    if (is_last_sh) {
      __threadfence();
      double fin[S_NUM];
#pragma unroll
      for (int k = 0; k < S_NUM; ++k) fin[k] = __ldcg(&sums[k]);
      ppo_finalize(a, h, U, g, TOKEN ? 1 : 0, fin);
      // self-cleaning workspace: the next call on this stream starts from zeros without a memset node
#pragma unroll
      for (int k = 0; k < S_NUM; ++k) sums[k] = 0.0;
      *reinterpret_cast<unsigned long long*>(sums + 31) = 0ull;
    }
  }
}

__device__ void ppo_finalize(const rb200_ppo_args& a, const Hyper& h, int U, int g, int token_mode, const double* sums) {
  const double n_units = (double)(a.bsz * U);
  const double n_elems = n_units * (token_mode ? g : 1);
  const bool has_mask = a.loss_mask != nullptr;
  const bool ratio_agg = has_mask && a.loss_mask_sum != nullptr && h.max_episode_steps > 0.0f;
  const double mcnt = has_mask ? sums[S_CNT] : 0.0;
  const bool all_masked = has_mask && mcnt == 0.0;
  // count_nonzero(loss_mask) or 1, at the preprocessed mask shape (units; ones_like(logprobs) if None)
  const double cnt = has_mask ? (mcnt > 0.0 ? mcnt : 1.0) : n_elems;
  // masked_mean denominators: the loss uses the un-expanded mask, the ratio metrics the expanded one
  const double d_loss = ratio_agg ? n_elems : (has_mask ? (all_masked ? 1.0 : mcnt) : n_elems);
  const double d_metric = has_mask ? (all_masked ? 1.0 : mcnt * (token_mode ? g : 1)) : n_elems;
  const double d_unit = ratio_agg ? n_units : (has_mask ? (all_masked ? 1.0 : mcnt) : n_units);
  const double d_ent = has_mask ? (all_masked ? 1.0 : mcnt) : n_units;

  float* M = a.metrics;
  for (int k = 0; k < RB200_NUM_METRICS; ++k) M[k] = 0.0f;
  double policy_loss = sums[S_L] / d_loss;
  if (h.critic_warmup) policy_loss = 0.0;
  M[RB200_M_POLICY_LOSS] = (float)policy_loss;
  M[RB200_M_POLICY_LOSS_ABS] = (float)(sums[S_LABS] / d_loss);
  M[RB200_M_RATIO] = (float)(sums[S_RATIO] / d_metric);
  M[RB200_M_RATIO_ABS] = (float)(sums[S_RABS] / d_metric);
  M[RB200_M_CLIPPED_RATIO] = (float)(sums[S_CLIPPED] / d_metric);
  M[RB200_M_DUAL_CLIPPED_RATIO] = (float)(sums[S_DUAL] / d_metric);
  M[RB200_M_APPROX_KL] = (float)(-sums[S_KL] / cnt);
  M[RB200_M_CLIP_FRACTION] = (float)(sums[S_CLIPFRAC] / cnt);
  M[RB200_M_TOKEN_NUM] = (float)(has_mask ? mcnt : n_elems);
  double total = policy_loss;
  if (a.with_critic) {
    const double vl = sums[S_VL] / d_unit;
    M[RB200_M_VALUE_LOSS] = (float)vl;
    M[RB200_M_VALUE_CLIP_RATIO] = (float)(sums[S_VCLIP] / n_units);
    M[RB200_M_EV_COUNT] = (float)sums[S_EV_N];
    M[RB200_M_EV_RET_SUM] = (float)sums[S_EV_R];
    M[RB200_M_EV_RET_SQ_SUM] = (float)sums[S_EV_R2];
    M[RB200_M_EV_ERR_SUM] = (float)sums[S_EV_E];
    M[RB200_M_EV_ERR_SQ_SUM] = (float)sums[S_EV_E2];
    total += vl;
  }
  if (a.entropy) {
    const double ent = sums[S_ENT] / d_ent;
    if (h.entropy_bonus > 0.0f && !h.critic_warmup) {
      M[RB200_M_ENTROPY] = (float)ent;
      total -= (double)h.entropy_bonus * ent;
    }
  }
  total *= (double)h.loss_scale;
  M[RB200_M_TOTAL_LOSS] = (float)total;
  if (a.loss) a.loss[0] = (float)total;
}

__global__ void __launch_bounds__(256) scale_kernel(float* __restrict__ x, int64_t n, float s) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) x[i] *= s;
}

__global__ void __launch_bounds__(256) scale_by_kernel(float* __restrict__ x, int64_t n, const float* __restrict__ s) {
  const float sv = *s;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) x[i] *= sv;
}

}  // namespace

extern "C" int rb200_ppo_loss(const rb200_ppo_args* args, rb200_stream_t stream) {
  if (!args) return RB200_E_NULL;
  const rb200_ppo_args& a = *args;
  if (!a.logprobs || !a.old_logprobs || !a.advantages || !a.metrics || !a.workspace) return RB200_E_NULL;
  if (a.bsz <= 0 || a.C <= 0 || a.A <= 0) return RB200_E_SHAPE;
  if (a.logprob_type < RB200_LOGPROB_TOKEN || a.logprob_type > RB200_LOGPROB_CHUNK) return RB200_E_ARG;
  if (a.with_critic && (!a.values || !a.returns || !a.prev_values)) return RB200_E_NULL;
  if (a.clip_ratio_c > 0.0 && !(a.clip_ratio_c > 1.0)) return RB200_E_ARG;  // losses.py:260 assert
  if (a.d_entropy && !a.entropy) return RB200_E_NULL;
  const int U = a.logprob_type == RB200_LOGPROB_CHUNK ? 1 : a.C;
  const int g = a.logprob_type == RB200_LOGPROB_CHUNK ? a.C * a.A : a.A;
  if (a.entropy && a.logprob_type == RB200_LOGPROB_CHUNK && a.C != 1) return RB200_E_UNSUPPORTED;

  Hyper h;
  h.clip_lo_bound = (float)(1.0 - a.clip_ratio_low);
  h.clip_hi_bound = (float)(1.0 + a.clip_ratio_high);
  h.dual_c = a.clip_ratio_c > 0.0 ? (float)a.clip_ratio_c : 0.0f;
  h.has_lr_min = a.has_clip_log_ratio_min;
  h.has_lr_max = a.has_clip_log_ratio_max;
  h.lr_min = (float)a.clip_log_ratio_min;
  h.lr_max = (float)a.clip_log_ratio_max;
  h.value_clip = (float)a.value_clip;
  h.huber_delta = (float)a.huber_delta;
  h.half_huber_delta = (float)(0.5 * a.huber_delta);
  h.max_episode_steps = a.max_episode_steps > 0 ? (float)a.max_episode_steps : 0.0f;
  h.critic_warmup = a.critic_warmup;
  h.entropy_bonus = (float)a.entropy_bonus;
  h.loss_scale = (float)a.loss_scale;
  h.adv_eps = a.adv_norm_eps;

  cudaStream_t st = rb::as_stream(stream);
  const int64_t n_units = a.bsz * U;
  int64_t blocks = (n_units + 255) / 256;
  const int64_t cap = (int64_t)rb::sm_count() * 3;  // one resident wave at 3 blocks / SM (80 registers)
  if (blocks > cap) blocks = cap;
  if (a.loss_mask) {
    mask_count_kernel<<<(int)blocks, 256, 0, st>>>(a.loss_mask, a.idx, a.bsz, U, a.workspace);
    rb::count_launch();
  }
  if (a.logprob_type == RB200_LOGPROB_TOKEN)
    ppo_main_kernel<true><<<(int)blocks, 256, 0, st>>>(a, h, U, g, a.workspace);
  else
    ppo_main_kernel<false><<<(int)blocks, 256, 0, st>>>(a, h, U, g, a.workspace);
  rb::count_launch();
  RB_RETURN_LAUNCH();
}

extern "C" int rb200_scale(float* x, int64_t n, float s, rb200_stream_t stream) {
  if (!x) return RB200_E_NULL;
  if (n <= 0) return RB200_E_SHAPE;
  int64_t blocks = (n + 255) / 256;
  const int64_t cap = (int64_t)rb::sm_count() * 8;
  if (blocks > cap) blocks = cap;
  scale_kernel<<<(int)blocks, 256, 0, rb::as_stream(stream)>>>(x, n, s); rb::count_launch();
  RB_RETURN_LAUNCH();
}

extern "C" int rb200_scale_by(float* x, int64_t n, const float* s_dev, rb200_stream_t stream) {
  if (!x || !s_dev) return RB200_E_NULL;
  if (n <= 0) return RB200_E_SHAPE;
  int64_t blocks = (n + 255) / 256;
  const int64_t cap = (int64_t)rb::sm_count() * 8;
  if (blocks > cap) blocks = cap;
  scale_by_kernel<<<(int)blocks, 256, 0, rb::as_stream(stream)>>>(x, n, s_dev); rb::count_launch();
  RB_RETURN_LAUNCH();
}
