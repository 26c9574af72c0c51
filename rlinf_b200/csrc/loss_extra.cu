// Remaining policy losses of LOSS_REGISTRY (SURVEY 8(f) rank 4), same fused forward+backward structure as ppo_loss.cu:
//   * "decoupled_actor_critic": compute_decoupled_ppo_actor_loss (rlinf/algorithms/losses.py:27-167) +
//     compute_ppo_critic_loss (:315-380), registered at :383-394 - PPO clipped around a PROXIMAL policy (given, or
//     interpolated between behaviour and current policy from the weight versions), importance weight
//     exp(proximal - old) towards the behaviour policy with an optional cut-off.
//   * "opd": compute_opd_actor_loss (:427-505) - -logp * stop_grad(dense reverse-KL reward).
// The decoupled loss also folds in the worker's entropy bonus (async_ppo_fsdp_worker.py:443-456), and its weight version
// is either a per-token tensor (rb200_decoupled_ppo_loss) or one scalar for the whole batch
// (rb200_decoupled_ppo_loss_scalar_version).
// One pre-pass (mask / behaviour-mask counts: the masked-mean denominators are needed by the gradient), one main pass
// whose last CTA forms loss + metrics and clears the workspace.
#include "common.cuh"

namespace {

enum DSlot {
  D_CNT = 0,   // count_nonzero(loss_mask) at the preprocessed (un-expanded) shape            [pre-pass]
  D_BCNT,      // count_nonzero(behav_mask) (expanded over tokens iff a threshold is given)    [pre-pass]
  D_L,         // sum of aggregated loss terms
  D_PR,        // sum prox_ratio * mask (elements)
  D_CPR,       // sum clipped * mask
  D_CLIP,      // count (l1 < l2) & mask
  D_DUAL,      // count dual_hit & mask
  D_PKL,       // sum where(mask, lp - prox, 0)
  D_BKL,       // sum where(bmask, prox - old, 0)
  D_VER,       // sum versions over mask (units)
  D_VL, D_VCLIP, D_EV_N, D_EV_R, D_EV_R2, D_EV_E, D_EV_E2,
  D_ENT,       // sum of per-unit entropy (summed over the unit's tokens) over the mask
  D_NUM
};
static_assert(D_NUM <= 31, "workspace is 32 doubles, slot 31 is the arrival counter");

struct DHyper {
  float clip_lo, clip_hi, dual_c;
  float value_clip, huber_delta, half_huber_delta, max_episode_steps;
  int critic_warmup;
  float loss_scale, entropy_bonus;
  int has_version, has_thr;
  float cur_version, prox_version, thr;
};

__device__ __forceinline__ float huber(float e, float delta, float half_delta) {
  const float a = fabsf(e);
  return a < delta ? __fmul_rn(0.5f, __fmul_rn(e, e)) : __fmul_rn(delta, __fsub_rn(a, half_delta));
}
__device__ __forceinline__ float huber_grad(float e, float delta) {
  const float a = fabsf(e);
  return a < delta ? e : (e > 0.0f ? delta : (e < 0.0f ? -delta : 0.0f));
}

// proximal log-prob of one (reduced) entry: given | old | old + alpha (lp - old) with alpha from the weight versions
__device__ __forceinline__ float proximal(float lp, float old, const float* prox_ptr, float prox_sum, float version,
                                          bool have_versions, const DHyper& h) {
  if (prox_ptr != nullptr) return prox_sum;
  if (!have_versions || !h.has_version) return old;
  const float diff = __fsub_rn(h.cur_version, version);
  const float gap = __fsub_rn(h.prox_version, version);
  float alpha = (diff > 0.0f && version >= 0.0f) ? __fdiv_rn(gap, diff) : 0.0f;
  alpha = fminf(fmaxf(alpha, 0.0f), 1.0f);
  return __fadd_rn(old, __fmul_rn(alpha, __fsub_rn(lp, old)));
}

struct DArgs {
  rb200_ppo_args b;
  const float* prox;
  const float* versions;  // per-token versions, or NULL
  int has_versions;       // versions != NULL, or the scalar `ver_scalar` stands for every token
  float ver_scalar;
};

// reduced (lp, old, prox-sum, version) of unit u / element k
template <bool TOKEN>
__device__ __forceinline__ void load_entry(const DArgs& a, int64_t u, int64_t so, int g, int k, float& lp, float& old,
                                           float& psum, float& ver) {
  const float* lp_cur = a.b.logprobs + u * g;
  const float* lp_old = a.b.old_logprobs + so * g;
  const float* pp = a.prox ? a.prox + so * g : nullptr;
  if (TOKEN) {
    lp = lp_cur[k];
    old = lp_old[k];
    psum = pp ? pp[k] : 0.0f;
    ver = a.versions ? a.versions[so * g + k] : a.ver_scalar;
  } else {
    lp = old = psum = 0.0f;
    for (int j = 0; j < g; ++j) {
      lp = __fadd_rn(lp, lp_cur[j]);
      old = __fadd_rn(old, lp_old[j]);
      if (pp) psum = __fadd_rn(psum, pp[j]);
    }
    ver = a.versions ? a.versions[so * g] : a.ver_scalar;  // versions[..., 0] / versions[:, 0, 0]
  }
}

template <bool TOKEN>
__global__ void __launch_bounds__(256) dppo_count_kernel(DArgs a, DHyper h, int U, int g, double* __restrict__ sums) {
  __shared__ double red[2 * 32];
  double v[2] = {0.0, 0.0};
  const int64_t n_units = a.b.bsz * U;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t u = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; u < n_units; u += stride) {
    const int64_t i = u / U;
    const int c = (int)(u - i * U);
    const int64_t row = a.b.idx ? a.b.idx[i] : i;
    const int64_t so = row * U + c;
    const bool m = a.b.loss_mask ? a.b.loss_mask[so] != 0 : true;
    // count_nonzero(loss_mask): un-expanded mask when given, ones_like(logprobs) (elements) when None
    v[0] += m ? ((a.b.loss_mask == nullptr && TOKEN) ? (double)g : 1.0) : 0.0;
    if (!h.has_thr) {
      v[1] += m ? ((a.b.loss_mask == nullptr && TOKEN) ? (double)g : 1.0) : 0.0;
    } else if (m) {
      const int reps = TOKEN ? g : 1;
      for (int k = 0; k < reps; ++k) {
        float lp, old, psum, ver;
        load_entry<TOKEN>(a, u, so, g, k, lp, old, psum, ver);
        const float px = proximal(lp, old, a.prox, psum, ver, a.has_versions != 0, h);
        const float bw = expf(__fsub_rn(px, old));
        v[1] += (bw <= h.thr) ? 1.0 : 0.0;
      }
    }
  }
  rb::block_sum<2>(v, red);
  if (threadIdx.x == 0) {
    if (v[0] != 0.0) atomicAdd(&sums[D_CNT], v[0]);
    if (v[1] != 0.0) atomicAdd(&sums[D_BCNT], v[1]);
  }
}

__device__ void dppo_finalize(const DArgs& a, const DHyper& h, int U, int g, int token_mode, const double* s) {
  const double n_units = (double)(a.b.bsz * U);
  const double n_elems = n_units * (token_mode ? g : 1);
  const bool has_mask = a.b.loss_mask != nullptr;
  const bool ratio_agg = has_mask && a.b.loss_mask_sum != nullptr && h.max_episode_steps > 0.0f;
  const double cnt = s[D_CNT] > 0.0 ? s[D_CNT] : 1.0;   // `count_nonzero() or 1`
  const double bcnt = s[D_BCNT] > 0.0 ? s[D_BCNT] : 1.0;
  // masked_mean(x, loss_mask): sum(x*mask) / sum(mask) with the mask at its own (un-expanded) shape
  const double d_mask = s[D_CNT] > 0.0 ? s[D_CNT] : 1.0;
  float* M = a.b.metrics;
  for (int k = 0; k < RB200_NUM_METRICS; ++k) M[k] = 0.0f;
  double policy_loss = ratio_agg ? s[D_L] / n_elems : (s[D_BCNT] > 0.0 ? s[D_L] / s[D_BCNT] : s[D_L]);
  if (h.critic_warmup) policy_loss = 0.0;
  M[RB200_DM_POLICY_LOSS] = (float)policy_loss;
  M[RB200_DM_PROXIMAL_RATIO] = (float)(s[D_PR] / d_mask);
  M[RB200_DM_CLIPPED_PROXIMAL_RATIO] = (float)(s[D_CPR] / d_mask);
  M[RB200_DM_CLIP_FRACTION] = (float)(s[D_CLIP] / cnt);
  M[RB200_DM_DUAL_CLIP_FRACTION] = (float)(s[D_DUAL] / cnt);
  M[RB200_DM_BEHAV_CLIP_FRACTION] = (float)(1.0 - (double)(float)(bcnt / cnt));
  M[RB200_DM_PROXIMAL_APPROX_KL] = (float)(-s[D_PKL] / cnt);
  M[RB200_DM_BEHAV_APPROX_KL] = (float)(-s[D_BKL] / bcnt);
  // actor/average_version: only when versions has the (preprocessed) loss-mask shape and the mask has a True entry
  const bool ver_shape_ok = a.has_versions && h.has_version && (!token_mode || !has_mask);
  if (ver_shape_ok && s[D_CNT] > 0.0) {
    M[RB200_DM_HAS_VERSION_METRICS] = 1.0f;
    M[RB200_DM_AVERAGE_VERSION] = (float)(s[D_VER] / s[D_CNT]);
    M[RB200_DM_CURRENT_VERSION] = h.cur_version;
  }
  M[RB200_DM_TOKEN_NUM] = (float)s[D_CNT];
  double total = policy_loss;
  if (a.b.with_critic) {
    const double d_unit = ratio_agg ? n_units : (has_mask ? (s[D_CNT] > 0.0 ? s[D_CNT] : 1.0) : n_units);
    const double vl = s[D_VL] / d_unit;
    M[RB200_DM_VALUE_LOSS] = (float)vl;
    M[RB200_DM_VALUE_CLIP_RATIO] = (float)(s[D_VCLIP] / n_units);
    M[RB200_DM_EV_COUNT] = (float)s[D_EV_N];
    M[RB200_DM_EV_COUNT + 1] = (float)s[D_EV_R];
    M[RB200_DM_EV_COUNT + 2] = (float)s[D_EV_R2];
    M[RB200_DM_EV_COUNT + 3] = (float)s[D_EV_E];
    M[RB200_DM_EV_COUNT + 4] = (float)s[D_EV_E2];
    total += vl;
  }
  // the worker's entropy term: loss -= entropy_bonus * masked_mean(entropy, loss_mask), outside critic warm-up only
  // chunk level with a mask: the reference's masked_mean broadcasts the [bsz] entropy against the [bsz, 1] mask, which
  // gives sum(entropy) * count / count, the sum over every unit (0 when no entry is valid)
  if (a.b.entropy && h.entropy_bonus > 0.0f && !h.critic_warmup) {
    const bool ent_bcast = has_mask && a.b.logprob_type == RB200_LOGPROB_CHUNK;
    const double d_ent = ent_bcast ? 1.0 : (has_mask ? (s[D_CNT] > 0.0 ? s[D_CNT] : 1.0) : n_units);
    const double ent = (ent_bcast && !(s[D_CNT] > 0.0)) ? 0.0 : s[D_ENT] / d_ent;
    M[RB200_DM_ENTROPY] = (float)ent;
    total -= (double)h.entropy_bonus * ent;
  }
  total *= (double)h.loss_scale;
  M[RB200_DM_TOTAL_LOSS] = (float)total;
  if (a.b.loss) a.b.loss[0] = (float)total;
}

template <bool TOKEN>
__global__ void __launch_bounds__(256, 2) dppo_main_kernel(DArgs a, DHyper h, int U, int g, double* __restrict__ sums) {
  __shared__ double red[D_NUM * 32];
  float acc[D_NUM];
#pragma unroll
  for (int k = 0; k < D_NUM; ++k) acc[k] = 0.0f;
  const int64_t n_units = a.b.bsz * U;
  const bool has_mask = a.b.loss_mask != nullptr;
  const bool ratio_agg = has_mask && a.b.loss_mask_sum != nullptr && h.max_episode_steps > 0.0f;
  const double n_elems = (double)n_units * (TOKEN ? g : 1);
  const double bcnt = sums[D_BCNT], mcnt = sums[D_CNT];
  // d loss / d term: masked_mean over behav_mask, or masked_mean_ratio ((v / ratio * mask).mean() over all elements)
  const float coef_actor = ratio_agg ? (float)(1.0 / n_elems) : (float)(1.0 / (bcnt > 0.0 ? bcnt : 1.0));
  const float coef_unit = ratio_agg ? (float)(1.0 / (double)n_units)
                                    : (has_mask ? (float)(1.0 / (mcnt > 0.0 ? mcnt : 1.0)) : (float)(1.0 / (double)n_units));
  // d masked_mean(entropy, loss_mask) / d entropy: the mask count whatever the policy-loss aggregation; 1 (or 0 with no
  // valid entry) for the chunk-level broadcast, see dppo_finalize
  const bool ent_bcast = has_mask && a.b.logprob_type == RB200_LOGPROB_CHUNK;
  const float coef_ent = ent_bcast ? (mcnt > 0.0 ? 1.0f : 0.0f)
                                   : (has_mask ? (float)(1.0 / (mcnt > 0.0 ? mcnt : 1.0)) : (float)(1.0 / (double)n_units));
  const float ent_grad = (h.entropy_bonus > 0.0f && !h.critic_warmup) ? -h.loss_scale * h.entropy_bonus * coef_ent : 0.0f;
  const float scale = h.loss_scale;

  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t u = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; u < n_units; u += stride) {
    const int64_t i = u / U;
    const int c = (int)(u - i * U);
    const int64_t row = a.b.idx ? a.b.idx[i] : i;
    const int64_t so = row * U + c;
    const bool m = has_mask ? (a.b.loss_mask[so] != 0) : true;
    const float mf = m ? 1.0f : 0.0f;
    const float adv = a.b.advantages[so];
    float w = 1.0f;
    if (ratio_agg) {
      const int64_t ms_row = a.b.mask_sum_row_mod > 0 ? (row % a.b.mask_sum_row_mod) : row;
      w = __fdiv_rn((float)a.b.loss_mask_sum[ms_row * U + c], h.max_episode_steps);
    }
    float* dlp = a.b.d_logprobs ? a.b.d_logprobs + u * g : nullptr;
    const int reps = TOKEN ? g : 1;
    float unit_grad = 0.0f;
    for (int k = 0; k < reps; ++k) {
      float lp, old, psum, ver;
      load_entry<TOKEN>(a, u, so, g, k, lp, old, psum, ver);
      const float px = proximal(lp, old, a.prox, psum, ver, a.has_versions != 0, h);
      const float lr = __fsub_rn(lp, px);
      const float ratio = m ? expf(lr) : 0.0f;
      const float clipped = fminf(fmaxf(ratio, h.clip_lo), h.clip_hi);
      const float nadv = -adv;
      const float l1 = __fmul_rn(nadv, ratio), l2 = __fmul_rn(nadv, clipped);
      float le = fmaxf(l1, l2);
      const bool in_range = (ratio >= h.clip_lo) && (ratio <= h.clip_hi);
      const float g1 = l1 > l2 ? 1.0f : (l1 == l2 ? 0.5f : 0.0f);
      const float g2 = l2 > l1 ? 1.0f : (l1 == l2 ? 0.5f : 0.0f);
      float dle = nadv * (g1 + (in_range ? g2 : 0.0f));
      bool dual_hit = false;
      if (h.dual_c > 0.0f) {
        const float sg = adv > 0.0f ? 1.0f : (adv < 0.0f ? -1.0f : 0.0f);
        const float l3 = __fmul_rn(__fmul_rn(sg, h.dual_c), adv);
        dual_hit = l3 < le;
        const float f = le < l3 ? 1.0f : (le == l3 ? 0.5f : 0.0f);
        le = fminf(le, l3);
        dle *= f;
      }
      const float bw = expf(__fsub_rn(px, old));
      const bool bm = m && (!h.has_thr || bw <= h.thr);
      const float bmf = bm ? 1.0f : 0.0f;
      const float term0 = __fmul_rn(le, bw);
      acc[D_L] += ratio_agg ? __fmul_rn(__fdiv_rn(term0, w), bmf) : __fmul_rn(term0, bmf);
      acc[D_PR] += ratio * mf;
      acc[D_CPR] += clipped * mf;
      acc[D_CLIP] += (l1 < l2 && m) ? 1.0f : 0.0f;
      acc[D_DUAL] += (dual_hit && m) ? 1.0f : 0.0f;
      acc[D_PKL] += m ? lr : 0.0f;
      acc[D_BKL] += bm ? __fsub_rn(px, old) : 0.0f;
      if (m && a.has_versions) acc[D_VER] += ver;
      const float cw = ratio_agg ? coef_actor / w : coef_actor;
      const float gval = (h.critic_warmup || !bm) ? 0.0f : scale * cw * bw * dle * ratio;
      if (TOKEN) {
        if (dlp) dlp[k] = gval;
      } else {
        unit_grad = gval;
      }
    }
    if (!TOKEN && dlp)
      for (int k = 0; k < g; ++k) dlp[k] = unit_grad;

    if (a.b.with_critic) {
      const float v = a.b.values[u], pv = a.b.prev_values[so], rt = a.b.returns[so];
      const float dv = __fsub_rn(v, pv);
      const float dvc = fminf(fmaxf(dv, -h.value_clip), h.value_clip);
      const float vpc = __fadd_rn(pv, dvc);
      const float e1 = __fsub_rn(rt, v), e2 = __fsub_rn(rt, vpc);
      const float lo = huber(e1, h.huber_delta, h.half_huber_delta);
      const float lc = huber(e2, h.huber_delta, h.half_huber_delta);
      const float vl = fmaxf(lo, lc);
      acc[D_VL] += has_mask ? (ratio_agg ? __fmul_rn(__fdiv_rn(vl, w), mf) : __fmul_rn(vl, mf)) : vl;
      acc[D_VCLIP] += (fabsf(__fsub_rn(vpc, pv)) > h.value_clip) ? 1.0f : 0.0f;
      if (m) {
        acc[D_EV_N] += 1.0f;
        acc[D_EV_R] += rt;
        acc[D_EV_R2] += __fmul_rn(rt, rt);
        acc[D_EV_E] += e1;
        acc[D_EV_E2] += __fmul_rn(e1, e1);
      }
      if (a.b.d_values) {
        const float g1 = lo > lc ? 1.0f : (lo == lc ? 0.5f : 0.0f);
        const float g2 = lc > lo ? 1.0f : (lo == lc ? 0.5f : 0.0f);
        const bool pass_c = (dv >= -h.value_clip) && (dv <= h.value_clip);
        const float dvl = -(g1 * huber_grad(e1, h.huber_delta)) - (pass_c ? g2 * huber_grad(e2, h.huber_delta) : 0.0f);
        const float cw = has_mask ? (ratio_agg ? coef_unit / w : coef_unit) * mf : coef_unit;
        a.b.d_values[u] = scale * cw * dvl;
      }
    }

    if (a.b.entropy) {
      const float* en = a.b.entropy + u * g;
      float es = 0.0f;
      for (int k = 0; k < g; ++k) es = __fadd_rn(es, en[k]);
      acc[D_ENT] += (has_mask && !ent_bcast) ? __fmul_rn(es, mf) : es;
      if (a.b.d_entropy) {
        float* de = a.b.d_entropy + u * g;
        const float gval = (has_mask && !ent_bcast) ? ent_grad * mf : ent_grad;
        for (int k = 0; k < g; ++k) de[k] = gval;
      }
    }
  }

  double accd[D_NUM];
#pragma unroll
  for (int k = 0; k < D_NUM; ++k) accd[k] = (double)acc[k];
  rb::block_sum<D_NUM>(accd, red);
  if (threadIdx.x == 0) {
#pragma unroll
    for (int k = D_L; k < D_NUM; ++k)
      if (accd[k] != 0.0) atomicAdd(&sums[k], accd[k]);
    __threadfence();
    const unsigned long long prev = atomicAdd(reinterpret_cast<unsigned long long*>(sums + 31), 1ull);
    if (prev == (unsigned long long)gridDim.x - 1ull) {
      __threadfence();
      double fin[D_NUM];
#pragma unroll
      for (int k = 0; k < D_NUM; ++k) fin[k] = __ldcg(&sums[k]);
      dppo_finalize(a, h, U, g, TOKEN ? 1 : 0, fin);
#pragma unroll
      for (int k = 0; k < D_NUM; ++k) sums[k] = 0.0;
      *reinterpret_cast<unsigned long long*>(sums + 31) = 0ull;
    }
  }
}

// ---- OPD ----------------------------------------------------------------------------------------------------------------
enum OSlot { O_CNT = 0, O_L, O_R, O_NUM };

__global__ void __launch_bounds__(256) opd_count_kernel(const uint8_t* __restrict__ mask, int64_t n_units,
                                                        double* __restrict__ sums) {
  __shared__ double red[32];
  double v[1] = {0.0};
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t u = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; u < n_units; u += stride) v[0] += mask[u] ? 1.0 : 0.0;
  rb::block_sum<1>(v, red);
  if (threadIdx.x == 0 && v[0] != 0.0) atomicAdd(&sums[O_CNT], v[0]);
}

// logprobs / advantages [n_units, g]; mask, mask_sum [n_units] (broadcast over the g tokens)
__global__ void __launch_bounds__(256) opd_main_kernel(const float* __restrict__ lp, const float* __restrict__ adv,
                                                       const uint8_t* __restrict__ mask,
                                                       const int64_t* __restrict__ mask_sum, int64_t n_units, int g,
                                                       float max_episode_steps, float loss_scale, float* __restrict__ loss,
                                                       float* __restrict__ metrics, float* __restrict__ dlp,
                                                       double* __restrict__ sums) {
  __shared__ double red[O_NUM * 32];
  double v[O_NUM] = {0.0, 0.0, 0.0};
  const bool ratio_agg = max_episode_steps > 0.0f;
  const double n_elems = (double)n_units * g;
  const double mcnt_e = sums[O_CNT] * g;  // expanded mask count
  const float coef = ratio_agg ? (float)(1.0 / n_elems) : (float)(1.0 / (mcnt_e > 0.0 ? mcnt_e : 1.0));
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t u = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; u < n_units; u += stride) {
    const bool m = mask[u] != 0;
    const float mf = m ? 1.0f : 0.0f;
    const float w = ratio_agg ? __fdiv_rn((float)mask_sum[u], max_episode_steps) : 1.0f;
    float sl = 0.0f, sr = 0.0f;
    for (int k = 0; k < g; ++k) {
      const float r = adv[u * g + k];
      const float t = __fmul_rn(-lp[u * g + k], r);
      sl += ratio_agg ? __fmul_rn(__fdiv_rn(t, w), mf) : __fmul_rn(t, mf);
      sr += __fmul_rn(r, mf);
      if (dlp) dlp[u * g + k] = m ? loss_scale * (ratio_agg ? coef / w : coef) * (-r) : 0.0f;
    }
    v[O_L] += (double)sl;
    v[O_R] += (double)sr;
  }
  rb::block_sum<O_NUM>(v, red);
  if (threadIdx.x == 0) {
    if (v[O_L] != 0.0) atomicAdd(&sums[O_L], v[O_L]);
    if (v[O_R] != 0.0) atomicAdd(&sums[O_R], v[O_R]);
    __threadfence();
    const unsigned long long prev = atomicAdd(reinterpret_cast<unsigned long long*>(sums + 31), 1ull);
    if (prev == (unsigned long long)gridDim.x - 1ull) {
      __threadfence();
      const double cnt_e = __ldcg(&sums[O_CNT]) * g, L = __ldcg(&sums[O_L]), R = __ldcg(&sums[O_R]);
      const double den = cnt_e > 0.0 ? cnt_e : 1.0;  // all-False mask: masked_mean returns the (zero) masked sum
      const double pl = ratio_agg ? L / n_elems : L / den;
      for (int k = 0; k < RB200_NUM_METRICS; ++k) metrics[k] = 0.0f;
      metrics[RB200_OM_POLICY_LOSS] = (float)pl;
      metrics[RB200_OM_OPD_REWARD] = (float)(R / den);
      metrics[RB200_OM_OPD_REVERSE_KL] = (float)(-R / den);
      metrics[RB200_OM_TOTAL_LOSS] = (float)(pl * (double)loss_scale);
      if (loss) loss[0] = (float)(pl * (double)loss_scale);
      sums[O_CNT] = 0.0;
      sums[O_L] = 0.0;
      sums[O_R] = 0.0;
      *reinterpret_cast<unsigned long long*>(sums + 31) = 0ull;
    }
  }
}

inline int grid_for(int64_t n) {
  int64_t blocks = (n + 255) / 256;
  const int64_t cap = (int64_t)rb::sm_count() * 3;
  if (blocks > cap) blocks = cap;
  return (int)(blocks < 1 ? 1 : blocks);
}

// shared by both decoupled entry points: versions != NULL (per token) or has_scalar (one version for every token)
int launch_decoupled(const rb200_ppo_args& b, const float* prox, const float* versions, int has_scalar,
                     double ver_scalar, int has_current_version, double current_version, int has_thr, double thr,
                     cudaStream_t st) {
  if (!b.logprobs || !b.old_logprobs || !b.advantages || !b.metrics || !b.workspace) return RB200_E_NULL;
  if (b.bsz <= 0 || b.C <= 0 || b.A <= 0) return RB200_E_SHAPE;
  if (b.logprob_type < RB200_LOGPROB_TOKEN || b.logprob_type > RB200_LOGPROB_CHUNK) return RB200_E_ARG;
  if (b.with_critic && (!b.values || !b.returns || !b.prev_values)) return RB200_E_NULL;
  if (b.clip_ratio_c > 0.0 && !(b.clip_ratio_c > 1.0)) return RB200_E_ARG;  // losses.py:106 assert
  if (b.d_entropy && !b.entropy) return RB200_E_NULL;
  if (b.adv_stats || b.has_clip_log_ratio_min || b.has_clip_log_ratio_max) return RB200_E_UNSUPPORTED;
  if (b.entropy && b.logprob_type == RB200_LOGPROB_CHUNK && b.C != 1) return RB200_E_UNSUPPORTED;
  const int U = b.logprob_type == RB200_LOGPROB_CHUNK ? 1 : b.C;
  const int g = b.logprob_type == RB200_LOGPROB_CHUNK ? b.C * b.A : b.A;
  DHyper h;
  h.clip_lo = (float)(1.0 - b.clip_ratio_low);
  h.clip_hi = (float)(1.0 + b.clip_ratio_high);
  h.dual_c = b.clip_ratio_c > 0.0 ? (float)b.clip_ratio_c : 0.0f;
  h.value_clip = (float)b.value_clip;
  h.huber_delta = (float)b.huber_delta;
  h.half_huber_delta = (float)(0.5 * b.huber_delta);
  h.max_episode_steps = b.max_episode_steps > 0 ? (float)b.max_episode_steps : 0.0f;
  h.critic_warmup = b.critic_warmup;
  h.loss_scale = (float)b.loss_scale;
  h.entropy_bonus = (float)b.entropy_bonus;
  h.has_version = has_current_version;
  h.cur_version = (float)current_version;
  h.prox_version = (float)(current_version - 1.0);
  h.has_thr = has_thr;
  h.thr = (float)thr;
  DArgs a{b, prox, versions, (versions != nullptr || has_scalar) ? 1 : 0, versions ? 0.0f : (float)ver_scalar};
  const int blocks = grid_for(b.bsz * U);
  const bool token = b.logprob_type == RB200_LOGPROB_TOKEN;
  if (token) dppo_count_kernel<true><<<blocks, 256, 0, st>>>(a, h, U, g, b.workspace);
  else dppo_count_kernel<false><<<blocks, 256, 0, st>>>(a, h, U, g, b.workspace);
  rb::count_launch();
  if (token) dppo_main_kernel<true><<<blocks, 256, 0, st>>>(a, h, U, g, b.workspace);
  else dppo_main_kernel<false><<<blocks, 256, 0, st>>>(a, h, U, g, b.workspace);
  rb::count_launch();
  RB_RETURN_LAUNCH();
}

}  // namespace

extern "C" int rb200_decoupled_ppo_loss(const rb200_dppo_args* args, rb200_stream_t stream) {
  if (!args) return RB200_E_NULL;
  return launch_decoupled(args->base, args->proximal_logprobs, args->versions, 0, 0.0, args->has_current_version,
                          args->current_version, args->has_behave_weight_threshold, args->behave_weight_threshold,
                          rb::as_stream(stream));
}

extern "C" int rb200_decoupled_ppo_loss_scalar_version(const rb200_dppo_scalar_version_args* args,
                                                       rb200_stream_t stream) {
  if (!args) return RB200_E_NULL;
  return launch_decoupled(args->base, args->proximal_logprobs, nullptr, 1, args->version, 1, args->current_version,
                          args->has_behave_weight_threshold, args->behave_weight_threshold, rb::as_stream(stream));
}

extern "C" int rb200_opd_loss(const float* logprobs, const float* advantages, const uint8_t* loss_mask,
                              const int64_t* loss_mask_sum, int64_t n_units, int tokens_per_unit, int max_episode_steps,
                              double loss_scale, double* workspace, float* loss, float* metrics, float* d_logprobs,
                              rb200_stream_t stream) {
  if (!logprobs || !advantages || !loss_mask || !loss_mask_sum || !workspace || !metrics) return RB200_E_NULL;
  if (n_units <= 0 || tokens_per_unit <= 0) return RB200_E_SHAPE;
  cudaStream_t st = rb::as_stream(stream);
  const int blocks = grid_for(n_units);
  opd_count_kernel<<<blocks, 256, 0, st>>>(loss_mask, n_units, workspace);
  rb::count_launch();
  opd_main_kernel<<<blocks, 256, 0, st>>>(logprobs, advantages, loss_mask, loss_mask_sum, n_units, tokens_per_unit,
                                          max_episode_steps > 0 ? (float)max_episode_steps : 0.0f, (float)loss_scale, loss,
                                          metrics, d_logprobs, workspace);
  rb::count_launch();
  RB_RETURN_LAUNCH();
}
