/*
 * rlinf_b200.h - C ABI of librlinf_b200.so: the H100-native (sm_90a) drop-in for the
 * data-parallel hot path of RLinf's actor-learner (advantages, PPO/GRPO loss,
 * MLP policy forward/backward, grad-clip + AdamW, rollout sampling).
 *
 * Conventions (SURVEY.md §8b):
 *  - plain pointers and sizes; every pointer is a DEVICE pointer unless the name ends in `_host`;
 *  - every entry point takes a `stream` (a cudaStream_t passed as void*), never synchronises
 *    the device, allocates nothing the caller can see, and owns no state except a lazily
 *    created per-device scratch (a few KB of reduction slots, TMA descriptors);
 *  - outputs are caller-allocated; inputs are never mutated;
 *  - return value: 0 = ok, <0 = invalid argument (RB200_E_*), >0 = a cudaError_t;
 *  - bool tensors are 1 byte per element (torch.bool / uint8), fp tensors are float32
 *    (the reference asserts fp32: rlinf/algorithms/losses.py:232-240).
 *
 * Each entry point cites the reference interface it replaces (file:line under the
 * RLinf v0.4.0 tree).  The reference is 100 % Python; the binding a maintainer
 * would add is a ctypes stub, shown in INTEGRATION.md.
 */
#ifndef RLINF_B200_H
#define RLINF_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define RB200_ABI_VERSION 2

/* error codes (<0); >0 is a cudaError_t */
#define RB200_OK 0
#define RB200_E_NULL (-1)      /* required pointer is NULL */
#define RB200_E_SHAPE (-2)     /* non-positive / inconsistent dimension */
#define RB200_E_ARG (-3)       /* bad scalar argument (e.g. clip_ratio_c <= 1) */
#define RB200_E_ALIGN (-4)     /* pointer not aligned as required */
#define RB200_E_UNSUPPORTED (-5)

typedef void* rb200_stream_t; /* cudaStream_t */

int rb200_abi_version(void);
const char* rb200_strerror(int code);
/* sm count / compute capability of the current device (host-side query). */
int rb200_device_info(int* sm_count, int* cc_major, int* cc_minor);
/* kernels launched by this library in this process so far (host counter; launches replayed from a
 * captured CUDA graph are counted once, at capture). */
uint64_t rb200_launch_count(void);

/* ------------------------------------------------------------------------------------------
 * K0  loss mask            replaces compute_loss_mask, rlinf/utils/metric_utils.py:516-537
 *   dones     bool  [(nc+1), B, C]
 *   mask      bool  [nc, B, C]        step valid while no done seen in rows [0..t]
 *   mask_sum  int64 [B]               per-env valid-step count (the reference expands it
 *                                     to mask's shape as a view; the shim does the same)
 * ---------------------------------------------------------------------------------------- */
int rb200_loss_mask(const uint8_t* dones, uint8_t* mask, int64_t* mask_sum,
                    int nc, int B, int C, rb200_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * K1  GAE scan (+ normalisation statistics)
 *   replaces compute_gae_advantages_and_returns, rlinf/algorithms/advantages.py:24-86
 *   (the T-iteration Python loop) and the statistics half of safe_normalize,
 *   rlinf/algorithms/utils.py:397-404.
 *   Step-major layout: rewards [T,B] f32, values [T+1,B] f32 (NULL = critic-free: gamma=lambda=1,
 *   delta=r), dones [T+1,B] bool, loss_mask [T,B] bool or NULL.
 *   adv, ret [T,B] f32 are the UN-normalised outputs, bit-identical to the reference's fp32
 *   sequential recurrence (each op rounded separately, no FMA contraction).
 *   stats (may be NULL): double[6] = {n, sum, sumsq} of adv over valid entries, then of ret.
 *   The caller zeroes nothing: the call resets stats itself.
 *   gamma / gae_lambda are doubles because the reference rounds fl32(gamma) for gamma*V but
 *   fl32(gamma*gae_lambda) (product taken in Python double) for the recurrence coefficient.
 * ---------------------------------------------------------------------------------------- */
int rb200_gae(const float* rewards, const float* values, const uint8_t* dones,
              const uint8_t* loss_mask, float* adv, float* ret, double* stats,
              int T, int B, double gamma, double gae_lambda, rb200_stream_t stream);

/* x <- (x - mean) / (std_unbiased + eps) with {n,sum,sumsq} = stats[0..2]; no-op if n == 0.
 * The apply half of safe_normalize (eps=1e-5, rlinf/algorithms/utils.py:397-404). In place. */
int rb200_normalize(float* x, const double* stats, int64_t n_elems, float eps,
                    rb200_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * K1' GRPO: first-episode scores + group normalisation + broadcast over T
 *   replaces calculate_scores, rlinf/algorithms/utils.py:134-152 (CPU-only reverse loop) and
 *   compute_grpo_advantages, rlinf/algorithms/advantages.py:89-121.
 *   rewards [T,B] f32, dones [T+1,B] bool -> scores [B] f32 (bit-identical reverse accumulation)
 *   scores [B] (groups of G consecutive envs), loss_mask [T,B] bool -> adv [T,B] f32
 * ---------------------------------------------------------------------------------------- */
int rb200_grpo_scores(const float* rewards, const uint8_t* dones, float* scores,
                      int T, int B, rb200_stream_t stream);
int rb200_grpo_advantages(const float* scores, const uint8_t* loss_mask, float* adv,
                          int T, int B, int G, float eps, rb200_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * a12 trajectory gather    replaces process_nested_dict_for_train's
 *   `value.reshape(-1, ...)[shuffle_id]`, rlinf/utils/nested_dict_process.py:272-285.
 *   dst[i, :] = src[idx[i], :] for rows of `row_bytes` bytes (any dtype). idx is int64.
 * ---------------------------------------------------------------------------------------- */
int rb200_gather_rows(const void* src, const int64_t* idx, void* dst, int64_t n_rows_out,
                      int64_t n_rows_src, int64_t row_bytes, rb200_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * K2  fused (gather +) PPO actor[-critic] loss, forward + backward in one pass
 *   replaces policy_loss, rlinf/algorithms/registry.py:77-92, preprocess_loss_inputs
 *   (algorithms/utils.py:280-376), compute_ppo_actor_loss (losses.py:170-312),
 *   compute_ppo_critic_loss (losses.py:315-380), the entropy term and 1/grad_accum scaling of
 *   embodied_fsdp_actor_worker.py:678-695, and autograd's backward of all of it.
 * ---------------------------------------------------------------------------------------- */
enum { RB200_LOGPROB_TOKEN = 0, RB200_LOGPROB_ACTION = 1, RB200_LOGPROB_CHUNK = 2 };

/* indices into the metrics vector written by rb200_ppo_loss */
enum {
  RB200_M_POLICY_LOSS = 0,      /* actor/policy_loss        */
  RB200_M_POLICY_LOSS_ABS = 1,  /* actor/policy_loss_abs    */
  RB200_M_RATIO = 2,            /* actor/ratio              */
  RB200_M_RATIO_ABS = 3,        /* actor/ratio_abs          */
  RB200_M_CLIPPED_RATIO = 4,    /* actor/clipped_ratio      */
  RB200_M_DUAL_CLIPPED_RATIO = 5, /* actor/dual_cliped_ratio (sic, reference spelling) */
  RB200_M_APPROX_KL = 6,        /* actor/approx_kl          */
  RB200_M_CLIP_FRACTION = 7,    /* actor/clip_fraction      */
  RB200_M_VALUE_LOSS = 8,       /* critic/value_loss        */
  RB200_M_VALUE_CLIP_RATIO = 9, /* critic/value_clip_ratio  */
  RB200_M_EV_COUNT = 10,        /* __sum__/_critic_explained_variance/count          */
  RB200_M_EV_RET_SUM = 11,      /*   .../returns_sum     */
  RB200_M_EV_RET_SQ_SUM = 12,   /*   .../returns_sq_sum  */
  RB200_M_EV_ERR_SUM = 13,      /*   .../errors_sum      */
  RB200_M_EV_ERR_SQ_SUM = 14,   /*   .../errors_sq_sum   */
  RB200_M_ENTROPY = 15,         /* actor/entropy_loss (masked mean entropy, before the bonus) */
  RB200_M_TOTAL_LOSS = 16,      /* actor/total_loss  (after entropy bonus and loss_scale)     */
  RB200_M_TOKEN_NUM = 17,       /* number of valid loss entries (count_nonzero of the mask)    */
  RB200_NUM_METRICS = 24
};

typedef struct rb200_ppo_args {
  /* shapes: bsz samples x C chunks x A action dims. A "unit" is one (sample, chunk) for
   * token/action level and one sample for chunk level; U = units per sample (C or 1). */
  int64_t bsz;
  int32_t C, A;
  int32_t logprob_type; /* RB200_LOGPROB_* */
  int32_t with_critic;  /* 1: actor_critic, 0: actor only */
  /* current policy outputs for this micro-batch (NOT gathered) */
  const float* logprobs; /* [bsz, C*A] */
  const float* values;   /* [bsz, U] or NULL */
  const float* entropy;  /* [bsz, C*A] or NULL (entropy bonus term, action-level reduction) */
  /* rollout data; row i of the micro-batch lives at row (idx ? idx[i] : i) */
  const int64_t* idx;          /* [bsz] or NULL */
  const float* old_logprobs;   /* [rows, C*A] */
  const float* advantages;     /* [rows, U] */
  const float* returns;        /* [rows, U] or NULL */
  const float* prev_values;    /* [rows, U] or NULL */
  const uint8_t* loss_mask;    /* [rows, U] or NULL */
  const int64_t* loss_mask_sum; /* [rows or mask_sum_rows, U] or NULL */
  int64_t mask_sum_row_mod;    /* >0: loss_mask_sum row = row % mask_sum_row_mod (per-env table) */
  /* deferred advantage normalisation: if non-NULL, advantages are normalised on the fly with
   * {n,sum,sumsq} = adv_stats[0..2] and eps adv_norm_eps (fusion of safe_normalize) */
  const double* adv_stats;
  float adv_norm_eps;
  /* hyper-parameters (losses.py:170-186, 315-325). Doubles: the reference holds them as Python
   * floats and rounds derived bounds (e.g. 1.0 - clip_ratio_low) once, from double. */
  double clip_ratio_low, clip_ratio_high;
  double clip_ratio_c;      /* <= 0: no dual clip; else must be > 1 */
  int32_t has_clip_log_ratio_min, has_clip_log_ratio_max;
  double clip_log_ratio_min, clip_log_ratio_max;
  double value_clip, huber_delta;
  int32_t max_episode_steps; /* >0 with mask+mask_sum: masked_mean_ratio aggregation */
  int32_t critic_warmup;     /* 1: policy loss := 0 (no actor grads) */
  double entropy_bonus;      /* 0: none */
  double loss_scale;         /* 1/gradient_accumulation */
  /* scratch: caller-provided, 32 doubles, ZERO before its first use; every call leaves it zeroed again (the last CTA
   * clears it), so one zero-initialised buffer per stream is reused without memset nodes. Calls sharing a workspace
   * must be stream-ordered. */
  double* workspace;
  /* outputs */
  float* loss;        /* [1] total loss (after entropy bonus and loss_scale) */
  float* metrics;     /* [RB200_NUM_METRICS] */
  float* d_logprobs;  /* [bsz, C*A] or NULL */
  float* d_values;    /* [bsz, U] or NULL */
  float* d_entropy;   /* [bsz, C*A] or NULL */
} rb200_ppo_args;

int rb200_ppo_loss(const rb200_ppo_args* args, rb200_stream_t stream);

/* "decoupled_actor_critic" (losses.py:27-167 + :315-380, registered :383-394): PPO clipped around a proximal policy.
 * `base` carries everything shared with rb200_ppo_loss (log-ratio clamps / adv_stats must be unset). The entropy
 * bonus is the worker's (async_ppo_fsdp_worker.py:443-456): base.entropy / d_entropy / entropy_bonus as in
 * rb200_ppo_loss, with the masked-mean entropy reported in RB200_DM_ENTROPY.  Metrics use the RB200_DM_* layout. */
enum {
  RB200_DM_POLICY_LOSS = 0,            /* actor/policy_loss            */
  RB200_DM_PROXIMAL_RATIO = 1,         /* actor/proximal_ratio         */
  RB200_DM_CLIPPED_PROXIMAL_RATIO = 2, /* actor/clipped_proximal_ratio */
  RB200_DM_CLIP_FRACTION = 3,          /* actor/clip_fraction          */
  RB200_DM_DUAL_CLIP_FRACTION = 4,     /* actor/dual_clip_fraction     */
  RB200_DM_BEHAV_CLIP_FRACTION = 5,    /* actor/behav_clip_fraction    */
  RB200_DM_PROXIMAL_APPROX_KL = 6,     /* actor/proximal_approx_kl     */
  RB200_DM_BEHAV_APPROX_KL = 7,        /* actor/behav_approx_kl        */
  RB200_DM_VALUE_LOSS = 8,             /* critic/value_loss            */
  RB200_DM_VALUE_CLIP_RATIO = 9,       /* critic/value_clip_ratio      */
  RB200_DM_EV_COUNT = 10,              /* 10..14: explained-variance sufficient statistics, as RB200_M_EV_* */
  RB200_DM_AVERAGE_VERSION = 15,       /* actor/average_version (valid iff slot 19 != 0) */
  RB200_DM_TOTAL_LOSS = 16,
  RB200_DM_TOKEN_NUM = 17,
  RB200_DM_CURRENT_VERSION = 18,       /* actor/current_version */
  RB200_DM_HAS_VERSION_METRICS = 19,
  RB200_DM_ENTROPY = 20                /* actor/entropy_loss (0 unless base.entropy, entropy_bonus > 0, no critic warm-up) */
};
typedef struct rb200_dppo_args {
  rb200_ppo_args base;
  const float* proximal_logprobs; /* [rows, C*A] or NULL: anchor = old_logprobs, or the version interpolation */
  const float* versions;          /* [rows, C*A] fp32 weight version that generated each token, or NULL */
  int32_t has_current_version;
  double current_version;
  int32_t has_behave_weight_threshold;
  double behave_weight_threshold;
} rb200_dppo_args;
int rb200_decoupled_ppo_loss(const rb200_dppo_args* args, rb200_stream_t stream);

/* The same loss for a batch generated by ONE weight version (one rollout between weight refreshes): the version is a
 * scalar, so no [rows, C*A] version tensor is built or gathered.  Identical results to rb200_decoupled_ppo_loss with
 * `versions` filled with `version` and has_current_version = 1. */
typedef struct rb200_dppo_scalar_version_args {
  rb200_ppo_args base;
  const float* proximal_logprobs; /* [rows, C*A] or NULL: the version interpolation */
  double version;                 /* weight version that generated every token of the batch */
  double current_version;
  int32_t has_behave_weight_threshold;
  double behave_weight_threshold;
} rb200_dppo_scalar_version_args;
int rb200_decoupled_ppo_loss_scalar_version(const rb200_dppo_scalar_version_args* args, rb200_stream_t stream);

/* "opd" (losses.py:427-505): loss = agg(-logprobs * stop_grad(advantages)) with the mask / mask_sum broadcast over the
 * tokens of a unit. logprobs, advantages: [n_units, tokens_per_unit]; loss_mask (uint8), loss_mask_sum: [n_units].
 * max_episode_steps > 0 selects masked_mean_ratio. workspace: as rb200_ppo_args.workspace. */
enum { RB200_OM_POLICY_LOSS = 0, RB200_OM_OPD_REWARD = 1, RB200_OM_OPD_REVERSE_KL = 2, RB200_OM_TOTAL_LOSS = 16 };
int rb200_opd_loss(const float* logprobs, const float* advantages, const uint8_t* loss_mask,
                   const int64_t* loss_mask_sum, int64_t n_units, int tokens_per_unit, int max_episode_steps,
                   double loss_scale, double* workspace, float* loss /*[1] or NULL*/,
                   float* metrics /*[RB200_NUM_METRICS]*/, float* d_logprobs /*or NULL*/, rb200_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Token-level PPO-clip actor loss of the reasoning workers (csrc/token_loss.cu): the loss block of
 *   FSDPActor.training_step (workers/actor/fsdp_actor_worker.py:700-780) and of the Megatron loss_func
 *   (megatron_actor_worker.py:194-293) for token log-probs [bsz, L]:
 *     advantages *= min(exp(recomputed - rollout), importance_sampling_clip)   (importance_sampling_fix)
 *     policy = compute_ppo_actor_loss (losses.py:170-312) aggregated with `agg`, fast_path_zero_loss_mask honoured
 *     entropy_loss = agg(entropy, mask);  kl_loss = agg(kl_penalty(x, y, kl_mode), mask)
 *     loss = policy - entropy_bonus * entropy_loss + kl_beta * kl_loss
 *   and the gradients of `loss` for a unit upstream gradient.  No host sync, no floating-point atomics: two identical
 *   calls give the same bits on any SM count.
 * Row i, token j of each input is at ptr[i * <name>_stride + j] (strides in elements, >= L), so slices such as
 *   log_probs[:, -L-1:-1] are read in place.  loss_mask is uint8 / bool; every other input is fp32.
 * Optional inputs (NULL = absent): entropy (the entropy term; its loss is reported even when entropy_bonus is 0),
 *   ref_logprobs (the KL term, added when kl_beta > 0), rollout_logprobs + recomputed_logprobs (the IS fix when
 *   importance_sampling_fix != 0, and RB200_TM_ROLLOUT_TRAIN_KL = masked_mean(|recomputed - rollout|)).
 * kl_order 0: kl_penalty(logprobs, ref_logprobs) (Megatron), 1: kl_penalty(ref_logprobs, logprobs) (FSDP).
 * fast_path_zero_loss_mask: if the FIRST row's mask is empty, the policy part and its metrics are 0 (decided on the
 *   device).  agg RB200_AGG_SEQ_MEAN_TOKEN_MEAN divides by each row's own count, so an empty row makes the loss NaN,
 *   as in the reference.
 * Outputs: loss [1], metrics [RB200_TM_NUM] (RB200_TM_*), d_logprobs / d_entropy [bsz, L] contiguous or NULL
 *   (d_entropy is zero unless entropy_bonus > 0).  workspace: rb200_token_loss_workspace_bytes(bsz, L) bytes,
 *   16-byte aligned, no initialisation needed (-1 = unsupported shape: bsz > 65535 or a non-positive dimension).
 * ---------------------------------------------------------------------------------------- */
enum { RB200_AGG_TOKEN_MEAN = 0, RB200_AGG_SEQ_MEAN_TOKEN_SUM = 1, RB200_AGG_SEQ_MEAN_TOKEN_MEAN = 2 };
enum {
  RB200_TM_POLICY_LOSS = 0,         /* actor/policy_loss        */
  RB200_TM_POLICY_LOSS_ABS = 1,     /* actor/policy_loss_abs    */
  RB200_TM_RATIO = 2,               /* actor/ratio              */
  RB200_TM_RATIO_ABS = 3,           /* actor/ratio_abs          */
  RB200_TM_CLIPPED_RATIO = 4,       /* actor/clipped_ratio      */
  RB200_TM_DUAL_CLIPPED_RATIO = 5,  /* actor/dual_cliped_ratio  */
  RB200_TM_APPROX_KL = 6,           /* actor/approx_kl          */
  RB200_TM_CLIP_FRACTION = 7,       /* actor/clip_fraction      */
  RB200_TM_ENTROPY_LOSS = 8,        /* actor/entropy_loss       */
  RB200_TM_KL_LOSS = 9,             /* actor/kl_loss            */
  RB200_TM_FINAL_LOSS = 10,         /* actor/final_loss (= loss[0]) */
  RB200_TM_ROLLOUT_TRAIN_KL = 11,   /* actor/rollout_train_kl   */
  RB200_TM_NUM = 16
};
typedef struct rb200_token_loss_args {
  int64_t bsz, L;
  const float* logprobs;            int64_t logprobs_stride;
  const float* old_logprobs;        int64_t old_logprobs_stride;
  const float* advantages;          int64_t advantages_stride;
  const uint8_t* loss_mask;         int64_t loss_mask_stride;
  const float* entropy;             int64_t entropy_stride;
  const float* ref_logprobs;        int64_t ref_logprobs_stride;
  const float* rollout_logprobs;    int64_t rollout_logprobs_stride;
  const float* recomputed_logprobs; int64_t recomputed_logprobs_stride;
  double clip_ratio_low, clip_ratio_high;
  double clip_ratio_c;              /* <= 0: no dual clip; else must be > 1 */
  double clip_log_ratio_min, clip_log_ratio_max;
  double entropy_bonus, kl_beta, importance_sampling_clip;
  int32_t has_clip_log_ratio_min, has_clip_log_ratio_max;
  int32_t agg;                      /* RB200_AGG_* */
  int32_t kl_mode;                  /* 0 k1/kl, 1 abs, 2 k2/mse, 3 k3/low_var_kl */
  int32_t kl_order;
  int32_t importance_sampling_fix;
  int32_t fast_path_zero_loss_mask;
  int32_t reserved;
  void* workspace;
  int64_t workspace_bytes;
  float* loss;
  float* metrics;
  float* d_logprobs;
  float* d_entropy;
} rb200_token_loss_args;
int64_t rb200_token_loss_workspace_bytes(int64_t bsz, int64_t L);
int rb200_token_ppo_loss(const rb200_token_loss_args* args, rb200_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Token-level PPO critic loss of the reasoning workers (csrc/token_critic_loss.cu): compute_ppo_critic_loss
 *   (losses.py:315-380) as MegatronCritic's loss_func calls it (workers/critic/megatron_critic_worker.py:92-123) on
 *   [bsz, L] values, returns, prev_values and a loss mask, with huber_delta and value_clip:
 *     vpc = prev + clamp(values - prev, -value_clip, value_clip)
 *     loss = masked_mean(max(huber(returns - values), huber(returns - vpc)), mask)  (the plain masked sum, i.e. 0,
 *            when every cell is masked: masked_mean, utils.py:321-328; the worker's loss_agg_func is not applied)
 *   and d loss / d values for a unit upstream gradient.  Row i, token j of each input is at ptr[i * <name>_stride + j]
 *   (strides in elements, >= L); loss_mask is uint8 / bool, the rest fp32.  Four launches (the token loss's mask
 *   counts and totals, then the critic's main and finish kernels), fp64 partials in fixed slots, no atomics, no host
 *   sync: two identical calls give the same bits on any SM count.
 * Outputs: loss [1], metrics [RB200_CM_NUM] (RB200_CM_*), d_values [bsz, L] contiguous or NULL.  workspace:
 *   rb200_token_loss_workspace_bytes(bsz, L) bytes, 16-byte aligned, no initialisation needed.
 * ---------------------------------------------------------------------------------------- */
enum {
  RB200_CM_VALUE_LOSS = 0,        /* critic/value_loss */
  RB200_CM_VALUE_CLIP_RATIO = 1,  /* critic/value_clip_ratio: unmasked mean over all bsz L cells */
  RB200_CM_EV_COUNT = 2,          /* __sum__/_critic_explained_variance/count (masked cells) */
  RB200_CM_EV_RET_SUM = 3,        /* .../returns_sum */
  RB200_CM_EV_RET_SQ_SUM = 4,     /* .../returns_sq_sum */
  RB200_CM_EV_ERR_SUM = 5,        /* .../errors_sum (errors = returns - values) */
  RB200_CM_EV_ERR_SQ_SUM = 6,     /* .../errors_sq_sum */
  RB200_CM_FINAL_VALUE_LOSS = 7,  /* critic/final_value_loss (= loss[0]) */
  RB200_CM_NUM = 8
};
typedef struct rb200_token_critic_loss_args {
  int64_t bsz, L;
  const float* values;       int64_t values_stride;
  const float* returns;      int64_t returns_stride;
  const float* prev_values;  int64_t prev_values_stride;
  const uint8_t* loss_mask;  int64_t loss_mask_stride;
  double value_clip, huber_delta;
  void* workspace;
  int64_t workspace_bytes;
  float* loss;
  float* metrics;
  float* d_values;
} rb200_token_critic_loss_args;
int rb200_token_critic_loss(const rb200_token_critic_loss_args* args, rb200_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Reasoning step bookkeeping (csrc/reasoning_stats.cu): the reasoning rollout metrics (rlinf/utils/distributed.py
 *   compute_rollout_metrics / compute_rollout_metrics_dynamic) and the tail of the Megatron workers' loss_func and
 *   _process_fwd_bwd_outputs, on the device.  No floating-point atomics; partials go to fixed slots and are added in a
 *   fixed order, so two identical calls give the same bits.
 *
 * rb200_reasoning_rollout_record: one rank's fixed-layout fp64 record [RB200_RR_NUM] (RB200_RR_*) from
 *   advantages [bsz, L] fp32 and the response mask [bsz, L] (uint8 / bool), both read through row strides (elements,
 *   >= L), optional values [bsz, L] fp32, and [bsz] prompt / response lengths (int64), rewards (fp32) and is_end
 *   (uint8); idx_to_traj [bsz] (int64) or NULL selects the multi-turn fields.  The SUM fields are rounded to fp32 as
 *   the reference rounds its reduction vector.  Two launches.  workspace: rb200_reasoning_record_workspace_bytes.
 * rb200_reasoning_rollout_finish: P records, gathered in rank order ([P, RB200_RR_NUM] fp64), -> the metric vector
 *   [RB200_RM_NUM + P] fp64 (RB200_RM_*, then each record's num_seq) with the reference's fp32 reduction and fp64
 *   host arithmetic.  values_world_sum:
 *   NULL = the values mean is averaged over the P records; else a device fp32 sum over the default group of
 *   world_size ranks' RB200_RR_VALUES_MEAN.  One launch.
 * ---------------------------------------------------------------------------------------- */
enum {
  RB200_RR_SUM_PLEN = 0, RB200_RR_SUM_RLEN = 1, RB200_RR_SUM_REWARDS = 2, RB200_RR_SUM_END = 3,
  RB200_RR_SUM_ADV = 4, RB200_RR_NUM_SEQ = 5, RB200_RR_N_VALID = 6, RB200_RR_SUM_TRAJ_REWARDS = 7,
  RB200_RR_NUM_TRAJ = 8,       /* 0-8: fp32-rounded SUM fields */
  RB200_RR_ADV_NEG_MIN = 9, RB200_RR_ADV_MAX = 10, RB200_RR_MAX_PLEN = 11, RB200_RR_MAX_RLEN = 12,
  RB200_RR_MAX_TOTAL = 13, RB200_RR_VAL_NEG_MIN = 14, RB200_RR_VAL_MAX = 15,  /* 9-15: fp32 MAX fields */
  RB200_RR_VALUES_MEAN = 16,   /* fp32 masked mean of this rank's values */
  RB200_RR_RLEN_SUM = 17, RB200_RR_RLEN_SQ_SUM = 18, RB200_RR_RLEN_MIN = 19, RB200_RR_RLEN_MAX = 20,  /* exact */
  RB200_RR_VERDICT = 21,       /* RB200_RV_* bits */
  RB200_RR_NUM = 24
};
enum { RB200_RV_EMPTY = 1, RB200_RV_BAD_TRAJ = 2 };  /* no valid advantage; idx_to_traj entry < 0 */
enum {
  RB200_RM_NUM_SEQ = 0, RB200_RM_PROMPT_LENGTH, RB200_RM_RESPONSE_LENGTH, RB200_RM_AVG_RESPONSE_LENGTH,
  RB200_RM_VAR_RESPONSE_LENGTH, RB200_RM_MAX_OF_RESPONSE_LENGTH, RB200_RM_MIN_OF_RESPONSE_LENGTH,
  RB200_RM_TOTAL_LENGTH, RB200_RM_REWARD_SCORES, RB200_RM_PROPERLY_ENDED, RB200_RM_ADV_MEAN, RB200_RM_ADV_MAX,
  RB200_RM_ADV_MIN, RB200_RM_VALUES_MEAN, RB200_RM_VALUES_MAX, RB200_RM_VALUES_MIN, RB200_RM_MAX_PROMPT_LENGTH,
  RB200_RM_MAX_RESPONSE_LENGTH, RB200_RM_MAX_TOTAL_LENGTH, RB200_RM_REWARD_SCORES_TRAJ, RB200_RM_REWARD_SCORES_TURN,
  RB200_RM_AVG_TURNS_PER_TRAJ, RB200_RM_VERDICT, RB200_RM_NUM_LENGTHS_MAX,  /* largest num_seq of a record */
  RB200_RM_NUM = 24
};
typedef struct rb200_reasoning_record_args {
  int64_t bsz, L;
  const float* advantages;    int64_t advantages_stride;
  const uint8_t* mask;        int64_t mask_stride;
  const float* values;        int64_t values_stride;  /* NULL: no values fields */
  const int64_t* prompt_lengths;
  const int64_t* response_lengths;
  const float* rewards;
  const uint8_t* is_end;
  const int64_t* idx_to_traj;  /* NULL: single-turn batch */
  void* workspace;
  int64_t workspace_bytes;
  double* record;              /* [RB200_RR_NUM] */
} rb200_reasoning_record_args;
int64_t rb200_reasoning_record_workspace_bytes(int64_t bsz, int64_t L);
int rb200_reasoning_rollout_record(const rb200_reasoning_record_args* args, rb200_stream_t stream);
int rb200_reasoning_rollout_finish(const double* records, int32_t P, const float* values_world_sum,
                                   int32_t world_size, double* metrics, rb200_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Megatron loss_func epilogue, one micro-batch (megatron_actor_worker.py:258-307, megatron_critic_worker.py:104-121),
 *   in two launches around ONE data-parallel SUM all-reduce of `pack` that the caller makes:
 * rb200_mb_epilogue_pack: pack[k] = *src[k] for the n_avg averaged keys then the n_sum SUM keys (the explained-
 *   variance sums); pack[final_slot] = loss s and pack[n_avg + n_sum] = (loss 0) s, where the scale
 *   s = fp32(fp32(fp32(mask_sum / global_valid_token) dp) num_microbatches) when global_valid_token is given, else 1;
 *   s goes to scale[0].  With global_valid_token the mask is counted (two more launches; workspace
 *   rb200_token_loss_workspace_bytes(bsz, L) bytes), else workspace needs RB200_EPI_WS_MIN bytes.
 * rb200_mb_epilogue_apply (after the all-reduce): averaged keys = pack / dp (Megatron's average), SUM keys = pack;
 *   early stop when has_early_stop and pack[ratio_slot] / dp > early_stop_imp_ratio (fp32 compare), in which case
 *   scale[0] = 0 and the final loss is the stopped variant; metrics [n_avg + n_sum] and row mb of step_acc
 *   [n_mb, n_avg + n_sum] get the reduced values.  One launch.
 * rb200_step_metrics_finish: _process_fwd_bwd_outputs (megatron_worker.py:550-599) for a training step: out[k] = the
 *   fp32 mean over the n_mb rows in index order for k < n_avg, the fp32 sum for the n_sum keys, and when n_sum == 5
 *   out[n_avg + 5] = compute_critic_explained_variance_from_stats in fp32 (NaN for count < 2 or a zero / NaN centred
 *   returns sum or a NaN centred errors sum).  One launch.
 * ---------------------------------------------------------------------------------------- */
#define RB200_EPI_MAX_KEYS 24
#define RB200_EPI_WS_MIN 64
typedef struct rb200_mb_epilogue_args {
  int32_t n_avg, n_sum;
  int32_t final_slot, ratio_slot;          /* indices among the averaged keys, -1 = none */
  const float* src[RB200_EPI_MAX_KEYS];    /* 0-dim fp32 device metrics: averaged keys, then the SUM keys */
  const float* loss;                       /* the unscaled loss, fp32 [1] */
  const uint8_t* mask;  int64_t mask_stride;  int64_t bsz, L;
  const float* global_valid_token;         /* fp32 [1] or NULL (no valid-token scale) */
  int32_t dp, num_microbatches;
  int32_t has_early_stop, mb;
  double early_stop_imp_ratio;
  void* workspace;
  int64_t workspace_bytes;
  float* pack;       /* [n_avg + n_sum + 1] */
  float* scale;      /* [1] */
  float* metrics;    /* [n_avg + n_sum] */
  float* step_acc;   /* [n_mb, n_avg + n_sum] */
  int32_t n_mb, reserved;
} rb200_mb_epilogue_args;
/* mask.to(float32).sum() of _setup_valid_token_scale (megatron_worker.py:640-654): out[0] = the mask count rounded
 * once to fp32.  workspace: rb200_token_loss_workspace_bytes(bsz, L) bytes.  Three launches. */
int rb200_mask_count_f32(const uint8_t* mask, int64_t mask_stride, int64_t bsz, int64_t L, void* workspace,
                         int64_t workspace_bytes, float* out, rb200_stream_t stream);
int rb200_mb_epilogue_pack(const rb200_mb_epilogue_args* args, rb200_stream_t stream);
int rb200_mb_epilogue_apply(const rb200_mb_epilogue_args* args, rb200_stream_t stream);
int rb200_step_metrics_finish(const float* step_acc, int32_t n_mb, int32_t n_avg, int32_t n_sum, float* out,
                              rb200_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Value head of the reasoning critic on a plan's rows (csrc/value_head.cu): the reference's LinearForLastLayer(H, 1)
 *   (a bf16 nn.Linear without bias, output cast with .float()) evaluated in place on rows of a hidden shard x
 *   (bf16, unit inner stride, row_stride elements between rows, a multiple of 8; 16-byte aligned), w [1, H] bf16.
 *   H % 64 == 0, 64 <= H <= 8192.
 * rb200_value_head_fwd: v[i] = float(bf16(sum_h x[rows[i], h] w[h])) for i < n (fp32 sum in a fixed order, one
 *   rounding to bf16), v[i] = 0 where rows[i] == -1 (a pad slot).  One launch; reads n H 2 bytes.
 * rb200_value_head_bwd: g [n] fp32, rounded to bf16 first (the backward of .float()); either output may be NULL.
 *   dx [T, H] bf16 contiguous: dx[t] = bf16(g_bf16[inv_map[t]] w), exact zeros where inv_map[t] == -1; every row
 *     written once.  One launch; writes T H 2 bytes.
 *   dw [H] bf16 = bf16(sum_i g_bf16[i] x[rows[i]]) over rows[i] != -1: fp32 partials over fixed chunks of rows, added
 *     in a fixed order (two launches; reads n H 2 bytes).  workspace: rb200_value_head_workspace_bytes(n, H) bytes,
 *     16-byte aligned (-1 = unsupported shape).
 *   No floating-point atomics and nothing that depends on the SM count: repeat calls give the same bits. */
int64_t rb200_value_head_workspace_bytes(int64_t n, int64_t H);
int rb200_value_head_fwd(const void* x, int64_t row_stride, const int64_t* rows, int64_t n, int64_t H, const void* w,
                         float* v, rb200_stream_t stream);
int rb200_value_head_bwd(const void* x, int64_t row_stride, const int64_t* rows, int64_t n, int64_t H, const float* g,
                         const void* w, const int64_t* inv_map, int64_t T, void* dx, void* dw, void* workspace,
                         int64_t workspace_bytes, rb200_stream_t stream);

/* x[i] *= s (device scalar-free helper for autograd's upstream scalar). */
int rb200_scale(float* x, int64_t n, float s, rb200_stream_t stream);
/* x[i] *= *s_dev  (the scalar lives on the device: no host sync in autograd's backward). */
int rb200_scale_by(float* x, int64_t n, const float* s_dev, rb200_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * K4  grad-norm clip + AdamW on one flat fp32 buffer
 *   replaces FSDPModelManager.optimizer_step, hybrid_engines/fsdp/fsdp_model_manager.py:429-463
 *   (clip_grad_norm_ of the no_shard path strategy/fsdp.py:363-369 = torch.nn.utils.clip_grad_norm_:
 *   coef = min(1, max_norm/(norm+1e-6)); non-finite norm => step skipped) and torch.optim.AdamW
 *   with the two lr groups of build_optimizer :501-590.
 *   group_end[k] = exclusive end offset of lr group k in the flat buffer (ascending).
 *   state: double[4] device = {step_count, last_grad_norm, last_clip_coef, skipped_flag}.
 * ---------------------------------------------------------------------------------------- */
int rb200_grad_sqnorm(const float* grads, int64_t n, double* out_sq /*[1], reset by kernel*/,
                      rb200_stream_t stream);
int rb200_adamw_step(float* params, const float* grads, float* exp_avg, float* exp_avg_sq,
                     int64_t n, const int64_t* group_end_host, const double* group_lr_host,
                     int n_groups, double beta1, double beta2, double eps, double weight_decay,
                     float max_grad_norm, float grad_scale, const double* grad_sq /*[1]*/,
                     double* state /*[4]*/, rb200_stream_t stream);
/* Same step with the per-group learning rates read from DEVICE memory (double[n_groups]) at execution time, so a
 * captured CUDA graph follows an LR schedule (LambdaLR stepped once per run_training,
 * workers/actor/embodied_fsdp_actor_worker.py:571, hybrid_engines/fsdp/utils.py:522) without re-capture.
 * In both entries lr < 0 marks a FROZEN group: its parameters and moments are left untouched - what
 * torch.optim.AdamW does for parameters outside its param groups (the actor during critic warm-up,
 * fsdp_model_manager.py:523-531) or whose grad is None. */
int rb200_adamw_step_dev(float* params, const float* grads, float* exp_avg, float* exp_avg_sq,
                         int64_t n, const int64_t* group_end_host, const double* group_lr_dev,
                         int n_groups, double beta1, double beta2, double eps, double weight_decay,
                         float max_grad_norm, float grad_scale, const double* grad_sq /*[1]*/,
                         double* state /*[4]*/, rb200_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * K3/K5  MLP policy (3x256 tanh backbone + mean head, state-independent log-std, 3x256 value
 *   MLP).  replaces MLPPolicy.default_forward, models/embodiment/mlp_policy/mlp_policy.py:202-236,
 *   ValueHead.forward, models/embodiment/modules/value_head.py:66, _generate_actions :256-293,
 *   and autograd's backward through them.  Declared in the second half of this header
 *   (rb200_mlp_*), see below.
 * ---------------------------------------------------------------------------------------- */

/* flat parameter layout, in the reference's named_parameters() order */
typedef struct rb200_mlp_layout {
  int32_t obs_dim, act_dim /* C*A outputs of the mean head */, value_dim, hidden /* 256 */;
  int64_t logstd;                         /* [act_dim] */
  int64_t vw0, vb0, vw1, vb1, vw2, vb2, vw3; /* value head: [H,obs],[H],[H,H],[H],[H,H],[H],[value_dim,H] */
  int64_t bw0, bb0, bw1, bb1, bw2, bb2;   /* backbone */
  int64_t mw, mb;                         /* actor_mean [act_dim,H],[act_dim] */
  int64_t total;                          /* number of floats */
} rb200_mlp_layout;

int rb200_mlp_layout_init(rb200_mlp_layout* L, int obs_dim, int act_dim, int value_dim, int hidden);

/* scratch sizes (floats) for n rows: `acts` and `work` of forward/backward/sample/value each need this many */
int64_t rb200_mlp_fwd_scratch_floats(const rb200_mlp_layout* L, int64_t n);

/* Tensor-core operand cache: packed fp16 (hi, lo) tiles of the hidden-layer weights (forward and dgrad packs).
 * rb200_mlp_wsplit_floats() floats; refresh with rb200_mlp_prepare_weights() after every parameter update.
 * Every MLP call below requires it: wsplit == NULL returns RB200_E_NULL. */
int64_t rb200_mlp_wsplit_floats(const rb200_mlp_layout* L);
int rb200_mlp_prepare_weights(const rb200_mlp_layout* L, const float* params, float* wsplit,
                              rb200_stream_t stream);

/* Forward for training: states [n,obs] (row i at idx?idx[i]:i), action [n,act] (same gather).
 * Writes logprobs [n,act], entropy [n,act] (NULL ok), values [n,value_dim] (NULL ok) and keeps
 * the activations needed by backward in `acts`. Hidden layers run on wgmma (2-way fp16 split); layer 0 does too when
 * obs is a multiple of 32 and idx == NULL (its weight gradient only for obs <= 256), and runs on the fp32 SIMT GEMM
 * otherwise. Activations are plain fp32; the
 * tensor-core kernels split them into fp16 (hi, lo) operands. */
int rb200_mlp_forward(const rb200_mlp_layout* L, const float* params, const float* wsplit,
                      const float* states, const float* action, const int64_t* idx, int64_t n,
                      float* logprobs, float* entropy, float* values, float* acts, float* work,
                      const float* states_amax, rb200_stream_t stream);
/* Layer 0 on the tensor cores scales the fp16 split of the states by powers of two where their range calls for it (any
 * finite observations keep fp32-level accuracy): by max|states| in the forward and by the max of each column in the
 * weight gradient.  states_amax: device maxima of the rows' batch as rb200_absmax writes them (4 + obs floats for
 * obs <= 256, else 1), e.g. over the whole batch once per update; NULL: rb200_mlp_forward computes them (one pass over
 * the rows).  rb200_absmax: out[0] = max|x| of x [rows, cols] (16-byte aligned, cols % 4 == 0) and, for cols <= 256,
 * out[4 + c] = max|x[:, c]|. */
int rb200_absmax(const float* x, int64_t rows, int cols, float* out, rb200_stream_t stream);

/* Backward: given d_logprobs [n,act], d_entropy [n,act] or NULL, d_values [n,value_dim] or NULL,
 * ACCUMULATES (+=) parameter gradients into grads (flat, same layout). `acts` from forward. */
int rb200_mlp_backward(const rb200_mlp_layout* L, const float* params, const float* wsplit,
                       const float* states, const float* action, const int64_t* idx, int64_t n,
                       const float* d_logprobs, const float* d_entropy, const float* d_values,
                       const float* acts, float* work, float* grads, rb200_stream_t stream);

/* Rollout step (inference): mean/value forward, action = mean + exp(logstd)*noise where noise is
 * either supplied ([n,act], parity mode) or drawn from Philox(seed, offset + *counter_dev) (noise == NULL;
 * counter_dev may be NULL); writes action [n,act], logprobs [n,act], values [n,value_dim]. */
int rb200_mlp_sample(const rb200_mlp_layout* L, const float* params, const float* wsplit,
                     const float* states, const float* noise, uint64_t seed, uint64_t offset,
                     const uint64_t* counter_dev, int64_t n, float* action, float* logprobs, float* values,
                     float* work, rb200_stream_t stream);

/* Unit-test entries of the fp16-split tensor-core GEMMs of the MLP towers (csrc/tc_gemm_h.cu, wgmma, fp32 in/out).
 * mode 0: C = A[M,K] . B[256,K]^T through the forward kernel the towers run (tc_h_fwd_kernel, csrc/tc_forward_h.cu, for
 * K <= 256; tc_h_gemm_kernel<0> above); mode 2: the same product through tc_h_gemm_kernel<0> for every K, the
 * reference mode 0 is compared against bit for bit; mode 1 (dgrad form, K = 256): C = A[M,256] . B[256,256].  amax: device float holding
 * max|A| (or max|Z|), NULL = no operand scaling.  work: >= 512*K floats (packed fp16 weight tiles: forward + dgrad pack). */
int rb200_tc_gemm_h(const float* A, const float* B, float* C, int64_t M, int K, int mode, const float* amax,
                    float* work, rb200_stream_t stream);
int rb200_tc_wgrad_h(const float* Z, const float* H, float* dW, int64_t n, int IN, const float* amax,
                     rb200_stream_t stream);
/* Backward through a square hidden layer (csrc/tc_backward_h.cu) for ngroups (1 or 2) towers stacked along the first
 * dimension: dW[g] += Z[g]^T . H[g];  dZprev[g] = (Z[g] . W[g]) * (1 - H[g]^2), colsum[g] += its column sums,
 * atomicMax(amax_out[g], max|dZprev[g]|).  Z, H, dZprev: [ngroups, n, 256]; W, dW: [ngroups, 256, 256]; colsum
 * [ngroups, 256], amax_in (max|Z[g]|) and amax_out [ngroups] are nullable.
 * work: >= ngroups * (131072 + 256 * ceil(n / 16)) floats. */
int rb200_tc_dgrad_wgrad_h(const float* Z, const float* W, const float* H, float* dZprev, float* dW, float* colsum,
                           const float* amax_in, float* amax_out, int64_t n, int ngroups, float* work,
                           rb200_stream_t stream);

/* Experiment switches (tests only; default 0 = the shipped kernels): 2 = round-1 layers in the fp32 SIMT fused rollout
 * (one-k-step weight prefetch); 4 = the hidden-layer backward of the MLP update as separate wgrad and dgrad kernels
 * instead of the fused one. */
int rb200_debug_set_flags(int flags);

/* Persistent rollouts: the whole T-step loop of one rank - MLP actor/critic inference, Normal sampling, synthetic-env
 * dynamics with auto-reset and the truncation bootstrap of rewards - in ONE kernel.  Replaces EnvWorker.interact /
 * MultiStepRolloutWorker.generate (rlinf/workers/env/env_worker.py:1059-1349,
 * rlinf/workers/rollout/hf/huggingface_worker.py:678-781) for the MLP-policy + device-resident env case, with the same
 * buffers, row alignment and random streams as the per-kernel path (rb200_mlp_sample + rb200_synth_env_step or
 * rb200_synth_env_chunk_step + rb200_mlp_value + rb200_bootstrap_rewards[_ld] per step).  Both kernels take everything
 * but the weights in one rb200_rollout_args (pointers, then 64-bit, then 32-bit integers, then doubles: no padding). */
typedef struct rb200_rollout_args {
  /* buffers; T = chunk steps, C = num_action_chunks, act = act_dim = C*A, obs = obs_dim */
  float* states;         /* [T+1,B,obs]: row 0 = the current observation (input), rows 1..T written */
  float* actions;        /* [T,B,act] */
  float* logprobs;       /* [T,B,act] */
  float* values;         /* [T+1,B,value_dim]; may be NULL in rb200_rollout_fused when value_dim == 0 */
  float* rewards;        /* [T,B,C], the truncation bootstrap gamma * V(final_obs) folded in */
  uint8_t* terminations; /* [T+1,B,C]: rows 1..T written; with C > 1 all-zero except the chunk's last column = any */
  uint8_t* truncations;  /* [T+1,B,C] */
  uint8_t* dones;        /* [T+1,B,C] */
  float* final_obs;      /* [B,obs]: observation before the auto-reset */
  float* final_values;   /* [B,value_dim]: V(final_obs); may be NULL as `values` */
  /* synthetic env dynamics, as rb200_synth_env_step */
  const float* w_s;      /* [obs,obs]; read by rb200_rollout_fused only (the tensor-core pack holds its own copy) */
  const float* w_a;      /* [A,obs] */
  int32_t* elapsed;      /* [B] env step counters, in/out */
  /* random streams: pre-drawn draws (parity mode) or NULL = Philox on the device */
  const float* policy_noise;      /* [T,B,act] or NULL */
  const float* env_noise;         /* [T,B,2*obs+2]; C > 1: [T,B,C*(obs+2)+obs] = per sub-step eps[obs] | eps_r | u,
                                     then the reset state; or NULL */
  /* device step counters, read once (chunk step t uses counter + t): the caller adds T to both afterwards
   * (rb200_counter_add) */
  const uint64_t* counter_policy;
  const uint64_t* counter_env;
  /* Training-rollout episode statistics: both NULL = off; exactly one NULL = RB200_E_NULL.  Buffers, flags and random
   * streams are the same with statistics on and off.  Per env step the raw reward (before the truncation bootstrap)
   * is added to the return; at a chunk's last sub-step
   *   auto_reset:  where the chunk is done, acc += {1, ret, elapsed, ret / (float)elapsed} with the pre-reset elapsed
   *                count, then ret = 0;
   *   otherwise:   at the rollout's last chunk step every env records its running episode the same way.
   * Replaces ManiskillEnv._record_metrics / _reset_metrics / _handle_auto_reset (rlinf/envs/maniskill/maniskill_env.py:
   * 243-272,377-391) with EnvWorker.env_interact_step's env_info and the should_record rule of
   * EnvWorker._run_interact_once (rlinf/workers/env/env_worker.py:507-522,1229-1235).  Reduce acc with
   * rb200_episode_stats_reduce. */
  float* episode_return; /* [B] fp32 running return, carried across rollouts; the caller zeroes it with every env reset */
  double* episode_acc;   /* [B,4] fp64 count, sum return, sum length, sum reward; zeroed by the caller per rollout */
  uint64_t seed_policy, seed_env, offset_policy;
  int32_t T, B;
  int32_t num_action_chunks; /* C: 1, or 2..8 in the tensor-core kernel */
  int32_t max_episode_steps, auto_reset;
  int32_t bootstrap_on_done; /* 1: bootstrap where done ("always"), 0: where truncated ("standard") */
  double gamma, p_term, noise_std, reward_noise_std;
} rb200_rollout_args;

/* fp32 SIMT kernel (csrc/rollout_fused.cu): CTA c owns environments [c*E, c*E+E) for all T steps.
 * rb200_rollout_fused_supported() == 0 iff hidden == 256, obs_dim % 4 == 0, obs_dim <= 256, value_dim <= 1 and
 * B <= 32 * #SM; rb200_rollout_fused() also needs num_action_chunks == 1 (else RB200_E_UNSUPPORTED).  `wt`
 * (rb200_rollout_fused_wt_floats floats) holds the transposed hidden weights; refresh it with
 * rb200_rollout_fused_prepare() after every parameter update. */
int64_t rb200_rollout_fused_wt_floats(const rb200_mlp_layout* L);
int rb200_rollout_fused_supported(const rb200_mlp_layout* L, int B);
int rb200_rollout_fused_prepare(const rb200_mlp_layout* L, const float* params, float* wt, rb200_stream_t stream);
int rb200_rollout_fused(const rb200_mlp_layout* L, const float* params, const float* wt, const rb200_rollout_args* a,
                        rb200_stream_t stream);

/* TENSOR-CORE kernel (csrc/rollout_tc.cu): every hidden layer of both towers and the env's s.W_s product run on wgmma
 * (fp16 in, 2-way fp16 split with fp32 accumulation, computed transposed: D[hidden unit, env] = W . X^T, 32 environments
 * per CTA, activations handed from the accumulator registers to the next layer's operand tile in shared memory); the
 * truncation bootstrap V(final_obs) rides in 32 extra MMA columns of the next step's value tower.  The weights are
 * streamed from a packed, pre-split, pre-swizzled copy (rb200_rollout_tc_pack_bytes bytes, 16-byte aligned) that
 * rb200_rollout_tc_prepare() rebuilds from the flat parameters and the env's w_s [obs,obs] after every parameter update.
 * Chunked policies (C = num_action_chunks > 1, act_dim = C*A): per chunk step one actor / value inference on obs_n,
 * then C synthetic-env sub-steps without reset (sub-step c uses action columns [cA, (c+1)A)), flags OR-ed over the
 * chunk, one auto-reset after the chunk and the truncation bootstrap on the last column - the semantics and random
 * streams of rb200_synth_env_chunk_step plus rb200_bootstrap_rewards_ld.
 * rb200_rollout_tc_supported(L, C, B) == 0 iff hidden == 256, obs_dim % 32 == 0, obs_dim <= 128, B > 0 and
 *   C == 1:  value_dim == 1, act_dim <= 8;
 *   C > 1:   2 <= C <= 8, act_dim = C*A with 1 <= A <= 8 and C*A <= 32, value_dim == C.
 * rb200_rollout_tc() checks it for (a->num_action_chunks, a->B) first. */
int rb200_rollout_tc_supported(const rb200_mlp_layout* L, int num_action_chunks, int B);
int64_t rb200_rollout_tc_pack_bytes(const rb200_mlp_layout* L);
int rb200_rollout_tc_prepare(const rb200_mlp_layout* L, const float* params, const float* w_s, void* pack,
                             rb200_stream_t stream);
int rb200_rollout_tc(const rb200_mlp_layout* L, const float* params, const void* pack, const rb200_rollout_args* a,
                     rb200_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * SURVEY 8(f)3: token log-probabilities and entropies straight from the logits (csrc/logits.cu).
 * Replaces compute_logprobs_from_logits (rlinf/utils/utils.py:454-492, = -cross_entropy) and
 * compute_entropy_from_logits (:495-512, = -sum p log p over log_softmax) together with what their callers do first:
 * logits.div_(temperature) (workers/actor/fsdp_actor_worker.py:478) and the OpenVLA action-bin window, every logit
 * outside [v_lo, v_hi) treated as -inf (models/embodiment/openvla_oft/rlinf/openvla_oft_action_model.py:546-551).
 * logits: dtype 0 = fp32, 1 = bf16; row r lives at logits + (r / L) * batch_stride + (r % L) * row_stride (elements),
 * so the `[:, -L-1:-1, :]` slice of a [bsz, S, V] tensor needs no copy.  Forward reads every logit once and writes
 * logprob / entropy / lse [N] fp32 (entropy, lse nullable); backward reads the logits once more and writes
 *   dlogits_i = inv_T * (g_lp * (1[i = target] - p_i) - g_H * p_i * (log p_i + H)),  0 outside the window,
 * in the logits' dtype with its own strides d_batch_stride / d_row_stride (grad_logprob / grad_entropy nullable = zero). */
int rb200_logits_logprob_entropy_fwd(const void* logits, int dtype, const int64_t* target, int64_t N, int64_t L,
                                     int64_t batch_stride, int64_t row_stride, int V, int v_lo, int v_hi,
                                     double inv_temperature, float* logprob, float* entropy, float* lse,
                                     rb200_stream_t stream);
int rb200_logits_logprob_entropy_bwd(const void* logits, int dtype, const int64_t* target, int64_t N, int64_t L,
                                     int64_t batch_stride, int64_t row_stride, int V, int v_lo, int v_hi,
                                     double inv_temperature, const float* lse, const float* entropy,
                                     const float* grad_logprob, const float* grad_entropy, void* dlogits,
                                     int64_t d_batch_stride, int64_t d_row_stride, rb200_stream_t stream);

/* The same log-probabilities and entropies fused into the LM-head GEMM (csrc/lmhead.cu): z = (X . W^T) * inv_T from
 * the last hidden states X (bf16, row r at hidden + (r / L) * batch_stride + (r % L) * row_stride, strides multiples of
 * 8 elements) and the LM-head weight W [V, H] (bf16 row-major, no bias), H % 64 == 0, 64 <= H <= 8192; the logits are
 * never stored.  Window, temperature, target handling and outputs as in rb200_logits_logprob_entropy_*.
 * workspace: device memory of workspace_bytes (16-byte aligned).  rb200_lmhead_workspace_bytes() returns what the
 * forward and a backward with vocabulary chunks of vocab_chunk columns (<= 0: the whole window) need, or -1 for an
 * unsupported shape.  The backward derives its chunk from workspace_bytes: the whole window when its bf16 dZ [N, window]
 * fits, else what fits after an fp32 [N, H] dX accumulator, in multiples of 256 columns (RB200_E_ARG below 256).
 * Backward: d_hidden [N, H] and d_weight [V, H] bf16, contiguous, either nullable (not computed); d_weight rows outside
 * the window are 0.  Deterministic: a fixed order, no atomics, nothing depends on the SM count. */
int64_t rb200_lmhead_workspace_bytes(int64_t N, int64_t L, int H, int V, int v_lo, int v_hi, int64_t vocab_chunk);
int rb200_lmhead_logprob_entropy_fwd(const void* hidden, const void* weight, const int64_t* target, int64_t N, int64_t L,
                                     int64_t batch_stride, int64_t row_stride, int H, int V, int v_lo, int v_hi,
                                     double inv_temperature, float* logprob, float* entropy, float* lse,
                                     void* workspace, int64_t workspace_bytes, rb200_stream_t stream);
int rb200_lmhead_logprob_entropy_bwd(const void* hidden, const void* weight, const int64_t* target, int64_t N, int64_t L,
                                     int64_t batch_stride, int64_t row_stride, int H, int V, int v_lo, int v_hi,
                                     double inv_temperature, const float* lse, const float* entropy,
                                     const float* grad_logprob, const float* grad_entropy, void* d_hidden,
                                     void* d_weight, void* workspace, int64_t workspace_bytes, rb200_stream_t stream);

/* Vocabulary-parallel (tensor-parallel) variants of the two ops above (csrc/vocab_parallel.cu, lmhead.cu, logits.cu).
 * Equal shards (Megatron's VocabUtility; the vocabulary is padded so that P divides it): rank k of P owns the global
 * vocabulary columns [vocab_start, vocab_start + Vs), vocab_start = k * Vs; its weight shard is W[k*Vs:(k+1)*Vs] [Vs, H],
 * its logits shard [..., Vs].  target holds global ids; [v_lo, v_hi) is the global window, 0 <= v_lo < v_hi <= P * Vs,
 * and each rank uses its intersection with the shard.
 * Record: each rank writes one 16-byte record per row, float4 {m, s, t, z_t} [N, 4] (16-byte aligned): the softmax
 * statistics of softmax_acc.cuh over the rank's part of the window (max m, s = sum e^(z-m), t = sum e^(z-m) (z-m)),
 * and z_t = the scaled logit of the target column if the rank owns it and it lies in the window, else 0.  A rank whose
 * shard misses the window writes {-inf, 0, 0, 0} and launches no row pass.
 * rb200_vp_combine: the gathered records [n_ranks, N, 4] (rank-major, rank 0 first) -> logprob / entropy / lse [N] as
 * the single-GPU ops write them (entropy, lse nullable).  Rows are merged in rank order and z_t comes from rank
 * target / Vs, so every rank that combines the same records gets the same bits; with one rank the results are
 * bit-identical to rb200_lmhead_logprob_entropy_fwd / rb200_logits_logprob_entropy_fwd.
 * rb200_lmhead_vp_logprob_entropy_bwd: the single-GPU backward on the shard, given the global lse / entropy of the
 * combine: d_weight_shard [Vs, H] bf16 (rows outside the window 0) and d_hidden_partial [N, H] **fp32**, the rank's
 * share of dX for the caller to sum over ranks (so the sum rounds once, in the caller's final bf16 cast); either
 * nullable.  Its vocabulary chunk comes from workspace_bytes as in rb200_lmhead_logprob_entropy_bwd, with no fp32
 * accumulator (d_hidden_partial is it).  rb200_lmhead_vp_workspace_bytes() sizes the workspace of both lmhead entries
 * (vocab_chunk 0: the shard's whole part of the window in one chunk; < 0: the forward's workspace only).
 * The logits-level backward is rb200_logits_logprob_entropy_bwd on the shard with the global lse / entropy, the local
 * window and the shard-local target (target - vocab_start; values outside [0, Vs) get no target term). */
int64_t rb200_lmhead_vp_workspace_bytes(int64_t N, int64_t L, int H, int Vs, int64_t vocab_start, int v_lo, int v_hi,
                                        int64_t vocab_chunk);
int rb200_lmhead_vp_partials_fwd(const void* hidden, const void* weight_shard, const int64_t* target, int64_t N,
                                 int64_t L, int64_t batch_stride, int64_t row_stride, int H, int Vs,
                                 int64_t vocab_start, int v_lo, int v_hi, double inv_temperature, float* record,
                                 void* workspace, int64_t workspace_bytes, rb200_stream_t stream);
int rb200_lmhead_vp_logprob_entropy_bwd(const void* hidden, const void* weight_shard, const int64_t* target,
                                        int64_t N, int64_t L, int64_t batch_stride, int64_t row_stride, int H, int Vs,
                                        int64_t vocab_start, int v_lo, int v_hi, double inv_temperature,
                                        const float* lse, const float* entropy, const float* grad_logprob,
                                        const float* grad_entropy, float* d_hidden_partial, void* d_weight_shard,
                                        void* workspace, int64_t workspace_bytes, rb200_stream_t stream);
int rb200_logits_vp_partials_fwd(const void* logits, int dtype, const int64_t* target, int64_t N, int64_t L,
                                 int64_t batch_stride, int64_t row_stride, int Vs, int64_t vocab_start, int v_lo,
                                 int v_hi, double inv_temperature, float* record, rb200_stream_t stream);
int rb200_vp_combine(const float* records, int n_ranks, int64_t N, const int64_t* target, int vocab_shard, int v_lo,
                     int v_hi, float* logprob, float* entropy, float* lse, rb200_stream_t stream);

/* Response-rows plan (csrc/response_rows.cu): the rows of the flattened [T, H] hidden states that the reasoning loss
 * reads, for one of three batch layouts, as int64 index maps for rb200_gather_rows.  Sequence b: response length
 * r_b = response_lengths[b] (0 <= r_b <= L), first response row a_b, first row s_b:
 *   layout 0 (padded, [bsz, S] left-padded prompt, right-padded response): s_b = b S, a_b = b S + S - L; T = bsz S.
 *   layout 1 (FSDP-packed): len0 = prompt lengths p_b <= S (S = max prompt length), s_b = sum_{i<b} (p_i + r_i),
 *            a_b = s_b + p_b.
 *   layout 2 (Megatron THD, cp 1): len0 = cu_seqlens_padded [bsz + 1], len1 = valid tokens n_b, s_b = len0[b],
 *            a_b = s_b + n_b - r_b.
 * Sequence b owns n_b = r_b + entropy_shift compact rows (none when r_b = 0), holding hidden rows a_b - 1 + k; compact
 * row o_b + j predicts response token j, and holds column j's entropy at o_b + j + entropy_shift.  R = sum n_b.
 * Outputs (sentinel -1: the zero row the caller appends to the gather's source):
 *   rows [R]: hidden row of each compact row;  targets [R]: the token at row + 1, or -1 (outside every window) where
 *   the log-prob is not needed;  cell_map [bsz, L]: compact row of the cell's log-prob, or -1;  hidden_map [T]: compact
 *   row of each hidden row, or -1;  cells [R + 1]: cells[0] = -1, cells[1 + c] = the cell b L + j whose log-prob
 *   compact row c holds, or -1;  status [2] int64: {R, RB200_RR_* error bits}.
 * Only the first min(R, capacity) compact rows are written.  The lengths and tokens are device pointers; the checks
 * run on the device and land in status[1].  bsz <= 8192.  One launch. */
enum {
  RB200_RR_RESPONSE = 1,   /* r_b < 0 or r_b > L */
  RB200_RR_PROMPT = 2,     /* a sequence has no prompt token (a_b - s_b < 1) */
  RB200_RR_BOUNDS = 4,     /* rows outside [0, T) */
  RB200_RR_ORDER = 8,      /* sequences overlap or are not ascending (or overrun their padded segment) */
  RB200_RR_MAX_PROMPT = 16, /* p_b > max prompt length */
  RB200_RR_CAPACITY = 32   /* R > capacity */
};
int rb200_response_rows_plan(int layout, const int64_t* len0, const int64_t* len1, const int64_t* response_lengths,
                             int64_t bsz, int64_t S, int64_t L, int64_t T, int entropy_shift, const int64_t* tokens,
                             int64_t capacity, int64_t* rows, int64_t* targets, int64_t* cell_map,
                             int64_t* hidden_map, int64_t* cells, int64_t* status, rb200_stream_t stream);

/* Response-rows plan under Megatron sequence (SP) and context (CP) parallelism (csrc/response_rows_mp.cu), for one
 * rank (tp_rank, cp_rank).  Lengths as rb200_response_rows_plan's layout 2: cu_seqlens_padded [bsz + 1] (N_b = its
 * differences, multiples of 2 cp when cp > 1), seq_lengths n_b, response_lengths r_b; responses [bsz, L] holds the
 * targets.  Ownership follows preprocess_packed_seqs: with cp = 1 sequence b sits at CP-local rows cu[b] + p; with
 * cp > 1, half = N_b / (2 cp), CP rank c holds positions [half c, half (c + 1)) at rows cu[b] / cp + ... and
 * [N_b - half (c + 1), N_b - half c) at rows cu[b] / cp + half + ...  T_c = rows of the CP-local stream; under SP TP
 * rank k holds rows [k Ts, (k + 1) Ts), Ts = T_c / tp.  Token j < r_b is predicted at position n_b - r_b - 1 + j.
 * A CP rank's R_c compact rows are its prediction rows in ascending local row; TP shard k holds cnt_k of them, starting
 * at off_k.  Rmax_k = max(1, max_k cnt_k) (SP), Rmax_c = max(1, max_c R_c).  Outputs (-1 = pad / zero row):
 *   rows [R_c]: CP-local row of each compact row;  targets [R_c]: responses[b, j];  cells [R_c]: b L + j;
 *   unpad [R_c]: row of the TP-gathered [tp, Rmax_k] buffer holding each compact row (SP; identity without);
 *   send [Rmax_k] (SP): the rank's compact rows as rows of its shard, -1 past cnt_k;
 *   slot_map [tp * Rmax_k] (SP): the compact row each slot of the reduce-scatter layout carries, or -1;
 *   cell_map [bsz L]: row of the CP-gathered [cp, Rmax_c] values holding cell (b, j), or -1 for j >= r_b;
 *   hidden_map [Ts] (SP: the slot of the reduce-scattered [Rmax_k] rows) or [T_c] (no SP: the compact row), or -1;
 *   status [1 + cp tp]: {RB200_RR_* bits, then cnt of every rank (c, k) in c-major order (R_c in every k without SP)}.
 * Only entries below capacity_c (R_c) and capacity_k (Rmax_k) are written.  tp * cp <= 64, bsz <= 8192.  One launch. */
enum {
  RB200_RR_SHARD = 64,     /* T_c < cu[bsz] / cp, or T_c not divisible by tp under SP */
  RB200_RR_CP_ALIGN = 128  /* cp > 1 and a padded length N_b (or cu[0]) is not a multiple of 2 cp */
};
int rb200_response_rows_mp_plan(const int64_t* cu_seqlens_padded, const int64_t* seq_lengths,
                                const int64_t* response_lengths, const int64_t* responses, int64_t bsz, int64_t L,
                                int64_t T_c, int tp_size, int cp_size, int sequence_parallel, int tp_rank, int cp_rank,
                                int64_t capacity_c, int64_t capacity_k, int64_t* rows, int64_t* send, int64_t* unpad,
                                int64_t* slot_map, int64_t* targets, int64_t* cell_map, int64_t* cells,
                                int64_t* hidden_map, int64_t* status, rb200_stream_t stream);
/* Backward tail: out [n_out, H] bf16 = dx [idx[i], :] fp32 rounded once to nearest even, zero rows where idx[i] < 0.
 * With the plan's slot_map it writes the [tp, Rmax_k, H] reduce-scatter send layout; with its hidden_map (no SP), dX
 * of the whole [T_c, H] input.  H % 8 == 0, 16-byte aligned pointers. */
int rb200_response_rows_mp_pack_grad(const float* dx, const int64_t* idx, void* out, int64_t n_out, int64_t H,
                                     rb200_stream_t stream);

/* Value tower only: values [n,value_dim] = ValueHead(states). Used for the bootstrap value of
 * final observations (get_bootstrap_values, workers/rollout/hf/huggingface_worker.py:612-627). */
int rb200_mlp_value(const rb200_mlp_layout* L, const float* params, const float* wsplit,
                    const float* states, int64_t n, float* values, float* work, rb200_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Rollout-side helpers (device-resident rollout loop; replaces the per-chunk-step Channel hops with
 * CPU staging of env_worker.py:1087-1202 / huggingface_worker.py:678-704).
 * ---------------------------------------------------------------------------------------- */
/* Synthetic vector env step implementing the chunk_step contract (C = 1):
 *   s' = tanh(s.W_s + a.W_a + noise_std*eps), r = -|s'|^2/obs + reward_noise_std*eps_r,
 *   term ~ Bernoulli(p_term), trunc at max_episode_steps, auto-reset to N(0,I).
 * w_s [obs,obs] (in,out), w_a [act,obs]; noise: optional pre-drawn [B, 2*obs+2] (parity mode), else
 * Philox(seed, *counter_dev). final_obs = observation before the reset. */
int rb200_synth_env_step(const float* w_s, const float* w_a, const float* state, const float* action,
                         const float* noise, float* next_state, float* final_obs, float* reward,
                         uint8_t* term, uint8_t* trunc, uint8_t* done, int32_t* elapsed, float* z_scratch,
                         int B, int obs, int act, int max_episode_steps, int auto_reset, float p_term,
                         float noise_std, float reward_noise_std, uint64_t seed,
                         const uint64_t* counter_dev, rb200_stream_t stream);
/* env.chunk_step for num_action_chunks = C > 1 (rlinf/envs/maniskill/maniskill_env.py:327-375): C sub-steps of the
 * synthetic env WITHOUT auto-reset (sub-step c takes columns [c*act, (c+1)*act) of chunk_actions [B, C*act]), rewards
 * [B,C] of every sub-step, terminations / truncations / dones [B,C] all-zero except the last column = any over the
 * chunk, ONE auto-reset after the chunk (final_obs = observation before it).  noise: optional pre-drawn
 * [B, C*(obs+2) + obs] = per sub-step eps[obs] | eps_r | u_term, then the reset state; else Philox(seed, counter).
 * scratch: 3*B*obs floats. */
int rb200_synth_env_chunk_step(const float* w_s, const float* w_a, const float* state, const float* chunk_actions,
                               const float* noise, float* next_state, float* final_obs, float* rewards,
                               uint8_t* term, uint8_t* trunc, uint8_t* done, int32_t* elapsed, float* scratch,
                               int B, int obs, int act, int C, int max_episode_steps, int auto_reset, float p_term,
                               float noise_std, float reward_noise_std, uint64_t seed, const uint64_t* counter_dev,
                               rb200_stream_t stream);
/* strided form of rb200_bootstrap_rewards for the last sub-step of a chunk:
 * rewards[b*ld_rewards] += gamma * final_values[b*value_dim] where flag[b*ld_flag]  (env_worker.py:736-758) */
int rb200_bootstrap_rewards_ld(float* rewards, int ld_rewards, const float* final_values, int value_dim,
                               const uint8_t* flag, int ld_flag, int B, double gamma, rb200_stream_t stream);
/* rewards[b] += gamma * final_values[b*value_dim] where flag[b]  (compute_bootstrap_rewards,
 * workers/env/env_worker.py:736-758; flag = truncations ("standard") or dones ("always")). */
int rb200_bootstrap_rewards(float* rewards, const float* final_values, const uint8_t* flag, int B,
                            int value_dim, double gamma, rb200_stream_t stream);
/* counter_dev[0] += inc (device-side RNG step counter so captured CUDA graphs replay fresh noise). */
int rb200_counter_add(uint64_t* counter_dev, uint64_t inc, rb200_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * Policy evaluation (csrc/eval.cu; EmbodiedRunner.evaluate, rlinf/runners/embodied_runner.py:193-206,308-329).
 * ---------------------------------------------------------------------------------------- */
/* Eval-mode inference, _generate_actions(mode="eval") (mlp_policy.py:256-293): actor tower and mean head only,
 * action [n,act] = mean; logprobs [n,act] = Normal(mean, exp(logstd)).log_prob(mean) (NULL = not computed);
 * values [n,value_dim] = ValueHead(states) (NULL = value tower skipped).  No sampling, no RNG.
 * work: rb200_mlp_fwd_scratch_floats(L, n) floats; wsplit as for rb200_mlp_sample. */
int rb200_mlp_mean(const rb200_mlp_layout* L, const float* params, const float* wsplit, const float* states,
                   int64_t n, float* action, float* logprobs, float* values, float* work, rb200_stream_t stream);
/* Episode statistics of one chunk step of an evaluation rollout, one thread per env (ManiskillEnv._record_metrics /
 * _reset_metrics / _handle_auto_reset, maniskill_env.py:225-271,327-390; EnvWorker.env_evaluate_step,
 * env_worker.py:557-620).  rewards [B,C] fp32, done [B,C] (column C-1 = the chunk's done flag):
 *   ret += rewards[c] for c = 0..C-1 in order (fp32);  len += C;
 *   newly = auto_reset ? done : done && !prev_done;  prev_done |= done;
 *   on newly: acc[b] += {1, ret, len, ret / (float)len} (fp64);
 *   then, if auto_reset && done: ret = len = 0.
 * ret [B] fp32, len [B] int32, prev_done [B] u8, acc [B,4] fp64 are zeroed by the caller at the start of an
 * evaluation (ret / len / prev_done also at every env reset).  episode [B,3] (nullable): (return, length, reward) of
 * the episode env b finished in this step, NaN in all three columns otherwise. */
int rb200_episode_stats_step(const float* rewards, const uint8_t* done, int B, int C, int auto_reset, float* ret,
                             int32_t* len, uint8_t* prev_done, double* acc, float* episode, rb200_stream_t stream);
/* out[4] = {count, sum return, sum length, sum reward} over the B rows of acc [B,4], summed in a fixed order by one
 * CTA (no atomics): repeated runs give bit-identical results. */
int rb200_episode_stats_reduce(const double* acc, int B, double* out, rb200_stream_t stream);
/* Training-rollout episode statistics of one chunk step of the per-kernel loop (run after the env step, before the
 * truncation bootstrap adds to rewards): the rb200_episode_stats_step update with the training record rule of the
 * persistent rollouts (rb200_rollout_args.episode_return) - auto_reset: every env whose chunk is done records and
 * restarts ret / len; otherwise every env records at the rollout's last chunk step (last_step != 0) and none before.
 * len [B] int32 is the env's elapsed count, zeroed with ret at every env reset.  Replaces the same reference lines. */
int rb200_train_episode_stats_step(const float* rewards, const uint8_t* done, int B, int C, int auto_reset,
                                   int last_step, float* ret, int32_t* len, double* acc, rb200_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * a10 reward filter: replaces the filter_rewards block of EmbodiedFSDPActor._process_received_rollout_batch,
 *   workers/actor/embodied_fsdp_actor_worker.py:236-282 (= preprocess_embodied_batch, rlinf/utils/utils.py:803-830).
 *   rewards f32 [nc,B,C]; loss_mask bool [nc,B,C] or NULL; keep_env bool [B] (scratch/out);
 *   out_mask bool [nc,B,C] (= keep & loss_mask) or [nc,B,1] when loss_mask is NULL.
 * ---------------------------------------------------------------------------------------- */
int rb200_reward_filter(const float* rewards, const uint8_t* loss_mask, uint8_t* out_mask, uint8_t* keep_env,
                        int nc, int B, int C, int group_size, float lower, float upper,
                        rb200_stream_t stream);

/* a18 kl_penalty (rlinf/algorithms/utils.py:26-64): mode 0 k1/kl, 1 abs, 2 k2/mse, 3 k3/low_var_kl.
 * out[n] = penalty, d_logprob[n] (NULL ok) = d penalty / d logprob. */
int rb200_kl_penalty(const float* logprob, const float* ref_logprob, float* out, float* d_logprob, int64_t n,
                     int mode, rb200_stream_t stream);

/* a24 masked statistics for compute_rollout_metrics (rlinf/utils/metric_utils.py:422-506):
 * out4 = {count, sum, min, max} of x[i] over entries with mask[i / mask_div] != 0 (mask NULL = all). */
int rb200_masked_stats(const float* x, const uint8_t* mask, int64_t n, int64_t mask_div, double* out4,
                       rb200_stream_t stream);

/* ------------------------------------------------------------------------------------------
 * SURVEY 8(f) rank 4 - the remaining advantage estimators of ADV_REGISTRY (rlinf/algorithms/advantages.py) and the
 * fp64 masked normalisations of rlinf/utils/distributed.py (a24).  Step-major [L,B] tensors, uint8 0/1 masks.
 * ---------------------------------------------------------------------------------------- */
/* masked_stats (distributed.py:942-954) and the three sums masked_normalization all-reduces (:903-933):
 * out3 = {count, sum x, sum x^2} over entries with mask != 0 (mask NULL = all), accumulated in fp64. */
/* Fixed summation order (per-CTA slots in the library's per-device scratch, one ordered pass): repeated calls give the
 * same bits. The scratch is per device, so calls on one device must be stream-ordered. */
int rb200_masked_moments(const float* x, const uint8_t* mask, int64_t n, double* out3 /*reset by the call*/,
                         rb200_stream_t stream);
/* Apply half, stats3 = (all-reduced) {count, sum, sumsq}:
 *  mode 0  masked_normalization(dim=None) :935-939  out = (x*mask - mean)/(sqrt(var[*n/(n-1)]) + eps), fp64 -> fp32
 *  mode 1  normalize_from_stats :957-965            out = (x - mean) * rsqrt(max(var,0) + 1e-5)
 *  mode 2  reinforce++ whitening, advantages.py:355-362   out = (x - mean) * rsqrt(max(var, eps)), biased var */
int rb200_masked_normalize(const float* x, const uint8_t* mask, float* out, int64_t n, const double* stats3,
                           int mode, double eps, int unbiased, rb200_stream_t stream);
/* "raw", advantages.py:410-438: adv[l,b] = scores[b] * mask[l,b]; stats3 (nullable) = {n, sum, sumsq} of the valid
 * entries for the optional safe_normalize-style normalisation (rb200_normalize, eps 1e-5). */
int rb200_raw_advantages(const float* scores /*[B]*/, const uint8_t* loss_mask /*[L,B]*/, float* adv /*[L,B]*/,
                         int L, int B, double* stats3, rb200_stream_t stream);
/* "reinpp", advantages.py:302-364: reward at the reference's eos index (its fliplr quirk reproduced), optional
 * -kl_beta * kl_penalty(logprob, ref_logprob) per token (kl_mode as rb200_kl_penalty), reverse cumulative sum over L
 * (fp64 accumulation as torch's CPU cumsum); stats3 = masked {n, sum, sumsq} of the returns for mode-2 whitening. */
int rb200_reinpp_returns(const float* rewards /*[B]*/, const uint8_t* loss_mask /*[L,B]*/, const float* logprob,
                         const float* ref_logprob, float* ret /*[L,B]*/, int L, int B, double kl_beta, int kl_mode,
                         double* stats3, rb200_stream_t stream);
/* "grpo_video", advantages.py:124-164: mode 0 = "frame", 1 = "video"; the mask is float in the reference (plain
 * product): pass it as mask_f32, or a 0/1 byte mask as mask_u8 (both NULL = no mask). */
int rb200_grpo_video_advantages(const float* rewards /*[S,B]*/, const float* mask_f32, const uint8_t* mask_u8,
                                float* adv /*[S,B]*/, int S, int B, int G, int mode, float eps, rb200_stream_t stream);
/* "grpo_dynamic", advantages.py:167-299: per-turn advantages [n] from per-turn rewards and the turn -> trajectory map
 * (int32, device); mode 0 = "trajectory", 1 = "turn".  The caller broadcasts over the sequence with the loss mask. */
int rb200_grpo_dynamic_turn_advantages(const float* rewards /*[n]*/, const int32_t* idx_to_traj /*[n]*/,
                                       float* turn_adv /*[n]*/, int n, int num_trajectories, int G, int mode,
                                       float eps, rb200_stream_t stream);
/* out = a - b, fp32 ("opd" advantages = teacher_logprobs - prev_logprobs, advantages.py:393). */
int rb200_sub(const float* a, const float* b, float* out, int64_t n, rb200_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* RLINF_B200_H */
