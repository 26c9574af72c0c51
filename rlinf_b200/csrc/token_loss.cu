// Token-level PPO-clip actor loss of the reasoning workers, forward and backward on the device with no host sync:
// the loss block of FSDPActor.training_step (rlinf/workers/actor/fsdp_actor_worker.py:700-780) and of the Megatron
// loss_func (megatron_actor_worker.py:194-293) - the importance-sampling fix, policy_loss(task_type="reasoning")
// = compute_ppo_actor_loss (rlinf/algorithms/losses.py:170-312) with its loss_agg_func and fast_path_zero_loss_mask,
// the entropy term, the KL-to-reference term and compute_rollout_train_kl (fsdp_actor_worker.py:75-93) - plus
// autograd's backward of all of it for a unit upstream gradient.
//
// Four launches, no floating-point atomics, nothing that depends on the SM count: rows are cut into segments of
// kSeg tokens and each (segment, row) is one CTA.
//   1. count_kernel: the mask count of each (segment, row), one int per slot.
//   2. totals_kernel (one CTA): row counts, the total count and the first-row-empty flag (the fast path).
//   3. main_kernel: the gradients (they need the denominators of step 2) and kNS fp64 partial sums per
//      (segment, row), written to fixed slots.
//   4. finalize_kernel (one CTA): adds the partials in a fixed order - per row over its segments, then over rows -
//      applies the aggregation and writes the loss and the metrics.
// Elementwise arithmetic is fp32 in the reference's op order (ppo_unit.cuh, kl_unit.cuh); sums are fp64.
#include "common.cuh"
#include "kl_unit.cuh"
#include "ppo_unit.cuh"
#include "token_counts.cuh"

namespace {

constexpr int kThreads = 256;
constexpr int kPerThread = 4;
constexpr int kSeg = kThreads * kPerThread;  // tokens per CTA

enum Slot { P_L = 0, P_LABS, P_RATIO, P_RABS, P_CLIPPED, P_DUAL, P_LR, P_CLIPFRAC, P_ENT, P_KL, P_RTKL, kNS };

struct Hyper {
  float clip_lo_bound, clip_hi_bound;  // fl32(1 - low), fl32(1 + high)
  float dual_c;                        // <= 0: off
  int has_lr_min, has_lr_max;
  float lr_min, lr_max;
};

// workspace layout
struct Totals {
  long long total;  // mask count of the micro-batch
  int first_empty;  // loss_mask[0].sum() == 0
};
struct WsLayout {
  int64_t seg_cnt, row_cnt, partials, bytes;
};
__host__ __device__ inline WsLayout ws_layout(int64_t bsz, int64_t nseg) {
  WsLayout w;
  w.seg_cnt = 64;
  w.row_cnt = w.seg_cnt + ((bsz * nseg * 4 + 15) / 16) * 16;
  w.partials = w.row_cnt + bsz * 8;
  w.bytes = w.partials + bsz * nseg * kNS * 8;
  return w;
}

__device__ __forceinline__ int block_sum_int(int v, int* smem) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if (lane == 0) smem[warp] = v;
  __syncthreads();
  int s = 0;
  if (threadIdx.x == 0)
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) s += smem[w];
  return s;
}

__global__ void __launch_bounds__(kThreads) count_kernel(const uint8_t* __restrict__ mask, int64_t mask_stride,
                                                         int64_t L, int* __restrict__ seg_cnt) {
  __shared__ int red[32];
  const int64_t row = blockIdx.y, seg = blockIdx.x;
  const int64_t j0 = seg * kSeg;
  int c = 0;
#pragma unroll
  for (int k = 0; k < kPerThread; ++k) {
    const int64_t j = j0 + k * kThreads + threadIdx.x;
    if (j < L) c += mask[row * mask_stride + j] != 0;
  }
  c = block_sum_int(c, red);
  if (threadIdx.x == 0) seg_cnt[row * gridDim.x + seg] = c;
}

__global__ void __launch_bounds__(1024) totals_kernel(const int* __restrict__ seg_cnt, int64_t bsz, int nseg,
                                                      long long* __restrict__ row_cnt, Totals* __restrict__ tot) {
  __shared__ long long red[32];
  long long acc = 0;
  for (int64_t i = threadIdx.x; i < bsz; i += blockDim.x) {
    long long c = 0;
    for (int s = 0; s < nseg; ++s) c += seg_cnt[i * nseg + s];
    row_cnt[i] = c;
    acc += c;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    long long t = 0;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) t += red[w];
    tot->total = t;
    tot->first_empty = row_cnt[0] == 0;
  }
}

// d (aggregated value) / d (element value) of a valid element of a row with `cnt` valid tokens
__device__ __forceinline__ float agg_coef(int agg, long long total, long long cnt, int64_t bsz) {
  if (agg == RB200_AGG_TOKEN_MEAN) return (float)(1.0 / (double)(total > 0 ? total : 1));
  if (agg == RB200_AGG_SEQ_MEAN_TOKEN_SUM) return (float)(1.0 / (double)bsz);
  return (float)(1.0 / ((double)bsz * (double)cnt));  // inf for an empty row: the reference's 0/0 NaN
}

__global__ void __launch_bounds__(kThreads) main_kernel(rb200_token_loss_args a, Hyper h,
                                                        const long long* __restrict__ row_cnt,
                                                        const Totals* __restrict__ tot,
                                                        double* __restrict__ partials) {
  __shared__ double red[kNS * 32];
  const int64_t row = blockIdx.y, seg = blockIdx.x;
  const int64_t L = a.L;
  const bool fast = a.fast_path_zero_loss_mask && tot->first_empty;
  const float c = agg_coef(a.agg, tot->total, row_cnt[row], a.bsz);
  const float ent_up = -(float)a.entropy_bonus * c;  // d loss / d (entropy * mask)
  const float kl_up = (float)a.kl_beta * c;          // d loss / d (kld * mask)
  const bool with_kl = a.ref_logprobs != nullptr && a.kl_beta > 0.0;
  const bool with_rr = a.rollout_logprobs != nullptr && a.recomputed_logprobs != nullptr;
  const float is_clip = (float)a.importance_sampling_clip;

  double acc[kNS];
#pragma unroll
  for (int k = 0; k < kNS; ++k) acc[k] = 0.0;

#pragma unroll
  for (int k = 0; k < kPerThread; ++k) {
    const int64_t j = seg * kSeg + k * kThreads + threadIdx.x;
    if (j >= L) break;
    const bool m = a.loss_mask[row * a.loss_mask_stride + j] != 0;
    const float mf = m ? 1.0f : 0.0f;
    const float lp = a.logprobs[row * a.logprobs_stride + j];
    float adv = a.advantages[row * a.advantages_stride + j];
    float rr_diff = 0.0f;
    if (with_rr)
      rr_diff = __fsub_rn(a.recomputed_logprobs[row * a.recomputed_logprobs_stride + j],
                          a.rollout_logprobs[row * a.rollout_logprobs_stride + j]);
    if (a.importance_sampling_fix) adv = __fmul_rn(adv, fminf(expf(rr_diff), is_clip));
    const rb::RatioOut o = rb::ratio_terms(lp, a.old_logprobs[row * a.old_logprobs_stride + j], adv, m, h);
    acc[P_L] += (double)__fmul_rn(o.loss_e, mf);
    acc[P_LABS] += (double)__fmul_rn(fabsf(o.loss_e), mf);
    acc[P_RATIO] += (double)__fmul_rn(o.ratio, mf);
    acc[P_RABS] += (double)__fmul_rn(fabsf(__fsub_rn(o.ratio, 1.0f)), mf);
    acc[P_CLIPPED] += (double)__fmul_rn(o.clipped, mf);
    acc[P_DUAL] += (double)o.dual_ratio;
    acc[P_LR] += (double)o.lr_kl;
    acc[P_CLIPFRAC] += (double)__fmul_rn(o.clip_hit, mf);
    float dlp = (m && !fast) ? o.dL_dlp * c : 0.0f;  // torch.where(mask, exp(lr), 0): masked tokens get 0
    if (a.entropy) {
      acc[P_ENT] += (double)__fmul_rn(a.entropy[row * a.entropy_stride + j], mf);
      if (a.d_entropy) a.d_entropy[row * L + j] = ent_up * mf;
    }
    if (with_kl) {
      const float ref = a.ref_logprobs[row * a.ref_logprobs_stride + j];
      const float x = a.kl_order ? ref : lp, y = a.kl_order ? lp : ref;
      float g;
      const float v = rb::kl_penalty_unit(x, y, a.kl_mode, g);
      acc[P_KL] += (double)__fmul_rn(v, mf);
      const float dv_dlp = a.kl_order ? -g : g;  // every kind is a function of x - y
      if (!rb::kl_penalty_blocked(x, y, a.kl_mode)) dlp += (kl_up * mf) * dv_dlp;
    }
    if (with_rr) acc[P_RTKL] += (double)__fmul_rn(fabsf(rr_diff), mf);
    if (a.d_logprobs) a.d_logprobs[row * L + j] = dlp;
  }

  rb::block_sum<kNS>(acc, red);
  if (threadIdx.x == 0) {
    double* p = partials + (row * gridDim.x + seg) * kNS;
#pragma unroll
    for (int k = 0; k < kNS; ++k) p[k] = acc[k];
  }
}

__global__ void __launch_bounds__(kThreads) finalize_kernel(rb200_token_loss_args a, int nseg,
                                                            const long long* __restrict__ row_cnt,
                                                            const Totals* __restrict__ tot,
                                                            const double* __restrict__ partials) {
  __shared__ double red[kNS * 32];
  double acc[kNS];
#pragma unroll
  for (int k = 0; k < kNS; ++k) acc[k] = 0.0;
  for (int64_t i = threadIdx.x; i < a.bsz; i += blockDim.x) {
    double rs[kNS];
#pragma unroll
    for (int k = 0; k < kNS; ++k) rs[k] = 0.0;
    for (int s = 0; s < nseg; ++s) {
      const double* p = partials + (i * nseg + s) * kNS;
#pragma unroll
      for (int k = 0; k < kNS; ++k) rs[k] += p[k];
    }
    if (a.agg == RB200_AGG_SEQ_MEAN_TOKEN_MEAN) {  // token-mean inside the row: 0/0 = NaN for an empty row
      const double cnt = (double)row_cnt[i];
      rs[P_L] /= cnt;
      rs[P_LABS] /= cnt;
      rs[P_ENT] /= cnt;
      rs[P_KL] /= cnt;
    }
#pragma unroll
    for (int k = 0; k < kNS; ++k) acc[k] += rs[k];
  }
  rb::block_sum<kNS>(acc, red);
  if (threadIdx.x != 0) return;

  const long long total = tot->total;
  const bool fast = a.fast_path_zero_loss_mask && tot->first_empty;
  // masked_mean: sum(v * m) / sum(m), or the plain sum when every token is masked; count_nonzero() or 1 likewise
  const double d_mean = total > 0 ? (double)total : 1.0;
  const double d_agg = a.agg == RB200_AGG_TOKEN_MEAN ? d_mean : (double)a.bsz;
  float* M = a.metrics;
  for (int k = 0; k < RB200_TM_NUM; ++k) M[k] = 0.0f;
  const double policy = fast ? 0.0 : acc[P_L] / d_agg;
  if (!fast) {
    M[RB200_TM_POLICY_LOSS] = (float)policy;
    M[RB200_TM_POLICY_LOSS_ABS] = (float)(acc[P_LABS] / d_agg);
    M[RB200_TM_RATIO] = (float)(acc[P_RATIO] / d_mean);
    M[RB200_TM_RATIO_ABS] = (float)(acc[P_RABS] / d_mean);
    M[RB200_TM_CLIPPED_RATIO] = (float)(acc[P_CLIPPED] / d_mean);
    M[RB200_TM_DUAL_CLIPPED_RATIO] = (float)(acc[P_DUAL] / d_mean);
    M[RB200_TM_APPROX_KL] = (float)(-acc[P_LR] / d_mean);
    M[RB200_TM_CLIP_FRACTION] = (float)(acc[P_CLIPFRAC] / d_mean);
  }
  double loss = policy;
  if (a.entropy) {
    const double ent = acc[P_ENT] / d_agg;
    M[RB200_TM_ENTROPY_LOSS] = (float)ent;
    if (a.entropy_bonus > 0.0) loss -= a.entropy_bonus * ent;
  }
  if (a.ref_logprobs && a.kl_beta > 0.0) {
    const double kl = acc[P_KL] / d_agg;
    M[RB200_TM_KL_LOSS] = (float)kl;
    loss += a.kl_beta * kl;
  }
  if (a.rollout_logprobs && a.recomputed_logprobs) M[RB200_TM_ROLLOUT_TRAIN_KL] = (float)(acc[P_RTKL] / d_mean);
  M[RB200_TM_FINAL_LOSS] = (float)loss;
  a.loss[0] = (float)loss;
}

int64_t num_segments(int64_t L) { return (L + kSeg - 1) / kSeg; }

}  // namespace

static_assert(kSeg == rb::kTokenSeg && kThreads == rb::kTokenThreads && kNS == rb::kTokenSlots,
              "token_counts.cuh describes this file's segments and workspace");

rb::TokenCounts rb::token_mask_counts(const uint8_t* mask, int64_t mask_stride, int64_t bsz, int64_t L,
                                      void* workspace, cudaStream_t st) {
  const int64_t nseg = num_segments(L);
  const WsLayout w = ws_layout(bsz, nseg);
  char* ws = static_cast<char*>(workspace);
  Totals* tot = reinterpret_cast<Totals*>(ws);
  int* seg_cnt = reinterpret_cast<int*>(ws + w.seg_cnt);
  long long* row_cnt = reinterpret_cast<long long*>(ws + w.row_cnt);
  count_kernel<<<dim3((unsigned)nseg, (unsigned)bsz), kThreads, 0, st>>>(mask, mask_stride, L, seg_cnt);
  rb::count_launch();
  totals_kernel<<<1, 1024, 0, st>>>(seg_cnt, bsz, (int)nseg, row_cnt, tot);
  rb::count_launch();
  return {nseg, row_cnt, &tot->total, reinterpret_cast<double*>(ws + w.partials)};
}

extern "C" int64_t rb200_token_loss_workspace_bytes(int64_t bsz, int64_t L) {
  if (bsz <= 0 || L <= 0 || bsz > 65535) return -1;
  const int64_t nseg = num_segments(L);
  if (nseg > 0x7fffffff) return -1;
  return ws_layout(bsz, nseg).bytes;
}

extern "C" int rb200_token_ppo_loss(const rb200_token_loss_args* args, rb200_stream_t stream) {
  if (!args) return RB200_E_NULL;
  const rb200_token_loss_args& a = *args;
  if (!a.logprobs || !a.old_logprobs || !a.advantages || !a.loss_mask || !a.loss || !a.metrics || !a.workspace)
    return RB200_E_NULL;
  const int64_t need = rb200_token_loss_workspace_bytes(a.bsz, a.L);
  if (need < 0) return RB200_E_SHAPE;
  if (a.workspace_bytes < need) return RB200_E_ARG;
  if ((reinterpret_cast<uintptr_t>(a.workspace) & 15) != 0) return RB200_E_ALIGN;
  if (a.agg < RB200_AGG_TOKEN_MEAN || a.agg > RB200_AGG_SEQ_MEAN_TOKEN_MEAN) return RB200_E_ARG;
  if (a.kl_mode < 0 || a.kl_mode > 3) return RB200_E_ARG;
  if (a.clip_ratio_c > 0.0 && !(a.clip_ratio_c > 1.0)) return RB200_E_ARG;  // losses.py:260 assert
  if (a.d_entropy && !a.entropy) return RB200_E_NULL;
  if (a.importance_sampling_fix && (!a.rollout_logprobs || !a.recomputed_logprobs)) return RB200_E_NULL;
  if (a.logprobs_stride < a.L || a.old_logprobs_stride < a.L || a.advantages_stride < a.L ||
      a.loss_mask_stride < a.L || (a.entropy && a.entropy_stride < a.L) ||
      (a.ref_logprobs && a.ref_logprobs_stride < a.L) || (a.rollout_logprobs && a.rollout_logprobs_stride < a.L) ||
      (a.recomputed_logprobs && a.recomputed_logprobs_stride < a.L))
    return RB200_E_SHAPE;

  Hyper h;
  h.clip_lo_bound = (float)(1.0 - a.clip_ratio_low);
  h.clip_hi_bound = (float)(1.0 + a.clip_ratio_high);
  h.dual_c = a.clip_ratio_c > 0.0 ? (float)a.clip_ratio_c : 0.0f;
  h.has_lr_min = a.has_clip_log_ratio_min;
  h.has_lr_max = a.has_clip_log_ratio_max;
  h.lr_min = (float)a.clip_log_ratio_min;
  h.lr_max = (float)a.clip_log_ratio_max;

  const int64_t nseg = num_segments(a.L);
  const WsLayout w = ws_layout(a.bsz, nseg);
  char* ws = static_cast<char*>(a.workspace);
  Totals* tot = reinterpret_cast<Totals*>(ws);
  int* seg_cnt = reinterpret_cast<int*>(ws + w.seg_cnt);
  long long* row_cnt = reinterpret_cast<long long*>(ws + w.row_cnt);
  double* partials = reinterpret_cast<double*>(ws + w.partials);

  cudaStream_t st = rb::as_stream(stream);
  const dim3 grid((unsigned)nseg, (unsigned)a.bsz);
  count_kernel<<<grid, kThreads, 0, st>>>(a.loss_mask, a.loss_mask_stride, a.L, seg_cnt);
  rb::count_launch();
  totals_kernel<<<1, 1024, 0, st>>>(seg_cnt, a.bsz, (int)nseg, row_cnt, tot);
  rb::count_launch();
  main_kernel<<<grid, kThreads, 0, st>>>(a, h, row_cnt, tot, partials);
  rb::count_launch();
  finalize_kernel<<<1, kThreads, 0, st>>>(a, (int)nseg, row_cnt, tot, partials);
  rb::count_launch();
  RB_RETURN_LAUNCH();
}
