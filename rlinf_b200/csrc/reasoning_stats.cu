// Reasoning step bookkeeping on the device: the reasoning rollout metrics (rlinf/utils/distributed.py:34-306,
// compute_rollout_metrics_dynamic and compute_rollout_metrics), the tail of the Megatron workers' loss_func
// (megatron_actor_worker.py:258-307, megatron_critic_worker.py:104-121) and the training branch of
// _process_fwd_bwd_outputs (megatron_worker.py:550-599).
//
// The reference syncs the host once per metric and makes one collective per key; here each stage is a short chain of
// launches with no host sync, and the collectives are the caller's: one all-gather of [P, RB200_RR_NUM] records for
// the rollout metrics and one SUM all-reduce of the packed metrics per micro-batch.
//
// No floating-point atomics and nothing that depends on the SM count: partials go to fixed slots and are added in a
// fixed order, so two identical calls give the same bits.
#include <limits.h>
#include <math.h>

#include "common.cuh"
#include "token_counts.cuh"

namespace {

constexpr int kThreads = 256;
constexpr int kPerThread = 4;
constexpr int kSeg = kThreads * kPerThread;  // tokens per (segment, row) CTA
constexpr int kFinishThreads = 1024;

enum Part { P_ADV = 0, P_NVALID, P_ADV_MIN, P_ADV_MAX, P_VAL, P_VAL_MIN, P_VAL_MAX, kNP = 8 };

int64_t num_segments(int64_t L) { return (L + kSeg - 1) / kSeg; }

struct MinOp {
  __device__ double operator()(double a, double b) const { return fmin(a, b); }
};
struct MaxOp {
  __device__ double operator()(double a, double b) const { return fmax(a, b); }
};
struct SumOp {
  template <typename T>
  __device__ T operator()(T a, T b) const { return a + b; }
};
struct MaxLL {
  __device__ long long operator()(long long a, long long b) const { return a > b ? a : b; }
};
struct MinLL {
  __device__ long long operator()(long long a, long long b) const { return a < b ? a : b; }
};

// Block-wide reduction in a fixed tree (shuffle-xor within warps, then warp 0 over the warp results); the result is
// returned to every thread.  smem: 32 elements of T; the call ends with a barrier so smem can be reused.
template <typename T, class Op>
__device__ T block_all(T v, T* smem, Op op, T identity) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarp = (blockDim.x + 31) >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = op(v, __shfl_xor_sync(0xffffffffu, v, o));
  if (lane == 0) smem[warp] = v;
  __syncthreads();
  if (warp == 0) {
    T x = lane < nwarp ? smem[lane] : identity;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) x = op(x, __shfl_xor_sync(0xffffffffu, x, o));
    if (lane == 0) smem[0] = x;
  }
  __syncthreads();
  const T r = smem[0];
  __syncthreads();
  return r;
}

// Per (segment, row): fp64 sum, count, min and max of the valid advantages, and of the valid values when given.
__global__ void __launch_bounds__(kThreads) record_cells_kernel(rb200_reasoning_record_args a,
                                                                double* __restrict__ partials) {
  __shared__ double red[32];
  const int64_t row = blockIdx.y, seg = blockIdx.x;
  double s_adv = 0.0, n = 0.0, s_val = 0.0;
  double a_min = INFINITY, a_max = -INFINITY, v_min = INFINITY, v_max = -INFINITY;
#pragma unroll
  for (int k = 0; k < kPerThread; ++k) {
    const int64_t j = seg * kSeg + k * kThreads + threadIdx.x;
    if (j >= a.L) break;
    if (a.mask[row * a.mask_stride + j] == 0) continue;
    const double x = (double)a.advantages[row * a.advantages_stride + j];
    s_adv += x;
    n += 1.0;
    a_min = fmin(a_min, x);
    a_max = fmax(a_max, x);
    if (a.values) {
      const double v = (double)a.values[row * a.values_stride + j];
      s_val += v;
      v_min = fmin(v_min, v);
      v_max = fmax(v_max, v);
    }
  }
  double out[kNP];
  out[P_ADV] = block_all(s_adv, red, SumOp(), 0.0);
  out[P_NVALID] = block_all(n, red, SumOp(), 0.0);
  out[P_ADV_MIN] = block_all(a_min, red, MinOp(), (double)INFINITY);
  out[P_ADV_MAX] = block_all(a_max, red, MaxOp(), -(double)INFINITY);
  out[P_VAL] = block_all(s_val, red, SumOp(), 0.0);
  out[P_VAL_MIN] = block_all(v_min, red, MinOp(), (double)INFINITY);
  out[P_VAL_MAX] = block_all(v_max, red, MaxOp(), -(double)INFINITY);
  out[7] = 0.0;
  if (threadIdx.x == 0) {
    double* p = partials + (row * gridDim.x + seg) * kNP;
#pragma unroll
    for (int k = 0; k < kNP; ++k) p[k] = out[k];
  }
}

// One CTA: adds the cell partials in a fixed order, reduces the per-sequence fields and writes the record.
__global__ void __launch_bounds__(kFinishThreads) record_finish_kernel(rb200_reasoning_record_args a, int64_t nparts,
                                                                       const double* __restrict__ partials) {
  __shared__ double red[32];
  __shared__ long long redl[32];
  double s_adv = 0.0, n = 0.0, s_val = 0.0;
  double a_min = INFINITY, a_max = -INFINITY, v_min = INFINITY, v_max = -INFINITY;
  for (int64_t i = threadIdx.x; i < nparts; i += blockDim.x) {
    const double* p = partials + i * kNP;
    s_adv += p[P_ADV];
    n += p[P_NVALID];
    s_val += p[P_VAL];
    a_min = fmin(a_min, p[P_ADV_MIN]);
    a_max = fmax(a_max, p[P_ADV_MAX]);
    v_min = fmin(v_min, p[P_VAL_MIN]);
    v_max = fmax(v_max, p[P_VAL_MAX]);
  }
  s_adv = block_all(s_adv, red, SumOp(), 0.0);
  n = block_all(n, red, SumOp(), 0.0);
  s_val = block_all(s_val, red, SumOp(), 0.0);
  a_min = block_all(a_min, red, MinOp(), (double)INFINITY);
  a_max = block_all(a_max, red, MaxOp(), -(double)INFINITY);
  v_min = block_all(v_min, red, MinOp(), (double)INFINITY);
  v_max = block_all(v_max, red, MaxOp(), -(double)INFINITY);

  long long plen = 0, rlen = 0, rlen2 = 0, ends = 0, max_p = LLONG_MIN, max_r = LLONG_MIN, max_t = LLONG_MIN;
  long long min_r = LLONG_MAX, max_idx = -1, min_idx = 0;
  double s_rew = 0.0;
  for (int64_t i = threadIdx.x; i < a.bsz; i += blockDim.x) {
    const long long p = a.prompt_lengths[i], r = a.response_lengths[i];
    plen += p;
    rlen += r;
    rlen2 += r * r;
    ends += a.is_end[i] != 0;
    max_p = p > max_p ? p : max_p;
    max_r = r > max_r ? r : max_r;
    min_r = r < min_r ? r : min_r;
    max_t = p + r > max_t ? p + r : max_t;
    s_rew += (double)a.rewards[i];
    if (a.idx_to_traj) {
      const long long t = a.idx_to_traj[i];
      max_idx = t > max_idx ? t : max_idx;
      min_idx = t < min_idx ? t : min_idx;
    }
  }
  plen = block_all(plen, redl, SumOp(), 0LL);
  rlen = block_all(rlen, redl, SumOp(), 0LL);
  rlen2 = block_all(rlen2, redl, SumOp(), 0LL);
  ends = block_all(ends, redl, SumOp(), 0LL);
  max_p = block_all(max_p, redl, MaxLL(), LLONG_MIN);
  max_r = block_all(max_r, redl, MaxLL(), LLONG_MIN);
  max_t = block_all(max_t, redl, MaxLL(), LLONG_MIN);
  min_r = block_all(min_r, redl, MinLL(), LLONG_MAX);
  max_idx = block_all(max_idx, redl, MaxLL(), -1LL);
  min_idx = block_all(min_idx, redl, MinLL(), 0LL);
  s_rew = block_all(s_rew, red, SumOp(), 0.0);

  // multi-turn: per-trajectory fp32 reward sums in turn order, divided by max(count, 1) (distributed.py:86-93)
  const long long ntraj = max_idx + 1;
  double s_traj = 0.0;
  if (a.idx_to_traj && min_idx >= 0) {
    for (long long t = threadIdx.x; t < ntraj; t += blockDim.x) {
      float s = 0.0f;
      long long c = 0;
      for (int64_t i = 0; i < a.bsz; ++i) {
        if (a.idx_to_traj[i] == t) {
          s = __fadd_rn(s, a.rewards[i]);
          ++c;
        }
      }
      s_traj += (double)__fdiv_rn(s, (float)(c > 1 ? c : 1));
    }
  }
  s_traj = block_all(s_traj, red, SumOp(), 0.0);
  if (threadIdx.x != 0) return;

  double* R = a.record;
  for (int k = 0; k < RB200_RR_NUM; ++k) R[k] = 0.0;
  R[RB200_RR_SUM_PLEN] = (double)(float)plen;
  R[RB200_RR_SUM_RLEN] = (double)(float)rlen;
  R[RB200_RR_SUM_REWARDS] = (double)(float)s_rew;
  R[RB200_RR_SUM_END] = (double)(float)ends;
  R[RB200_RR_SUM_ADV] = (double)(float)s_adv;
  R[RB200_RR_NUM_SEQ] = (double)(float)a.bsz;
  R[RB200_RR_N_VALID] = (double)(float)n;
  R[RB200_RR_SUM_TRAJ_REWARDS] = (double)(float)s_traj;
  R[RB200_RR_NUM_TRAJ] = (double)(float)ntraj;
  R[RB200_RR_ADV_NEG_MIN] = (double)(-(float)a_min);
  R[RB200_RR_ADV_MAX] = (double)(float)a_max;
  R[RB200_RR_MAX_PLEN] = (double)(float)max_p;
  R[RB200_RR_MAX_RLEN] = (double)(float)max_r;
  R[RB200_RR_MAX_TOTAL] = (double)(float)max_t;
  R[RB200_RR_VAL_NEG_MIN] = (double)(-(float)v_min);
  R[RB200_RR_VAL_MAX] = (double)(float)v_max;
  R[RB200_RR_VALUES_MEAN] = n > 0.0 ? (double)(float)(s_val / n) : (double)NAN;
  R[RB200_RR_RLEN_SUM] = (double)rlen;
  R[RB200_RR_RLEN_SQ_SUM] = (double)rlen2;
  R[RB200_RR_RLEN_MIN] = (double)min_r;
  R[RB200_RR_RLEN_MAX] = (double)max_r;
  R[RB200_RR_VERDICT] = (double)((n > 0.0 ? 0 : RB200_RV_EMPTY) | (a.idx_to_traj && min_idx < 0 ? RB200_RV_BAD_TRAJ : 0));
}

// One thread: the P records in rank order -> the metric vector.  The SUM fields are added in fp32 (the reference's
// fp32 all-reduce), the MAX fields take the max, and the metrics are formed in fp64 as the reference's host code does.
__global__ void rollout_finish_kernel(const double* __restrict__ rec, int P, const float* __restrict__ world_sum,
                                      int world, double* __restrict__ M) {
  if (threadIdx.x != 0) return;
  float S[RB200_RR_NUM_TRAJ + 1];
  for (int k = 0; k <= RB200_RR_NUM_TRAJ; ++k) S[k] = 0.0f;
  float X[RB200_RR_VAL_MAX + 1];
  for (int k = RB200_RR_ADV_NEG_MIN; k <= RB200_RR_VAL_MAX; ++k) X[k] = -INFINITY;
  float vsum = 0.0f;
  double rl_sum = 0.0, rl_sq = 0.0, rl_min = INFINITY, rl_max = -INFINITY, nmax = 0.0;
  long long verdict = 0;
  for (int r = 0; r < P; ++r) {
    const double* R = rec + (int64_t)r * RB200_RR_NUM;
    for (int k = 0; k <= RB200_RR_NUM_TRAJ; ++k) S[k] = __fadd_rn(S[k], (float)R[k]);
    for (int k = RB200_RR_ADV_NEG_MIN; k <= RB200_RR_VAL_MAX; ++k) X[k] = fmaxf(X[k], (float)R[k]);
    vsum = __fadd_rn(vsum, (float)R[RB200_RR_VALUES_MEAN]);
    rl_sum += R[RB200_RR_RLEN_SUM];
    rl_sq += R[RB200_RR_RLEN_SQ_SUM];
    rl_min = fmin(rl_min, R[RB200_RR_RLEN_MIN]);
    rl_max = fmax(rl_max, R[RB200_RR_RLEN_MAX]);
    nmax = fmax(nmax, R[RB200_RR_NUM_SEQ]);
    verdict |= (long long)R[RB200_RR_VERDICT];
  }
  const double nseq = (double)S[RB200_RR_NUM_SEQ];
  const double ntraj = (double)S[RB200_RR_NUM_TRAJ];
  M[RB200_RM_NUM_SEQ] = nseq;
  M[RB200_RM_PROMPT_LENGTH] = (double)S[RB200_RR_SUM_PLEN] / nseq;
  M[RB200_RM_RESPONSE_LENGTH] = (double)S[RB200_RR_SUM_RLEN] / nseq;
  M[RB200_RM_TOTAL_LENGTH] = ((double)S[RB200_RR_SUM_PLEN] + (double)S[RB200_RR_SUM_RLEN]) / nseq;
  M[RB200_RM_REWARD_SCORES] = (double)S[RB200_RR_SUM_REWARDS] / nseq;
  M[RB200_RM_PROPERLY_ENDED] = (double)S[RB200_RR_SUM_END] / nseq;
  M[RB200_RM_ADV_MEAN] = (double)S[RB200_RR_SUM_ADV] / (double)S[RB200_RR_N_VALID];
  M[RB200_RM_ADV_MAX] = (double)X[RB200_RR_ADV_MAX];
  M[RB200_RM_ADV_MIN] = -(double)X[RB200_RR_ADV_NEG_MIN];
  M[RB200_RM_VALUES_MEAN] = world_sum ? (double)__fdiv_rn(*world_sum, (float)world) : (double)__fdiv_rn(vsum, (float)P);
  M[RB200_RM_VALUES_MAX] = (double)X[RB200_RR_VAL_MAX];
  M[RB200_RM_VALUES_MIN] = -(double)X[RB200_RR_VAL_NEG_MIN];
  M[RB200_RM_MAX_PROMPT_LENGTH] = (double)X[RB200_RR_MAX_PLEN];
  M[RB200_RM_MAX_RESPONSE_LENGTH] = (double)X[RB200_RR_MAX_RLEN];
  M[RB200_RM_MAX_TOTAL_LENGTH] = (double)X[RB200_RR_MAX_TOTAL];
  M[RB200_RM_REWARD_SCORES_TRAJ] = (double)S[RB200_RR_SUM_TRAJ_REWARDS] / ntraj;
  M[RB200_RM_REWARD_SCORES_TURN] = (double)S[RB200_RR_SUM_REWARDS] / nseq;
  M[RB200_RM_AVG_TURNS_PER_TRAJ] = nseq / ntraj;
  // statistics of the gathered decode lengths: total_decode_lengths.float().mean() / .var() / .aminmax()
  // (distributed.py:225-228) from exact integer sums; the variance is formed exactly and rounded once
  double count = 0.0;
  for (int r = 0; r < P; ++r) count += rec[(int64_t)r * RB200_RR_NUM + RB200_RR_NUM_SEQ];
  M[RB200_RM_AVG_RESPONSE_LENGTH] = (double)__fdiv_rn((float)rl_sum, (float)count);
  if (count > 1.0) {
    const __int128 cn = (__int128)(long long)count, s = (__int128)(long long)rl_sum, s2 = (__int128)(long long)rl_sq;
    const __int128 num = cn * s2 - s * s;  // n^2 (n - 1) / n  times the unbiased variance, exact
    M[RB200_RM_VAR_RESPONSE_LENGTH] = (double)(float)((double)num / (count * (count - 1.0)));
  } else {
    M[RB200_RM_VAR_RESPONSE_LENGTH] = (double)NAN;
  }
  M[RB200_RM_MAX_OF_RESPONSE_LENGTH] = (double)(float)rl_max;
  M[RB200_RM_MIN_OF_RESPONSE_LENGTH] = (double)(float)rl_min;
  M[RB200_RM_VERDICT] = (double)verdict;
  M[RB200_RM_NUM_LENGTHS_MAX] = nmax;
  for (int r = 0; r < P; ++r) M[RB200_RM_NUM + r] = rec[(int64_t)r * RB200_RR_NUM + RB200_RR_NUM_SEQ];
}

// mask.to(float32).sum() of _setup_valid_token_scale: the exact count, rounded once to fp32
__global__ void count_to_f32_kernel(const long long* __restrict__ total, float* __restrict__ out) {
  if (threadIdx.x == 0) out[0] = (float)*total;
}

// ---- Megatron loss_func epilogue ----------------------------------------------------------------------------------

__global__ void epilogue_pack_kernel(rb200_mb_epilogue_args a, const long long* __restrict__ mask_total) {
  if (threadIdx.x != 0) return;
  const int n = a.n_avg + a.n_sum;
  for (int k = 0; k < n; ++k) a.pack[k] = (k == a.final_slot) ? 0.0f : *a.src[k];
  float s = 1.0f;
  if (a.global_valid_token) {  // mask.sum() / global_valid_token * dp * num_microbatches, each step in fp32
    s = __fdiv_rn((float)*mask_total, *a.global_valid_token);
    s = __fmul_rn(s, (float)a.dp);
    s = __fmul_rn(s, (float)a.num_microbatches);
  }
  const float loss = *a.loss;
  if (a.final_slot >= 0) a.pack[a.final_slot] = __fmul_rn(loss, s);
  a.pack[n] = __fmul_rn(__fmul_rn(loss, 0.0f), s);  // the final loss of an early-stopped micro-batch
  a.scale[0] = s;
}

__global__ void epilogue_apply_kernel(rb200_mb_epilogue_args a) {
  if (threadIdx.x != 0) return;
  const int n = a.n_avg + a.n_sum;
  const float dp = (float)a.dp;
  bool stop = false;
  if (a.has_early_stop && a.ratio_slot >= 0) stop = __fdiv_rn(a.pack[a.ratio_slot], dp) > (float)a.early_stop_imp_ratio;
  float* row = a.step_acc + (int64_t)a.mb * n;
  for (int k = 0; k < n; ++k) {
    float v = a.pack[k];
    if (k == a.final_slot && stop) v = a.pack[n];
    if (k < a.n_avg) v = __fdiv_rn(v, dp);
    a.metrics[k] = v;
    row[k] = v;
  }
  if (stop) a.scale[0] = 0.0f;
}

__global__ void step_finish_kernel(const float* __restrict__ acc, int n_mb, int n_avg, int n_sum,
                                   float* __restrict__ out) {
  const int n = n_avg + n_sum;
  for (int k = threadIdx.x; k < n; k += blockDim.x) {
    float s = 0.0f;
    for (int m = 0; m < n_mb; ++m) s = __fadd_rn(s, acc[(int64_t)m * n + k]);
    out[k] = k < n_avg ? __fdiv_rn(s, (float)n_mb) : s;
  }
  __syncthreads();
  if (threadIdx.x != 0 || n_sum != 5) return;
  // compute_critic_explained_variance_from_stats (metric_utils.py:261-290), fp32, no contraction
  const float* e = out + n_avg;
  const float count = e[0], rs = e[1], rsq = e[2], es = e[3], esq = e[4];
  float ev = NAN;
  if (!(count < 2.0f)) {
    const float rc = __fsub_rn(rsq, __fdiv_rn(__fmul_rn(rs, rs), count));
    if (!isnan(rc) && rc != 0.0f) {
      const float ec = __fsub_rn(esq, __fdiv_rn(__fmul_rn(es, es), count));
      if (!isnan(ec)) ev = __fsub_rn(1.0f, __fdiv_rn(ec, rc));
    }
  }
  out[n] = ev;
}

}  // namespace

extern "C" int64_t rb200_reasoning_record_workspace_bytes(int64_t bsz, int64_t L) {
  if (bsz <= 0 || L <= 0 || bsz > 65535) return -1;
  const int64_t nseg = num_segments(L);
  if (nseg > 0x7fffffff) return -1;
  return bsz * nseg * kNP * (int64_t)sizeof(double);
}

extern "C" int rb200_reasoning_rollout_record(const rb200_reasoning_record_args* args, rb200_stream_t stream) {
  if (!args) return RB200_E_NULL;
  const rb200_reasoning_record_args& a = *args;
  if (!a.advantages || !a.mask || !a.prompt_lengths || !a.response_lengths || !a.rewards || !a.is_end ||
      !a.workspace || !a.record)
    return RB200_E_NULL;
  const int64_t need = rb200_reasoning_record_workspace_bytes(a.bsz, a.L);
  if (need < 0) return RB200_E_SHAPE;
  if (a.workspace_bytes < need) return RB200_E_ARG;
  if ((reinterpret_cast<uintptr_t>(a.workspace) & 15) != 0) return RB200_E_ALIGN;
  if (a.advantages_stride < a.L || a.mask_stride < a.L || (a.values && a.values_stride < a.L)) return RB200_E_SHAPE;
  cudaStream_t st = rb::as_stream(stream);
  const int64_t nseg = num_segments(a.L);
  double* partials = static_cast<double*>(a.workspace);
  record_cells_kernel<<<dim3((unsigned)nseg, (unsigned)a.bsz), kThreads, 0, st>>>(a, partials);
  rb::count_launch();
  record_finish_kernel<<<1, kFinishThreads, 0, st>>>(a, a.bsz * nseg, partials);
  rb::count_launch();
  RB_RETURN_LAUNCH();
}

extern "C" int rb200_reasoning_rollout_finish(const double* records, int32_t P, const float* values_world_sum,
                                              int32_t world_size, double* metrics, rb200_stream_t stream) {
  if (!records || !metrics) return RB200_E_NULL;
  if (P <= 0 || (values_world_sum && world_size <= 0)) return RB200_E_SHAPE;
  rollout_finish_kernel<<<1, 32, 0, rb::as_stream(stream)>>>(records, P, values_world_sum, world_size, metrics);
  rb::count_launch();
  RB_RETURN_LAUNCH();
}

static int epilogue_check(const rb200_mb_epilogue_args* args) {
  if (!args) return RB200_E_NULL;
  const rb200_mb_epilogue_args& a = *args;
  if (a.n_avg < 0 || a.n_sum < 0 || a.n_avg + a.n_sum <= 0 || a.n_avg + a.n_sum > RB200_EPI_MAX_KEYS)
    return RB200_E_SHAPE;
  if (a.final_slot >= a.n_avg || a.ratio_slot >= a.n_avg || a.final_slot < -1 || a.ratio_slot < -1) return RB200_E_ARG;
  if (a.dp <= 0 || a.num_microbatches <= 0 || a.n_mb <= 0 || a.mb < 0 || a.mb >= a.n_mb) return RB200_E_ARG;
  if (!a.loss || !a.pack || !a.scale || !a.metrics || !a.step_acc || !a.workspace) return RB200_E_NULL;
  for (int k = 0; k < a.n_avg + a.n_sum; ++k)
    if (!a.src[k] && k != a.final_slot) return RB200_E_NULL;
  return RB200_OK;
}

extern "C" int rb200_mask_count_f32(const uint8_t* mask, int64_t mask_stride, int64_t bsz, int64_t L, void* workspace,
                                    int64_t workspace_bytes, float* out, rb200_stream_t stream) {
  if (!mask || !workspace || !out) return RB200_E_NULL;
  const int64_t need = rb200_token_loss_workspace_bytes(bsz, L);
  if (need < 0 || mask_stride < L) return RB200_E_SHAPE;
  if (workspace_bytes < need) return RB200_E_ARG;
  if ((reinterpret_cast<uintptr_t>(workspace) & 15) != 0) return RB200_E_ALIGN;
  cudaStream_t st = rb::as_stream(stream);
  const rb::TokenCounts c = rb::token_mask_counts(mask, mask_stride, bsz, L, workspace, st);
  count_to_f32_kernel<<<1, 32, 0, st>>>(c.total, out);
  rb::count_launch();
  RB_RETURN_LAUNCH();
}

extern "C" int rb200_mb_epilogue_pack(const rb200_mb_epilogue_args* args, rb200_stream_t stream) {
  const int rc = epilogue_check(args);
  if (rc != RB200_OK) return rc;
  const rb200_mb_epilogue_args& a = *args;
  cudaStream_t st = rb::as_stream(stream);
  const long long* total = nullptr;
  if (a.global_valid_token) {
    if (!a.mask) return RB200_E_NULL;
    const int64_t need = rb200_token_loss_workspace_bytes(a.bsz, a.L);
    if (need < 0 || a.mask_stride < a.L) return RB200_E_SHAPE;
    if (a.workspace_bytes < need) return RB200_E_ARG;
    if ((reinterpret_cast<uintptr_t>(a.workspace) & 15) != 0) return RB200_E_ALIGN;
    total = rb::token_mask_counts(a.mask, a.mask_stride, a.bsz, a.L, a.workspace, st).total;
  } else if (a.workspace_bytes < RB200_EPI_WS_MIN) {
    return RB200_E_ARG;
  }
  epilogue_pack_kernel<<<1, 32, 0, st>>>(a, total);
  rb::count_launch();
  RB_RETURN_LAUNCH();
}

extern "C" int rb200_mb_epilogue_apply(const rb200_mb_epilogue_args* args, rb200_stream_t stream) {
  const int rc = epilogue_check(args);
  if (rc != RB200_OK) return rc;
  epilogue_apply_kernel<<<1, 32, 0, rb::as_stream(stream)>>>(*args);
  rb::count_launch();
  RB_RETURN_LAUNCH();
}

extern "C" int rb200_step_metrics_finish(const float* step_acc, int32_t n_mb, int32_t n_avg, int32_t n_sum,
                                         float* out, rb200_stream_t stream) {
  if (!step_acc || !out) return RB200_E_NULL;
  if (n_mb <= 0 || n_avg < 0 || n_sum < 0 || n_avg + n_sum <= 0 || n_avg + n_sum > RB200_EPI_MAX_KEYS)
    return RB200_E_SHAPE;
  step_finish_kernel<<<1, 32, 0, rb::as_stream(stream)>>>(step_acc, n_mb, n_avg, n_sum, out);
  rb::count_launch();
  RB_RETURN_LAUNCH();
}
