// Remaining advantage estimators of the registry (SURVEY 8(f) rank 4) and the fp64 masked normalisations (a24).
// Reference: rlinf/algorithms/advantages.py - grpo_video :124-164, grpo_dynamic :167-299, reinpp :302-364,
// opd :367-407, raw :410-438; rlinf/utils/distributed.py - masked_normalization :866-939, masked_stats :942-954,
// normalize_from_stats :957-965.
// Layout everywhere: step-major [L, B] (B fastest), loss_mask as uint8 0/1 (NULL = all valid).
#include "common.cuh"
#include "kl_unit.cuh"

namespace {

// ---- {count, sum, sumsq} of x over the mask, fp64 (masked_stats; masked_normalization's factor / x_sum / x_sum_sq) --
// Fixed order, so repeated calls agree bit for bit: each CTA writes its partial sums to its own slot; the last CTA to
// arrive adds the slots in CTA order (thread t takes CTAs t, t + 256, ... in order, then the fixed block tree) and
// clears the arrival counter.  `scratch` is the per-device rb::device_scratch (zero-initialised): the arrival counter in
// its first 8 bytes, then 3 doubles per CTA.  Calls on one device are therefore stream-ordered.
__global__ void __launch_bounds__(256) masked_moments_kernel(const float* __restrict__ x, const uint8_t* __restrict__ mask,
                                                             int64_t n, double* __restrict__ out3,
                                                             double* __restrict__ scratch) {
  unsigned long long* arrived = reinterpret_cast<unsigned long long*>(scratch);
  double* part = scratch + 1;
  __shared__ double red[3 * 32];
  __shared__ int is_last;
  double v[3] = {0.0, 0.0, 0.0};
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    if (mask == nullptr || mask[i]) {
      const double xi = (double)x[i];
      v[0] += 1.0;
      v[1] += xi;
      v[2] += xi * xi;
    }
  }
  rb::block_sum<3>(v, red);
  if (threadIdx.x == 0) {
    part[blockIdx.x * 3 + 0] = v[0];
    part[blockIdx.x * 3 + 1] = v[1];
    part[blockIdx.x * 3 + 2] = v[2];
    __threadfence();
    is_last = atomicAdd(arrived, 1ull) == (unsigned long long)gridDim.x - 1ull;
  }
  __syncthreads();
  if (!is_last) return;
  __threadfence();
  double w[3] = {0.0, 0.0, 0.0};
  for (int b = threadIdx.x; b < (int)gridDim.x; b += blockDim.x) {
    w[0] += __ldcg(&part[b * 3 + 0]);
    w[1] += __ldcg(&part[b * 3 + 1]);
    w[2] += __ldcg(&part[b * 3 + 2]);
  }
  __syncthreads();  // `red` is reused
  rb::block_sum<3>(w, red);
  if (threadIdx.x == 0) {
    out3[0] = w[0];
    out3[1] = w[1];
    out3[2] = w[2];
    *arrived = 0ull;
  }
}

// mode 0  masked_normalization (distributed.py:903-939, dim=None): xm = x*mask; mean = S/n; var = SS/n - mean^2
//         [* n/(n-1) if unbiased]; out = (xm - mean) / (sqrt(var) + eps)           (fp64, rounded once to fp32)
// mode 1  normalize_from_stats (:957-965): n' = max(n,1); out = (x - S/n') * rsqrt(max(SS/n' - mean^2, 0) + 1e-5)
// mode 2  reinforce++ whitening (advantages.py:355-362): mean = S/n (0 if n == 0: masked_mean of an all-False mask is
//         the plain masked sum); var = SS/n - mean^2; out = (x - mean) * rsqrt(max(var, eps))   with eps = 1e-8
__global__ void __launch_bounds__(256) masked_normalize_kernel(const float* __restrict__ x,
                                                               const uint8_t* __restrict__ mask, float* __restrict__ out,
                                                               int64_t n, const double* __restrict__ stats3, int mode,
                                                               double eps, int unbiased) {
  const double cnt = stats3[0], S = stats3[1], SS = stats3[2];
  double mean, scale;  // out = (v - mean) * scale
  if (mode == 0) {
    mean = S / cnt;
    double var = SS / cnt - mean * mean;
    if (unbiased) var *= cnt / (cnt - 1.0);
    scale = 1.0 / (sqrt(var) + eps);
  } else if (mode == 1) {
    const double c = cnt < 1.0 ? 1.0 : cnt;
    mean = S / c;
    const double var = SS / c - mean * mean;
    scale = rsqrt((var < 0.0 ? 0.0 : var) + 1e-5);
  } else {
    const double c = cnt > 0.0 ? cnt : 1.0;
    mean = S / c;
    const double var = SS / c - mean * mean;
    // the reference works in fp32 here: clamp(min=1e-8).rsqrt() on an fp32 variance
    const float var_f = fmaxf((float)var, (float)eps);
    scale = (double)(1.0f / sqrtf(var_f));
    mean = (double)(float)mean;
  }
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    double v = (double)x[i];
    if (mode == 0 && mask != nullptr && !mask[i]) v = 0.0;
    if (mode == 2) out[i] = __fmul_rn(__fsub_rn(x[i], (float)mean), (float)scale);
    else out[i] = (float)((v - mean) * scale);
  }
}

// ---- raw (advantages.py:410-438): adv[l,b] = score[b] * mask[l,b]; optional {n, sum, sumsq} over the valid entries ----
constexpr int kCols = 32, kRowsPar = 8;
__global__ void __launch_bounds__(kCols* kRowsPar) raw_adv_kernel(const float* __restrict__ scores,
                                                                   const uint8_t* __restrict__ mask,
                                                                   float* __restrict__ adv, int L, int B,
                                                                   double* __restrict__ stats3) {
  __shared__ double red[3 * 32];
  const int tx = threadIdx.x & (kCols - 1), ty = threadIdx.x / kCols;
  const int b = blockIdx.x * kCols + tx;
  double v[3] = {0.0, 0.0, 0.0};
  if (b < B) {
    const float s = scores[b];
    for (int l = ty; l < L; l += kRowsPar) {
      const size_t o = (size_t)l * B + b;
      const bool m = mask ? mask[o] != 0 : true;
      const float a = __fmul_rn(s, m ? 1.0f : 0.0f);
      adv[o] = a;
      if (m) {
        v[0] += 1.0;
        v[1] += (double)a;
        v[2] += (double)a * (double)a;
      }
    }
  }
  if (stats3 != nullptr) {
    rb::block_sum<3>(v, red);
    if (threadIdx.x == 0 && v[0] != 0.0) {
      atomicAdd(&stats3[0], v[0]);
      atomicAdd(&stats3[1], v[1]);
      atomicAdd(&stats3[2], v[2]);
    }
  }
}

// ---- reinforce++ (advantages.py:302-364) ----------------------------------------------------------------------------
// r[l,b] = reward[b] at l = eos[b], minus kl_beta * kld[l,b]; ret = reverse cumulative sum over L; masked {n,S,SS}.
// eos[b] reproduces the reference's quirk: `loss_mask.long().fliplr().argmax(dim=0)` flips the BATCH dimension of the
// [L,B] mask, so column b uses the FIRST valid row of column B-1-b:  eos[b] = L-1 - argmax_l mask[l, B-1-b].
// The cumulative sum follows torch's CPU cumsum: sequential from the last row, accumulated in fp64 (acc_type of float
// on CPU), each prefix rounded to fp32.  kl terms: mode as rb200_kl_penalty (k1 / abs / k2 / k3).
__device__ __forceinline__ float kl_term(float a, float b, int mode) {
  float g;
  return rb::kl_penalty_unit(a, b, mode, g);
}

__global__ void __launch_bounds__(128) reinpp_scan_kernel(const float* __restrict__ rewards,
                                                          const uint8_t* __restrict__ mask,
                                                          const float* __restrict__ logprob,
                                                          const float* __restrict__ ref_logprob, float* __restrict__ ret,
                                                          int L, int B, float kl_beta, int kl_mode,
                                                          double* __restrict__ stats3) {
  __shared__ double red[3 * 32];
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  double v[3] = {0.0, 0.0, 0.0};
  if (b < B) {
    const int src = B - 1 - b;
    int first = 0;  // argmax of an all-zero column is 0
    for (int l = 0; l < L; ++l)
      if (mask[(size_t)l * B + src]) {
        first = l;
        break;
      }
    const int eos = L - 1 - first;
    const float rew = rewards[b];
    double acc = 0.0;
    for (int l = L - 1; l >= 0; --l) {
      const size_t o = (size_t)l * B + b;
      float r = (l == eos) ? rew : 0.0f;
      if (kl_beta > 0.0f) r = __fsub_rn(r, __fmul_rn(kl_beta, kl_term(logprob[o], ref_logprob[o], kl_mode)));
      acc += (double)r;
      const float out = (float)acc;
      ret[o] = out;
      if (mask[o]) {
        v[0] += 1.0;
        v[1] += (double)out;
        v[2] += (double)out * (double)out;
      }
    }
  }
  rb::block_sum<3>(v, red);
  if (threadIdx.x == 0 && v[0] != 0.0) {
    atomicAdd(&stats3[0], v[0]);
    atomicAdd(&stats3[1], v[1]);
    atomicAdd(&stats3[2], v[2]);
  }
}

// ---- grpo_video (advantages.py:124-164): rewards [S, B], groups of G consecutive envs -----------------------------------
// mode 0 "frame": mean / unbiased std over the G samples of each (step, group); mode 1 "video": over all S*G entries of
// the group.  adv = (r - mean) / (std + 1e-6) * mask (mask is a float tensor in the reference: a plain product).
// One warp per group (video) or per (step, group) (frame); two-pass mean / M2 in fp64.
__global__ void __launch_bounds__(256) grpo_video_kernel(const float* __restrict__ rewards, const float* __restrict__ maskf,
                                                         const uint8_t* __restrict__ mask8, float* __restrict__ adv,
                                                         int S, int B, int G, int mode, float eps) {
  const int lane = threadIdx.x & 31;
  const int64_t w = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int n_groups = B / G;
  const int64_t n_items = mode == 0 ? (int64_t)S * n_groups : n_groups;
  if (w >= n_items) return;
  const int grp = (int)(mode == 0 ? w % n_groups : w);
  const int s0 = mode == 0 ? (int)(w / n_groups) : 0, s1 = mode == 0 ? s0 + 1 : S;
  const int cnt = (s1 - s0) * G;
  double sum = 0.0;
  for (int i = lane; i < cnt; i += 32) sum += (double)rewards[(size_t)(s0 + i / G) * B + grp * G + i % G];
  sum = rb::warp_sum(sum);
  const double mean_d = sum / (double)cnt;
  double m2 = 0.0;
  for (int i = lane; i < cnt; i += 32) {
    const double d = (double)rewards[(size_t)(s0 + i / G) * B + grp * G + i % G] - mean_d;
    m2 += d * d;
  }
  m2 = rb::warp_sum(m2);
  const float mean = (float)mean_d;
  const float den = __fadd_rn((float)sqrt(m2 / (double)(cnt - 1)), eps);  // cnt == 1 -> NaN like torch.std
  for (int i = lane; i < cnt; i += 32) {
    const size_t o = (size_t)(s0 + i / G) * B + grp * G + i % G;
    const float a = __fdiv_rn(__fsub_rn(rewards[o], mean), den);
    const float m = maskf ? maskf[o] : (mask8 ? (mask8[o] ? 1.0f : 0.0f) : 1.0f);
    adv[o] = __fmul_rn(a, m);
  }
}

// ---- grpo_dynamic (advantages.py:167-299): multi-turn GRPO --------------------------------------------------------------
// rewards[n] per turn, idx_to_traj[n] (turn -> global trajectory), G trajectories per question.
// mode 0 "trajectory": trajectory reward = mean of its turns' rewards (sequential fp32 sum in turn order / count);
//   per question (mean, unbiased std) over its G trajectory rewards; every turn gets its trajectory's normalised reward.
// mode 1 "turn": per question (mean, unbiased std) over ALL its turns.
// One CTA per question; n is small (turns of one dynamic batch) so each CTA scans the whole index list.
__global__ void __launch_bounds__(128) grpo_dynamic_kernel(const float* __restrict__ rewards,
                                                           const int32_t* __restrict__ idx_to_traj, float* __restrict__ turn_adv,
                                                           int n, int G, int mode, float eps) {
  extern __shared__ float traj_sh[];  // [G] trajectory rewards (mode 0)
  __shared__ double red[2 * 32];
  __shared__ float stat_sh[2];
  const int q = blockIdx.x;
  if (mode == 0) {
    // per-trajectory mean, accumulated in turn order like the reference's Python loop (one thread per trajectory)
    for (int k = threadIdx.x; k < G; k += blockDim.x) {
      const int traj = q * G + k;
      float s = 0.0f;
      int c = 0;
      for (int i = 0; i < n; ++i)
        if (idx_to_traj[i] == traj) {
          s = __fadd_rn(s, rewards[i]);
          ++c;
        }
      traj_sh[k] = __fdiv_rn(s, (float)(c < 1 ? 1 : c));
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      double sum = 0.0;
      for (int k = 0; k < G; ++k) sum += (double)traj_sh[k];
      const double mean = sum / (double)G;
      double m2 = 0.0;
      for (int k = 0; k < G; ++k) m2 += ((double)traj_sh[k] - mean) * ((double)traj_sh[k] - mean);
      stat_sh[0] = (float)mean;
      stat_sh[1] = __fadd_rn((float)sqrt(m2 / (double)(G - 1)), eps);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
      const int traj = idx_to_traj[i];
      if (traj / G == q) turn_adv[i] = __fdiv_rn(__fsub_rn(traj_sh[traj - q * G], stat_sh[0]), stat_sh[1]);
    }
  } else {
    double v[2] = {0.0, 0.0};
    for (int i = threadIdx.x; i < n; i += blockDim.x)
      if (idx_to_traj[i] / G == q) {
        v[0] += 1.0;
        v[1] += (double)rewards[i];
      }
    rb::block_sum<2>(v, red);
    __shared__ double mean_sh, cnt_sh;
    if (threadIdx.x == 0) {
      cnt_sh = v[0];
      mean_sh = v[0] > 0.0 ? v[1] / v[0] : 0.0;
    }
    __syncthreads();
    double w[2] = {0.0, 0.0};
    for (int i = threadIdx.x; i < n; i += blockDim.x)
      if (idx_to_traj[i] / G == q) {
        const double d = (double)rewards[i] - mean_sh;
        w[0] += d * d;
      }
    __syncthreads();
    rb::block_sum<2>(w, red);
    if (threadIdx.x == 0) {
      stat_sh[0] = (float)mean_sh;
      stat_sh[1] = __fadd_rn((float)sqrt(w[0] / (cnt_sh - 1.0)), eps);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < n; i += blockDim.x)
      if (idx_to_traj[i] / G == q) turn_adv[i] = __fdiv_rn(__fsub_rn(rewards[i], stat_sh[0]), stat_sh[1]);
  }
}

// ---- opd (advantages.py:367-407): dense reverse-KL reward teacher_logp - student_logp ---------------------------------------
__global__ void __launch_bounds__(256) sub_kernel(const float* __restrict__ a, const float* __restrict__ b,
                                                  float* __restrict__ out, int64_t n) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) out[i] = __fsub_rn(a[i], b[i]);
}

inline int grid_for(int64_t n, int per_sm = 8) {
  int64_t blocks = (n + 255) / 256;
  const int64_t cap = (int64_t)rb::sm_count() * per_sm;
  if (blocks > cap) blocks = cap;
  return (int)(blocks < 1 ? 1 : blocks);
}

}  // namespace

extern "C" int rb200_masked_moments(const float* x, const uint8_t* mask, int64_t n, double* out3, rb200_stream_t stream) {
  if (!x || !out3) return RB200_E_NULL;
  if (n < 0) return RB200_E_SHAPE;
  cudaStream_t st = rb::as_stream(stream);
  if (n == 0) {
    RB_CHECK_CUDA(cudaMemsetAsync(out3, 0, 3 * sizeof(double), st));
    return RB200_OK;
  }
  const int blocks = grid_for(n, 4);
  double* scratch = rb::device_scratch(1 + 3 * blocks);
  if (!scratch) return RB200_E_UNSUPPORTED;
  masked_moments_kernel<<<blocks, 256, 0, st>>>(x, mask, n, out3, scratch);  // writes all of out3
  rb::count_launch();
  RB_RETURN_LAUNCH();
}

extern "C" int rb200_masked_normalize(const float* x, const uint8_t* mask, float* out, int64_t n, const double* stats3,
                                      int mode, double eps, int unbiased, rb200_stream_t stream) {
  if (!x || !out || !stats3) return RB200_E_NULL;
  if (n <= 0) return RB200_E_SHAPE;
  if (mode < 0 || mode > 2) return RB200_E_ARG;
  masked_normalize_kernel<<<grid_for(n), 256, 0, rb::as_stream(stream)>>>(x, mask, out, n, stats3, mode, eps, unbiased);
  rb::count_launch();
  RB_RETURN_LAUNCH();
}

extern "C" int rb200_raw_advantages(const float* scores, const uint8_t* loss_mask, float* adv, int L, int B,
                                    double* stats3, rb200_stream_t stream) {
  if (!scores || !adv) return RB200_E_NULL;
  if (L <= 0 || B <= 0) return RB200_E_SHAPE;
  cudaStream_t st = rb::as_stream(stream);
  if (stats3) RB_CHECK_CUDA(cudaMemsetAsync(stats3, 0, 3 * sizeof(double), st));
  raw_adv_kernel<<<(B + kCols - 1) / kCols, kCols * kRowsPar, 0, st>>>(scores, loss_mask, adv, L, B, stats3);
  rb::count_launch();
  RB_RETURN_LAUNCH();
}

extern "C" int rb200_reinpp_returns(const float* rewards, const uint8_t* loss_mask, const float* logprob,
                                    const float* ref_logprob, float* ret, int L, int B, double kl_beta, int kl_mode,
                                    double* stats3, rb200_stream_t stream) {
  if (!rewards || !loss_mask || !ret || !stats3) return RB200_E_NULL;
  if (L <= 0 || B <= 0) return RB200_E_SHAPE;
  if (kl_beta > 0.0 && (!logprob || !ref_logprob)) return RB200_E_NULL;
  if (kl_mode < 0 || kl_mode > 3) return RB200_E_ARG;
  cudaStream_t st = rb::as_stream(stream);
  RB_CHECK_CUDA(cudaMemsetAsync(stats3, 0, 3 * sizeof(double), st));
  reinpp_scan_kernel<<<(B + 127) / 128, 128, 0, st>>>(rewards, loss_mask, logprob, ref_logprob, ret, L, B,
                                                      (float)kl_beta, kl_mode, stats3);
  rb::count_launch();
  RB_RETURN_LAUNCH();
}

extern "C" int rb200_grpo_video_advantages(const float* rewards, const float* mask_f32, const uint8_t* mask_u8, float* adv,
                                           int S, int B, int G, int mode, float eps, rb200_stream_t stream) {
  if (!rewards || !adv) return RB200_E_NULL;
  if (S <= 0 || B <= 0 || G <= 0 || B % G != 0) return RB200_E_SHAPE;
  if (mode != 0 && mode != 1) return RB200_E_ARG;
  const int64_t items = mode == 0 ? (int64_t)S * (B / G) : (B / G);
  const int blocks = (int)((items + 7) / 8);
  grpo_video_kernel<<<blocks, 256, 0, rb::as_stream(stream)>>>(rewards, mask_f32, mask_u8, adv, S, B, G, mode, eps);
  rb::count_launch();
  RB_RETURN_LAUNCH();
}

extern "C" int rb200_grpo_dynamic_turn_advantages(const float* rewards, const int32_t* idx_to_traj, float* turn_adv,
                                                  int n, int num_trajectories, int G, int mode, float eps,
                                                  rb200_stream_t stream) {
  if (!rewards || !idx_to_traj || !turn_adv) return RB200_E_NULL;
  if (n <= 0 || G <= 0 || num_trajectories <= 0 || num_trajectories % G != 0) return RB200_E_SHAPE;
  if (mode != 0 && mode != 1) return RB200_E_ARG;
  if (G * (int)sizeof(float) > 48 * 1024) return RB200_E_UNSUPPORTED;
  grpo_dynamic_kernel<<<num_trajectories / G, 128, G * sizeof(float), rb::as_stream(stream)>>>(
      rewards, idx_to_traj, turn_adv, n, G, mode, eps);
  rb::count_launch();
  RB_RETURN_LAUNCH();
}

extern "C" int rb200_sub(const float* a, const float* b, float* out, int64_t n, rb200_stream_t stream) {
  if (!a || !b || !out) return RB200_E_NULL;
  if (n <= 0) return RB200_E_SHAPE;
  sub_kernel<<<grid_for(n), 256, 0, rb::as_stream(stream)>>>(a, b, out, n);
  rb::count_launch();
  RB_RETURN_LAUNCH();
}
