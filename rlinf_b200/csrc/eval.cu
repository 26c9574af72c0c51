// Policy evaluation: eval-mode action generation and per-episode statistics of evaluation rollouts.
// Reference: EmbodiedRunner.evaluate / _maybe_eval_and_checkpoint, rlinf/runners/embodied_runner.py:193-206,308-329;
// MLPPolicy._generate_actions(mode="eval"), rlinf/models/embodiment/mlp_policy/mlp_policy.py:256-293 (action = mean);
// ManiskillEnv._record_metrics / _reset_metrics / _handle_auto_reset, rlinf/envs/maniskill/maniskill_env.py:225-271,
// 327-390 and EnvWorker.env_evaluate_step, rlinf/workers/env/env_worker.py:557-620 (episode return / length / mean
// reward of every newly finished episode); compute_evaluate_metrics, rlinf/utils/metric_utils.py:372-419.
//
// The statistics never leave the device during an evaluation: per-env running return (fp32, summed sub-step by
// sub-step like `self.returns += step_reward`) and length, and per-env fp64 sums over finished episodes.  One
// fixed-order reduction produces [count, sum return, sum length, sum reward] - no float atomics, so two runs of the
// same evaluation give bit-identical metrics.
#include "common.cuh"
#include "episode_stats.cuh"

namespace rb {
int mlp_mean_forward(const rb200_mlp_layout* L, const float* params, const float* wsplit, const float* states,
                     int64_t n, float* action, float* logprobs, float* values, float* work, cudaStream_t st);
}

namespace {

constexpr int kReduceThreads = 512;

struct StatsArgs {
  const float* rewards;   // [B,C]
  const uint8_t* done;    // [B,C]; column C-1 is the chunk's done flag
  float* ret;             // [B]
  int32_t* len;           // [B]
  uint8_t* prev_done;     // [B]; read and written by kNewlyDone only
  double* acc;            // [B,4]: count, sum return, sum length, sum reward
  float* episode;         // [B,3] or null: (return, length, reward) of the episode finished this step, else NaN
  int B, C, auto_reset;
  int rule;               // which envs record an episode this step (Record)
};

// Record rules.  Evaluation (EnvWorker.env_evaluate_step): kDone with auto-reset, else kNewlyDone.  Training
// (EnvWorker._run_interact_once with should_record / env_interact_step): kDone with auto-reset; without it every env
// records its running episode at the rollout's last chunk step (kAll) and none before (kNone).
enum Record { kDone = 0, kNewlyDone = 1, kNone = 2, kAll = 3 };

__global__ void __launch_bounds__(256) episode_stats_step_kernel(StatsArgs p) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= p.B) return;
  float r = p.ret[b];
  for (int c = 0; c < p.C; ++c) r = __fadd_rn(r, p.rewards[(size_t)b * p.C + c]);
  // ManiSkill's elapsed_steps keeps counting through a termination inside a chunk
  const int32_t l = p.len[b] + p.C;
  const bool done = p.done[(size_t)b * p.C + p.C - 1] != 0;
  bool newly = p.rule == kAll || (p.rule == kDone && done);
  if (p.rule == kNewlyDone) {
    const bool prev = p.prev_done[b] != 0;
    newly = done && !prev;
    p.prev_done[b] = prev || done;
  }
  float* ep = p.episode ? p.episode + (size_t)b * 3 : nullptr;
  if (newly) {
    const float rew = rb::episode_finish(p.acc + (size_t)b * 4, r, l);
    if (ep) {
      ep[0] = r;
      ep[1] = (float)l;
      ep[2] = rew;
    }
  } else if (ep) {
    ep[0] = ep[1] = ep[2] = __int_as_float(0x7fc00000);
  }
  const bool reset = p.auto_reset && done;  // _handle_auto_reset -> _reset_metrics(env_idx)
  p.ret[b] = reset ? 0.f : r;
  p.len[b] = reset ? 0 : l;
}

// one block: thread t sums envs t, t + nthreads, ... in order, then a fixed tree over the threads
__global__ void __launch_bounds__(kReduceThreads) episode_stats_reduce_kernel(const double* __restrict__ acc, int B,
                                                                             double* __restrict__ out) {
  __shared__ double sm[4][kReduceThreads];
  double s[4] = {0.0, 0.0, 0.0, 0.0};
  for (int b = threadIdx.x; b < B; b += blockDim.x)
    for (int k = 0; k < 4; ++k) s[k] += acc[(size_t)b * 4 + k];
  for (int k = 0; k < 4; ++k) sm[k][threadIdx.x] = s[k];
  __syncthreads();
  for (int h = blockDim.x / 2; h > 0; h >>= 1) {
    if (threadIdx.x < h)
      for (int k = 0; k < 4; ++k) sm[k][threadIdx.x] += sm[k][threadIdx.x + h];
    __syncthreads();
  }
  if (threadIdx.x < 4) out[threadIdx.x] = sm[threadIdx.x][0];
}

}  // namespace

extern "C" int rb200_mlp_mean(const rb200_mlp_layout* L, const float* params, const float* wsplit,
                              const float* states, int64_t n, float* action, float* logprobs, float* values,
                              float* work, rb200_stream_t stream) {
  if (!L || !params || !wsplit || !states || !action || !work) return RB200_E_NULL;
  if (n <= 0) return RB200_E_SHAPE;
  if (values && L->value_dim == 0) return RB200_E_SHAPE;
  return rb::mlp_mean_forward(L, params, wsplit, states, n, action, logprobs, values, work, rb::as_stream(stream));
}

extern "C" int rb200_episode_stats_step(const float* rewards, const uint8_t* done, int B, int C, int auto_reset,
                                        float* ret, int32_t* len, uint8_t* prev_done, double* acc, float* episode,
                                        rb200_stream_t stream) {
  if (!rewards || !done || !ret || !len || !prev_done || !acc) return RB200_E_NULL;
  if (B <= 0 || C <= 0) return RB200_E_SHAPE;
  StatsArgs p{};
  p.rewards = rewards; p.done = done; p.ret = ret; p.len = len; p.prev_done = prev_done; p.acc = acc;
  p.episode = episode; p.B = B; p.C = C; p.auto_reset = auto_reset; p.rule = auto_reset ? kDone : kNewlyDone;
  episode_stats_step_kernel<<<(B + 255) / 256, 256, 0, rb::as_stream(stream)>>>(p);
  rb::count_launch();
  RB_RETURN_LAUNCH();
}

extern "C" int rb200_train_episode_stats_step(const float* rewards, const uint8_t* done, int B, int C, int auto_reset,
                                              int last_step, float* ret, int32_t* len, double* acc,
                                              rb200_stream_t stream) {
  if (!rewards || !done || !ret || !len || !acc) return RB200_E_NULL;
  if (B <= 0 || C <= 0) return RB200_E_SHAPE;
  StatsArgs p{};
  p.rewards = rewards; p.done = done; p.ret = ret; p.len = len; p.acc = acc; p.B = B; p.C = C;
  p.auto_reset = auto_reset; p.rule = auto_reset ? kDone : (last_step ? kAll : kNone);
  episode_stats_step_kernel<<<(B + 255) / 256, 256, 0, rb::as_stream(stream)>>>(p);
  rb::count_launch();
  RB_RETURN_LAUNCH();
}

extern "C" int rb200_episode_stats_reduce(const double* acc, int B, double* out, rb200_stream_t stream) {
  if (!acc || !out) return RB200_E_NULL;
  if (B <= 0) return RB200_E_SHAPE;
  episode_stats_reduce_kernel<<<1, kReduceThreads, 0, rb::as_stream(stream)>>>(acc, B, out);
  rb::count_launch();
  RB_RETURN_LAUNCH();
}
