// Rollout-side kernels: synthetic vector env step (chunk_step contract), truncation bootstrap of rewards,
// value-only forward, device step counter.
// Reference: EnvWorker.env_interact_step / compute_bootstrap_rewards, rlinf/workers/env/env_worker.py:464-560,
// 719-758 (r[:, -1] += gamma * V(final_obs) where truncated - or done when bootstrap_type != "standard");
// env contract: chunk_step -> (obs, rewards [B,C], terminations, truncations, infos{final_observation}),
// rlinf/envs/maniskill/maniskill_env.py:327-375; MultiStepRolloutWorker.get_bootstrap_values,
// rlinf/workers/rollout/hf/huggingface_worker.py:612-627.
//
// The synthetic env is the benchmark workload of SURVEY.md §8(d)/BASELINE.md §4 (device resident):
//   s' = tanh(s.W_s + a.W_a + noise_std*eps),  r = -||s'||^2/obs + reward_noise_std*eps_r,
//   termination ~ Bernoulli(p_term), truncation at max_episode_steps, auto-reset to s ~ N(0, I).
#include <curand_kernel.h>

#include "common.cuh"
#include "sgemm.cuh"

namespace {

using namespace rb::gemm;

struct EnvArgs {
  const float* z;        // [B,obs] = s . W_s  (GEMM output)
  const float* action;   // [B,act]
  const float* w_a;      // [act,obs]
  const float* noise;    // optional pre-drawn [B, 2*obs+2]: eps[obs] | eps_r | u_term | reset[obs]
  float* next_state;     // [B,obs]
  float* final_obs;      // [B,obs]  (observation BEFORE the auto-reset)
  float* reward;         // [B]
  uint8_t* term;         // [B]
  uint8_t* trunc;        // [B]
  uint8_t* done;         // [B]
  int32_t* elapsed;      // [B] in/out
  const uint64_t* counter;  // device step counter (may be null)
  uint64_t seed;
  int B, obs, act, max_episode_steps, auto_reset;
  float p_term, noise_std, reward_noise_std;
};

// one warp per env
__global__ void __launch_bounds__(256) env_finish_kernel(EnvArgs p) {
  const int lane = threadIdx.x & 31;
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= p.B) return;
  const uint64_t ctr = p.counter ? p.counter[0] : 0ull;
  curandStatePhilox4_32_10_t st;
  if (!p.noise) curand_init(p.seed, (unsigned long long)row * 32ull + lane, ctr * 64ull, &st);
  const float* nz = p.noise ? p.noise + (size_t)row * (2 * p.obs + 2) : nullptr;
  float sq = 0.f;
  for (int j = lane; j < p.obs; j += 32) {
    float z = p.z[(size_t)row * p.obs + j];
    for (int a = 0; a < p.act; ++a) z = fmaf(p.action[(size_t)row * p.act + a], p.w_a[a * p.obs + j], z);
    const float eps = nz ? nz[j] : curand_normal(&st);
    const float s = tanhf(z + p.noise_std * eps);
    p.final_obs[(size_t)row * p.obs + j] = s;
    sq += s * s;
  }
  sq = rb::warp_sum(sq);
  float eps_r = 0.f, u = 1.f;
  if (lane == 0) {
    eps_r = nz ? nz[p.obs] : curand_normal(&st);
    u = nz ? nz[p.obs + 1] : curand_uniform(&st);
  }
  eps_r = __shfl_sync(0xffffffffu, eps_r, 0);
  u = __shfl_sync(0xffffffffu, u, 0);
  const int el = p.elapsed[row] + 1;
  const bool term = u < p.p_term;
  const bool trunc = p.max_episode_steps > 0 && el >= p.max_episode_steps;
  const bool done = term || trunc;
  if (lane == 0) {
    p.reward[row] = -sq / (float)p.obs + p.reward_noise_std * eps_r;
    p.term[row] = term;
    p.trunc[row] = trunc;
    p.done[row] = done;
    p.elapsed[row] = (done && p.auto_reset) ? 0 : el;
  }
  const bool reset = done && p.auto_reset;
  for (int j = lane; j < p.obs; j += 32) {
    float s = p.final_obs[(size_t)row * p.obs + j];  // written by this same lane above
    if (reset) s = nz ? nz[p.obs + 2 + j] : curand_normal(&st);
    p.next_state[(size_t)row * p.obs + j] = s;
  }
}

// ---- chunked stepping (num_action_chunks = C > 1): env.chunk_step of rlinf/envs/maniskill/maniskill_env.py:327-375 ----
// C sub-steps WITHOUT auto-reset, raw flags OR-ed over the chunk and reported on its last sub-step only, one auto-reset
// after the chunk (final_obs = observation before that reset); rewards [B,C] keep every sub-step.
struct SubArgs {
  const float* z;        // [B,obs] = s . W_s
  const float* action;   // [B, C*act]: sub-step c uses columns [c*act, (c+1)*act)
  const float* w_a;      // [act,obs]
  const float* noise;    // optional [B, C*(obs+2) + obs]: per sub-step eps[obs] | eps_r | u_term, then reset[obs]
  float* out_state;      // [B,obs] state after this sub-step (no reset)
  float* reward;         // [B,C]
  uint8_t* raw_term;     // [B,C] raw flags of every sub-step (rewritten by chunk_finish_kernel)
  uint8_t* raw_trunc;
  int32_t* elapsed;
  const uint64_t* counter;
  uint64_t seed;
  int B, obs, act, C, c, max_episode_steps;
  float p_term, noise_std, reward_noise_std;
};

__global__ void __launch_bounds__(256) env_substep_kernel(SubArgs p) {
  const int lane = threadIdx.x & 31;
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= p.B) return;
  const uint64_t ctr = p.counter ? p.counter[0] : 0ull;
  curandStatePhilox4_32_10_t st;
  if (!p.noise) curand_init(p.seed, (unsigned long long)row * 32ull + lane, (ctr * (uint64_t)p.C + p.c) * 64ull, &st);
  const float* nz = p.noise ? p.noise + (size_t)row * (p.C * (p.obs + 2) + p.obs) + (size_t)p.c * (p.obs + 2) : nullptr;
  const float* act = p.action + (size_t)row * p.C * p.act + (size_t)p.c * p.act;
  float sq = 0.f;
  for (int j = lane; j < p.obs; j += 32) {
    float z = p.z[(size_t)row * p.obs + j];
    for (int a = 0; a < p.act; ++a) z = fmaf(act[a], p.w_a[a * p.obs + j], z);
    const float eps = nz ? nz[j] : curand_normal(&st);
    const float s = tanhf(z + p.noise_std * eps);
    p.out_state[(size_t)row * p.obs + j] = s;
    sq += s * s;
  }
  sq = rb::warp_sum(sq);
  if (lane == 0) {
    const float eps_r = nz ? nz[p.obs] : curand_normal(&st);
    const float u = nz ? nz[p.obs + 1] : curand_uniform(&st);
    const int el = p.elapsed[row] + 1;
    p.elapsed[row] = el;
    p.reward[(size_t)row * p.C + p.c] = -sq / (float)p.obs + p.reward_noise_std * eps_r;
    p.raw_term[(size_t)row * p.C + p.c] = u < p.p_term;
    p.raw_trunc[(size_t)row * p.C + p.c] = p.max_episode_steps > 0 && el >= p.max_episode_steps;
  }
}

struct ChunkFinishArgs {
  const float* last_state;  // [B,obs] state after the last sub-step
  const float* noise;
  float* next_state;        // [B,obs]
  float* final_obs;         // [B,obs]
  uint8_t* term;            // [B,C] in: raw flags; out: zeros except the last column = any over the chunk
  uint8_t* trunc;
  uint8_t* done;
  int32_t* elapsed;
  const uint64_t* counter;
  uint64_t seed;
  int B, obs, C, auto_reset;
};

__global__ void __launch_bounds__(256) chunk_finish_kernel(ChunkFinishArgs p) {
  const int lane = threadIdx.x & 31;
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= p.B) return;
  bool t = false, tr = false;
  for (int c = 0; c < p.C; ++c) {
    t |= p.term[(size_t)row * p.C + c] != 0;
    tr |= p.trunc[(size_t)row * p.C + c] != 0;
  }
  const bool done = t || tr;
  const bool reset = done && p.auto_reset;
  __syncwarp();
  if (lane == 0) {
    for (int c = 0; c < p.C; ++c) {
      const bool last = c == p.C - 1;
      p.term[(size_t)row * p.C + c] = last && t;
      p.trunc[(size_t)row * p.C + c] = last && tr;
      p.done[(size_t)row * p.C + c] = last && done;
    }
    if (reset) p.elapsed[row] = 0;
  }
  const uint64_t ctr = p.counter ? p.counter[0] : 0ull;
  curandStatePhilox4_32_10_t st;
  // reset draws: same (row, lane) stream as the sub-steps, 32 outputs behind the last sub-step's window
  if (reset && !p.noise)
    curand_init(p.seed, (unsigned long long)row * 32ull + lane, (ctr * (uint64_t)p.C + (p.C - 1)) * 64ull + 32ull, &st);
  const float* nz = p.noise ? p.noise + (size_t)row * (p.C * (p.obs + 2) + p.obs) + (size_t)p.C * (p.obs + 2) : nullptr;
  for (int j = lane; j < p.obs; j += 32) {
    float s = p.last_state[(size_t)row * p.obs + j];
    p.final_obs[(size_t)row * p.obs + j] = s;
    if (reset) s = nz ? nz[j] : curand_normal(&st);
    p.next_state[(size_t)row * p.obs + j] = s;
  }
}

// rewards[b*ld_r] += gamma * vfinal[b*vdim] where flag[b*ld_f]  (compute_bootstrap_rewards, env_worker.py:736-758;
// ld = 1 for one-step actions, ld = C at the last sub-step of a chunk)
__global__ void __launch_bounds__(256) bootstrap_ld_kernel(float* __restrict__ rewards, int ld_r, const float* __restrict__ vfinal,
                                                           int vdim, const uint8_t* __restrict__ flag, int ld_f, int B,
                                                           float gamma) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  if (flag[(size_t)b * ld_f])
    rewards[(size_t)b * ld_r] = __fadd_rn(rewards[(size_t)b * ld_r], __fmul_rn(gamma, vfinal[(size_t)b * vdim]));
}

__global__ void counter_add_kernel(uint64_t* ctr, uint64_t inc) {
  if (threadIdx.x == 0 && blockIdx.x == 0) ctr[0] += inc;
}

}  // namespace

extern "C" int rb200_synth_env_step(const float* w_s, const float* w_a, const float* state, const float* action,
                                    const float* noise, float* next_state, float* final_obs, float* reward,
                                    uint8_t* term, uint8_t* trunc, uint8_t* done, int32_t* elapsed, float* z_scratch,
                                    int B, int obs, int act, int max_episode_steps, int auto_reset, float p_term,
                                    float noise_std, float reward_noise_std, uint64_t seed,
                                    const uint64_t* counter_dev, rb200_stream_t stream) {
  if (!w_s || !w_a || !state || !action || !next_state || !final_obs || !reward || !term || !trunc || !done ||
      !elapsed || !z_scratch)
    return RB200_E_NULL;
  if (B <= 0 || obs <= 0 || act <= 0) return RB200_E_SHAPE;
  cudaStream_t st = rb::as_stream(stream);
  GemmArgs g{};
  g.A = state; g.lda = obs; g.B = w_s; g.ldb = obs; g.C = z_scratch; g.ldc = obs;
  g.M = B; g.N = obs; g.K = obs; g.k_per_split = 1 << 30;
  int e = launch_gemm<A_KCONTIG, B_NCONTIG, EPI_STORE>(g, 1, st);  // z = s . W_s   (W_s is [obs_in, obs_out])
  if (e) return e;
  EnvArgs p{};
  p.z = z_scratch; p.action = action; p.w_a = w_a; p.noise = noise; p.next_state = next_state; p.final_obs = final_obs;
  p.reward = reward; p.term = term; p.trunc = trunc; p.done = done; p.elapsed = elapsed; p.counter = counter_dev;
  p.seed = seed; p.B = B; p.obs = obs; p.act = act; p.max_episode_steps = max_episode_steps; p.auto_reset = auto_reset;
  p.p_term = p_term; p.noise_std = noise_std; p.reward_noise_std = reward_noise_std;
  env_finish_kernel<<<(B + 7) / 8, 256, 0, st>>>(p); rb::count_launch();
  RB_RETURN_LAUNCH();
}

extern "C" int rb200_counter_add(uint64_t* counter_dev, uint64_t inc, rb200_stream_t stream) {
  if (!counter_dev) return RB200_E_NULL;
  counter_add_kernel<<<1, 32, 0, rb::as_stream(stream)>>>(counter_dev, inc); rb::count_launch();
  RB_RETURN_LAUNCH();
}

extern "C" int rb200_synth_env_chunk_step(const float* w_s, const float* w_a, const float* state, const float* chunk_actions,
                                          const float* noise, float* next_state, float* final_obs, float* rewards,
                                          uint8_t* term, uint8_t* trunc, uint8_t* done, int32_t* elapsed,
                                          float* scratch, int B, int obs, int act, int C, int max_episode_steps,
                                          int auto_reset, float p_term, float noise_std, float reward_noise_std,
                                          uint64_t seed, const uint64_t* counter_dev, rb200_stream_t stream) {
  if (!w_s || !w_a || !state || !chunk_actions || !next_state || !final_obs || !rewards || !term || !trunc || !done ||
      !elapsed || !scratch)
    return RB200_E_NULL;
  if (B <= 0 || obs <= 0 || act <= 0 || C <= 0) return RB200_E_SHAPE;
  cudaStream_t st = rb::as_stream(stream);
  const size_t n = (size_t)B * obs;
  float* z = scratch;                       // [B,obs]
  float* ping[2] = {scratch + n, scratch + 2 * n};  // states between sub-steps
  const float* cur = state;
  for (int c = 0; c < C; ++c) {
    GemmArgs g{};
    g.A = cur; g.lda = obs; g.B = w_s; g.ldb = obs; g.C = z; g.ldc = obs;
    g.M = B; g.N = obs; g.K = obs; g.k_per_split = 1 << 30;
    int e = launch_gemm<A_KCONTIG, B_NCONTIG, EPI_STORE>(g, 1, st);
    if (e) return e;
    SubArgs p{};
    p.z = z; p.action = chunk_actions; p.w_a = w_a; p.noise = noise; p.out_state = ping[c & 1]; p.reward = rewards;
    p.raw_term = term; p.raw_trunc = trunc; p.elapsed = elapsed; p.counter = counter_dev; p.seed = seed; p.B = B;
    p.obs = obs; p.act = act; p.C = C; p.c = c; p.max_episode_steps = max_episode_steps; p.p_term = p_term;
    p.noise_std = noise_std; p.reward_noise_std = reward_noise_std;
    env_substep_kernel<<<(B + 7) / 8, 256, 0, st>>>(p); rb::count_launch();
    cur = ping[c & 1];
  }
  ChunkFinishArgs f{};
  f.last_state = cur; f.noise = noise; f.next_state = next_state; f.final_obs = final_obs; f.term = term; f.trunc = trunc;
  f.done = done; f.elapsed = elapsed; f.counter = counter_dev; f.seed = seed; f.B = B; f.obs = obs; f.C = C;
  f.auto_reset = auto_reset;
  chunk_finish_kernel<<<(B + 7) / 8, 256, 0, st>>>(f); rb::count_launch();
  RB_RETURN_LAUNCH();
}

extern "C" int rb200_bootstrap_rewards_ld(float* rewards, int ld_rewards, const float* final_values, int value_dim,
                                          const uint8_t* flag, int ld_flag, int B, double gamma, rb200_stream_t stream) {
  if (!rewards || !final_values || !flag) return RB200_E_NULL;
  if (B <= 0 || value_dim <= 0 || ld_rewards <= 0 || ld_flag <= 0) return RB200_E_SHAPE;
  bootstrap_ld_kernel<<<(B + 255) / 256, 256, 0, rb::as_stream(stream)>>>(rewards, ld_rewards, final_values, value_dim,
                                                                           flag, ld_flag, B, (float)gamma);
  rb::count_launch();
  RB_RETURN_LAUNCH();
}
