// Per-episode statistics shared by the evaluation statistics kernel (eval.cu), the training statistics step and the
// persistent rollout kernels (rollout_tc.cu, rollout_fused.cu).
// Reference: ManiskillEnv._record_metrics, rlinf/envs/maniskill/maniskill_env.py:259-272 (return, episode_len = the
// env's elapsed steps, reward = return / episode_len); compute_evaluate_metrics, rlinf/utils/metric_utils.py:372-419.
#pragma once

#include <cstdint>

namespace rb {

// Finish one episode into an env's fp64 sums acc[4] = {count, sum return, sum length, sum reward}; returns the
// episode's reward (return / length, rounded like the reference's fp32 division).
__device__ __forceinline__ float episode_finish(double* acc, float ret, int32_t len) {
  const float rew = __fdiv_rn(ret, (float)len);
  acc[0] += 1.0;
  acc[1] += (double)ret;
  acc[2] += (double)len;
  acc[3] += (double)rew;
  return rew;
}

}  // namespace rb
