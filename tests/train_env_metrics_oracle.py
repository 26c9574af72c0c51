"""CPU restatement of the training rollouts' episode statistics (env/* metrics; test infrastructure, like
tests/eval_oracle.py).

RunnerOracle.rollout drives the synthetic env with pre-drawn noise; this class wraps that env's `reset` / `chunk_step`
with the bookkeeping of ManiskillEnv (_record_metrics / _reset_metrics / _handle_auto_reset, rlinf/envs/maniskill/
maniskill_env.py:243-272,377-391) and the record rule of EnvWorker._run_interact_once / env_interact_step
(rlinf/workers/env/env_worker.py:507-522,1229-1235): every sub-step adds its raw reward to the fp32 running return, the
episode length is the env's elapsed step count (pre-reset), with auto_reset every env whose chunk is done records
(return, length, return / length) and restarts its return, without it every env records at the rollout's last chunk
step.  The return and the length carry over between rollouts; both restart where the env is reset.
"""
from __future__ import annotations

import torch

from eval_oracle import metrics_from_records
from oracle.runner_oracle import RunnerOracle

KEYS = ("return", "episode_len", "reward")


def oracle_cfg(B, T, C, obs, A, auto_reset, always, mes, p_term, env_seed, gamma=0.97):
    return {
        "algorithm": {"gamma": gamma, "bootstrap_type": "always" if always else "standard", "adv_type": "gae"},
        "env": {"train": {"auto_reset": bool(auto_reset), "max_episode_steps": mes, "total_num_envs": B,
                          "max_steps_per_rollout_epoch": T, "p_term": p_term, "seed": env_seed}},
        "actor": {"seed": 1, "model": {"obs_dim": obs, "action_dim": A, "num_action_chunks": C},
                  "optim": {"lr": 1e-3, "clip_grad": 1.0}},
    }


class TrainEnvMetricsOracle:
    """One rank's training rollouts with episode records.  initial_states [resets, B, obs]: the observations of the
    env's full resets in order (the first rollout's, and without auto_reset every rollout's)."""

    def __init__(self, cfg, params, initial_states):
        self.runner = RunnerOracle(cfg, params=params)
        env = self.runner.env
        self.C, self.nc = self.runner.num_action_chunks, self.runner.n_chunk_steps
        self.auto_reset = bool(cfg["env"]["train"]["auto_reset"])
        self.returns = torch.zeros(env.B, dtype=torch.float32)
        self._init = list(initial_states)
        self._n = 0
        self._recs = None
        chunk_step = env.chunk_step

        def reset():
            env.state = self._init.pop(0).clone()
            env.elapsed.zero_()
            self.returns.zero_()  # _reset_metrics
            return {"states": env.state}, {}

        def recording_chunk_step(chunk_actions, noise=None):
            length = env.elapsed + self.C  # no reset inside a chunk: the elapsed count at its last sub-step
            out = chunk_step(chunk_actions, noise)
            self._record(out[1], (out[2] | out[3])[:, -1], length)
            return out

        env.reset, env.chunk_step = reset, recording_chunk_step

    def _record(self, rewards, done, length):
        for c in range(self.C):
            self.returns = self.returns + rewards[:, c]  # _record_metrics: self.returns += step_reward
        episode = {"return": self.returns.clone(), "episode_len": length.clone()}
        episode["reward"] = episode["return"] / episode["episode_len"]
        if self.auto_reset:
            rec = done
            self.returns = torch.where(done, torch.zeros_like(self.returns), self.returns)
        else:
            rec = torch.full_like(done, self._n == self.nc - 1)
        for k in KEYS:
            self._recs[k].append(episode[k][rec])
        self._n += 1

    @torch.no_grad()
    def rollout(self, policy_noise, env_noise):
        """One rollout with the given draws (RunnerOracle.rollout); returns (records, batch): the episodes recorded, in
        the order env_interact_step reports them (chunk step by chunk step, env index within a step)."""
        self._n, self._recs = 0, {k: [] for k in KEYS}
        batch = self.runner.rollout(policy_noise=policy_noise, env_noise=env_noise)
        return {k: torch.cat(v) for k, v in self._recs.items()}, batch


def env_metrics(per_rank_records):
    """compute_evaluate_metrics over the ranks' records with the env/ prefix of EmbodiedRunner._log_step_metrics."""
    return {k.replace("eval/", "env/"): v for k, v in metrics_from_records(per_rank_records).items()}
