"""CPU restatement of EmbodiedRunner.evaluate on the synthetic env (test infrastructure, like oracle/runner_oracle.py).

The loop follows EnvWorker.evaluate / env_evaluate_step (rlinf/workers/env/env_worker.py:557-620,1374-1461) with the
policy in mode="eval" (action = mean, mlp_policy.py:256-293) and the episode bookkeeping of ManiskillEnv
(_record_metrics / _reset_metrics / _handle_auto_reset / chunk_step, rlinf/envs/maniskill/maniskill_env.py:225-271,
327-390): every sub-step adds its reward to the fp32 running return, the episode length is the env's elapsed step count,
and a chunk whose sub-steps terminated or truncated reports (return, length, return / length) of that env - once per
episode with auto_reset, only the first time per env and epoch without it.  Metrics are compute_evaluate_metrics
(rlinf/utils/metric_utils.py:372-419): the fp32 mean of each per-episode key and the number of episodes.
"""
from __future__ import annotations

import torch

from oracle import rl_oracle as O
from oracle.runner_oracle import SyntheticEnvCPU


def eval_env_params(cfg):
    """(num envs of the whole eval set, SyntheticEnvCPU kwargs) of cfg.env.eval, train values as defaults."""
    et, ev = cfg["env"]["train"], cfg["env"]["eval"]
    p_term = 0.0 if ev.get("ignore_terminations", False) else ev.get("p_term", et.get("p_term", 0.005))
    return ev["total_num_envs"], dict(max_episode_steps=ev["max_episode_steps"], auto_reset=ev["auto_reset"],
                                      p_term=p_term, noise_std=ev.get("noise_std", et.get("noise_std", 0.1)),
                                      reward_noise_std=ev.get("reward_noise_std", et.get("reward_noise_std", 0.01)))


class EvalOracle:
    """One rank's evaluation: `B` eval envs with the train env's dynamics (W_s / W_a from env.train.seed)."""

    def __init__(self, cfg, params, B=None):
        m, et, ev = cfg["actor"]["model"], cfg["env"]["train"], cfg["env"]["eval"]
        total, kw = eval_env_params(cfg)
        self.B = B or total
        self.C = m.get("num_action_chunks", 1)
        self.A = m["action_dim"]
        self.params = {k: v.detach().cpu() for k, v in params.items()}
        self.env = SyntheticEnvCPU(self.B, m["obs_dim"], self.A, seed=et.get("seed", 1234), **kw)
        self.auto_reset = bool(ev["auto_reset"])
        self.rollout_epoch = ev.get("rollout_epoch", 1)
        self.n_chunk_steps = ev["max_steps_per_rollout_epoch"] // self.C

    @torch.no_grad()
    def mean_action(self, states):
        return O.mlp_forward(self.params, states, None, want_entropy=False, want_values=False)["mean"]

    @torch.no_grad()
    def evaluate(self, env_noise, initial_states):
        """env_noise [rollout_epoch, n_chunk_steps, B, C*(obs+2)+obs]; initial_states [resets, B, obs].
        Returns (metrics, records): records = {"return", "episode_len", "reward"} per finished episode, in the order
        env_evaluate_step reports them (step by step, env index within a step)."""
        env, B, C, obs = self.env, self.B, self.C, self.env.obs_dim
        recs = {"return": [], "episode_len": [], "reward": []}
        resets = 0
        state = returns = prev_done = None
        for e in range(self.rollout_epoch):
            if e == 0 or not self.auto_reset:
                state = initial_states[resets].clone()
                resets += 1
                env.elapsed.zero_()
                returns = torch.zeros(B, dtype=torch.float32)
                prev_done = torch.zeros(B, dtype=torch.bool)
            for n in range(self.n_chunk_steps):
                noise = env_noise[e][n]
                action = self.mean_action(state).reshape(B, C, self.A)
                terms, truncs = [], []
                for c in range(C):
                    state, r, t, tr = env.substep_given_noise(state, action[:, c], noise[:, c * (obs + 2):(c + 1) * (obs + 2)])
                    returns = returns + r  # _record_metrics: self.returns += step_reward
                    terms.append(t)
                    truncs.append(tr)
                episode = {"return": returns.clone(), "episode_len": env.elapsed.clone()}
                episode["reward"] = episode["return"] / episode["episode_len"]
                done = torch.stack(terms, 1).any(1) | torch.stack(truncs, 1).any(1)
                if self.auto_reset:
                    newly = done
                    state = torch.where(done.unsqueeze(-1), noise[:, C * (obs + 2):], state)
                    env.elapsed[done] = 0
                    returns = torch.where(done, torch.zeros_like(returns), returns)
                else:
                    newly = done & ~prev_done
                    prev_done = prev_done | done
                for k in recs:
                    recs[k].append(episode[k][newly])
        records = {k: torch.cat(v) for k, v in recs.items()}
        return metrics_from_records([records]), records


def metrics_from_records(per_rank_records):
    """compute_evaluate_metrics over the ranks' record dicts, keys prefixed with eval/ as _maybe_eval_and_checkpoint
    does; with no finished episode only the count remains (an env_info key without entries is never created)."""
    count = sum(int(r["return"].numel()) for r in per_rank_records)
    if count == 0:
        return {"eval/num_trajectories": 0}
    out = {}
    for k in ("return", "episode_len", "reward"):
        stacked = torch.cat([r[k] for r in per_rank_records]).float()
        out[f"eval/{k}"] = float(stacked.mean())
    out["eval/num_trajectories"] = count
    return out


def draw_eval_noise(cfg, B, generator):
    """(env_noise [rollout_epoch, n, B, C*(obs+2)+obs], initial_states [resets, B, obs]) for one rank."""
    m, ev = cfg["actor"]["model"], cfg["env"]["eval"]
    C, obs = m.get("num_action_chunks", 1), m["obs_dim"]
    E, n = ev.get("rollout_epoch", 1), ev["max_steps_per_rollout_epoch"] // C
    parts = []
    for _ in range(C):
        parts += [torch.randn(E, n, B, obs + 1, generator=generator), torch.rand(E, n, B, 1, generator=generator)]
    parts.append(torch.randn(E, n, B, obs, generator=generator))
    resets = 1 if ev["auto_reset"] else E
    return torch.cat(parts, -1), torch.randn(resets, B, obs, generator=generator)
