"""Device-resident synthetic vector env implementing the reference's `chunk_step` contract.

Contract (rlinf/envs/maniskill/maniskill_env.py:327-375, consumed by EnvWorker.env_interact_step,
rlinf/workers/env/env_worker.py:464-560): `reset() -> (obs, infos)`;
`chunk_step(chunk_actions [B,C,A]) -> (obs_list, rewards [B,C], terminations [B,C], truncations [B,C],
infos_list)` with `infos["final_observation"]` holding the pre-reset observation when auto_reset.
Dynamics are the benchmark workload of SURVEY.md §8(d): s' = tanh(s.W_s + a.W_a + 0.1 eps),
r = -|s'|^2/obs + 0.01 eps_r, termination ~ Bernoulli(p), truncation at max_episode_steps.
All state lives in HBM; one env step = one fp32 GEMM + one fused elementwise kernel.
"""
from __future__ import annotations

import math

import torch

from .. import _lib as L


class SyntheticVectorEnv:
    def __init__(self, num_envs, obs_dim, action_dim, max_episode_steps, auto_reset=True, p_term=0.005,
                 noise_std=0.1, reward_noise_std=0.01, seed=1234, device=None):
        self.num_envs, self.obs_dim, self.action_dim = int(num_envs), int(obs_dim), int(action_dim)
        self.max_episode_steps, self.auto_reset = int(max_episode_steps), bool(auto_reset)
        self.p_term, self.noise_std, self.reward_noise_std = float(p_term), float(noise_std), float(reward_noise_std)
        self.seed = int(seed)
        self.device = device or L.default_device()
        g = torch.Generator().manual_seed(self.seed)  # fixed dynamics, same on CPU (oracle) and device
        self.w_s = (torch.randn(obs_dim, obs_dim, generator=g) / math.sqrt(obs_dim)).to(self.device)
        self.w_a = (torch.randn(action_dim, obs_dim, generator=g) / math.sqrt(action_dim)).to(self.device)
        B = self.num_envs
        self.state = torch.zeros(B, obs_dim, device=self.device)
        self.elapsed = torch.zeros(B, dtype=torch.int32, device=self.device)
        self._z = torch.empty(B, obs_dim, device=self.device)
        self.counter = torch.zeros(1, dtype=torch.int64, device=self.device)  # device RNG step counter
        self._reset_gen = torch.Generator(device=self.device).manual_seed(self.seed + 1)
        self._chunk_scratch = None

    def reset(self):
        self.state.normal_(generator=self._reset_gen)  # one-off initialisation, not on the hot path
        self.elapsed.zero_()
        return {"states": self.state}, {}

    def state_dict(self) -> dict:
        """What the env carries between steps: the state written by the last reset, the elapsed step counts, the
        device random-stream counter and the reset generator.  The dynamics (w_s, w_a) come from the config."""
        return {"state": self.state, "elapsed": self.elapsed, "counter": self.counter,
                "reset_generator": self._reset_gen.get_state()}

    def load_state_dict(self, sd: dict) -> None:
        """In place: captured rollout graphs keep pointing at these tensors."""
        self.state.copy_(sd["state"])
        self.elapsed.copy_(sd["elapsed"])
        self.counter.copy_(sd["counter"])
        self._reset_gen.set_state(sd["reset_generator"])

    def step_into(self, state, action, next_state, final_obs, reward, term, trunc, done, noise=None):
        """One env step written straight into caller-provided (rollout-buffer) rows."""
        lib = L.load()
        L.check(lib.rb200_synth_env_step(
            L.ptr(self.w_s), L.ptr(self.w_a), L.ptr(state), L.ptr(action), L.ptr(noise), L.ptr(next_state),
            L.ptr(final_obs), L.ptr(reward), L.ptr(term), L.ptr(trunc), L.ptr(done), L.ptr(self.elapsed),
            L.ptr(self._z), self.num_envs, self.obs_dim, self.action_dim, self.max_episode_steps,
            int(self.auto_reset), self.p_term, self.noise_std, self.reward_noise_std, self.seed,
            L.ptr(self.counter), L.stream_ptr()), "synth_env_step")
        L.check(lib.rb200_counter_add(L.ptr(self.counter), 1, L.stream_ptr()), "counter_add")

    def chunk_step_into(self, state, chunk_actions, next_state, final_obs, rewards, term, trunc, done, noise=None):
        """num_action_chunks = C > 1 (maniskill_env.py:327-375): C sub-steps without auto-reset, flags any-reduced onto
        the last sub-step, one auto-reset after the chunk.  chunk_actions [B, C*A]; rewards / term / trunc / done [B, C]
        rows of the rollout buffer; noise: optional pre-drawn [B, C*(obs+2) + obs]."""
        lib = L.load()
        B, CA = chunk_actions.shape
        Cn = CA // self.action_dim
        if self._chunk_scratch is None:
            self._chunk_scratch = torch.empty(3, B, self.obs_dim, device=self.device)
        L.check(lib.rb200_synth_env_chunk_step(
            L.ptr(self.w_s), L.ptr(self.w_a), L.ptr(state), L.ptr(chunk_actions), L.ptr(noise), L.ptr(next_state),
            L.ptr(final_obs), L.ptr(rewards), L.ptr(term), L.ptr(trunc), L.ptr(done), L.ptr(self.elapsed),
            L.ptr(self._chunk_scratch), self.num_envs, self.obs_dim, self.action_dim, Cn, self.max_episode_steps,
            int(self.auto_reset), self.p_term, self.noise_std, self.reward_noise_std, self.seed, L.ptr(self.counter),
            L.stream_ptr()), "synth_env_chunk_step")
        L.check(lib.rb200_counter_add(L.ptr(self.counter), 1, L.stream_ptr()), "counter_add")

    def chunk_step(self, chunk_actions, noise=None):
        B, C, A = chunk_actions.shape
        dev = self.device
        if C != 1:
            nxt = torch.empty_like(self.state)
            final = torch.empty_like(self.state)
            rew = torch.empty(B, C, dtype=torch.float32, device=dev)
            term = torch.empty(B, C, dtype=torch.uint8, device=dev)
            trunc, done = torch.empty_like(term), torch.empty_like(term)
            self.chunk_step_into(self.state, chunk_actions.reshape(B, C * A).contiguous(), nxt, final, rew, term, trunc,
                                 done, noise)
            self.state = nxt
            return ([{"states": nxt}], rew, term.view(torch.bool), trunc.view(torch.bool),
                    [{"final_observation": {"states": final}}])
        nxt = torch.empty_like(self.state)
        final = torch.empty_like(self.state)
        rew = torch.empty(B, dtype=torch.float32, device=dev)
        term = torch.empty(B, dtype=torch.uint8, device=dev)
        trunc = torch.empty_like(term)
        done = torch.empty_like(term)
        self.step_into(self.state, chunk_actions.reshape(B, A).contiguous(), nxt, final, rew, term, trunc, done, noise)
        self.state = nxt
        infos = {"final_observation": {"states": final}}
        return ([{"states": nxt}], rew.view(B, 1), term.view(torch.bool).view(B, 1), trunc.view(torch.bool).view(B, 1),
                [infos])
