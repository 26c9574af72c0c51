"""Device-resident rollout: buffer layout and the T-step env/policy loop.

Replaces, for one rank, the ping-pong of EnvWorker._run_interact_once
(rlinf/workers/env/env_worker.py:1059-1349) and MultiStepRolloutWorker.generate_one_epoch
(rlinf/workers/rollout/hf/huggingface_worker.py:678-781): per chunk step the reference does two
Channel hops with CPU staging and appends [B,...] CPU tensors to Python lists that are later
`torch.stack`ed (rlinf/data/schema/embodied_trajectory_builder.py:72-231).  Here the trajectory rows
are written by the kernels directly into one `[T(+1), B, ...]` buffer in HBM - the layout
`convert_trajectories_to_batch` would produce (rlinf/data/schema/embodied_types.py:500):
  rewards / actions / prev_logprobs / forward_inputs{states,action}: T rows,
  dones / terminations / truncations / prev_values: T+1 rows (one bootstrap row)  [SURVEY A12].
Row alignment (env_worker.py:1120-1202): row t holds the action/logprob/value computed from obs_t,
`dones[t]` = done flags produced by step t-1 (row 0 all False), `rewards[t]` = reward of step t with the
truncation bootstrap gamma*V(final_obs) already folded in (SURVEY A14).
Three implementations of the same loop: the persistent tensor-core kernel (`rb200_rollout_tc`, one launch per rollout,
the default whenever it supports the problem), the persistent fp32 SIMT kernel (`rb200_rollout_fused`,
`rollout.fused_kernel: true`) and the per-kernel loop (`rollout.fused_kernel: false`)
captured once in a CUDA graph (rollout.enable_cuda_graph) and replayed - any env exposing `step_into` works there.
Each of the three also keeps the episode statistics of the rollout (the reference's `env/*` metrics) on the device.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass, field
from typing import Optional

import torch

from . import _lib as L


@dataclass
class Trajectory:
    """Field-for-field counterpart of rlinf.data.schema.embodied_types.Trajectory (:380-398) for the tensors this path
    produces.  Instances handed out by RolloutBuffer are VIEWS of the device buffer (no stack / cat / .cpu())."""

    max_episode_length: int = 0
    model_weights_id: str = ""
    actions: Optional[torch.Tensor] = None
    intervene_flags: Optional[torch.Tensor] = None
    rewards: Optional[torch.Tensor] = None
    terminations: Optional[torch.Tensor] = None
    truncations: Optional[torch.Tensor] = None
    dones: Optional[torch.Tensor] = None
    prev_logprobs: Optional[torch.Tensor] = None
    prev_values: Optional[torch.Tensor] = None
    versions: Optional[torch.Tensor] = None
    forward_inputs: dict = field(default_factory=dict)
    curr_obs: dict = field(default_factory=dict)
    next_obs: dict = field(default_factory=dict)


_TRAJ_TENSOR_FIELDS = ("actions", "intervene_flags", "rewards", "terminations", "truncations", "dones", "prev_logprobs",
                       "prev_values", "versions")


def _adjacent_views(parts) -> Optional[torch.Tensor]:
    """If `parts` are consecutive column slices [:, lo:hi] of ONE tensor, return that parent slice (zero copy)."""
    first = parts[0]
    if any(p.dim() < 2 or p.stride() != first.stride() or p.shape[0] != first.shape[0] or p.dtype != first.dtype or
           p.shape[2:] != first.shape[2:] for p in parts):
        return None
    step = first.stride(1) * first.element_size()
    ptr, cols = first.data_ptr(), 0
    for p in parts:
        if p.data_ptr() != ptr + cols * step or p.untyped_storage().data_ptr() != first.untyped_storage().data_ptr():
            return None
        cols += p.shape[1]
    return first.as_strided((first.shape[0], cols, *first.shape[2:]), first.stride(), first.storage_offset())


def convert_trajectories_to_batch(trajectories: list) -> dict:
    """[T, B, ...] batch dict from a list of trajectories (embodied_types.py:500-559: torch.cat over dim 1).  Parts that
    are adjacent views of the rollout buffer are re-joined without copying."""
    if not trajectories:
        return {}

    def join(parts):
        parts = [p for p in parts if p is not None]
        if not parts:
            return None
        if len(parts) == 1:
            return parts[0]
        joined = _adjacent_views(parts)
        return joined if joined is not None else torch.cat(parts, dim=1)

    batch: dict = {}
    for group in ("curr_obs", "next_obs", "forward_inputs"):
        if getattr(trajectories[0], group):
            keys = []
            for t in trajectories:
                keys += [k for k in getattr(t, group) if k not in keys]
            batch[group] = {k: join([getattr(t, group).get(k) for t in trajectories]) for k in keys}
    for name in _TRAJ_TENSOR_FIELDS:
        if isinstance(getattr(trajectories[0], name), torch.Tensor):
            batch[name] = join([getattr(t, name) for t in trajectories])
    return batch


class RolloutBuffer:
    def __init__(self, T, B, obs_dim, act_dim, value_dim=1, device=None, num_action_chunks=1):
        """T = CHUNK steps (n_chunk_steps = env steps // num_action_chunks); act_dim = num_action_chunks * action_dim.
        rewards / dones / terminations / truncations carry one column per sub-step of a chunk (SURVEY A12)."""
        dev = device or L.default_device()
        self.T, self.B, self.obs_dim, self.act_dim, self.value_dim = T, B, obs_dim, act_dim, value_dim
        self.num_action_chunks = Cn = int(num_action_chunks)
        f32, u8 = torch.float32, torch.uint8
        self.states = torch.zeros(T + 1, B, obs_dim, dtype=f32, device=dev)  # row T = bootstrap observation
        self.actions = torch.zeros(T, B, act_dim, dtype=f32, device=dev)
        self.prev_logprobs = torch.zeros(T, B, act_dim, dtype=f32, device=dev)
        self.prev_values = torch.zeros(T + 1, B, value_dim, dtype=f32, device=dev)
        self.rewards = torch.zeros(T, B, Cn, dtype=f32, device=dev)
        self.dones = torch.zeros(T + 1, B, Cn, dtype=u8, device=dev)
        self.terminations = torch.zeros(T + 1, B, Cn, dtype=u8, device=dev)
        self.truncations = torch.zeros(T + 1, B, Cn, dtype=u8, device=dev)
        self.final_obs = torch.zeros(B, obs_dim, dtype=f32, device=dev)
        self.final_values = torch.zeros(B, value_dim, dtype=f32, device=dev)

    def as_batch(self) -> dict:
        """The rollout batch dict the actor consumes (keys of Trajectory / convert_trajectories_to_batch)."""
        return {
            "rewards": self.rewards,
            "dones": self.dones.view(torch.bool),
            "terminations": self.terminations.view(torch.bool),
            "truncations": self.truncations.view(torch.bool),
            "prev_values": self.prev_values,
            "prev_logprobs": self.prev_logprobs,
            "forward_inputs": {"states": self.states[: self.T], "action": self.actions},
        }

    def to_trajectory(self, max_episode_length: int = 0, version: Optional[int] = None) -> Trajectory:
        """EmbodiedTrajectoryBuilder.to_trajectory (embodied_trajectory_builder.py:176-230) as views of the buffer."""
        b = self.as_batch()
        traj = Trajectory(max_episode_length=max_episode_length, actions=self.actions, rewards=b["rewards"],
                          terminations=b["terminations"], truncations=b["truncations"], dones=b["dones"],
                          prev_logprobs=b["prev_logprobs"], prev_values=b["prev_values"],
                          forward_inputs=dict(b["forward_inputs"]))
        if version is not None:
            traj.model_weights_id = str(version)
        return traj

    def to_splited_trajectories(self, split_size: int, max_episode_length: int = 0) -> list:
        """to_splited_trajectories (embodied_trajectory_builder.py:232-283): torch.chunk over the env dimension - here
        `split_size` column views of the same buffer (the reference makes each chunk contiguous, i.e. copies)."""
        full = self.to_trajectory(max_episode_length)
        if self.B % split_size != 0:
            raise ValueError(f"{self.B} envs cannot be split into {split_size} equal trajectories")
        w = self.B // split_size
        parts = []
        for i in range(split_size):
            sl = slice(i * w, (i + 1) * w)
            p = Trajectory(max_episode_length=full.max_episode_length, model_weights_id=full.model_weights_id)
            for name in _TRAJ_TENSOR_FIELDS:
                v = getattr(full, name)
                if v is not None:
                    setattr(p, name, v[:, sl])
            p.forward_inputs = {k: v[:, sl] for k, v in full.forward_inputs.items()}
            parts.append(p)
        return parts

    def nbytes(self) -> int:
        return sum(t.numel() * t.element_size() for t in (
            self.states[: self.T], self.actions, self.prev_logprobs, self.prev_values, self.rewards, self.dones,
            self.terminations, self.truncations))


# thresholds of rollout.fused_kernel: auto, carried over from an earlier GPU; not re-measured on the H100
FUSED_AUTO_MAX_ENVS_PER_CTA = 16
TC_AUTO_MIN_ENVS = 640


def select_rollout_impl(fused_kernel, num_action_chunks: int, B: int, sm_count: int, tc_supported: bool,
                        simt_supported: bool) -> str:
    """The rollout implementation for rollout.fused_kernel = "auto" | "tc" | True / "simt" | False: "tc" (persistent
    tensor-core kernel), "simt" (persistent fp32 SIMT kernel) or "graph" (per-kernel loop).  tc_supported /
    simt_supported: the env dynamics are on the device and rb200_rollout_tc_supported / rb200_rollout_fused_supported
    accept the problem."""
    Cn = num_action_chunks
    if Cn > 1 and fused_kernel in ("simt", True):
        raise ValueError("the persistent fp32 SIMT rollout kernel implements num_action_chunks == 1; chunked "
                         "policies use the tensor-core kernel (rollout.fused_kernel: tc / auto) or the per-kernel "
                         "loop (rollout.fused_kernel: false)")
    if fused_kernel == "tc" and not tc_supported:
        if Cn > 1:
            raise ValueError("rollout.fused_kernel='tc' with num_action_chunks > 1 needs hidden 256, obs_dim % 32 "
                             "== 0, obs_dim <= 128, 2 <= num_action_chunks <= 8, 1 <= action_dim <= 8, "
                             "num_action_chunks * action_dim <= 32 and one value per sub-step "
                             "(rb200_rollout_tc_supported)")
        raise ValueError("rollout.fused_kernel='tc' needs hidden 256, a value head, act_dim <= 8, obs_dim % 32 "
                         "== 0 and obs_dim <= 128 (rb200_rollout_tc_supported)")
    if tc_supported and (fused_kernel == "tc" or (fused_kernel == "auto" and Cn == 1 and B >= TC_AUTO_MIN_ENVS)):
        return "tc"
    # chunked: `auto` keeps the per-kernel loop, measured faster than the kernel at 256-4096 environments on an
    # H100 80GB HBM3 at 700 W (DESIGN.md §6)
    if Cn > 1 or not simt_supported:
        return "graph"
    if fused_kernel == "auto":
        return "simt" if -(-B // sm_count) <= FUSED_AUTO_MAX_ENVS_PER_CTA else "graph"
    return "simt" if fused_kernel else "graph"


def _capture_graph(fn):
    """(CUDA graph of fn(), kernels this library launched while capturing it = kernels replayed per replay)."""
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    n0 = L.load().rb200_launch_count()
    with torch.cuda.graph(g):
        fn()
    return g, int(L.load().rb200_launch_count() - n0)


class RolloutWorker:
    """One rank's env + policy replica.

    Episode statistics of the training rollouts (ManiskillEnv._record_metrics / _reset_metrics / _handle_auto_reset
    with the should_record rule of EnvWorker._run_interact_once, rlinf/envs/maniskill/maniskill_env.py:243-272,377-391,
    rlinf/workers/env/env_worker.py:507-522,1229-1235): every env step adds its raw reward (before the truncation
    bootstrap) to a per-env fp32 running return `ep_ret`.  With auto_reset an env whose chunk is done records
    (return, episode length, return / length) and restarts its return; return and length carry over between rollouts.
    Without auto_reset every env records its running episode at the rollout's last chunk step.  The records are summed
    per env into `ep_acc` [B,4] fp64 inside whichever rollout implementation runs, and `episode_sums` [4] fp64 =
    [count, sum return, sum length, sum reward] is reduced from it in a fixed order after every rollout.
    `episode_stats=False` runs the rollouts without statistics (for comparisons).
    `impl` is the implementation every rollout runs (select_rollout_impl)."""

    def __init__(self, cfg, policy, env, buffer: RolloutBuffer, episode_stats: bool = True):
        self.cfg, self.policy, self.env, self.buf = cfg, policy, env, buffer
        self.gamma = float(cfg.algorithm.get("gamma", 1))
        self.bootstrap_type = cfg.algorithm.get("bootstrap_type", "standard")
        self.auto_reset = bool(cfg.env.train.auto_reset)
        self.seed = int(cfg.actor.seed)
        self.counter = torch.zeros(1, dtype=torch.int64, device=policy.device)
        self._graph = None
        self._use_graph = bool(cfg.rollout.get("enable_cuda_graph", True))
        self.started = False
        self._calls = 0
        self.graph_kernel_count = 0  # kernels replayed per rollout once the CUDA graph exists
        # V(final_obs) of step t (bootstrap of truncated episodes) only feeds rewards[t]: it runs on a side stream,
        # concurrently with the policy inference of step t+1 (both are 32-CTA GEMM chains on a 132-SM device)
        self._side = torch.cuda.Stream(device=policy.device) if policy.device.type == "cuda" else None
        # the persistent kernels need the synthetic env's dynamics (w_s, w_a) on the device and a supported MLP shape
        self.num_action_chunks = Cn = int(getattr(buffer, "num_action_chunks", 1))
        B, lay = int(buffer.B), C.byref(policy.layout)
        on_dev_env = policy.device.type == "cuda" and hasattr(env, "w_s") and hasattr(env, "w_a")
        tc_ok = on_dev_env and L.load().rb200_rollout_tc_supported(lay, Cn, B) == 0
        simt_ok = on_dev_env and Cn == 1 and L.load().rb200_rollout_fused_supported(lay, B) == 0
        sms = torch.cuda.get_device_properties(policy.device).multi_processor_count if on_dev_env else 0
        self.impl = select_rollout_impl(cfg.rollout.get("fused_kernel", "auto"), Cn, B, sms, tc_ok, simt_ok)
        self.episode_stats = bool(episode_stats)
        dev = policy.device
        self.ep_ret = torch.zeros(buffer.B, dtype=torch.float32, device=dev)  # running return, carried across rollouts
        self.ep_len = torch.zeros(buffer.B, dtype=torch.int32, device=dev)    # elapsed steps (per-kernel loop only)
        self.ep_acc = torch.zeros(buffer.B, 4, dtype=torch.float64, device=dev)
        self.episode_sums = torch.zeros(4, dtype=torch.float64, device=dev)

    @property
    def _tc(self) -> bool:
        """The persistent tensor-core kernel runs the rollouts."""
        return self.impl == "tc"

    @property
    def _fused(self) -> bool:
        """The persistent fp32 SIMT kernel runs the rollouts."""
        return self.impl == "simt"

    def state_dict(self) -> dict:
        """What carries from one rollout to the next: the policy-sampling counter, whether the envs were reset, the
        last observation (row T, the next rollout's row 0 with auto_reset) and the running episode return / length.
        Device tensors, not copies; the env saves its own state."""
        return {"counter": self.counter, "started": bool(self.started), "last_obs": self.buf.states[self.buf.T],
                "ep_ret": self.ep_ret, "ep_len": self.ep_len}

    def load_state_dict(self, sd: dict) -> None:
        """In place: a captured rollout graph keeps pointing at these tensors."""
        self.counter.copy_(sd["counter"])
        self.started = bool(sd["started"])
        self.buf.states[self.buf.T].copy_(sd["last_obs"])
        self.ep_ret.copy_(sd["ep_ret"])
        self.ep_len.copy_(sd["ep_len"])

    def _stats_step(self, rewards, dones, C, last):
        """Episode statistics of one chunk step of the per-kernel loop: after the env step, before the bootstrap."""
        if self.episode_stats:
            L.check(L.load().rb200_train_episode_stats_step(
                L.ptr(rewards), L.ptr(dones), self.buf.B, C, int(self.auto_reset), int(last), L.ptr(self.ep_ret),
                L.ptr(self.ep_len), L.ptr(self.ep_acc), L.stream_ptr()), "train_episode_stats_step")

    def _kernel_rollout(self, policy_noise, env_noise):
        """The whole T-step loop in one persistent kernel: tensor-core (csrc/rollout_tc.cu; T = chunk steps when
        num_action_chunks > 1) or fp32 SIMT (csrc/rollout_fused.cu)."""
        lib = L.load()
        buf, pol, env = self.buf, self.policy, self.env
        st = L.stream_ptr()
        lay = C.byref(pol.layout)
        if self.impl == "tc":
            nbytes = int(lib.rb200_rollout_tc_pack_bytes(lay))
            weights = pol._buf("rollout_tc_pack", (nbytes + 3) // 4)
            L.check(lib.rb200_rollout_tc_prepare(lay, L.ptr(pol.flat_params), L.ptr(env.w_s), L.ptr(weights), st),
                    "rollout_tc_prepare")
            entry, what = lib.rb200_rollout_tc, "rollout_tc"
        else:
            weights = pol._buf("rollout_wt", lib.rb200_rollout_fused_wt_floats(lay))
            L.check(lib.rb200_rollout_fused_prepare(lay, L.ptr(pol.flat_params), L.ptr(weights), st),
                    "rollout_fused_prepare")
            entry, what = lib.rb200_rollout_fused, "rollout_fused"
        has_v, stats = pol.value_dim > 0, self.episode_stats
        a = L.RolloutArgs(
            states=L.ptr(buf.states), actions=L.ptr(buf.actions), logprobs=L.ptr(buf.prev_logprobs),
            values=L.ptr(buf.prev_values) if has_v else None, rewards=L.ptr(buf.rewards),
            terminations=L.ptr(buf.terminations), truncations=L.ptr(buf.truncations), dones=L.ptr(buf.dones),
            final_obs=L.ptr(buf.final_obs), final_values=L.ptr(buf.final_values) if has_v else None,
            w_s=L.ptr(env.w_s), w_a=L.ptr(env.w_a), elapsed=L.ptr(env.elapsed), policy_noise=L.ptr(policy_noise),
            env_noise=L.ptr(env_noise), counter_policy=L.ptr(self.counter), counter_env=L.ptr(env.counter),
            episode_return=L.ptr(self.ep_ret) if stats else None, episode_acc=L.ptr(self.ep_acc) if stats else None,
            seed_policy=self.seed, seed_env=env.seed, offset_policy=0, T=buf.T, B=buf.B,
            num_action_chunks=self.num_action_chunks, max_episode_steps=env.max_episode_steps,
            auto_reset=int(self.auto_reset), bootstrap_on_done=int(self.bootstrap_type != "standard"), gamma=self.gamma,
            p_term=env.p_term, noise_std=env.noise_std, reward_noise_std=env.reward_noise_std)
        L.check(entry(lay, L.ptr(pol.flat_params), L.ptr(weights), C.byref(a), st), what)
        L.check(lib.rb200_counter_add(L.ptr(self.counter), buf.T, st), "counter_add")
        L.check(lib.rb200_counter_add(L.ptr(env.counter), buf.T, st), "counter_add")

    def _one_rollout(self, policy_noise=None, env_noise=None):
        """policy_noise [T,B,act] / env_noise [T,B,2*obs+2]: pre-drawn N(0,1)/U(0,1) draws (parity tests);
        None -> Philox on the device."""
        if self.impl != "graph":
            return self._kernel_rollout(None if policy_noise is None else policy_noise.contiguous(),
                                        None if env_noise is None else env_noise.contiguous())
        lib = L.load()
        buf, pol, env = self.buf, self.policy, self.env
        T, B = buf.T, buf.B
        st = L.stream_ptr()
        pol.mark_params_changed()  # the weight split refresh is always part of the (captured) rollout
        if self.num_action_chunks > 1:
            return self._chunked_rollout(policy_noise, env_noise)
        main, side = torch.cuda.current_stream(), self._side
        side_busy = False
        for t in range(T):
            # policy/value inference on obs_t -> action, logprob, value rows t  (predict_action_batch)
            pol.sample(buf.states[t], noise=None if policy_noise is None else policy_noise[t], seed=self.seed,
                       offset=0, counter=self.counter, out=(buf.actions[t], buf.prev_logprobs[t], buf.prev_values[t]))
            L.check(lib.rb200_counter_add(L.ptr(self.counter), 1, st), "counter_add")
            if side_busy:  # V(final_obs) of step t-1 must have read final_obs before this step overwrites it
                main.wait_stream(side)
                side_busy = False
            # env.chunk_step: writes obs_{t+1} (row t+1), reward t, flags row t+1
            env.step_into(buf.states[t], buf.actions[t], buf.states[t + 1], buf.final_obs,
                          buf.rewards[t].view(B), buf.terminations[t + 1].view(B), buf.truncations[t + 1].view(B),
                          buf.dones[t + 1].view(B), noise=None if env_noise is None else env_noise[t])
            self._stats_step(buf.rewards[t], buf.dones[t + 1], 1, t == T - 1)
            # compute_bootstrap_rewards (env_worker.py:719-758): r += gamma * V(final_obs) where truncated/done
            if self.auto_reset and pol.value_dim > 0:
                flag = buf.truncations[t + 1] if self.bootstrap_type == "standard" else buf.dones[t + 1]
                side.wait_stream(main)
                with torch.cuda.stream(side):
                    pol.value(buf.final_obs, out=buf.final_values)
                    L.check(lib.rb200_bootstrap_rewards_ld(L.ptr(buf.rewards[t]), 1, L.ptr(buf.final_values),
                                                           pol.value_dim, L.ptr(flag.view(B)), 1, B, self.gamma,
                                                           L.stream_ptr()), "bootstrap_rewards_ld")
                side_busy = True
        if side_busy:
            main.wait_stream(side)
        # final extra inference for the bootstrap value row T (env_worker.py:1237-1306)
        if pol.value_dim > 0:
            pol.value(buf.states[T], out=buf.prev_values[T])

    def _chunked_rollout(self, policy_noise=None, env_noise=None):
        """num_action_chunks = C > 1: one policy inference per CHUNK step, C env sub-steps per chunk (chunk_step contract,
        maniskill_env.py:327-375), bootstrap on the chunk's last sub-step (compute_bootstrap_rewards, env_worker.py:
        719-758).  policy_noise [nc, B, C*A], env_noise [nc, B, C*(obs+2) + obs]."""
        lib = L.load()
        buf, pol, env = self.buf, self.policy, self.env
        nc, B, Cn = buf.T, buf.B, self.num_action_chunks
        st = L.stream_ptr()
        for n in range(nc):
            pol.sample(buf.states[n], noise=None if policy_noise is None else policy_noise[n], seed=self.seed, offset=0,
                       counter=self.counter, out=(buf.actions[n], buf.prev_logprobs[n], buf.prev_values[n]))
            L.check(lib.rb200_counter_add(L.ptr(self.counter), 1, st), "counter_add")
            env.chunk_step_into(buf.states[n], buf.actions[n], buf.states[n + 1], buf.final_obs, buf.rewards[n],
                                buf.terminations[n + 1], buf.truncations[n + 1], buf.dones[n + 1],
                                noise=None if env_noise is None else env_noise[n])
            self._stats_step(buf.rewards[n], buf.dones[n + 1], Cn, n == nc - 1)
            if self.auto_reset and pol.value_dim > 0:
                flag = buf.truncations[n + 1] if self.bootstrap_type == "standard" else buf.dones[n + 1]
                pol.value(buf.final_obs, out=buf.final_values)
                L.check(lib.rb200_bootstrap_rewards_ld(
                    C.c_void_p(buf.rewards[n].data_ptr() + 4 * (Cn - 1)), Cn, L.ptr(buf.final_values), pol.value_dim,
                    C.c_void_p(flag.data_ptr() + (Cn - 1)), Cn, B, self.gamma, st), "bootstrap_rewards_ld")
        if pol.value_dim > 0:
            pol.value(buf.states[nc], out=buf.prev_values[nc])

    def generate(self):
        """One rollout epoch of T steps into the buffer (all on the current stream, no host sync)."""
        buf = self.buf
        if not self.started or not self.auto_reset:
            # bootstrap_step (env_worker.py:908-935): with auto_reset off the envs are reset at EVERY rollout epoch
            # (elapsed back to 0, fresh initial states); with auto_reset on only once, at the very beginning
            obs, _ = self.env.reset()
            buf.states[0].copy_(obs["states"])
            self.ep_ret.zero_()  # ManiskillEnv.reset -> _reset_metrics
            self.ep_len.zero_()
            self.started = True
        else:
            buf.states[0].copy_(buf.states[buf.T])  # last obs of the previous rollout (bootstrap_step)
        self.ep_acc.zero_()
        # dones row 0 = zeros (env_worker.py:899-945): never written by the loop, stays zero
        if self.impl != "graph" or not self._use_graph or self._calls == 0:
            self._one_rollout()  # first call runs eagerly (also allocates every scratch buffer)
        else:
            self._replay()
        self._calls += 1
        if self.episode_stats:
            L.check(L.load().rb200_episode_stats_reduce(L.ptr(self.ep_acc), buf.B, L.ptr(self.episode_sums),
                                                        L.stream_ptr()), "episode_stats_reduce")

    def _replay(self):
        if self._graph is None:
            self._graph, self.graph_kernel_count = _capture_graph(self._one_rollout)
        self._graph.replay()


class EvalWorker:
    """Deterministic evaluation rollouts of one rank: EnvWorker.evaluate / env_evaluate_step (rlinf/workers/env/
    env_worker.py:557-620,1374-1461) against MultiStepRolloutWorker.evaluate with predict_action_batch(mode="eval").

    Per chunk step: action = policy mean (rb200_mlp_mean, no value tower), one env chunk step, then the episode
    statistics (rb200_episode_stats_step).  Nothing of the trajectory is kept: two [B,obs] state tensors used in turn
    and one [B,C*A] / [B,C] row set.  The env is reset at the first eval epoch and, with auto_reset off, at every epoch
    (running return / length / prev_done reset with it); with auto_reset on its state carries over between epochs.
    The statistics stay on the device until `run()` has reduced them to [count, sum return, sum length, sum reward]."""

    def __init__(self, cfg, policy, env, num_action_chunks=1):
        ev = cfg.env.eval
        self.policy, self.env = policy, env
        self.num_action_chunks = Cn = int(num_action_chunks)
        T = int(ev.max_steps_per_rollout_epoch)
        if T % Cn != 0:
            raise ValueError(f"env.eval.max_steps_per_rollout_epoch {T} is not a multiple of num_action_chunks {Cn}")
        self.n_chunk_steps = T // Cn
        self.rollout_epoch = int(ev.get("rollout_epoch", 1))
        self.auto_reset = bool(ev.auto_reset)
        self._use_graph = bool(cfg.rollout.get("enable_cuda_graph", True))
        B, obs, dev = env.num_envs, env.obs_dim, policy.device
        f32, u8 = torch.float32, torch.uint8
        self.B = B
        self.states = torch.zeros(2, B, obs, dtype=f32, device=dev)
        self.final_obs = torch.zeros(B, obs, dtype=f32, device=dev)
        self.actions = torch.zeros(B, policy.act_dim, dtype=f32, device=dev)
        self.rewards = torch.zeros(B, Cn, dtype=f32, device=dev)
        self.terminations = torch.zeros(B, Cn, dtype=u8, device=dev)
        self.truncations = torch.zeros(B, Cn, dtype=u8, device=dev)
        self.dones = torch.zeros(B, Cn, dtype=u8, device=dev)
        self.ret = torch.zeros(B, dtype=f32, device=dev)
        self.len = torch.zeros(B, dtype=torch.int32, device=dev)
        self.prev_done = torch.zeros(B, dtype=u8, device=dev)
        self.acc = torch.zeros(B, 4, dtype=torch.float64, device=dev)  # count, sum return, sum length, sum reward
        self.sums = torch.zeros(4, dtype=torch.float64, device=dev)
        self._graph = None
        self._calls = 0
        self.graph_kernel_count = 0

    def _reset(self, initial_states=None):
        obs, _ = self.env.reset()
        self.states[0].copy_(obs["states"] if initial_states is None else initial_states)
        self.ret.zero_()
        self.len.zero_()
        self.prev_done.zero_()

    def _epoch(self, env_noise=None, episodes=None):
        """One eval epoch of n_chunk_steps chunk steps from states[0]; leaves the last observation in states[0].
        env_noise [n, B, ...] (layout of the env's step); episodes [n, B, 3] receives the per-step episode records."""
        lib = L.load()
        pol, env, B, Cn = self.policy, self.env, self.B, self.num_action_chunks
        st = L.stream_ptr()
        pol.mark_params_changed()  # the weight split refresh is part of the (captured) epoch
        for n in range(self.n_chunk_steps):
            s, s_next = self.states[n & 1], self.states[(n + 1) & 1]
            noise = None if env_noise is None else env_noise[n]
            pol.mean(s, calculate_logprobs=False, calculate_values=False, out=self.actions, work_key="eval")
            if Cn == 1:
                env.step_into(s, self.actions, s_next, self.final_obs, self.rewards.view(B),
                              self.terminations.view(B), self.truncations.view(B), self.dones.view(B), noise=noise)
            else:
                env.chunk_step_into(s, self.actions, s_next, self.final_obs, self.rewards, self.terminations,
                                    self.truncations, self.dones, noise=noise)
            L.check(lib.rb200_episode_stats_step(
                L.ptr(self.rewards), L.ptr(self.dones), B, Cn, int(self.auto_reset), L.ptr(self.ret), L.ptr(self.len),
                L.ptr(self.prev_done), L.ptr(self.acc), None if episodes is None else L.ptr(episodes[n]), st),
                "episode_stats_step")
        if self.n_chunk_steps % 2:
            self.states[0].copy_(self.states[1])

    def run(self, env_noise=None, initial_states=None, episodes=None) -> torch.Tensor:
        """All eval epochs; returns the device tensor [count, sum return, sum length, sum reward] (fp64).
        env_noise [rollout_epoch, n, B, ...] / initial_states [number of resets, B, obs]: pre-drawn draws (parity
        tests; they run eagerly); episodes [rollout_epoch, n, B, 3]: optional per-step episode records."""
        self.acc.zero_()
        resets = 0
        for e in range(self.rollout_epoch):
            if e == 0 or not self.auto_reset:  # EnvWorker.evaluate: reset at the first epoch / every epoch
                self._reset(None if initial_states is None else initial_states[resets])
                resets += 1
            eager = (env_noise is not None or episodes is not None or not self._use_graph or self._calls == 0)
            if eager:
                self._epoch(None if env_noise is None else env_noise[e], None if episodes is None else episodes[e])
                continue
            if self._graph is None:
                self._graph, self.graph_kernel_count = _capture_graph(self._epoch)
            self._graph.replay()
        L.check(L.load().rb200_episode_stats_reduce(L.ptr(self.acc), self.B, L.ptr(self.sums), L.stream_ptr()),
                "episode_stats_reduce")
        self._calls += 1
        return self.sums
