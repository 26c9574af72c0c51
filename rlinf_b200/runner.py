"""Single-process-per-GPU driver loop - mirror of EmbodiedRunner.run().

Reference: rlinf/runners/embodied_runner.py:478-563 (set_global_step, update_rollout_weights,
env.interact || rollout.generate || actor.recv_rollout_trajectories, compute_advantages_and_returns,
run_training, metrics).  Not a port of the Ray worker stack: one process per GPU owns the env shard,
the rollout policy replica and the learner; experience shards over ranks by environment.
"""
from __future__ import annotations

import time

import torch
import torch.distributed as dist

from . import _lib as L
from . import checkpoint as ckpt
from .actor import EmbodiedActor
from .config import wrap
from .envs import SyntheticVectorEnv
from .rollout import EvalWorker, RolloutBuffer, RolloutWorker


def max_steps(runner_cfg) -> int:
    """EmbodiedRunner.set_max_steps (embodied_runner.py:655-660): runner.max_epochs, capped by runner.max_steps >= 0."""
    n = int(runner_cfg.max_epochs)
    cap = int(runner_cfg.get("max_steps", -1))
    return min(n, cap) if cap >= 0 else n


def should_evaluate(step: int, max_steps: int, val_check_interval: int) -> bool:
    """The validation half of check_progress (rlinf/utils/runner_utils.py:31-61): evaluate when val_check_interval > 0
    and either step is a positive multiple of it or step == max_steps (the last step)."""
    if val_check_interval <= 0:
        return False
    return (step != 0 and step % val_check_interval == 0) or step == max_steps


def check_eval_config(cfg) -> int:
    """runner.val_check_interval (0 / absent / negative = no evaluation); evaluating needs an env.eval section with the
    keys the eval loop reads.  Returns the interval."""
    interval = int(cfg.runner.get("val_check_interval", 0) or 0)
    ev = cfg.env.get("eval")
    if interval > 0 and ev is None:
        raise ValueError(f"runner.val_check_interval={interval} needs an env.eval section")
    if ev is not None:
        missing = [k for k in ("total_num_envs", "max_episode_steps", "max_steps_per_rollout_epoch", "auto_reset")
                   if k not in ev]
        if missing:
            raise ValueError(f"env.eval is missing {missing}")
    return interval


def should_save(step: int, max_steps: int, val_check_interval: int, save_interval: int) -> bool:
    """The save half of check_progress (rlinf/utils/runner_utils.py:31-61): save when save_interval > 0 and either step
    is a positive multiple of it or step == max_steps (the last step).  With evaluation on, save_interval must be
    negative or a multiple of val_check_interval (ValueError otherwise, the reference's assertion)."""
    if val_check_interval > 0 and not (save_interval < 0 or save_interval % val_check_interval == 0):
        raise ValueError(f"runner.save_interval={save_interval} must be divisible by "
                         f"runner.val_check_interval={val_check_interval}")
    if save_interval <= 0:
        return False
    return (step != 0 and step % save_interval == 0) or step == max_steps


def check_save_config(cfg, val_check_interval: int) -> int:
    """runner.save_interval (0 / absent / negative = no checkpoints); saving needs runner.logger.log_path and
    runner.logger.experiment_name.  Returns the interval."""
    interval = int(cfg.runner.get("save_interval", 0) or 0)
    should_save(0, 0, val_check_interval, interval)  # the interval check only
    if interval > 0:
        ckpt.checkpoint_dir(cfg.runner, 0)
    return interval


def eval_metrics_from_sums(sums, prefix: str = "eval") -> dict:
    """compute_evaluate_metrics (rlinf/utils/metric_utils.py:372-419) for an env without `success`, from the reduced
    [count, sum return, sum length, sum reward]: means over recorded episodes and their number; only the count when
    no episode was recorded (there is no per-episode entry to average then).  Keys are `{prefix}/...`: `eval` for
    evaluation, `env` for the training rollouts (EmbodiedRunner._log_step_metrics)."""
    count, s_ret, s_len, s_rew = (float(x) for x in sums)
    n = int(count)
    if n == 0:
        return {f"{prefix}/num_trajectories": 0}
    return {f"{prefix}/return": s_ret / n, f"{prefix}/episode_len": s_len / n, f"{prefix}/reward": s_rew / n,
            f"{prefix}/num_trajectories": n}


def records_train_episodes(env_train_cfg) -> bool:
    """Whether the training rollouts report env/* metrics: always, except with auto_reset off and
    ignore_terminations on, which the synthetic training env does not implement."""
    return bool(env_train_cfg.auto_reset) or not env_train_cfg.get("ignore_terminations", False)


class EmbodiedRunner:
    def __init__(self, cfg, rank=None, world_size=None, process_group=None):
        self.cfg = cfg = wrap(cfg)
        self.val_check_interval = check_eval_config(cfg)
        self.save_interval = check_save_config(cfg, self.val_check_interval)
        self.max_steps = max_steps(cfg.runner)
        self._dist = dist.is_available() and dist.is_initialized()
        self.rank = rank if rank is not None else (dist.get_rank() if self._dist else 0)
        self.world_size = world_size if world_size is not None else (dist.get_world_size() if self._dist else 1)
        et, m = cfg.env.train, cfg.actor.model
        from .dist_utils import shard_envs
        self.env_start, self.B = shard_envs(et.total_num_envs, self.world_size, self.rank,
                                            cfg.algorithm.get("group_size", 1))  # envs owned by this rank
        self.T = et.max_steps_per_rollout_epoch
        Cn = int(m.get("num_action_chunks", 1))
        if self.T % Cn != 0:
            raise ValueError(f"max_steps_per_rollout_epoch {self.T} is not a multiple of num_action_chunks {Cn}")
        self.n_chunk_steps = self.T // Cn  # env_worker.py: n_chunk_steps = max_steps_per_rollout_epoch // num_action_chunks
        self.actor = EmbodiedActor(cfg, rank=self.rank, world_size=self.world_size, process_group=process_group)
        pol = self.actor.model
        self.env = SyntheticVectorEnv(self.B, m.obs_dim, m.action_dim,  # the env takes ONE action per sub-step
                                      et.max_episode_steps, auto_reset=et.auto_reset, p_term=et.get("p_term", 0.005),
                                      noise_std=et.get("noise_std", 0.1),
                                      reward_noise_std=et.get("reward_noise_std", 0.01),
                                      seed=et.get("seed", 1234) + 1000 * self.rank)
        # dynamics are identical on every rank (same W_s / W_a), only the noise stream differs
        g = torch.Generator().manual_seed(et.get("seed", 1234))
        import math
        self.env.w_s.copy_(torch.randn(m.obs_dim, m.obs_dim, generator=g) / math.sqrt(m.obs_dim))
        self.env.w_a.copy_(torch.randn(m.action_dim, m.obs_dim, generator=g) / math.sqrt(m.action_dim))
        self.buffer = RolloutBuffer(self.n_chunk_steps, self.B, m.obs_dim, pol.act_dim, max(pol.value_dim, 1),
                                    num_action_chunks=Cn)
        self.rollout = RolloutWorker(cfg, pol, self.env, self.buffer, episode_stats=records_train_episodes(et))
        ev = cfg.env.get("eval")
        self.eval_env, self.evaluator = None, None
        if ev is not None:
            self.eval_env = self._build_eval_env(ev, et, m)
            self.evaluator = EvalWorker(cfg, pol, self.eval_env, Cn)
        self.global_step = 0
        if cfg.runner.get("ckpt_path"):  # policy weights only (embodied_fsdp_actor_worker.py:122-124)
            pol.load_state_dict(ckpt.load_weights(cfg.runner.ckpt_path), strict=True)
        if self.world_size > 1:  # same initial weights everywhere (rank 0's)
            dist.broadcast(pol.flat_params, src=0, group=process_group)
        self._pg = process_group
        if cfg.runner.get("resume_dir"):  # the end of init_workers (embodied_runner.py:175-185)
            self.load_checkpoint(cfg.runner.resume_dir)

    def _build_eval_env(self, ev, et, m):
        """The eval env set (cfg.env.eval): same task as the train env (its W_s / W_a), own state, step counter and
        reset generator, so the training random streams are untouched.  Noise parameters and seed default to the train
        values; ignore_terminations: True -> p_term = 0 (the termination draw is still made, so the noise stream is
        the same; terminations of this env only feed the done flags, maniskill_env.py:312-318)."""
        from .dist_utils import shard_envs
        _, B = shard_envs(ev.total_num_envs, self.world_size, self.rank)
        p_term = 0.0 if ev.get("ignore_terminations", False) else ev.get("p_term", et.get("p_term", 0.005))
        env = SyntheticVectorEnv(B, m.obs_dim, m.action_dim, ev.max_episode_steps, auto_reset=ev.auto_reset,
                                 p_term=p_term, noise_std=ev.get("noise_std", et.get("noise_std", 0.1)),
                                 reward_noise_std=ev.get("reward_noise_std", et.get("reward_noise_std", 0.01)),
                                 seed=ev.get("seed", et.get("seed", 1234)) + 1000 * self.rank)
        env.w_s.copy_(self.env.w_s)
        env.w_a.copy_(self.env.w_a)
        return env

    def evaluate(self, env_noise=None, initial_states=None) -> dict:
        """EmbodiedRunner.evaluate after update_rollout_weights (embodied_runner.py:193-206,308-329): the policy mean
        on the eval envs for env.eval.rollout_epoch epochs; {"eval/return", "eval/episode_len", "eval/reward",
        "eval/num_trajectories"} over the episodes finished on all ranks (one all-reduce of 4 doubles, one
        device-to-host copy).  env_noise / initial_states: pre-drawn draws for parity tests (EvalWorker.run)."""
        if self.evaluator is None:
            raise ValueError("evaluate() needs an env.eval section in the config")
        self.update_rollout_weights()
        sums = self.evaluator.run(env_noise=env_noise, initial_states=initial_states)
        if self.world_size > 1:
            sums = sums.clone()
            dist.all_reduce(sums, op=dist.ReduceOp.SUM, group=self._pg)
        return eval_metrics_from_sums(sums.cpu().tolist())

    def env_metrics(self) -> dict:
        """env/return, env/episode_len, env/reward, env/num_trajectories of the last training rollout on all ranks
        (one all-reduce of 4 doubles, one device-to-host copy); {} when the config records no training episodes."""
        if not self.rollout.episode_stats:
            return {}
        sums = self.rollout.episode_sums
        if self.world_size > 1:
            sums = sums.clone()
            dist.all_reduce(sums, op=dist.ReduceOp.SUM, group=self._pg)
        return eval_metrics_from_sums(sums.cpu().tolist(), "env")

    def update_rollout_weights(self):
        self.actor.sync_model_to_rollout(self.rollout.policy.flat_params)

    def rollout_phase(self):
        self.rollout.generate()

    def update_phase(self, batch=None):
        self.actor.recv_rollout_trajectories(batch if batch is not None else self.buffer.as_batch())
        rollout_metrics = self.actor.compute_advantages_and_returns()
        metrics = self.actor.run_training()
        metrics.update({f"rollout/{k}": v for k, v in rollout_metrics.items()})
        return metrics

    def run_iteration(self):
        self.actor.version = self.global_step
        if self.global_step % self.cfg.runner.get("weight_sync_interval", 1) == 0:
            self.update_rollout_weights()
        self.rollout_phase()
        metrics = self.update_phase()
        metrics.update(self.env_metrics())
        self.global_step += 1
        # _maybe_eval_and_checkpoint (embodied_runner.py:308-329), on the incremented step count
        if should_evaluate(self.global_step, self.max_steps, self.val_check_interval):
            metrics.update(self.evaluate())
        if should_save(self.global_step, self.max_steps, self.val_check_interval, self.save_interval):
            self.save_checkpoint()
        return metrics

    def run(self, max_epochs=None):
        """`max_epochs` iterations; by default the iterations left until runner.max_epochs, so a resumed run stops
        where an uninterrupted one would."""
        out = []
        for _ in range(max_epochs or max(0, int(self.cfg.runner.max_epochs) - self.global_step)):
            out.append(self.run_iteration())
        return out

    # ---- checkpoint --------------------------------------------------------------------------------
    def fingerprint(self) -> dict:
        """The shapes and the sharding a checkpoint must agree with (checkpoint.FINGERPRINT_FIELDS)."""
        et, ev, pol = self.cfg.env.train, self.cfg.env.get("eval"), self.actor.model
        return {"obs_dim": pol.obs_dim, "action_dim": pol.action_dim, "num_action_chunks": pol.num_action_chunks,
                "value_dim": pol.value_dim, "world_size": self.world_size, "total_num_envs": int(et.total_num_envs),
                "max_steps_per_rollout_epoch": int(self.T), "rollout_epoch": int(et.get("rollout_epoch", 1)),
                "eval_total_num_envs": int(ev.total_num_envs) if ev is not None else 0}

    def _barrier(self):
        if self.world_size > 1:
            dist.barrier(group=self._pg)

    def save_checkpoint(self, path=None) -> str:
        """Save everything an exact resume needs (checkpoint.py has the layout) to `path`, by default
        checkpoints/global_step_{global_step} under runner.logger; returns the directory.  Call it on every rank.
        One device synchronisation: all device tensors are copied to pinned host memory, then the stream is waited on."""
        path = path or ckpt.checkpoint_dir(self.cfg.runner, self.global_step)
        pol = self.actor.model
        rank_state = {"global_step": int(self.global_step), "env": self.env.state_dict(),
                      "rollout": self.rollout.state_dict()}
        if self.eval_env is not None:
            rank_state["eval_env"] = self.eval_env.state_dict()
        tree = {"rank": rank_state, "grads_nonzero": torch.count_nonzero(pol.flat_grads)}
        if self.rank == 0:
            tree["weights"] = dict(pol.named_parameters())
            tree["trainer"] = {"actor": self.actor.state_dict(), "fingerprint": self.fingerprint()}
        host = ckpt.to_host(tree)
        torch.cuda.current_stream().synchronize()
        # run_training ends with zero_grad: no gradient is carried between iterations
        assert int(host["grads_nonzero"]) == 0, "save_checkpoint() between iterations only: gradients are not zero"
        return ckpt.write(path, self.rank, host["rank"], host.get("weights"), host.get("trainer"), self._barrier)

    def load_checkpoint(self, path) -> None:
        """Restore a checkpoint written by save_checkpoint() at the same world size, env count and shapes; the next
        iteration continues exactly where the saved run left off.  Everything is copied into the existing tensors, so
        captured rollout, evaluation and optimiser-step graphs stay valid."""
        path = str(path)
        step = ckpt.step_from_path(path)
        weights, trainer, rank_state = ckpt.read(path, self.rank)
        ckpt.check_fingerprint(trainer["fingerprint"], self.fingerprint())
        if int(rank_state["global_step"]) != step:
            raise ValueError(f"{path} names step {step} but holds the state of step {rank_state['global_step']}")
        self.actor.model.load_state_dict(weights, strict=True)
        self.actor.load_state_dict(trainer["actor"])  # also refreshes the weight split and the frozen groups
        self.env.load_state_dict(rank_state["env"])
        self.rollout.load_state_dict(rank_state["rollout"])
        if self.eval_env is not None:
            self.eval_env.load_state_dict(rank_state["eval_env"])
        self.global_step = step
