"""Checkpoint layout, config fingerprint and file I/O of EmbodiedRunner.

What is saved is decided by the owners (`MLPPolicy`, `EmbodiedActor`, `SyntheticVectorEnv`, `RolloutWorker` each
provide `state_dict()` / `load_state_dict()`); this module only knows where it goes:

    {runner.logger.log_path}/{runner.logger.experiment_name}/checkpoints/global_step_{N}/
        actor/model_state_dict/full_weights.pt   {name: CPU fp32 tensor}, the reference's file (rank 0)
        actor/trainer_state.pt                   optimiser, LR schedule, critic warm-up, fingerprint (rank 0)
        rank_{r}/runner_state.pt                 global_step, env and rollout state of rank r (every rank)

The directory layout and the `global_step_{N}` naming follow the reference (embodied_runner.py:644-653,
hybrid_engines/fsdp/strategy/base.py:250-263).  Every file loads with `torch.load(..., weights_only=True)`.  A save
writes into a temporary sibling directory that is renamed only after every rank has written, so an interrupted save
never leaves a partial checkpoint under the final name.
"""
from __future__ import annotations

import os
import shutil
from typing import Callable, Optional

import torch

STEP_PREFIX = "global_step_"
WEIGHTS_FILE = os.path.join("actor", "model_state_dict", "full_weights.pt")
TRAINER_FILE = os.path.join("actor", "trainer_state.pt")
RANK_FILE = "runner_state.pt"

# fields of the fingerprint; a resume into a runner whose values differ is refused
FINGERPRINT_FIELDS = ("obs_dim", "action_dim", "num_action_chunks", "value_dim", "world_size", "total_num_envs",
                      "max_steps_per_rollout_epoch", "rollout_epoch", "eval_total_num_envs")


def checkpoint_dir(runner_cfg, step: int) -> str:
    """`{logger.log_path}/{logger.experiment_name}/checkpoints/global_step_{step}` (EmbodiedRunner._save_checkpoint)."""
    lg = runner_cfg.get("logger") or {}
    missing = [k for k in ("log_path", "experiment_name") if lg.get(k) is None]
    if missing:
        raise ValueError(f"saving checkpoints needs runner.logger.{' and runner.logger.'.join(missing)}")
    return os.path.join(str(lg["log_path"]), str(lg["experiment_name"]), "checkpoints", f"{STEP_PREFIX}{int(step)}")


def step_from_path(path: str) -> int:
    """The global step a checkpoint directory names: `path.split("global_step_")[-1]`, as the reference's resume
    reads it (embodied_runner.py:185); a trailing separator is ignored."""
    tail = os.path.normpath(str(path)).split(STEP_PREFIX)[-1]
    try:
        return int(tail)
    except ValueError:
        raise ValueError(f"checkpoint directory {path!r} is not named {STEP_PREFIX}<step>") from None


def rank_dir(path: str, rank: int) -> str:
    return os.path.join(path, f"rank_{int(rank)}")


def check_fingerprint(saved: dict, current: dict) -> None:
    """Raise ValueError naming the first field whose saved value differs from this runner's."""
    for k in FINGERPRINT_FIELDS:
        if saved.get(k) != current.get(k):
            raise ValueError(f"checkpoint does not match this run: {k} is {saved.get(k)!r} in the checkpoint and "
                             f"{current.get(k)!r} here")


def to_host(tree):
    """Device tensors of a nested dict copied to (pinned) host memory without waiting; the caller synchronises once."""
    if isinstance(tree, dict):
        return {k: to_host(v) for k, v in tree.items()}
    if isinstance(tree, torch.Tensor) and tree.device.type == "cuda":
        out = torch.empty(tree.shape, dtype=tree.dtype, pin_memory=True)
        out.copy_(tree, non_blocking=True)
        return out
    if isinstance(tree, torch.Tensor):
        return tree.clone()
    return tree


def write(path: str, rank: int, rank_state: dict, weights: Optional[dict] = None, trainer: Optional[dict] = None,
          barrier: Callable[[], None] = lambda: None) -> str:
    """Write one rank's share of a checkpoint (host tensors) to `path`.  Every rank calls this with the same `path`;
    rank 0 also passes `weights` and `trainer`.  `barrier` synchronises the ranks (a no-op with one rank)."""
    path = os.path.normpath(str(path))
    parent, name = os.path.split(path)
    tmp = os.path.join(parent, f".{name}.tmp")
    if rank == 0:
        shutil.rmtree(tmp, ignore_errors=True)  # left over from an interrupted save
        os.makedirs(tmp)
    barrier()
    os.makedirs(rank_dir(tmp, rank), exist_ok=True)
    torch.save(rank_state, os.path.join(rank_dir(tmp, rank), RANK_FILE))
    if rank == 0:
        os.makedirs(os.path.dirname(os.path.join(tmp, WEIGHTS_FILE)), exist_ok=True)
        torch.save(weights, os.path.join(tmp, WEIGHTS_FILE))
        torch.save(trainer, os.path.join(tmp, TRAINER_FILE))
    barrier()
    if rank == 0:
        if os.path.isdir(path):  # the reference overwrites a checkpoint of the same step
            shutil.rmtree(path)
        os.replace(tmp, path)
    barrier()
    return path


def _load(path: str):
    return torch.load(path, map_location="cpu", weights_only=True)


def read(path: str, rank: int) -> tuple[dict, dict, dict]:
    """(full weights, trainer state, this rank's state) of the checkpoint at `path`."""
    rfile = os.path.join(rank_dir(path, rank), RANK_FILE)
    if not os.path.isfile(rfile):
        raise ValueError(f"{path} holds no runner state for rank {rank} ({rfile} is missing), so training cannot "
                         f"resume from it; to start from its policy weights only, set runner.ckpt_path to "
                         f"{os.path.join(path, WEIGHTS_FILE)}")
    return _load(os.path.join(path, WEIGHTS_FILE)), _load(os.path.join(path, TRAINER_FILE)), _load(rfile)


def load_weights(path: str) -> dict:
    """A `{name: tensor}` policy state dict (runner.ckpt_path)."""
    return _load(str(path))
