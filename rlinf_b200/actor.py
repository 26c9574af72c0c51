"""Actor (learner) for the embodied PPO/GRPO path - host-side mirror of EmbodiedFSDPActor.

Reference: rlinf/workers/actor/embodied_fsdp_actor_worker.py - `recv_rollout_trajectories` (:187),
`_process_received_rollout_batch` (:209-284), `compute_advantages_and_returns` (:287-321),
`run_training` (:484-589: seeded randperm shuffle :511-518, update_epoch / global-batch / micro-batch
loops :529-571, lr step, metric reduction :573-589), `train_micro_batch` (:591-699).
Same method names, same config keys, same metric keys; the arithmetic is librlinf_b200.so:
one process per GPU, data-parallel over environments, ONE NCCL all-reduce on the flat gradient buffer
per optimiser step (FSDP no_shard semantics: gradients averaged over ranks).
"""
from __future__ import annotations

from typing import Optional

import numpy as np
import torch
import torch.distributed as dist

from . import _lib as L
from . import dist_utils as D
from . import ops
from .algorithms import calculate_adv_and_returns
from .config import wrap
from .lr_scheduler import LRSchedule
from .policy import FlatAdamW, MLPPolicy

EV_KEY = "critic/explained_variance"
_T_PLUS_ONE_KEYS = ("dones", "terminations", "truncations", "prev_values")


def process_nested_dict_for_adv(nested, rollout_epoch):
    """[E*nc, B, ...] -> [nc, E*B, ...] (rlinf/utils/nested_dict_process.py:251-269); views/reshapes only."""
    out = {}
    for k, v in nested.items():
        if isinstance(v, dict):
            out[k] = process_nested_dict_for_adv(v, rollout_epoch)
        elif isinstance(v, torch.Tensor):
            x = v.reshape(rollout_epoch, -1, *v.shape[1:]).transpose(0, 1)
            out[k] = x.reshape(x.shape[0], -1, *x.shape[3:])
    return out


def process_nested_dict_for_train(nested, shuffle_id):
    """Drop the bootstrap row of the T+1-row tensors, flatten [T,B,..] -> [T*B,..] (row t*B+b) and gather by
    `shuffle_id` with the row-gather kernel (rlinf/utils/nested_dict_process.py:272-285)."""
    out = {}
    for k, v in nested.items():
        if v is None:
            out[k] = None
        elif isinstance(v, dict):
            out[k] = process_nested_dict_for_train(v, shuffle_id)
        elif isinstance(v, torch.Tensor):
            if k in _T_PLUS_ONE_KEYS:
                v = v[:-1]
            flat = v.reshape(-1, *v.shape[2:])
            if any(s == 0 for s in flat.stride()) and flat.numel() > 1:
                flat = flat.contiguous()  # expanded view (loss_mask_sum)
            as_bool = flat.dtype == torch.bool
            src = flat.contiguous()
            res = ops.gather_rows(src.view(torch.uint8) if as_bool else src, shuffle_id)
            out[k] = res.view(torch.bool) if as_bool else res
    return out


class EmbodiedActor:
    def __init__(self, cfg, policy: Optional[MLPPolicy] = None, rank: Optional[int] = None,
                 world_size: Optional[int] = None, process_group=None):
        self.cfg = wrap(cfg)
        self.pg = process_group
        self._dist = dist.is_available() and dist.is_initialized()
        self._rank = rank if rank is not None else (dist.get_rank() if self._dist else 0)
        self._world_size = world_size if world_size is not None else (dist.get_world_size() if self._dist else 1)
        m = self.cfg.actor.model
        self.device = L.default_device()
        self.model = policy or MLPPolicy(m.obs_dim, m.action_dim, m.get("num_action_chunks", 1),
                                         add_value_head=m.get("add_value_head", True), device=self.device,
                                         seed=self.cfg.actor.seed)
        o = self.cfg.actor.optim
        self.optimizer = FlatAdamW(self.model, lr=o.lr, value_lr=o.get("value_lr", o.lr),
                                   betas=(o.get("adam_beta1", 0.9), o.get("adam_beta2", 0.999)),
                                   eps=o.get("adam_eps", 1e-8), weight_decay=o.get("weight_decay", 1e-2),
                                   clip_grad=o.get("clip_grad", 1.0))
        self.optimizer_steps = 0
        # critic warm-up (fsdp_model_manager.py:88-93, 304-310, 451-459): for the first `critic_warmup_steps` optimiser
        # steps only the value head is optimised (actor parameters frozen: no update, no weight decay, no moments),
        # lr_list reports 0.0; then optimiser AND lr scheduler are rebuilt (fresh moments / step count / schedule)
        self.critic_warmup_steps = int(o.get("critic_warmup_steps", 0) or 0) if self.model.value_dim > 0 else 0
        self._with_critic = self.cfg.algorithm.adv_type == "gae"
        self._set_frozen_groups()
        self.lr_schedule = LRSchedule(o, base_lr=o.lr)
        self.optimizer.lr_scale = self.lr_schedule.multiplier()
        self.rollout_batch: dict = {}
        self._perm_cache: dict = {}
        self.version = 0
        # actor.cuda_graph_update: replay one CUDA graph per optimiser step instead of ~35 ctypes launches
        self._graph_update = self.cfg.actor.get("cuda_graph_update", False)  # True / False / "auto"
        # Multi-rank graphed steps are EXPERIMENTAL and off unless actor.cuda_graph_multi_rank is set.
        self._graph_multi_rank = bool(self.cfg.actor.get("cuda_graph_multi_rank", False))
        self._capture_nccl = bool(self.cfg.actor.get("cuda_graph_capture_nccl", True))
        self._static_batch: dict = {}
        self._step_graphs: dict = {}
        self._train_calls = 0

    # ---- rollout intake ---------------------------------------------------------------------------
    def recv_rollout_trajectories(self, batch: dict) -> None:
        """Take a rollout batch (device tensors from the on-device rollout buffer, or HOST tensors as the
        reference's channel delivers them - those are copied H2D here, once)."""
        def to_dev(d):
            return {k: (to_dev(v) if isinstance(v, dict) else L.to_device(v, self.device)) for k, v in d.items()
                    if v is not None}

        self.rollout_batch = self._process_received_rollout_batch(to_dev(batch))

    def _process_received_rollout_batch(self, rollout_batch: dict) -> dict:
        cfg = self.cfg
        rollout_epoch = cfg.env.train.get("rollout_epoch", 1)
        if rollout_epoch != 1:
            rollout_batch = process_nested_dict_for_adv(rollout_batch, rollout_epoch)
        if not cfg.env.train.auto_reset and not cfg.env.train.get("ignore_terminations", False):
            loss_mask, loss_mask_sum = ops.loss_mask(rollout_batch["dones"])
            if cfg.algorithm.reward_type == "chunk_level":
                loss_mask = loss_mask.any(dim=-1, keepdim=True)
                loss_mask_sum = loss_mask_sum[..., -1:]
            rollout_batch["loss_mask"] = loss_mask
            rollout_batch["loss_mask_sum"] = loss_mask_sum
        if cfg.algorithm.get("filter_rewards", False):
            rollout_batch["loss_mask"] = ops.reward_filter(
                rollout_batch["rewards"], rollout_batch.get("loss_mask", None), cfg.algorithm.group_size,
                cfg.algorithm.rewards_lower_bound, cfg.algorithm.rewards_upper_bound)
        return rollout_batch

    # ---- advantages -------------------------------------------------------------------------------
    def compute_advantages_and_returns(self) -> dict:
        cfg, rb = self.cfg, self.rollout_batch
        kwargs = {
            "task_type": cfg.runner.task_type, "adv_type": cfg.algorithm.adv_type, "rewards": rb["rewards"],
            "dones": rb["dones"], "values": rb.get("prev_values", None), "prev_logprobs": rb.get("prev_logprobs", None),
            "teacher_logprobs": None, "num_action_chunks": cfg.actor.model.get("num_action_chunks", 1),
            "gamma": cfg.algorithm.get("gamma", 1), "gae_lambda": cfg.algorithm.get("gae_lambda", 1),
            "group_size": cfg.algorithm.get("group_size", 8), "reward_type": cfg.algorithm.reward_type,
            "loss_mask": rb.get("loss_mask", None), "loss_mask_sum": rb.get("loss_mask_sum", None),
            "advantage_mode": cfg.algorithm.get("advantage_mode", None),
        }
        rb.update(calculate_adv_and_returns(**kwargs))
        if not cfg.runner.get("rollout_metrics", True):
            return {}
        from .metric_utils import compute_rollout_metrics

        return compute_rollout_metrics(rb, self._world_size, self.pg)

    # ---- training ---------------------------------------------------------------------------------
    def _shuffle_id(self, n: int) -> torch.Tensor:
        """torch.randperm(n, generator=CPU mt19937 seeded actor.seed + rank) - the reference re-seeds
        identically at every run_training call (embodied_fsdp_actor_worker.py:511-513), so the permutation
        is computed once per size and cached on the device."""
        key = (n, self.cfg.actor.seed + self._rank)
        if key not in self._perm_cache:
            g = torch.Generator()
            g.manual_seed(D.shuffle_seed(self.cfg.actor.seed, self._rank))
            self._perm_cache[key] = torch.randperm(n, generator=g).to(self.device)
        return self._perm_cache[key]

    def run_training(self) -> dict:
        cfg = self.cfg
        rb = self.rollout_batch
        rollout_size = rb["prev_logprobs"].shape[0] * rb["prev_logprobs"].shape[1]
        shuffle_id = self._shuffle_id(rollout_size)
        batch = process_nested_dict_for_train(rb, shuffle_id)
        self.rollout_batch = batch
        mbs = cfg.actor.micro_batch_size
        batch_size_per_rank, self.gradient_accumulation, n_global = D.per_rank_batch(
            cfg.actor.global_batch_size, self._world_size, mbs, rollout_size)
        update_epoch = cfg.algorithm.get("update_epoch", 1)
        n_steps = update_epoch * n_global
        n_micro = n_steps * self.gradient_accumulation
        metric_rows = torch.zeros(n_micro, L.NUM_METRICS, dtype=torch.float32, device=self.device)
        step_rows = torch.zeros(n_steps, 4, dtype=torch.float64, device=self.device)
        lr_rows = []
        mi = si = 0
        use_graph = self._graph_update
        if use_graph == "auto":  # small per-rank mini-batches: the step is short enough for launch gaps to matter
            use_graph = batch_size_per_rank <= 65536
        if self._world_size > 1 and not self._graph_multi_rank:
            use_graph = False
        graphed = bool(use_graph) and self._train_calls > 0  # the first call runs eagerly (lazy initialisation)
        self._train_calls += 1
        if graphed:
            batch = self._persist_batch(batch)
            self.rollout_batch = batch
        for _ in range(update_epoch):
            for gb in range(n_global):
                if graphed:
                    lr_rows.append(self._graphed_step(batch, gb, batch_size_per_rank, mbs,
                                                      metric_rows[mi: mi + self.gradient_accumulation], step_rows[si]))
                    mi += self.gradient_accumulation
                    si += 1
                    continue
                self.optimizer.zero_grad()
                for k in range(self.gradient_accumulation):
                    lo = gb * batch_size_per_rank + k * mbs
                    self.train_micro_batch(batch, lo, lo + mbs, metric_rows[mi])
                    mi += 1
                grad_norm_state, lr_list = self.optimizer_step()
                step_rows[si].copy_(grad_norm_state)
                lr_rows.append(lr_list)
                si += 1
        self.optimizer.lr_scale = self.lr_schedule.step()  # "put LR scheduler step here" (:571)
        self.optimizer.zero_grad()
        return self._reduce_metrics(metric_rows, step_rows, lr_rows)

    # ---- experimental: CUDA-graphed optimiser step -------------------------------------------------
    def _persist_batch(self, batch: dict, prefix: str = "") -> dict:
        """Copy the shuffled training batch into buffers with stable addresses (graphs bake pointers)."""
        out = {}
        for k, v in batch.items():
            key = prefix + k
            if isinstance(v, dict):
                out[k] = self._persist_batch(v, key + "/")
            elif isinstance(v, torch.Tensor):
                buf = self._static_batch.get(key)
                if buf is None or buf.shape != v.shape or buf.dtype != v.dtype:
                    buf = torch.empty_like(v)
                    self._static_batch[key] = buf
                    self._step_graphs.clear()  # addresses changed
                buf.copy_(v)
                out[k] = buf
            else:
                out[k] = v
        return out

    def _graphed_step(self, batch, gb, batch_size_per_rank, mbs, metric_out, state_out):
        """One optimiser step as CUDA-graph replays: zero_grad + micro-batches + gradient all-reduce + clip + AdamW in ONE
        graph when the NCCL all-reduce can be captured (torch.distributed supports capture of NCCL collectives), else
        graph A | eager all-reduce | graph B.  Learning rates / frozen groups are read from a device table, so LR
        schedules and the end of critic warm-up do not force a re-capture of the optimiser node."""
        warm = self.optimizer_steps < self.critic_warmup_steps
        accum = self.gradient_accumulation
        key = (gb, warm, accum, mbs, batch_size_per_rank, self._world_size)
        self.optimizer.sync_lr_table()  # outside capture: replays read the device copy
        entry = self._step_graphs.get(key)
        if entry is None:
            stage_m = torch.zeros(accum, L.NUM_METRICS, dtype=torch.float32, device=self.device)
            stage_s = torch.zeros(4, dtype=torch.float64, device=self.device)
            scale = 1.0 / self._world_size

            def fwd_bwd():
                self.optimizer.zero_grad()
                for k in range(accum):
                    lo = gb * batch_size_per_rank + k * mbs
                    self.train_micro_batch(batch, lo, lo + mbs, stage_m[k])

            def opt():
                self.optimizer.step(grad_scale=scale)
                stage_s.copy_(self.optimizer.state)

            graphs = None
            if self._world_size > 1 and self._capture_nccl:
                try:
                    torch.cuda.synchronize()
                    self.model.mark_params_changed()  # the weight-split refresh must be part of the graph
                    g_all = torch.cuda.CUDAGraph()
                    with torch.cuda.graph(g_all):
                        fwd_bwd()
                        dist.all_reduce(self.model.flat_grads, op=dist.ReduceOp.SUM, group=self.pg)
                        opt()
                    graphs = (g_all, None)
                except Exception as e:  # pragma: no cover - depends on the NCCL / torch build
                    self._capture_nccl = False
                    self._capture_nccl_error = repr(e)
                    torch.cuda.synchronize()
            if graphs is None:
                torch.cuda.synchronize()
                self.model.mark_params_changed()
                g_a = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g_a):
                    fwd_bwd()
                g_b = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g_b, pool=g_a.pool()):
                    opt()
                graphs = (g_a, g_b)
            entry = (graphs, stage_m, stage_s)
            self._step_graphs[key] = entry
        (g_a, g_b), stage_m, stage_s = entry
        g_a.replay()
        self.optimizer_steps += 1
        if g_b is not None:
            D.allreduce_flat_grads(self.model.flat_grads, self._world_size, self.pg)
            g_b.replay()
        self.model.mark_params_changed()
        metric_out.copy_(stage_m)
        state_out.copy_(stage_s)
        return self._after_optimizer_step()

    def train_micro_batch(self, batch, lo, hi, metric_out) -> None:
        cfg = self.cfg
        fi = batch["forward_inputs"]
        with_critic = self._with_critic
        ent_bonus = float(cfg.algorithm.get("entropy_bonus", 0) or 0)
        warm = self.optimizer_steps < self.critic_warmup_steps
        out = self.model.forward_train(fi["states"][lo:hi], fi["action"][lo:hi], compute_entropy=ent_bonus > 0,
                                       compute_values=with_critic)
        A = cfg.actor.model.get("action_dim", 7)
        Cc = out["logprobs"].shape[1] // A
        U = 1 if cfg.algorithm.logprob_type == "chunk_level" else Cc
        n = hi - lo

        def unit(key):
            t = batch.get(key)
            return None if t is None else t[lo:hi].reshape(n, U)

        loss, metrics, d_lp, d_v, d_e = ops.ppo_loss(
            logprobs=out["logprobs"], values=out.get("values") if with_critic else None,
            entropy=out.get("entropy"), old_logprobs=batch["prev_logprobs"][lo:hi].reshape(n, Cc * A),
            advantages=unit("advantages"), returns=unit("returns") if with_critic else None,
            prev_values=unit("prev_values") if with_critic else None, loss_mask=unit("loss_mask"),
            loss_mask_sum=unit("loss_mask_sum"), C_chunks=Cc, A_dim=A, logprob_type=cfg.algorithm.logprob_type,
            clip_ratio_low=cfg.algorithm.clip_ratio_low, clip_ratio_high=cfg.algorithm.clip_ratio_high,
            value_clip=cfg.algorithm.get("value_clip", None), huber_delta=cfg.algorithm.get("huber_delta", None),
            max_episode_steps=cfg.env.train.max_episode_steps if batch.get("loss_mask_sum") is not None else None,
            critic_warmup=warm, entropy_bonus=ent_bonus, loss_scale=1.0 / self.gradient_accumulation)
        metric_out.copy_(metrics)
        self.model.backward(d_lp, d_v if with_critic else None, d_e)

    def _set_frozen_groups(self):
        frozen = set()
        if self.critic_warmup_steps > 0:
            frozen.add("actor")
        if not self._with_critic:
            # the value head receives no gradient (compute_values=False): torch.optim.AdamW skips parameters whose
            # grad is None - no decay, no moment update
            frozen.add("critic")
        self.optimizer.frozen = frozen

    def _after_optimizer_step(self):
        """Bookkeeping of FSDPModelManager.optimizer_step after the step itself (:451-463): returns lr_list."""
        if self.critic_warmup_steps > 0:
            lr_list = [0.0 for _ in self.optimizer.lr_list()]
            if self.optimizer_steps >= self.critic_warmup_steps:
                self.critic_warmup_steps = 0
                self._set_frozen_groups()
                self.optimizer.reset_state(carry_grads=True)
                self.lr_schedule = LRSchedule(self.cfg.actor.optim, base_lr=self.cfg.actor.optim.lr)
                self.optimizer.lr_scale = self.lr_schedule.multiplier()
            return lr_list
        return self.optimizer.lr_list()

    def optimizer_step(self):
        """all-reduce(SUM) of the flat gradient buffer over the data-parallel ranks, then one fused
        norm / clip / AdamW pass that also applies the 1/world_size average."""
        self.optimizer_steps += 1
        scale = D.allreduce_flat_grads(self.model.flat_grads, self._world_size, self.pg)
        self.optimizer.step(grad_scale=scale)
        state = self.optimizer.state.clone()
        return state, self._after_optimizer_step()

    def _reduce_metrics(self, metric_rows, step_rows, lr_rows) -> dict:
        """np.mean over micro-batches, AVG all-reduce over ranks, explained variance from SUM-reduced
        sufficient statistics (embodied_fsdp_actor_worker.py:573-589). One device->host copy."""
        with_critic = self.cfg.algorithm.adv_type == "gae"
        mean_vec = metric_rows.mean(dim=0)
        ev_sum = metric_rows[:, 10:15].sum(dim=0)
        grad_norm = step_rows[:, 1].mean().to(torch.float32)
        packed = D.reduce_metric_pack(mean_vec, ev_sum, grad_norm, self._world_size, self.pg)
        host = packed.tolist()
        out = {}
        slots = L.ACTOR_SLOTS + ((8, 9) if with_critic else ()) + (15, 16)
        for s in slots:
            out[L.M_KEYS[s]] = host[s]
        out["actor/grad_norm"] = host[-1]
        out["actor/lr"] = float(np.mean([r[0] for r in lr_rows]))
        second = [r[1] for r in lr_rows if len(r) > 1]  # absent while the warm-up optimiser has one param group
        if second:
            out["critic/lr"] = float(np.mean(second))
        if with_critic:
            cnt, rs, rss, es, ess = host[L.NUM_METRICS: L.NUM_METRICS + 5]
            ev = float("nan")
            if cnt >= 2:
                rc = rss - rs * rs / cnt
                ec = ess - es * es / cnt
                if rc == rc and rc != 0 and ec == ec:
                    ev = 1 - ec / rc
            out[EV_KEY] = ev
        return out

    # ---- weight sync ------------------------------------------------------------------------------
    def sync_model_to_rollout(self, rollout_params: Optional[torch.Tensor] = None, src: int = 0):
        """Actor -> rollout replica parameter hand-off (embodied_fsdp_actor_worker.py:132-154). With one
        process per GPU holding both roles the rollout policy reads the SAME flat buffer (no-op); a
        separate replica buffer gets a device copy; across ranks one NCCL broadcast of the flat buffer."""
        if rollout_params is not None and rollout_params.data_ptr() != self.model.flat_params.data_ptr():
            rollout_params.copy_(self.model.flat_params)
        if self.cfg.runner.get("broadcast_params", True):
            from .weight_sync import broadcast_flat

            self.rollout_version = broadcast_flat(self.model, self.version, src, self.pg)
        self.model.mark_params_changed()
