"""Registered policy losses (CUDA-backed), surface of rlinf/algorithms/losses.py.

`compute_ppo_actor_critic_loss` ("actor_critic", losses.py:396-424) and `compute_grpo_actor_loss_fn`
("actor", :508-535) take the kwargs produced by preprocess_loss_inputs (so they can be dropped into
the REFERENCE's own LOSS_REGISTRY); `fused_embodied_policy_loss` is what this package's `policy_loss`
uses for the embodied task type: it skips the torch-side reduction and hands the raw [bsz, C*A]
log-probs to the kernel.  Either way: one fused forward+backward kernel group, gradients delivered to
autograd through a Function whose backward only rescales the stored gradients.
"""
from __future__ import annotations

from typing import Optional

import torch

from .. import _lib as L
from .. import ops
from .registry import register_policy_loss

_HP_KEYS = ("clip_ratio_low", "clip_ratio_high", "clip_ratio_c", "clip_log_ratio_min", "clip_log_ratio_max",
            "value_clip", "huber_delta", "max_episode_steps", "critic_warmup")


class _FusedPpoLoss(torch.autograd.Function):
    """forward: launch the fused kernel (loss, metrics AND gradients); backward: grads x upstream scalar."""

    @staticmethod
    def forward(ctx, logprobs, values, entropy, cfg):
        cfg = dict(cfg)
        loss, metrics, d_lp, d_v, d_e = ops.ppo_loss(
            logprobs=logprobs.detach(), values=None if values is None else values.detach(),
            entropy=None if entropy is None else entropy.detach(), want_grads=True, **cfg)
        ctx.grads = (d_lp, d_v, d_e)
        ctx.shapes = (logprobs.shape, None if values is None else values.shape,
                      None if entropy is None else entropy.shape)
        ctx.mark_non_differentiable(metrics)
        return loss.reshape(()), metrics

    @staticmethod
    def backward(ctx, g_loss, _g_metrics):
        d_lp, d_v, d_e = ctx.grads
        ctx.grads = None
        outs = []
        for g, shp in zip((d_lp, d_v, d_e), ctx.shapes):
            if g is None or shp is None:
                outs.append(None)
            else:
                outs.append(ops.scale_by_(g, g_loss).view(shp))
        return outs[0], outs[1], outs[2], None


def _check_fp32(**named):
    for k, v in named.items():
        if v is not None and v.dtype != torch.float32:
            raise AssertionError(f"{k} must be float32 to keep numerical stability")  # losses.py:232-240


def _metrics_dict(metrics: torch.Tensor, with_critic: bool, as_float: bool) -> dict:
    slots = L.ACTOR_SLOTS + (L.CRITIC_SLOTS if with_critic else ())
    if as_float:
        host = metrics.tolist()  # ONE device->host copy for all metrics
        return {L.M_KEYS[s]: host[s] for s in slots}
    return {L.M_KEYS[s]: metrics[s] for s in slots}


def _decoupled_metrics_dict(metrics: torch.Tensor, as_float: bool) -> dict:
    host = metrics.tolist() if as_float else None
    get = (lambda s: host[s]) if as_float else (lambda s: metrics[s])
    out = {k: get(s) for s, k in L.DM_KEYS.items()}
    has_ver = (host[19] if as_float else float(metrics[19])) != 0
    if has_ver:
        out["actor/average_version"] = get(15)
        out["actor/current_version"] = get(18)
    return out


def preprocess_loss_inputs(logprobs, old_logprobs, advantages, logprob_type=None, single_action_dim=None,
                           loss_mask=None, loss_mask_sum=None, values=None, prev_values=None, returns=None,
                           reward_type=None, versions=None, **kwargs) -> dict:
    """rlinf/algorithms/utils.py:280-376 for loss functions a USER registers (the built-in entries never come here:
    their reduction happens inside the fused kernels).  Layout work only - reshapes, the per-action / per-chunk sums
    that carry autograd history, trailing-dimension expansion."""
    def flat(t):
        return None if t is None else t.flatten()

    def rank_up(t, shape):
        if t is None:
            return None
        while t.dim() < len(shape) and t.shape != shape:
            t = t.unsqueeze(-1)
        return t

    if reward_type == "chunk_level":
        advantages, loss_mask, loss_mask_sum = flat(advantages), flat(loss_mask), flat(loss_mask_sum)
        values, prev_values, returns = flat(values), flat(prev_values), flat(returns)
    bsz = logprobs.shape[0]
    proximal = kwargs.get("proximal_logprobs", None)
    A = single_action_dim

    def per(t):
        return None if t is None else t.reshape(bsz, -1, A)

    if logprob_type == "token_level":
        logprobs, old_logprobs, proximal, versions = per(logprobs), per(old_logprobs), per(proximal), per(versions)
        if kwargs.get("loss_type") == "opd":
            assert advantages.shape == logprobs.shape, (
                f"OPD advantages shape {advantages.shape} must match logprobs shape {logprobs.shape}.")
        else:
            advantages = advantages.unsqueeze(-1)
        loss_mask = None if loss_mask is None else loss_mask.unsqueeze(-1)
        loss_mask_sum = None if loss_mask_sum is None else loss_mask_sum.unsqueeze(-1)
    elif logprob_type == "action_level":
        logprobs, old_logprobs = per(logprobs).sum(dim=-1), per(old_logprobs).sum(dim=-1)
        proximal = None if proximal is None else per(proximal).sum(dim=-1)
        versions = None if versions is None else per(versions)[..., 0]
    elif logprob_type == "chunk_level":
        logprobs, old_logprobs = per(logprobs).sum(dim=[1, 2]), per(old_logprobs).sum(dim=[1, 2])
        proximal = None if proximal is None else per(proximal).sum(dim=[1, 2])
        versions = None if versions is None else per(versions)[:, 0, 0]
    shape = logprobs.shape
    kwargs.update({
        "logprobs": logprobs, "old_logprobs": old_logprobs, "proximal_logprobs": proximal,
        "versions": rank_up(versions, shape), "advantages": rank_up(advantages, shape),
        "loss_mask": rank_up(loss_mask, shape), "loss_mask_sum": rank_up(loss_mask_sum, shape),
        "values": rank_up(values, shape), "prev_values": rank_up(prev_values, shape), "returns": rank_up(returns, shape),
        "logprob_type": logprob_type, "single_action_dim": single_action_dim, "reward_type": reward_type,
    })
    return kwargs


def postprocess_loss_metric(metrics_data: dict) -> dict:
    """rlinf/algorithms/utils.py:379-385."""
    for k, v in metrics_data.items():
        if isinstance(v, torch.Tensor):
            metrics_data[k] = v.detach().item()
    return metrics_data


def _run(logprobs, values, entropy, cfg, with_critic, as_float, decoupled=False):
    needs_grad = torch.is_grad_enabled() and (
        logprobs.requires_grad or (values is not None and values.requires_grad)
        or (entropy is not None and entropy.requires_grad))
    if needs_grad:
        loss, metrics = _FusedPpoLoss.apply(logprobs, values, entropy, cfg)
    else:
        loss, metrics, *_ = ops.ppo_loss(logprobs=logprobs.detach(), values=None if values is None else values.detach(),
                                         entropy=entropy, want_grads=False, **cfg)
        loss = loss.reshape(())
    if decoupled:
        return loss, _decoupled_metrics_dict(metrics, as_float), metrics
    return loss, _metrics_dict(metrics, with_critic, as_float), metrics


def fused_embodied_policy_loss(**kwargs):
    """policy_loss for task_type == "embodied" (registry.py:77-92 + utils.py:280-376 fused).
    kwargs are the ones EmbodiedFSDPActor.train_micro_batch builds
    (workers/actor/embodied_fsdp_actor_worker.py:642-676)."""
    loss_type = kwargs["loss_type"]
    logprobs = kwargs["logprobs"]
    dev = logprobs.device if logprobs.is_cuda else L.default_device()
    logprobs = logprobs if logprobs.is_cuda else logprobs.to(dev)
    decoupled = loss_type == "decoupled_actor_critic"
    with_critic = loss_type in ("actor_critic", "decoupled_actor_critic")
    values = kwargs.get("values") if with_critic else None
    _check_fp32(logprobs=logprobs, old_logprobs=kwargs["old_logprobs"], advantages=kwargs["advantages"])
    A = int(kwargs.get("single_action_dim") or logprobs.shape[-1])
    bsz = logprobs.shape[0]
    total = logprobs[0].numel()
    if total % A != 0:
        raise RuntimeError(f"logprobs row of {total} entries is not a multiple of single_action_dim={A}")
    Cc = total // A
    logprob_type = kwargs.get("logprob_type")
    if logprob_type not in L.LOGPROB_TYPES:
        raise ValueError(f"unsupported logprob_type {logprob_type!r}")
    U = 1 if logprob_type == "chunk_level" else Cc

    def per_unit(t, name):
        if t is None:
            return None
        t = L.to_device(t, dev)
        if t.numel() != bsz * U:
            raise RuntimeError(f"{name} has {t.numel()} entries, expected bsz*{U}={bsz * U} "
                               f"(logprob_type={logprob_type}, reward_type={kwargs.get('reward_type')})")
        return t.reshape(bsz, U)

    lms = kwargs.get("loss_mask_sum")
    cfg = dict(
        old_logprobs=L.to_device(kwargs["old_logprobs"], dev).reshape(bsz, Cc * A),
        advantages=per_unit(kwargs["advantages"], "advantages"),
        returns=per_unit(kwargs.get("returns"), "returns") if with_critic else None,
        prev_values=per_unit(kwargs.get("prev_values"), "prev_values") if with_critic else None,
        loss_mask=per_unit(kwargs.get("loss_mask"), "loss_mask"),
        loss_mask_sum=per_unit(lms, "loss_mask_sum"),
        C_chunks=Cc, A_dim=A, logprob_type=logprob_type,
    )
    for k in _HP_KEYS:
        if kwargs.get(k) is not None:
            cfg[k] = kwargs[k]
    if with_critic and values is not None:
        values = values if values.is_cuda else values.to(dev)
        _check_v = per_unit(values.detach(), "values")  # shape check only
        del _check_v
    # Extension kwargs (absent in the reference's call, where the WORKER subtracts the entropy bonus and divides by the
    # gradient accumulation after policy_loss returns - embodied_fsdp_actor_worker.py:678-695): when given, both are
    # folded into the same fused launch and `actor/entropy_loss` / `actor/total_loss` are reported.
    if decoupled:
        def full(t, name):
            if t is None:
                return None
            t = L.to_device(t, dev, torch.float32)
            if t.numel() != bsz * Cc * A:
                raise RuntimeError(f"{name} has {t.numel()} entries, expected {bsz * Cc * A}")
            return t.reshape(bsz, Cc * A)

        cfg["_decoupled"] = dict(proximal_logprobs=full(kwargs.get("proximal_logprobs"), "proximal_logprobs"),
                                 versions=full(kwargs.get("versions"), "versions"),
                                 current_version=kwargs.get("current_version"),
                                 behave_weight_threshold=kwargs.get("behave_weight_threshold"))
        for k in ("clip_log_ratio_min", "clip_log_ratio_max"):
            cfg.pop(k, None)  # compute_decoupled_ppo_actor_loss has no log-ratio clamps (they fall into **kwargs)
    entropy = kwargs.get("entropy")
    ent_bonus = float(kwargs.get("entropy_bonus", 0.0) or 0.0)
    if entropy is not None:
        ent_type = kwargs.get("entropy_type", "action_level")
        want = "chunk_level" if logprob_type == "chunk_level" else "action_level"
        if ent_type != want:
            raise NotImplementedError(f"entropy_type={ent_type!r} with logprob_type={logprob_type!r}: the fused kernel "
                                      f"reduces the entropy over the same unit as the log-probs ({want})")
        entropy = (entropy if entropy.is_cuda else entropy.to(dev)).reshape(bsz, Cc * A)
        cfg["entropy_bonus"] = ent_bonus
    if kwargs.get("loss_scale") is not None:
        cfg["loss_scale"] = float(kwargs["loss_scale"])
    loss, metrics, raw = _run(logprobs.reshape(bsz, Cc * A), None if values is None else values.reshape(bsz, U), entropy,
                              cfg, with_critic, as_float=True, decoupled=decoupled)
    if entropy is not None or kwargs.get("loss_scale") is not None:
        host = raw.tolist()
        metrics["actor/entropy_loss"] = host[L.DM_ENTROPY if decoupled else 15]
        metrics["actor/total_loss"] = host[16]
    return loss, metrics


def _from_preprocessed(kwargs, with_critic):
    """Map the kwargs of preprocess_loss_inputs (already-reduced log-probs) onto kernel arguments."""
    logprobs = kwargs["logprobs"]
    old = kwargs["old_logprobs"]
    adv = kwargs["advantages"]
    _check_fp32(logprobs=logprobs, old_logprobs=old, advantages=adv)
    dev = logprobs.device if logprobs.is_cuda else L.default_device()
    if adv.shape == logprobs.shape or adv.numel() == logprobs.numel():
        g, mode = 1, "action_level"  # one ratio per entry
    elif adv.dim() == logprobs.dim() and adv.shape[-1] == 1:
        g, mode = logprobs.shape[-1], "token_level"
    else:
        raise RuntimeError(f"advantages {tuple(adv.shape)} cannot be matched to logprobs {tuple(logprobs.shape)}")
    n_units = logprobs.numel() // g

    def unit(t):
        if t is None:
            return None
        t = L.to_device(t, dev)
        if t.numel() != n_units:
            t = t.expand(adv.shape)
        return t.reshape(n_units, 1)

    cfg = dict(old_logprobs=L.to_device(old, dev).reshape(n_units, g), advantages=unit(adv),
               returns=unit(kwargs.get("returns")) if with_critic else None,
               prev_values=unit(kwargs.get("prev_values")) if with_critic else None,
               loss_mask=unit(kwargs.get("loss_mask")), loss_mask_sum=unit(kwargs.get("loss_mask_sum")),
               C_chunks=1, A_dim=g, logprob_type=mode)
    for k in _HP_KEYS:
        if kwargs.get(k) is not None:
            cfg[k] = kwargs[k]
    values = kwargs.get("values") if with_critic else None
    lp2 = (logprobs if logprobs.is_cuda else logprobs.to(dev)).reshape(n_units, g)
    v2 = None if values is None else (values if values.is_cuda else values.to(dev)).reshape(n_units, 1)
    return lp2, v2, cfg


@register_policy_loss("actor_critic")
def compute_ppo_actor_critic_loss(**kwargs) -> tuple[torch.Tensor, dict]:
    """PPO actor + critic loss, no value coefficient (losses.py:396-424). Metrics are 0-dim tensors
    (the caller - registry.policy_loss - converts them for the embodied task type)."""
    lp, v, cfg = _from_preprocessed(kwargs, True)
    loss, metrics, _ = _run(lp, v, None, cfg, True, as_float=False)
    return loss, metrics


@register_policy_loss("actor")
def compute_grpo_actor_loss_fn(**kwargs) -> tuple[torch.Tensor, dict]:
    """PPO-clip actor loss for GRPO (losses.py:508-535)."""
    lp, _, cfg = _from_preprocessed(kwargs, False)
    loss, metrics, _ = _run(lp, None, None, cfg, False, as_float=False)
    return loss, metrics


def compute_ppo_actor_loss(**kwargs):
    """losses.py:170-312 - same kernel, actor half only."""
    return compute_grpo_actor_loss_fn(**kwargs)


@register_policy_loss("decoupled_actor_critic")
def compute_decoupled_ppo_actor_critic_loss(**kwargs) -> tuple[torch.Tensor, dict]:
    """Decoupled PPO actor + critic loss (losses.py:27-167, 383-394) on preprocess_loss_inputs kwargs."""
    lp, v, cfg = _from_preprocessed(kwargs, True)
    n_units, g = lp.shape

    def elem(t):
        if t is None:
            return None
        t = L.to_device(t, lp.device, torch.float32)
        if t.numel() == n_units * g:
            return t.reshape(n_units, g)
        if g == 1 or t.numel() != n_units:
            raise RuntimeError(f"cannot match a tensor of {t.numel()} entries to {n_units} x {g} log-probs")
        return t.reshape(n_units, 1).expand(n_units, g).contiguous()

    cfg["_decoupled"] = dict(proximal_logprobs=elem(kwargs.get("proximal_logprobs")), versions=elem(kwargs.get("versions")),
                             current_version=kwargs.get("current_version"),
                             behave_weight_threshold=kwargs.get("behave_weight_threshold"))
    for k in ("clip_log_ratio_min", "clip_log_ratio_max"):
        cfg.pop(k, None)
    loss, metrics, _ = _run(lp, v, None, cfg, True, as_float=False, decoupled=True)
    return loss, metrics


# loss_agg_func of the reasoning workers (get_loss_agg_func, rlinf/utils/utils.py:359-381), matched by function name
_AGG_BY_NAME = {"masked_mean": "token-mean", "seq_mean_token_sum": "seq-mean-token-sum",
                "seq_mean_token_mean": "seq-mean-token-mean"}


def loss_agg_mode(loss_agg_func) -> str:
    """The aggregation a reasoning worker's loss_agg_func selects: None or masked_mean -> "token-mean", the reference's
    seq_mean_token_sum / seq_mean_token_mean by name; a string is one of get_loss_agg_func's names.  Any other callable
    raises ValueError naming what is supported."""
    if loss_agg_func is None:
        return "token-mean"
    if isinstance(loss_agg_func, str):
        if loss_agg_func not in L.AGG_MODES:
            raise ValueError(f"Unsupported loss aggregation method: {loss_agg_func}")
        return loss_agg_func
    mode = _AGG_BY_NAME.get(getattr(loss_agg_func, "__name__", None))
    if mode is None:
        raise ValueError(f"loss_agg_func {loss_agg_func!r} is not supported: pass masked_mean, seq_mean_token_sum or "
                         f"seq_mean_token_mean (rlinf.utils.utils.get_loss_agg_func)")
    return mode


def token_level_actor_loss(**kwargs) -> tuple[torch.Tensor, dict]:
    """policy_loss(task_type != "embodied", loss_type="actor") with a seq-mean loss_agg_func: compute_ppo_actor_loss
    (losses.py:170-312) on [bsz, L] token log-probs through the token-level kernel, fast_path_zero_loss_mask honoured.
    Metrics: the eight actor/* keys as 0-dim device tensors."""
    if kwargs.get("critic_warmup"):
        raise ValueError("critic_warmup is not supported with a seq-mean loss_agg_func")
    loss, metrics = ops.token_policy_loss(
        kwargs["logprobs"], kwargs["old_logprobs"], kwargs["advantages"], kwargs.get("loss_mask"),
        loss_agg=loss_agg_mode(kwargs.get("loss_agg_func")), clip_ratio_low=kwargs["clip_ratio_low"],
        clip_ratio_high=kwargs["clip_ratio_high"], clip_ratio_c=kwargs.get("clip_ratio_c"),
        clip_log_ratio_min=kwargs.get("clip_log_ratio_min"), clip_log_ratio_max=kwargs.get("clip_log_ratio_max"),
        fast_path_zero_loss_mask=bool(kwargs.get("fast_path_zero_loss_mask", False)))
    return loss, {k: metrics[k] for k in (L.TM_KEYS[s] for s in L.ACTOR_SLOTS)}


def reasoning_actor_loss(logprobs, advantages, loss_mask, *, old_logprobs=None, recomputed_logprobs=None,
                         rollout_logprobs=None, ref_logprobs=None, entropy=None, loss_agg_func=None,
                         clip_ratio_low: float = 0.2, clip_ratio_high: float = 0.2, clip_ratio_c: Optional[float] = 3.0,
                         clip_log_ratio_min: Optional[float] = None, clip_log_ratio_max: Optional[float] = None,
                         entropy_bonus: float = 0.0, kl_beta: float = 0.0, kl_penalty_type: str = "kl",
                         kl_order: str = "fsdp", importance_sampling_fix: bool = False,
                         importance_sampling_clip: Optional[float] = None,
                         fast_path_zero_loss_mask: bool = True) -> tuple[torch.Tensor, dict]:
    """The whole loss block of the reasoning actor in one device pass: FSDPActor.training_step
    (workers/actor/fsdp_actor_worker.py:700-780, kl_order="fsdp") or the Megatron loss_func
    (megatron_actor_worker.py:194-293, kl_order="megatron"), with the worker's own variables.

    old_logprobs defaults to recomputed_logprobs, else rollout_logprobs (the workers' choice).  loss_agg_func is the
    worker's self.loss_agg_func (or a get_loss_agg_func name).  entropy: pass it when the worker has calculate_entropy
    (actor/entropy_loss is then reported); entropy_bonus > 0 adds the term to the loss (calculate_entropy_loss).
    ref_logprobs with kl_beta > 0 adds kl_beta * kl_loss.  rollout and recomputed log-probs also give
    actor/rollout_train_kl (compute_rollout_train_kl, fsdp_actor_worker.py:75-93).

    Returns (loss, metrics): loss before 1/gradient_accumulation (and before Megatron's early-stop and valid-token
    scales: algorithms.MegatronLossEpilogue applies them and the data-parallel metric average on the device),
    differentiable w.r.t. logprobs and entropy; metrics are 0-dim device tensors under the workers' keys,
    actor/final_loss, actor/entropy_loss and actor/kl_loss included.  No host sync."""
    if old_logprobs is None:
        old_logprobs = recomputed_logprobs if recomputed_logprobs is not None else rollout_logprobs
    if old_logprobs is None:
        raise ValueError("reasoning_actor_loss needs old_logprobs, recomputed_logprobs or rollout_logprobs")
    return ops.token_policy_loss(
        logprobs, old_logprobs, advantages, loss_mask, entropy=entropy, ref_logprobs=ref_logprobs,
        rollout_logprobs=rollout_logprobs, recomputed_logprobs=recomputed_logprobs,
        loss_agg=loss_agg_mode(loss_agg_func), clip_ratio_low=clip_ratio_low, clip_ratio_high=clip_ratio_high,
        clip_ratio_c=clip_ratio_c, clip_log_ratio_min=clip_log_ratio_min, clip_log_ratio_max=clip_log_ratio_max,
        entropy_bonus=entropy_bonus, kl_beta=kl_beta, kl_penalty=kl_penalty_type, kl_order=kl_order,
        importance_sampling_fix=importance_sampling_fix, importance_sampling_clip=importance_sampling_clip,
        fast_path_zero_loss_mask=fast_path_zero_loss_mask)


def reasoning_critic_loss(values, returns, prev_values, loss_mask, *, value_clip: float,
                          huber_delta: float = 10000.0) -> tuple[torch.Tensor, dict]:
    """The loss block of the reasoning critic (MegatronCritic's loss_func, workers/critic/megatron_critic_worker.py:
    92-123) in one device pass, with the worker's own variables: values = vpreds [bsz, L] (e.g. from
    ops.megatron_response_values), returns and prev_values = batch["returns"] / batch["values"], loss_mask =
    response_mask[:, -L:], value_clip = the worker's value_clip; huber_delta is the worker's fixed 10000.  The
    aggregation is masked_mean whatever the worker's loss_agg_func, as in compute_ppo_critic_loss.

    Returns (loss, metrics): loss differentiable w.r.t. values; metrics are 0-dim device tensors under the worker's keys
    (critic/value_loss, critic/value_clip_ratio, the five __sum__/_critic_explained_variance/* sums and
    critic/final_value_loss), before Megatron's data-parallel reductions (algorithms.MegatronLossEpilogue("critic")
    makes them in one all-reduce, and algorithms.step_metrics finishes the explained variance).  No host sync."""
    return ops.token_critic_loss(values, returns, prev_values, loss_mask, value_clip=value_clip,
                                 huber_delta=huber_delta)


class _FusedOpdLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, logprobs, cfg):
        loss, metrics, d_lp = ops.opd_loss(logprobs=logprobs.detach(), want_grads=True, **cfg)
        ctx.grad = d_lp
        ctx.shape = logprobs.shape
        ctx.mark_non_differentiable(metrics)
        return loss.reshape(()), metrics

    @staticmethod
    def backward(ctx, g_loss, _g_metrics):
        g, ctx.grad = ctx.grad, None
        return ops.scale_by_(g, g_loss).view(ctx.shape), None


@register_policy_loss("opd")
def compute_opd_actor_loss(logprobs: torch.Tensor, advantages: torch.Tensor, loss_mask: Optional[torch.Tensor] = None,
                           loss_agg_func=None, max_episode_steps: Optional[int] = None,
                           loss_mask_sum: Optional[torch.Tensor] = None, **kwargs) -> tuple[torch.Tensor, dict]:
    """VLA-OPD actor loss with stop-gradient dense rewards (losses.py:427-505): agg(-logprobs * advantages)."""
    _check_fp32(logprobs=logprobs, advantages=advantages)
    assert advantages.shape == logprobs.shape, (
        f"OPD advantages shape {advantages.shape} must match logprobs shape {logprobs.shape}.")
    assert loss_mask is not None, "OPD actor loss requires loss_mask."
    assert loss_mask_sum is not None, "OPD actor loss requires loss_mask_sum."
    dev = logprobs.device if logprobs.is_cuda else L.default_device()
    lp = logprobs if logprobs.is_cuda else logprobs.to(dev)
    tok = lp.shape[-1]
    n_units = lp.numel() // tok

    def unit(t, name):
        t = L.to_device(t, dev)
        if t.dim() == lp.dim() - 1:
            t = t.unsqueeze(-1)
        assert t.dim() == lp.dim(), f"OPD {name} rank {t.dim()} must match logprobs rank {lp.dim()}."
        assert t.shape[:-1] == lp.shape[:-1], (
            f"OPD {name} shape {t.shape} must match logprobs shape {lp.shape} except the token dimension.")
        if t.shape[-1] != 1:
            assert t.shape[-1] == tok, (
                f"OPD {name} token dimension {t.shape[-1]} must be 1 or match logprobs token dimension {tok}.")
            # a per-token mask: one unit per token
            return t.reshape(-1), True
        return t.reshape(n_units), False

    m, m_tok = unit(loss_mask, "loss_mask")
    ms, ms_tok = unit(loss_mask_sum, "loss_mask_sum")
    if m_tok != ms_tok:  # bring both to per-token granularity
        if not m_tok:
            m = m.reshape(n_units, 1).expand(n_units, tok).reshape(-1)
        if not ms_tok:
            ms = ms.reshape(n_units, 1).expand(n_units, tok).reshape(-1)
        m_tok = True
    lp2 = lp.reshape(-1, 1) if m_tok else lp.reshape(n_units, tok)
    cfg = dict(advantages=L.to_device(advantages, dev, torch.float32).reshape(lp2.shape), loss_mask=m, loss_mask_sum=ms,
               max_episode_steps=max_episode_steps)
    if torch.is_grad_enabled() and logprobs.requires_grad:
        loss, metrics = _FusedOpdLoss.apply(lp2, cfg)
    else:
        loss, metrics, _ = ops.opd_loss(logprobs=lp2.detach(), want_grads=False, **cfg)
        loss = loss.reshape(())
    return loss, {"actor/policy_loss": metrics[0], "actor/opd_reward": metrics[1], "actor/opd_reverse_kl": metrics[2]}


# built-in entries: for task_type == "embodied" registry.policy_loss hands them the RAW worker kwargs through this marker
# (one fused launch group); a callable a user registers under the same name has no marker and takes the generic route
compute_ppo_actor_critic_loss._rb200_fused_embodied = fused_embodied_policy_loss
compute_grpo_actor_loss_fn._rb200_fused_embodied = fused_embodied_policy_loss
compute_decoupled_ppo_actor_critic_loss._rb200_fused_embodied = fused_embodied_policy_loss
