"""Plugin registries and the two operator entry points, with the reference's surface.

Mirror of rlinf/algorithms/registry.py: `ADV_REGISTRY` (:30), `register_advantage` (:33),
`get_adv_and_returns` (:47), `LOSS_REGISTRY` (:56), `register_policy_loss` (:59),
`get_policy_loss` (:71), `policy_loss` (:77-92), `calculate_adv_and_returns` (:95-124).
Same names, kwargs, return conventions (embodied -> dict, reasoning -> tuple) and error behaviour;
the registered callables launch the sm_90a kernels of librlinf_b200.so.
"""
from __future__ import annotations

from typing import Callable, Optional

import torch

from .utils import (
    calculate_scores,
    postprocess_embodied_advantages_outputs,
    postprocess_reasoning_advantages_outputs,
    preprocess_embodied_advantages_inputs,
    preprocess_reasoning_advantages_inputs,
)

ADV_REGISTRY: dict[str, Callable] = {}
LOSS_REGISTRY: dict[str, Callable] = {}


def _registrar(table: dict):
    """Decorator factory shared by both tables; keys are stored lower-cased, as the reference does."""

    def register(name: str):
        def bind(fn):
            table[name.lower()] = fn
            return fn

        return bind

    return register


register_advantage = _registrar(ADV_REGISTRY)      # registry.py:33
register_policy_loss = _registrar(LOSS_REGISTRY)   # registry.py:59


def get_adv_and_returns(name: str) -> Callable:
    """Case-insensitive lookup (registry.py:47); unknown names raise the reference's message."""
    fn = ADV_REGISTRY.get(name.lower())
    if fn is None:
        raise ValueError(f"Advantage '{name}' not registered. Available: {list(ADV_REGISTRY.keys())}")
    return fn


def get_policy_loss(name: str):
    """Exact-key lookup (registry.py:71: no lower-casing on this side)."""
    try:
        return LOSS_REGISTRY[name]
    except KeyError:
        raise ValueError(f"Loss {name} not registered") from None


def policy_loss(**kwargs) -> tuple[torch.Tensor, dict]:
    """Unified loss entry (registry.py:77-92).

    For the embodied task type the whole chain preprocess_loss_inputs -> loss fn -> autograd backward
    is one fused kernel group (the logprob reduction happens inside the kernel), and the metric dict
    holds Python floats obtained with ONE device->host copy (the reference does one .item() per metric).
    """
    from . import losses

    loss_type = kwargs["loss_type"]
    get_policy_loss(loss_type)  # same "not registered" error
    task_type = kwargs["task_type"]
    loss_fn = LOSS_REGISTRY[loss_type]
    # Built-in entries carry a marker: for them the embodied chain preprocess -> loss -> backward is ONE fused launch
    # group. A callable a user registered under the same name has no marker and takes the reference's generic route.
    fused = getattr(loss_fn, "_rb200_fused_embodied", None)
    if task_type == "embodied" and fused is not None:
        return fused(**kwargs)
    if task_type != "embodied" and fused is not None:
        # the reasoning workers pass loss_agg_func (fsdp_actor_worker.py:737-751, megatron_actor_worker.py:225-243);
        # the built-in kernels aggregate as masked_mean, the token-level kernel also as the two seq-mean variants
        mode = losses.loss_agg_mode(kwargs.get("loss_agg_func"))
        ratio_agg = all(kwargs.get(k) is not None for k in ("max_episode_steps", "loss_mask_sum", "loss_mask"))
        if mode != "token-mean" and not ratio_agg:  # masked_mean_ratio overrides loss_agg_func (losses.py:221-227)
            if loss_type != "actor":
                raise ValueError(f"loss_agg_func {mode!r} is supported with loss_type='actor' only; "
                                 f"{loss_type!r} aggregates as token-mean (masked_mean)")
            return losses.token_level_actor_loss(**kwargs)
    if task_type == "embodied":
        kwargs = losses.preprocess_loss_inputs(**kwargs)
    loss, metrics_data = loss_fn(**kwargs)
    if task_type == "embodied":
        metrics_data = losses.postprocess_loss_metric(metrics_data)
    return loss, metrics_data


def calculate_adv_and_returns(**kwargs):
    """Unified advantage entry (registry.py:95-124)."""
    adv_type = kwargs["adv_type"]
    fn = get_adv_and_returns(adv_type)
    task_type = kwargs["task_type"]
    if task_type == "embodied":
        if adv_type == "opd":  # registry.py:106-110: no layout pre/post-processing for the dense OPD rewards
            advantages, returns = fn(**kwargs)
            res = {"advantages": advantages}
            if returns is not None:
                res["returns"] = returns
            return res
        kwargs = preprocess_embodied_advantages_inputs(**kwargs)
        if adv_type not in ("gae", "grpo_video"):
            kwargs = calculate_scores(**kwargs)
        advantages, returns = fn(**kwargs)
        res = postprocess_embodied_advantages_outputs(advantages=advantages, returns=returns, **kwargs)
    else:
        kwargs = preprocess_reasoning_advantages_inputs(**kwargs)
        advantages, returns = fn(**kwargs)
        res = postprocess_reasoning_advantages_outputs(advantages, returns)
    return res
