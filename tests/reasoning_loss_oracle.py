"""CPU oracle of the reasoning actor's loss block (test infrastructure, not product code): a torch-on-CPU restatement
of what ops.token_policy_loss / algorithms.reasoning_actor_loss compute, in the reference's op order so that in fp32
it reproduces tests/golden/golden_reasoning_loss.npz bit for bit, and in fp64 it is the bar the GPU tests use.

  - the importance-sampling fix of both workers (fsdp_actor_worker.py:722-735, megatron_actor_worker.py:208-221);
  - compute_ppo_actor_loss (rlinf/algorithms/losses.py:170-312) with its loss_agg_func and fast path (:204-217);
  - the entropy and KL terms (fsdp_actor_worker.py:753-765 / megatron_actor_worker.py:245-256) with kl_penalty
    (rlinf/algorithms/utils.py:26-64) in either argument order;
  - masked_mean, seq_mean_token_sum, seq_mean_token_mean (rlinf/utils/utils.py:323-349);
  - compute_rollout_train_kl (fsdp_actor_worker.py:75-93).
Gradients come from autograd."""
from __future__ import annotations

import torch


def masked_mean(values, mask):
    """rlinf/utils/utils.py:323-330."""
    if (~mask).all():
        return (values * mask).sum()
    return (values * mask).sum() / mask.sum()


def seq_mean_token_sum(values, mask):
    """rlinf/utils/utils.py:338-341."""
    return torch.mean(torch.sum(values * mask, dim=-1))


def seq_mean_token_mean(values, mask):
    """rlinf/utils/utils.py:344-349: 0/0 = NaN for a row without a valid token."""
    return torch.mean(torch.sum(values * mask, dim=-1) / torch.sum(mask, dim=-1))


AGG = {"token-mean": masked_mean, "seq-mean-token-sum": seq_mean_token_sum, "seq-mean-token-mean": seq_mean_token_mean}


def kl_penalty(logprob, ref_logprob, kind):
    """rlinf/algorithms/utils.py:26-64."""
    if kind in ("kl", "k1"):
        return logprob - ref_logprob
    if kind == "abs":
        return (logprob - ref_logprob).abs()
    if kind in ("mse", "k2"):
        return 0.5 * (logprob - ref_logprob).square()
    if kind in ("low_var_kl", "k3"):
        kl = torch.clamp(ref_logprob - logprob, min=-20, max=20)
        return torch.clamp(torch.exp(kl) - kl - 1, min=-10, max=10)
    raise NotImplementedError(kind)


def ppo_actor_loss(logprobs, old_logprobs, advantages, loss_mask, agg, clip_ratio_low, clip_ratio_high,
                   clip_ratio_c=None, clip_log_ratio_min=None, clip_log_ratio_max=None, fast_path=False):
    """compute_ppo_actor_loss (losses.py:170-312) on [bsz, L] tokens; returns (loss, metrics) with the normal key set
    in both branches (the fast path's values are 0)."""
    zero = torch.zeros((), dtype=logprobs.dtype)
    keys = ("actor/policy_loss", "actor/policy_loss_abs", "actor/ratio", "actor/ratio_abs", "actor/clipped_ratio",
            "actor/dual_cliped_ratio", "actor/approx_kl", "actor/clip_fraction")
    if fast_path and loss_mask[0].sum() == 0.0:
        return zero, {k: zero for k in keys}
    cnt = loss_mask.count_nonzero() or 1
    log_ratio = logprobs - old_logprobs
    if clip_log_ratio_min is not None:
        log_ratio = torch.clamp(log_ratio, min=clip_log_ratio_min)
    if clip_log_ratio_max is not None:
        log_ratio = torch.clamp(log_ratio, max=clip_log_ratio_max)
    ratio = torch.where(loss_mask, torch.exp(log_ratio), 0)
    approx_kl = torch.where(loss_mask, log_ratio.detach(), 0.0)
    clipped = torch.clamp(ratio, 1.0 - clip_ratio_low, 1.0 + clip_ratio_high)
    l1, l2 = -advantages * ratio, -advantages * clipped
    loss_e = torch.max(l1, l2)
    if clip_ratio_c is not None:
        l3 = torch.sign(advantages) * clip_ratio_c * advantages
        dual = l3.detach() < loss_e.detach()
        loss_e = torch.min(loss_e, l3)
    else:
        dual = torch.zeros_like(loss_mask)
    loss_abs = agg(loss_e.abs(), loss_mask)
    loss = agg(loss_e, loss_mask)
    clip_hit = l1.detach() < l2.detach()
    dual = (dual * loss_mask).bool()
    clip_fraction = (clip_hit * loss_mask).sum() / float(cnt)
    approx_kl = -torch.sum(approx_kl) / float(cnt)
    rd = ratio.detach()
    values = (loss.detach(), loss_abs.detach(), masked_mean(rd, loss_mask), masked_mean((rd - 1).abs(), loss_mask),
              masked_mean(clipped.detach(), loss_mask), masked_mean(torch.where(dual, ratio, 0).detach(), loss_mask),
              approx_kl.detach(), clip_fraction.detach())
    return loss, dict(zip(keys, values))


def reasoning_actor_loss(logprobs, advantages, loss_mask, old_logprobs, *, entropy=None, ref_logprobs=None,
                         rollout_logprobs=None, recomputed_logprobs=None, loss_agg="token-mean", clip_ratio_low=0.2,
                         clip_ratio_high=0.2, clip_ratio_c=3.0, clip_log_ratio_min=None, clip_log_ratio_max=None,
                         entropy_bonus=0.0, kl_beta=0.0, kl_penalty_type="kl", kl_order="fsdp",
                         importance_sampling_fix=False, importance_sampling_clip=None, fast_path=True):
    """One micro-batch of the worker's loss block.  Returns (loss, metrics, d_logprobs, d_entropy); the gradients
    are autograd's for a unit upstream gradient (zeros where the loss does not depend on the input)."""
    agg = AGG[loss_agg]
    lp = logprobs.detach().clone().requires_grad_(True)
    ent = entropy.detach().clone().requires_grad_(True) if entropy is not None else None
    if importance_sampling_fix:
        advantages = advantages * torch.clamp((recomputed_logprobs - rollout_logprobs).exp(),
                                              max=importance_sampling_clip)
    loss, metrics = ppo_actor_loss(lp, old_logprobs, advantages, loss_mask, agg, clip_ratio_low, clip_ratio_high,
                                   clip_ratio_c, clip_log_ratio_min, clip_log_ratio_max, fast_path)
    zero = torch.zeros((), dtype=logprobs.dtype)
    entropy_loss = zero
    if ent is not None:
        entropy_loss = agg(ent, loss_mask)
        if entropy_bonus > 0:
            loss = loss - entropy_bonus * entropy_loss
    kl_loss = zero
    if kl_beta > 0 and ref_logprobs is not None:
        kld = kl_penalty(ref_logprobs, lp, kl_penalty_type) if kl_order == "fsdp" else \
            kl_penalty(lp, ref_logprobs, kl_penalty_type)
        kl_loss = agg(kld, loss_mask)
        loss = loss + kl_loss * kl_beta
    metrics.update({"actor/final_loss": loss.detach(), "actor/entropy_loss": entropy_loss.detach(),
                    "actor/kl_loss": kl_loss.detach()})
    if rollout_logprobs is not None and recomputed_logprobs is not None:
        metrics["actor/rollout_train_kl"] = masked_mean(torch.abs(recomputed_logprobs - rollout_logprobs), loss_mask)
    if loss.requires_grad:
        loss.backward()
    d_lp = lp.grad if lp.grad is not None else torch.zeros_like(logprobs)
    d_ent = None
    if entropy is not None:
        d_ent = ent.grad if ent.grad is not None else torch.zeros_like(entropy)
    return loss.detach(), metrics, d_lp, d_ent
