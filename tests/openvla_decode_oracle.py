"""Restatement of plain OpenVLA's generate step over the action window (openvla_action_model.py:453-471 and HF's
processor order: the user processors, then TemperatureLogitsWarper, then TopKLogitsWarper), beside
tests/action_sample_oracle.py, which it reuses for the greedy step and the de-tokenisation."""
from __future__ import annotations

import torch

import action_sample_oracle as O


def processed_scores(window_logits, do_sample: bool, T: float = 1.0, k: int = 0) -> torch.Tensor:
    """generate's `scores` over the window [..., W] from the raw fp32 logits' window: VLALogitsProcessor leaves the
    window as it is, then with do_sample `scores / T` and, for 0 < k, -inf below the k-th largest scaled score (ties
    kept), in fp32 as HF computes them."""
    z = torch.as_tensor(window_logits).float()
    if not do_sample:
        return z.clone()
    z = z / T
    if 0 < k < z.shape[-1]:
        thr = torch.topk(z, k, dim=-1).values[..., -1:]
        z = z.masked_fill(z < thr, float("-inf"))
    return z


def step_logprobs(window_logits, do_sample: bool, T: float = 1.0, k: int = 0) -> torch.Tensor:
    """fp64 log-probabilities over the window of one generate step, as the sampler forms them (top-k on the unscaled
    values, then / T): the same kept set as processed_scores wherever dividing by T merges no two values."""
    return O.window_logprobs(window_logits, 0, torch.as_tensor(window_logits).shape[-1], do_sample, T, k)


def greedy_step(window_logits, lo: int) -> torch.Tensor:
    """The greedy token of each row as an absolute vocabulary id (lowest index on ties)."""
    x = torch.as_tensor(window_logits)
    return O.greedy_tokens(x, 0, x.shape[-1]) + lo
