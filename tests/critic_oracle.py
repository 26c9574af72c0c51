"""CPU oracle of the reasoning PPO critic (test infrastructure, not product code), written from the reference's
documented computation:

  values   LinearForLastLayer(H, 1): a bf16 Linear without bias, cast with .float(), read at log_probs[:, -L-1:-1]:
           the value of response token j < r_b of sequence b is the head at position n_b - r_b - 1 + j, 0 past r_b.
  loss     compute_ppo_critic_loss (rlinf/algorithms/losses.py:315-380) with masked_mean (utils.py:321-328) and the
           explained-variance sums (metric_utils.py:232-258), MegatronCritic's critic/final_value_loss added.

`critic_loss` keeps the reference's fp32 elementwise op order; `sums="fp64"` adds in fp64 (what the kernel's fixed
partials approximate), `sums="fp32"` as torch's fp32 sums do (the fixture's bits)."""
from __future__ import annotations

import torch

import response_rows_mp_oracle as O

KEYS = ("critic/value_loss", "critic/value_clip_ratio",
        "__sum__/_critic_explained_variance/count",
        "__sum__/_critic_explained_variance/returns_sum",
        "__sum__/_critic_explained_variance/returns_sq_sum",
        "__sum__/_critic_explained_variance/errors_sum",
        "__sum__/_critic_explained_variance/errors_sq_sum",
        "critic/final_value_loss")


def huber(e, delta):
    a = e.abs()
    return torch.where(a < delta, 0.5 * e * e, delta * (a - 0.5 * delta))


def critic_loss(values, returns, prev_values, mask, value_clip, huber_delta, sums="fp64"):
    """(loss, metrics {KEYS}, d loss / d values) of fp32 [bsz, L] inputs."""
    v = values.detach().float().clone().requires_grad_(True)
    m = mask.bool()
    vpc = prev_values + (v - prev_values).clamp(-value_clip, value_clip)
    vl = torch.max(huber(returns - v, huber_delta), huber(returns - vpc, huber_delta))
    acc = torch.float64 if sums == "fp64" else torch.float32
    s = (vl.to(acc) * m).sum()
    cnt = m.sum()
    loss = s if bool((~m).all()) else s / cnt
    loss.backward()
    with torch.no_grad():
        clip = ((vpc - prev_values).abs() > value_clip).to(acc).mean()
        r, e = returns[m].to(acc), (returns - v)[m].to(acc)
        if sums == "fp64":
            sq_r, sq_e = r * r, e * e
        else:
            sq_r, sq_e = returns[m] * returns[m], (returns - v)[m] * (returns - v)[m]
        vals = (loss.detach(), clip, cnt.to(acc), r.sum(), sq_r.sum(), e.sum(), sq_e.sum(), loss.detach())
    return loss.detach(), dict(zip(KEYS, vals)), v.grad


def clip_count(values, prev_values, value_clip):
    """The number of cells whose clipped prediction moved by more than value_clip (all cells, masked or not)."""
    vpc = prev_values + (values - prev_values).clamp(-value_clip, value_clip)
    return int(((vpc - prev_values).abs() > value_clip).sum())


def head_values(streams, w, cu, n, r, cp, L):
    """[bsz, L] fp32 values from each CP rank's full [T_c, H] bf16 stream: F.linear in bf16, .float(), placed at the
    response cells of the prediction rows the rank holds (zeros past r_b)."""
    out = torch.zeros(len(n), L)
    for c, rows in enumerate(O.prediction_rows(cu, n, r, cp)):
        v = torch.nn.functional.linear(streams[c], w).float()[:, 0]
        for t, b, j in rows:
            out[b, j] = v[t]
    return out
