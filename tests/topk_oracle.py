"""fp64 torch oracle of the top-k filtered log-probabilities and entropies (csrc/topk.cu), forward and the closed-form
gradient, with the reference's semantics (TopKLogitsWarper over the whole row, then the action-bin window, then
compute_logprobs_from_logits / compute_entropy_from_logits):
  thr = the k-th largest logit of the row (with multiplicity), selected on the unscaled logits;
  column i is kept iff lo <= i < hi and x_i >= thr (ties at the k-th value are all kept);
  lse / logprob / entropy over the kept columns; a target that is not kept -> logprob -inf;
  a row with no kept column -> logprob NaN, entropy -0.0 and a zero gradient;
  grad_i = inv_T (g_lp (1[i = t] - p_i) - g_H p_i (log p_i + H)) at kept columns, 0 elsewhere;
  a kept -inf logit (thr = -inf once k reaches past the finite logits) has p_i = 0, and p_i log p_i is taken as 0
  there, as the reference's where(p > 0, ., 0), in the entropy and in the gradient.
top_k <= 0 or >= V: no filtering (the window only)."""
from __future__ import annotations

import torch


def topk_logprobs_entropy(logits, target, temperature=1.0, window=None, top_k=0, g_lp=None, g_h=None):
    """logits [..., V] (any float dtype, taken exactly into fp64), target [...] -> dict of fp64 tensors:
    lp, ent, lse, thr (the unscaled k-th value, -inf without filtering), kept [..., V] bool, and grad [..., V]
    when g_lp or g_h is given (None entries count as zero)."""
    x = logits.detach().to(torch.float64)
    V = x.shape[-1]
    lo, hi = (0, V) if window is None else (int(window[0]), int(window[1]))
    cols = torch.arange(V, device=x.device)
    kept = ((cols >= lo) & (cols < hi)).expand_as(x).clone()
    if 0 < top_k < V:
        thr = torch.topk(x, top_k, dim=-1).values[..., -1]
        kept &= x >= thr.unsqueeze(-1)
    else:
        thr = torch.full(x.shape[:-1], -float("inf"), dtype=torch.float64, device=x.device)
    z = torch.where(kept, x / float(temperature), torch.tensor(-float("inf"), dtype=torch.float64))
    empty = ~kept.any(-1)
    lse = torch.logsumexp(z, dim=-1)
    logp = torch.where(kept, z - lse.unsqueeze(-1), torch.tensor(-float("inf"), dtype=torch.float64))
    p = torch.where(kept, logp.exp(), torch.zeros((), dtype=torch.float64))
    # a kept -inf logit (thr = -inf when k reaches past the finite columns) has p = 0 and logp = -inf: it adds 0, as
    # the reference's where(p > 0, ., 0), not 0 * -inf
    plogp = torch.where(p > 0, p * logp, torch.zeros((), dtype=torch.float64))
    ent = -plogp.sum(-1)
    t = target.to(torch.int64).to(x.device)
    lp = torch.gather(logp, -1, t.clamp(0, V - 1).unsqueeze(-1)).squeeze(-1)
    lp = torch.where((t >= 0) & (t < V), lp, torch.tensor(-float("inf"), dtype=torch.float64))
    lp = torch.where(empty, torch.tensor(float("nan"), dtype=torch.float64), lp)
    ent = torch.where(empty, torch.tensor(-0.0, dtype=torch.float64), ent)
    out = {"lp": lp, "ent": ent, "lse": lse, "thr": thr, "kept": kept}
    if g_lp is not None or g_h is not None:
        glp = torch.zeros(x.shape[:-1], dtype=torch.float64) if g_lp is None else g_lp.to(torch.float64)
        gh = torch.zeros(x.shape[:-1], dtype=torch.float64) if g_h is None else g_h.to(torch.float64)
        glp, gh = glp.to(x.device), gh.to(x.device)
        onehot = torch.nn.functional.one_hot(t.clamp(0, V - 1), V).to(torch.float64)
        g = glp.unsqueeze(-1) * (onehot - p) - gh.unsqueeze(-1) * (plogp + p * ent.unsqueeze(-1))
        g = torch.where(kept, g / float(temperature), torch.zeros((), dtype=torch.float64))
        out["grad"] = torch.where(empty.unsqueeze(-1), torch.zeros((), dtype=torch.float64), g)
    return out
