"""CPU oracle of the response-rows plans (test infrastructure, not product code): where each layout's response tokens
sit in the flattened hidden states, and the [bsz, L] log-probs / entropies a reasoning loss reads, as
ops.response_logprobs_entropy computes them (zeros at j >= r_b).  In fp32, with the reference's per-row arithmetic on
the same full logits, it reproduces tests/golden/golden_response_rows.npz bit for bit on every response column.

  padded        a_b = b S + S - L                    fsdp_actor_worker.py:492-495
  fsdp_packed   a_b = sum_{i<b} (p_i + r_i) + p_b    hybrid_engines/fsdp/utils.py:918-1022; entropy one row later
  megatron_thd  a_b = cu_padded[b] + n_b - r_b       hybrid_engines/megatron/utils.py:27-170, cp 1
"""
from __future__ import annotations

import torch
import torch.nn.functional as F


def first_rows(layout, response_lengths, *, S=None, L=None, prompt_lengths=None, cu_seqlens_padded=None,
               seq_lengths=None):
    """a_b of every sequence, as Python ints."""
    r = [int(x) for x in response_lengths]
    if layout == "padded":
        return [b * S + S - L for b in range(len(r))]
    if layout == "fsdp_packed":
        out, c = [], 0
        for p, rb in zip(prompt_lengths, r):
            out.append(c + int(p))
            c += int(p) + rb
        return out
    if layout == "megatron_thd":
        return [int(cu_seqlens_padded[b]) + int(seq_lengths[b]) - r[b] for b in range(len(r))]
    raise ValueError(layout)


def num_rows(response_lengths, shift):
    return sum(int(r) + shift for r in response_lengths if int(r) > 0)


def rows_and_targets(a, response_lengths, tokens, shift):
    """Compact rows in order and their targets (-1 where the log-prob is not read): what the plan kernel writes."""
    rows, targets = [], []
    for ab, rb in zip(a, response_lengths):
        rb = int(rb)
        for k in range(rb + shift if rb > 0 else 0):
            rows.append(ab - 1 + k)
            targets.append(int(tokens[ab + k]) if k < rb else -1)
    return rows, targets


def to_cells(row_values, a, response_lengths, L, shift=0):
    """[T] per-row values -> [bsz, L]: cell (b, j) = row a_b - 1 + j + shift, zero at j >= r_b."""
    bsz = len(a)
    out = torch.zeros(bsz, L, dtype=row_values.dtype)
    for b in range(bsz):
        rb = int(response_lengths[b])
        if rb:
            out[b, :rb] = row_values[a[b] - 1 + shift:a[b] - 1 + shift + rb]
    return out


def fsdp_row_values(hidden, W, tokens, temperature):
    """Per-row log-prob of the next token and entropy, as the FSDP worker computes them: logits = hidden @ W^T in the
    model's shape, divided in place by the temperature, -cross_entropy and compute_entropy_from_logits per row."""
    logits = hidden @ W.T
    logits.div_(temperature)
    z = logits.reshape(-1, logits.shape[-1])
    tok = tokens.reshape(-1)
    nxt = torch.cat([tok[1:], tok[-1:]])  # the last row's target is never read
    lp = -F.cross_entropy(z, nxt, reduction="none").float()
    logp = F.log_softmax(z, dim=-1)
    p = logp.exp()
    ent = -torch.where(p > 0, p * logp, 0.0).sum(dim=-1)
    return lp, ent


def megatron_row_values(hidden, W, tokens, temperature, P, targets=None):
    """Per-row log-prob of the next token (or of `targets`, one per row) and entropy, as the vocabulary-parallel
    reference computes them over P equal shards (fp32; the cross-rank reductions of two ranks are exact sums / maxima)."""
    Vtot = W.shape[0]
    Vs = Vtot // P
    full = hidden @ W.T
    shards = [full[..., k * Vs:(k + 1) * Vs].contiguous() for k in range(P)]
    for s in shards:
        s /= temperature
    tok = tokens.reshape(1, -1)
    nxt = torch.cat([tok[:, 1:], tok[:, -1:]], 1) if targets is None else targets.reshape(1, -1)
    mx = torch.stack([s.max(dim=-1, keepdim=True).values for s in shards]).amax(0)
    norm = [s - mx for s in shards]
    exps = [n.exp() for n in norm]
    sums = [e.sum(dim=-1, keepdim=True) for e in exps]
    se = sums[0]
    for x in sums[1:]:
        se = se + x
    soft = [e.div_(se) for e in exps]
    st = [(sm * s).sum(dim=-1, keepdim=True) for sm, s in zip(soft, shards)]
    sst = st[0]
    for x in st[1:]:
        sst = sst + x
    ent = mx.squeeze(-1) + se.log().squeeze(-1) - sst.squeeze(-1)
    pred = torch.zeros_like(nxt, dtype=torch.float32)
    for k in range(P):
        own = (nxt >= k * Vs) & (nxt < (k + 1) * Vs)
        loc = torch.where(own, nxt - k * Vs, torch.zeros_like(nxt))
        v = norm[k].reshape(-1, Vs)[torch.arange(loc.numel()), loc.reshape(-1)].view_as(nxt)
        pred = pred + torch.where(own, v, torch.zeros_like(v))
    lp = -(se.log().squeeze(-1) - pred)
    return lp.reshape(-1), ent.reshape(-1)
