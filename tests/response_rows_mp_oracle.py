"""CPU oracle of the response-rows plan under Megatron sequence and context parallelism (test infrastructure, not
product code), written position by position from preprocess_packed_seqs' chunking (rlinf/hybrid_engines/megatron/
utils.py:27-102) and Megatron's sequence-parallel split of dim 0:

  cp = 1   sequence b's position p sits at CP-local row cu[b] + p
  cp > 1   half = N_b / (2 cp); CP rank c holds positions [half c, half (c + 1)) at rows cu[b] / cp + ... and
           [N_b - half (c + 1), N_b - half c) at rows cu[b] / cp + half + ...
  SP       TP rank k holds CP-local rows [k T_c / tp, (k + 1) T_c / tp)

Response token j < r_b of sequence b is predicted at position n_b - r_b - 1 + j; its target is responses[b, j].
`rank_maps` gives every map the plan kernel writes for one rank, `owner` the (cp rank, local row) of every position."""
from __future__ import annotations

import torch


def owner(cu, n, cp):
    """{(b, p): (c, local row)} for every valid position p < n_b."""
    out = {}
    for b in range(len(n)):
        N, nb, s = int(cu[b + 1]) - int(cu[b]), int(n[b]), int(cu[b])
        for p in range(nb):
            if cp == 1:
                out[b, p] = (0, s + p)
                continue
            half, start = N // (2 * cp), s // cp
            q = p // half
            if q < cp:
                out[b, p] = (q, start + p - half * q)
            else:
                c = 2 * cp - 1 - q
                out[b, p] = (c, start + half + p - (N - half * (c + 1)))
    return out


def prediction_rows(cu, n, r, cp):
    """Per CP rank: [(local row, b, j)] of its prediction rows, ascending in local row."""
    own = owner(cu, n, cp)
    per = [[] for _ in range(cp)]
    for b in range(len(n)):
        for j in range(int(r[b])):
            c, t = own[b, int(n[b]) - int(r[b]) - 1 + j]
            per[c].append((t, b, j))
    return [sorted(x) for x in per]


def rank_maps(cu, n, r, responses, L, tp, cp, sp, T_c, k, c):
    """Every map of the plan kernel for rank (k, c), as Python lists."""
    per = prediction_rows(cu, n, r, cp)
    Ts = T_c // tp if sp else T_c
    counts = []
    for cc in range(cp):
        if sp:
            counts.append(tuple(sum(1 for t, _, _ in per[cc] if kk * Ts <= t < (kk + 1) * Ts) for kk in range(tp)))
        else:
            counts.append((len(per[cc]),) * tp)
    R_of = [sum(x) if sp else x[0] for x in counts]
    Rmax_c = max(1, max(R_of))
    Rmax_k = max(1, max(counts[c])) if sp else R_of[c]
    mine = per[c]
    off = [sum(counts[c][:kk]) for kk in range(tp)] if sp else [0] * tp
    m = dict(R=R_of[c], Rmax_k=Rmax_k, Rmax_c=Rmax_c, counts=tuple(counts))
    m["rows"] = [t for t, _, _ in mine]
    m["targets"] = [int(responses[b][j]) for _, b, j in mine]
    m["cells"] = [b * L + j for _, b, j in mine]
    if sp:
        m["unpad"] = [(t // Ts) * Rmax_k + i - off[t // Ts] for i, (t, _, _) in enumerate(mine)]
        send = [t - k * Ts for t, _, _ in mine if k * Ts <= t < (k + 1) * Ts]
        m["send"] = send + [-1] * (Rmax_k - len(send))
        m["slot_map"] = [off[kk] + s if s < counts[c][kk] else -1 for kk in range(tp) for s in range(Rmax_k)]
        slot = {t - k * Ts: i - off[k] for i, (t, _, _) in enumerate(mine) if k * Ts <= t < (k + 1) * Ts}
        m["hidden_map"] = [slot.get(x, -1) for x in range(Ts)]
    else:
        m["unpad"] = list(range(len(mine)))
        compact = {t: i for i, (t, _, _) in enumerate(mine)}
        m["hidden_map"] = [compact.get(x, -1) for x in range(T_c)]
    cell_map = [-1] * (len(n) * L)
    for cc in range(cp):
        for i, (_, b, j) in enumerate(per[cc]):
            cell_map[b * L + j] = cc * Rmax_c + i
    m["cell_map"] = cell_map
    return m


def local_stream(seq_values, cu, n, cp, c, T_c):
    """CP rank c's packed [T_c, ...] stream of per-position values seq_values[b] [n_b, ...] (zeros elsewhere), as
    preprocess_packed_seqs lays out input ids."""
    ref = seq_values[0]
    out = torch.zeros((T_c, *ref.shape[1:]), dtype=ref.dtype, device=ref.device)
    for (b, p), (cc, t) in owner(cu, n, cp).items():
        if cc == c:
            out[t] = seq_values[b][p]
    return out
