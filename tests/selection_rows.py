"""Rows on which a radix top-k select goes wrong, shared by the selection tests (test_selection_oracle_cpu.py,
test_gpu_selection_edges.py): -inf columns (with k past the finite count, so that the k-th value is -inf), small
integers that tie thousands of times at the k-th value, all-equal rows, and +0.0 / -0.0 at the k-th value.  Every value
is exact in bf16, so the fp32 and bf16 rows are the same numbers."""
from __future__ import annotations

import torch

KINDS = ("neginf_few", "neginf_half", "int_ties", "all_equal", "zero_mixed", "zero_pos")


def _zero_row(V, lo, hi, k, g, mixed):
    """+1 at about k / 2 columns, zeros past the k-th largest, -1 elsewhere: the k-th value is a zero.  `mixed`: zeros of
    both signs; otherwise every zero is +0.0 except the window's, which are -0.0 (so the k-th key is +0.0's key while
    the window holds only -0.0).  A few zeros are always in the window."""
    kk = k if 0 < k < V else V // 2
    n_pos = kk // 2
    n_zero = min(V - n_pos, kk - n_pos + max(8, kk // 8))
    vals = torch.cat([torch.ones(n_pos), torch.zeros(n_zero), -torch.ones(V - n_pos - n_zero)])
    row = vals[torch.randperm(V, generator=g)]
    zeros = (row == 0).nonzero()[:, 0]
    outside = zeros[(zeros < lo) | (zeros >= hi)]
    for j in range(min(4, hi - lo, outside.numel())):  # swap zeros into the window's first columns
        row[outside[j]], row[lo + j] = row[lo + j].clone(), 0.0
    zeros = row == 0
    if mixed:
        sign = torch.rand(V, generator=g) < 0.5
    else:
        sign = torch.zeros(V, dtype=torch.bool)
        sign[lo:hi] = True
    return torch.where(zeros & sign, torch.tensor(-0.0), row)


def hard_row(kind, V, lo, hi, k, g):
    """One fp32 row [V] of `kind` for the window [lo, hi) and top_k = k (0 = no filter)."""
    if kind == "neginf_few":  # fewer finite columns than k (when k > 1), one of them in the window: thr = -inf
        F = max(1, min(k // 2, V - 1))
        pos = torch.randperm(V, generator=g)[:F]
        pos[0] = lo + int(torch.randint(hi - lo, (1,), generator=g))
        row = torch.full((V,), float("-inf"))
        row[pos] = torch.randint(-8, 9, (F,), generator=g).float()
        return row
    if kind == "neginf_half":
        row = (torch.randn(V, generator=g) * 2).to(torch.bfloat16).float()
        row[torch.rand(V, generator=g) < 0.5] = float("-inf")
        row[lo + int(torch.randint(hi - lo, (1,), generator=g))] = 1.0  # a finite column in the window
        return row
    if kind == "int_ties":  # 7 values, each about V / 7 times
        return torch.randint(-3, 4, (V,), generator=g).float()
    if kind == "all_equal":
        return torch.full((V,), 1.25)
    if kind in ("zero_mixed", "zero_pos"):
        return _zero_row(V, lo, hi, k, g, kind == "zero_mixed")
    raise ValueError(kind)


def hard_rows(V, lo, hi, k, seed=0, reps=2):
    """fp32 [len(KINDS) * reps, V] (CPU), each kind `reps` times with different draws, and the kind of each row."""
    g = torch.Generator().manual_seed(seed)
    rows, kinds = [], []
    for kind in KINDS:
        for _ in range(reps):
            rows.append(hard_row(kind, V, lo, hi, k, g))
            kinds.append(kind)
    return torch.stack(rows), kinds
