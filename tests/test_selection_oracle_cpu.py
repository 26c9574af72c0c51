"""The fp64 selection oracles (tests/topk_oracle.py, tests/action_sample_oracle.py) on the rows where a top-k select goes
wrong (tests/selection_rows.py), against a plain restatement of the reference chain: masked_fill(x < topk(x, k)[..., -1:],
-inf), the action-bin window, log_softmax and where(p > 0, p * logp, 0).  Also the greedy tie-break (lowest index, as
torch.argmax)."""
from __future__ import annotations

import pytest
import torch

import action_sample_oracle as A
import selection_rows as S
import topk_oracle as O

NEG = float("-inf")


def _chain(x, target, T, lo, hi, k):
    """The reference chain in fp64, differentiable in x: (lp, ent, kept).  Selection on the unscaled x, as the kernels
    select (DESIGN §2).  The entropy's p * logp goes through a second where so that autograd, like the value, never
    forms 0 * -inf at a column with p = 0."""
    V = x.shape[-1]
    xm = x.masked_fill(x < torch.topk(x, k, dim=-1).values[..., -1:], NEG) if 0 < k < V else x
    cols = torch.arange(V)
    outside = (cols < lo) | (cols >= hi)
    z = (xm / T).masked_fill(outside, NEG)
    logp = torch.log_softmax(z, dim=-1)
    p = logp.exp()
    ent = -torch.where(p > 0, p * logp.masked_fill(p == 0, 0.0), 0.0).sum(-1)
    lp = logp.gather(-1, target.unsqueeze(-1)).squeeze(-1)
    kept = ~outside & ~(x < torch.topk(x, k, dim=-1).values[..., -1:]) if 0 < k < V else ~outside.expand_as(x)
    return lp, ent, kept


def _case(V, lo, hi, k, seed):
    x, _ = S.hard_rows(V, lo, hi, k, seed=seed)
    g = torch.Generator().manual_seed(seed + 1)
    tgt = torch.randint(lo, hi, (x.shape[0],), generator=g)
    return x.double(), tgt, torch.randn(x.shape[0], generator=g, dtype=torch.float64), \
        torch.randn(x.shape[0], generator=g, dtype=torch.float64)


V = 300
WINDOWS = [(0, V), (V - 69, V - 5)]


@pytest.mark.parametrize("win", WINDOWS)
@pytest.mark.parametrize("k", [0, 1, 5, 37, 150, V - 1])
@pytest.mark.parametrize("T", [1.0, 0.7])
def test_topk_oracle_on_hard_rows_matches_the_chain(win, k, T):
    lo, hi = win
    x, tgt, g_lp, g_h = _case(V, lo, hi, k, seed=k)
    o = O.topk_logprobs_entropy(x, tgt, T, win, k, g_lp=g_lp, g_h=g_h)
    xr = x.clone().requires_grad_(True)
    lp, ent, kept = _chain(xr, tgt, T, lo, hi, k)
    assert torch.equal(o["kept"], kept)
    assert torch.equal(torch.isnan(o["lp"]), torch.isnan(lp)) and torch.equal(torch.isneginf(o["lp"]), torch.isneginf(lp))
    fin = torch.isfinite(lp)
    torch.testing.assert_close(o["lp"][fin], lp[fin], rtol=1e-12, atol=1e-12)
    assert torch.isfinite(o["ent"]).all()
    torch.testing.assert_close(o["ent"], ent.detach(), rtol=1e-12, atol=1e-12)
    assert torch.equal(torch.signbit(o["ent"]), torch.signbit(ent.detach()))  # -0.0 on rows with no kept column
    # the closed form against autograd through the chain: g_lp through the log-probs (no NaN there: log_softmax's
    # backward at a -inf column is g (1[t] - 0)), g_H through the entropy
    (d_lp,) = torch.autograd.grad(lp, xr, grad_outputs=torch.where(torch.isnan(lp), 0.0, g_lp), retain_graph=True)
    (d_h,) = torch.autograd.grad(ent, xr, grad_outputs=g_h)
    assert torch.isfinite(o["grad"]).all()
    assert (o["grad"][~o["kept"]] == 0).all()
    torch.testing.assert_close(o["grad"], d_lp + d_h, rtol=1e-10, atol=1e-12)


def test_topk_oracle_k_past_the_finite_columns():
    """k = 14 on 16 columns of which 3 are -inf: the k-th value is -inf, every column is kept, the -inf ones with p = 0;
    the entropy and the gradient are finite and the -inf columns only get the target's g_lp."""
    x = torch.randn(2, 16, generator=torch.Generator().manual_seed(0), dtype=torch.float64)
    x[:, [2, 9, 15]] = NEG
    tgt = torch.tensor([9, 4])
    o = O.topk_logprobs_entropy(x, tgt, 1.0, None, 14, g_lp=torch.ones(2, dtype=torch.float64),
                                g_h=torch.ones(2, dtype=torch.float64))
    assert torch.isneginf(o["thr"]).all() and o["kept"].all()
    assert torch.isneginf(o["lp"][0]) and torch.isfinite(o["lp"][1])
    assert torch.isfinite(o["ent"]).all() and torch.isfinite(o["grad"]).all()
    fin = x[:, [0, 1, 3, 4, 5, 6, 7, 8, 10, 11, 12, 13, 14]]
    torch.testing.assert_close(o["ent"], -(fin.softmax(-1) * fin.log_softmax(-1)).sum(-1), rtol=1e-12, atol=0)
    assert o["grad"][0, 9] == 1.0 and (o["grad"][0, [2, 15]] == 0).all() and (o["grad"][1, [2, 9, 15]] == 0).all()


W = 64
LO = 200


def _window_chain(x, lo, hi, do_sample, T, k):
    """predict_action_batch's chain: -inf outside the window, then (sampling) / T and TopK over the whole row (selected
    on the unscaled values), log_softmax; greedy: log_softmax of the window at T = 1."""
    V = x.shape[-1]
    cols = torch.arange(V)
    z = x.masked_fill((cols < lo) | (cols >= hi), NEG)
    if do_sample:
        if 0 < k < V:
            z = z.masked_fill(z < torch.topk(z, k, dim=-1).values[..., -1:], NEG)
        z = z / T
    return torch.log_softmax(z, dim=-1)[..., lo:hi]


@pytest.mark.parametrize("do_sample,T", [(False, 1.0), (True, 1.0), (True, 0.7)])
@pytest.mark.parametrize("k", [0, 1, 5, W - 1, W, W + 3])
def test_window_logprobs_on_hard_rows_matches_the_chain(do_sample, T, k):
    rows, _ = S.hard_rows(W, 0, W, k if 0 < k < W else 0, seed=3 + k)
    x = torch.full((rows.shape[0], 320), float("nan"), dtype=torch.float64)
    x[:, LO:LO + W] = rows.double()
    got = A.window_logprobs(x, LO, LO + W, do_sample, T, k if 0 < k < W else 0)
    want = _window_chain(torch.nan_to_num(x, nan=0.0, neginf=NEG), LO, LO + W, do_sample, T, k)
    assert torch.equal(torch.isneginf(got), torch.isneginf(want)) and not torch.isnan(got).any()
    fin = torch.isfinite(want)
    torch.testing.assert_close(got[fin], want[fin], rtol=1e-12, atol=1e-12)
    assert (fin.sum(-1) > 0).all()


def test_greedy_tokens_break_ties_at_the_lowest_index():
    lo, hi = 100, 100 + 1024
    x = torch.zeros(6, 1200, dtype=torch.bfloat16)
    ties = [(31, 32), (32, 31 + 64), (0, hi - lo - 1), (5, 37, 69, 1023), (257, 256), (700, 900, 1000)]
    for r, cols in enumerate(ties):
        x[r, [lo + c for c in cols]] = 3.0
    x[:, :lo] = 9.0  # larger values outside the window do not count
    got = A.greedy_tokens(x, lo, hi)
    assert got.tolist() == [lo + min(c) for c in ties]
    for r in range(x.shape[0]):  # the same as a plain first-maximum scan
        w = x[r, lo:hi].tolist()
        assert int(got[r]) == lo + w.index(max(w))
