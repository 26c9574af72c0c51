"""Action-token sampling fused into the LM head (csrc/lmhead_sample.cu, ops.linear_sample_action_tokens): bit identity
with the logits-level sampler where fp32 accumulation is exact, fp64 log-probs and a chi-square test at OFT's rollout
shape, weight rows outside the window never read, determinism and no host sync."""
from __future__ import annotations

import numpy as np
import pytest
import torch
from scipy import stats

import action_sample_oracle as O

pytestmark = pytest.mark.gpu

V_VLA = 32064
WIN_VLA = (32000 - 256, 32000)


def _ops():
    from rlinf_b200 import ops

    return ops


def _bins():
    edges = np.linspace(-1, 1, 256)
    mask = np.ones(7, dtype=bool)
    mask[6] = False
    return _ops().ActionBins(32000, (edges[:-1] + edges[1:]) / 2, np.linspace(-1.0, -0.2, 7), np.linspace(0.3, 1.5, 7),
                             mask)


def _bits(t):
    return t.view(torch.int32) if t.dtype == torch.float32 else t.view(torch.int64)


def _int_grid(bsz, L, H, V, seed):
    """hidden [bsz, L + 2, H] and W [V, H] on a small-integer bf16 grid: every fp32 dot product is exact."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    hidden = torch.randint(-3, 4, (bsz, L + 2, H), device="cuda", generator=g).to(torch.bfloat16)
    w = torch.randint(-3, 4, (V, H), device="cuda", generator=g).to(torch.bfloat16)
    return hidden, w


@pytest.mark.parametrize("bsz,L,H,win", [(4, 56, 256, WIN_VLA), (3, 7, 128, (31700, 32050)), (300, 14, 64, (5, 6))])
@pytest.mark.parametrize("mode", [dict(do_sample=False), dict(do_sample=True), dict(do_sample=True, top_k=50,
                                                                                     temperature=0.7)])
def test_fused_equals_logits_level_on_exact_grid(bsz, L, H, win, mode):
    ops = _ops()
    hidden, w = _int_grid(bsz, L, H, V_VLA, seed=bsz + H)
    h = hidden[:, 1:-1]  # the in-place slice of the last hidden state
    logits = (h.double() @ w.double().T).float()
    bins = _bins() if L % 7 == 0 else None
    a = ops.linear_sample_action_tokens(h, w, win, seed=17, offset=3, bins=bins, **mode)
    b = ops.sample_action_tokens(logits, win, seed=17, offset=3, bins=bins, **mode)
    assert torch.equal(a[0], b[0]) and torch.equal(_bits(a[1]), _bits(b[1]))
    assert (a[2] is None and b[2] is None) or torch.equal(_bits(a[2]), _bits(b[2]))


def test_fused_at_rollout_shape_vs_fp64():
    """bsz 256 x 56 positions, H = 4096, V = 32064: log-probs against fp64 and the draws against their probabilities."""
    ops = _ops()
    g = torch.Generator(device="cuda").manual_seed(9)
    N, H = 256 * 56, 4096
    hidden = (torch.randn(256, 56, H, device="cuda", generator=g) * 0.5).to(torch.bfloat16)
    w = (torch.randn(V_VLA, H, device="cuda", generator=g) * 0.05).to(torch.bfloat16)
    tok, lp, _ = ops.linear_sample_action_tokens(hidden, w, WIN_VLA, do_sample=True, top_k=50, seed=2, offset=0)
    z = hidden.reshape(N, H).double() @ w[WIN_VLA[0]:WIN_VLA[1]].double().T  # [N, 256] fp64 logits of the window
    logp = O.window_logprobs(z, 0, 256, True, 1.0, 50)
    col = tok.reshape(N) - WIN_VLA[0]
    assert ((col >= 0) & (col < 256)).all()
    at = logp.gather(1, col[:, None])[:, 0]
    fin = torch.isfinite(at)
    assert fin.float().mean() > 0.999  # a near-tie at the 50th value can differ between fp32 and fp64
    torch.testing.assert_close(lp.reshape(N).double()[fin], at[fin], rtol=1e-4, atol=1e-4)
    # aggregated chi-square: counts per column against the summed per-row probabilities
    p = logp.exp().sum(0).cpu().numpy()
    counts = torch.bincount(col, minlength=256).cpu().numpy().astype(np.float64)
    keep = p >= 5
    e = np.append(p[keep], p[~keep].sum())
    c = np.append(counts[keep], counts[~keep].sum())
    if e[-1] < 5:
        e, c = e[:-1], c[:-1]
    assert stats.chisquare(c, e * c.sum() / e.sum()).pvalue > 1e-6


def test_fused_reads_only_the_window_rows():
    ops = _ops()
    hidden, w = _int_grid(8, 56, 256, V_VLA, seed=1)
    h = hidden[:, 1:-1]
    w_nan = torch.full_like(w, float("nan"))
    w_nan[WIN_VLA[0]:WIN_VLA[1]] = w[WIN_VLA[0]:WIN_VLA[1]]
    for mode in (dict(do_sample=False), dict(do_sample=True, top_k=8)):
        a = ops.linear_sample_action_tokens(h, w, WIN_VLA, seed=4, offset=4, bins=_bins(), **mode)
        b = ops.linear_sample_action_tokens(h, w_nan, WIN_VLA, seed=4, offset=4, bins=_bins(), **mode)
        for u, v in zip(a, b):
            assert torch.equal(_bits(u), _bits(v))


def test_fused_deterministic_and_no_host_sync():
    ops = _ops()
    hidden, w = _int_grid(16, 56, 512, V_VLA, seed=2)
    h = hidden[:, 1:-1]
    bins = _bins()
    a = ops.linear_sample_action_tokens(h, w, WIN_VLA, do_sample=True, seed=8, offset=1, bins=bins)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        b = ops.linear_sample_action_tokens(h, w, WIN_VLA, do_sample=True, seed=8, offset=1, bins=bins)
        c = ops.linear_sample_action_tokens(h, w, WIN_VLA, do_sample=True, seed=8, offset=2, bins=bins)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert torch.equal(a[0], b[0]) and torch.equal(_bits(a[1]), _bits(b[1])) and torch.equal(a[2], b[2])
    assert not torch.equal(a[0], c[0])
