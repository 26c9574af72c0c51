"""Action-token sampling of the OpenVLA-OFT rollout from the logits (csrc/action_sample.cu, ops.sample_action_tokens):
the reference fixture (tests/golden/golden_action_sample.npz) through the in-place slice in greedy and sample mode,
chi-square tests of the draws against fp64 probabilities at OpenVLA's vocabulary in fp32 and bf16, window-only reads,
determinism in (seed, offset) and no host sync."""
from __future__ import annotations

import os
import sys

import numpy as np
import pytest
import torch
from scipy import stats

import action_sample_oracle as O

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
import make_golden_action_sample as G  # noqa: E402

pytestmark = pytest.mark.gpu

V_VLA = 32064
WIN_VLA = (32000 - 256, 32000)
ROWS = 1 << 16


def _ops():
    from rlinf_b200 import ops

    return ops


@pytest.fixture(scope="module")
def fx():
    return dict(np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "golden_action_sample.npz")))


def _bins(fx):
    return _ops().ActionBins(G.VOCAB, fx["bin_centers"], fx["q01"], fx["q99"], fx["mask"])


def _inplace(fx, C):
    """The fixture's logits as a [:, 1:-1] slice of a wider tensor, so the op reads it in place."""
    x = torch.from_numpy(fx[f"c{C}_logits"]).cuda()
    full = torch.full((x.shape[0], x.shape[1] + 2, G.V), float("nan"), device="cuda")
    full[:, 1:-1] = x
    return full[:, 1:-1]


@pytest.mark.parametrize("C", G.CHUNKS)
def test_fixture_greedy(fx, C):
    tok, lp, act = _ops().sample_action_tokens(_inplace(fx, C), (G.LO, G.HI), do_sample=False, seed=0, offset=0,
                                               bins=_bins(fx))
    assert tok.dtype == torch.int64 and lp.dtype == torch.float32 and act.dtype == torch.float64
    assert np.array_equal(tok.cpu().numpy(), fx[f"c{C}_greedy_tokens"])
    assert np.array_equal(act.cpu().numpy(), fx[f"c{C}_greedy_actions"])
    np.testing.assert_allclose(lp.cpu().numpy(), fx[f"c{C}_greedy_logprob"], rtol=1e-5, atol=1e-5)


@pytest.mark.parametrize("C,T,k", [(C, T, k) for C in G.CHUNKS for T, k in G.CASES])
def test_fixture_sampling(fx, C, T, k):
    tok, lp, act = _ops().sample_action_tokens(_inplace(fx, C), (G.LO, G.HI), do_sample=True, temperature=T, top_k=k,
                                               seed=11, offset=C, bins=_bins(fx))
    tok = tok.cpu().numpy()
    table = fx[f"{G.case_name(C, T, k)}_table"]
    assert ((tok >= G.LO) & (tok < G.HI)).all()
    at = np.take_along_axis(table, (tok - G.LO)[..., None], -1)[..., 0]
    assert np.isfinite(at).all()
    np.testing.assert_allclose(lp.cpu().numpy(), at, rtol=1e-5, atol=1e-5)
    want = O.detokenize(tok, G.VOCAB, fx["bin_centers"], fx["q01"], fx["q99"], fx["mask"])
    assert np.array_equal(act.cpu().numpy(), want)


def _planted(dtype, seed=0):
    """One OpenVLA logits row: a spread distribution over the window, larger values outside it."""
    g = torch.Generator().manual_seed(seed)
    row = torch.randn(V_VLA, generator=g) * 1.5
    row[:WIN_VLA[0]] += 6.0
    row[WIN_VLA[1]:] += 6.0
    return row.to(dtype)


def _chi2(counts, p):
    """p-value of a chi-square test of counts against probabilities p, bins with an expected count below 5 merged."""
    n = counts.sum()
    order = np.argsort(p)
    e, c = n * p[order], counts[order]
    groups, acc_e, acc_c = [], 0.0, 0
    for ei, ci in zip(e, c):
        acc_e += ei
        acc_c += ci
        if acc_e >= 5:
            groups.append((acc_e, acc_c))
            acc_e, acc_c = 0.0, 0
    if acc_e > 0 and groups:
        ge, gc = groups.pop()
        groups.append((ge + acc_e, gc + acc_c))
    ge = np.array([a for a, _ in groups])
    gc = np.array([b for _, b in groups], dtype=np.float64)
    if len(ge) < 2:
        return 1.0
    return stats.chisquare(gc, ge * n / ge.sum()).pvalue


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("k", [0, 1, 50, 255, 256])
def test_distribution_matches_fp64(dtype, k):
    """2^16 copies of one row (a stride-0 batch: distinct Philox subsequences of the same values)."""
    ops = _ops()
    T = 1.0 if k != 50 else 0.8
    row = _planted(dtype, seed=k)
    x = row.cuda().view(1, 1, V_VLA).expand(ROWS, 1, V_VLA)
    tok, lp, _ = ops.sample_action_tokens(x, WIN_VLA, do_sample=True, temperature=T, top_k=k, seed=1234, offset=7)
    tok, lp = tok.view(-1).cpu(), lp.view(-1).cpu()
    logp = O.window_logprobs(row.double(), *WIN_VLA, True, T, k)
    p = logp.exp().numpy()
    col = (tok - WIN_VLA[0]).numpy()
    assert ((col >= 0) & (col < 256)).all()
    assert np.isfinite(logp.numpy()[col]).all()  # filtered tokens never appear
    np.testing.assert_allclose(lp.numpy(), logp.numpy()[col], rtol=1e-5, atol=1e-5)
    if k == 1:
        am = int(row[WIN_VLA[0]:WIN_VLA[1]].float().argmax())
        assert (col == am).all() and (lp == 0).all()
        return
    counts = np.bincount(col, minlength=256)
    assert _chi2(counts, p) > 1e-6


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_reads_only_the_window(dtype):
    ops = _ops()
    g = torch.Generator(device="cuda").manual_seed(3)
    x = torch.randn(8, 56, V_VLA, device="cuda", generator=g).to(dtype)
    y = torch.full_like(x, float("nan"))
    y[..., WIN_VLA[0]:WIN_VLA[1]] = x[..., WIN_VLA[0]:WIN_VLA[1]]
    for kw in (dict(do_sample=False), dict(do_sample=True, top_k=50, temperature=0.7), dict(do_sample=True)):
        a = ops.sample_action_tokens(x, WIN_VLA, seed=5, offset=9, **kw)
        b = ops.sample_action_tokens(y, WIN_VLA, seed=5, offset=9, **kw)
        assert torch.equal(a[0], b[0]) and torch.equal(a[1].view(torch.int32), b[1].view(torch.int32))


def test_deterministic_in_seed_and_offset():
    ops = _ops()
    g = torch.Generator(device="cuda").manual_seed(4)
    x = torch.randn(64, 56, V_VLA, device="cuda", generator=g, dtype=torch.bfloat16)
    a = ops.sample_action_tokens(x, WIN_VLA, do_sample=True, top_k=50, seed=3, offset=100)
    b = ops.sample_action_tokens(x, WIN_VLA, do_sample=True, top_k=50, seed=3, offset=100)
    c = ops.sample_action_tokens(x, WIN_VLA, do_sample=True, top_k=50, seed=3, offset=101)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1].view(torch.int32), b[1].view(torch.int32))
    assert not torch.equal(a[0], c[0])
    # a row's draw depends only on (seed, offset, row, its values): the same rows inside a larger batch draw the same
    d = ops.sample_action_tokens(torch.cat([x, x]), WIN_VLA, do_sample=True, top_k=50, seed=3, offset=100)
    assert torch.equal(d[0][:64], a[0])


def test_no_host_sync(fx):
    ops = _ops()
    bins = _bins(fx)
    x = torch.randn(4, 14, V_VLA, device="cuda")
    ops.sample_action_tokens(x, WIN_VLA, do_sample=True, seed=0, offset=0, bins=bins)  # the table reaches the device
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for do_sample in (True, False):
            ops.sample_action_tokens(x, WIN_VLA, do_sample=do_sample, top_k=50, seed=0, offset=1, bins=bins)
    finally:
        torch.cuda.set_sync_debug_mode("default")
