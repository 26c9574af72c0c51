"""Plain OpenVLA's generate step on the device (ops.sample_action_tokens / ops.linear_sample_action_tokens with
out= / column= and counter=): the transformers-generate fixture (tests/golden/golden_openvla_decode.npz) greedy and
sampled, logits-level and fused; the device counter against host offsets; a whole 7-step decode and the OFT call in one
CUDA graph; and fp64 at the rollout geometry (B = 256, H = 4096, V = 32064)."""
from __future__ import annotations

import os
import sys

import numpy as np
import pytest
import torch
from scipy import stats

import action_sample_oracle as O

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_golden_openvla_decode as G  # noqa: E402

V = 32064
WIN = (G.LO, G.HI)
A = G.ADIM
SAMPLED = [("T1_k0", 1.0, 0), ("T1_k50", 1.0, 50), ("T0.6_k50", 0.6, 50), ("tie_T1_k50", 1.0, 50)]


def _ops():
    from rlinf_b200 import ops

    return ops


@pytest.fixture(scope="module")
def fx():
    return dict(np.load(os.path.join(HERE, "golden", "golden_openvla_decode.npz")))


def _bins(fx):
    return _ops().ActionBins(G.VOCAB, fx["bin_centers"], fx["q01"], fx["q99"], fx["mask"])


def _bits(t):
    return t.view(torch.int32) if t.dtype == torch.float32 else t.view(torch.int64)


def _buffers(bsz, bins=True):
    return (torch.empty(bsz, A, dtype=torch.int64, device="cuda"), torch.empty(bsz, A, device="cuda"),
            torch.empty(bsz, A, dtype=torch.float64, device="cuda") if bins else None)


def _full(window_rows):
    """[n, 1, V] fp32 logits: the window rows in [LO, HI), NaN everywhere else (never read)."""
    w = torch.as_tensor(window_rows, device="cuda")
    x = torch.full((w.shape[0], 1, V), float("nan"), device="cuda")
    x[:, 0, G.LO:G.HI] = w
    return x


def _weight(w_window):
    """[V, 64] bf16 lm_head.weight: the window rows, NaN outside."""
    w = torch.full((V, G.HID), float("nan"), dtype=torch.bfloat16, device="cuda")
    w[G.LO:G.HI] = torch.as_tensor(w_window, device="cuda").to(torch.bfloat16)
    return w


@pytest.mark.parametrize("n", ["greedy", "tie_greedy"])
def test_greedy_logits_level_matches_generate(fx, n):
    ops = _ops()
    bins = _bins(fx)
    out = _buffers(G.B)
    for j in range(A):
        r = ops.sample_action_tokens(_full(fx[f"{n}_logits"][:, j]), WIN, do_sample=False, seed=0, offset=0, bins=bins,
                                     out=out, column=j)
        assert r is out or all(a is b for a, b in zip(r, out))
    assert np.array_equal(out[0].cpu().numpy(), fx[f"{n}_tokens"])
    assert np.array_equal(out[2].cpu().numpy().view(np.int64), fx[f"{n}_actions"].view(np.int64))
    np.testing.assert_allclose(out[1].cpu().numpy(), fx[f"{n}_logprob"], rtol=1e-6, atol=4e-6)


@pytest.mark.parametrize("n", ["greedy", "tie_greedy"])
def test_greedy_fused_matches_generate(fx, n):
    ops = _ops()
    bins = _bins(fx)
    ww = fx[("tie_" if n.startswith("tie") else "") + "w_window"]
    w = _weight(ww)
    hidden = torch.as_tensor(fx[f"{n}_hidden"], device="cuda").to(torch.bfloat16)
    out = _buffers(G.B)
    ctr = torch.zeros(1, dtype=torch.int64, device="cuda")
    for j in range(A):
        ops.linear_sample_action_tokens(hidden[:, j], w, WIN, do_sample=False, seed=0, counter=ctr, bins=bins, out=out,
                                        column=j)
    assert int(ctr) == A
    assert np.array_equal(out[0].cpu().numpy(), fx[f"{n}_tokens"])
    assert np.array_equal(out[2].cpu().numpy().view(np.int64), fx[f"{n}_actions"].view(np.int64))
    # the fp32 accumulator against fp64 on the same bf16 inputs, and against generate's bf16-rounded logits
    z = hidden.double() @ torch.as_tensor(ww, device="cuda").double().T
    want = torch.log_softmax(z, -1).gather(-1, out[0][..., None] - G.LO)[..., 0]
    torch.testing.assert_close(out[1].double(), want, rtol=1e-4, atol=1e-4)
    # a log-softmax moves by at most twice the largest change of its inputs: here generate's bf16 rounding of the logits
    dz = (z - torch.as_tensor(fx[f"{n}_logits"], device="cuda").double()).abs().amax(-1)
    ref = torch.as_tensor(fx[f"{n}_logprob"], device="cuda").double()
    assert ((out[1].double() - ref).abs() <= 2 * dz + 1e-5).all()


@pytest.mark.parametrize("n,T,k", SAMPLED)
def test_sampled_draws_lie_in_the_kept_set(fx, n, T, k):
    """R draws per (step, row) through the counter: every token has a finite processed score, and its log-prob is
    log_softmax(processed scores)[token]."""
    ops = _ops()
    bins = _bins(fx)
    R = 512
    rows = np.repeat(fx[f"{n}_logits"], R, axis=0)  # [B R, 7, 256]
    out = _buffers(G.B * R)
    ctr = torch.full((1,), 1 << 40, dtype=torch.int64, device="cuda")
    for j in range(A):
        ops.sample_action_tokens(_full(rows[:, j]), WIN, do_sample=True, temperature=T, top_k=k, seed=21, counter=ctr,
                                 bins=bins, out=out, column=j)
    assert int(ctr) == (1 << 40) + A
    scores = torch.as_tensor(np.repeat(fx[f"{n}_scores"], R, axis=0), device="cuda").double()
    col = out[0] - G.LO
    assert ((col >= 0) & (col < 256)).all()
    at = scores.gather(-1, col[..., None])[..., 0]
    assert torch.isfinite(at).all()
    want = torch.log_softmax(scores, -1).gather(-1, col[..., None])[..., 0]
    torch.testing.assert_close(out[1].double(), want, rtol=1e-5, atol=1e-5)
    act = O.detokenize(out[0].cpu().numpy(), G.VOCAB, fx["bin_centers"], fx["q01"], fx["q99"], fx["mask"])
    assert np.array_equal(out[2].cpu().numpy().view(np.int64), act.view(np.int64))


@pytest.mark.parametrize("n,T,k", SAMPLED)
def test_sampled_distribution_chi_square(fx, n, T, k):
    ops = _ops()
    D = 1 << 16
    row = fx[f"{n}_logits"][1, 3]
    ctr = torch.full((1,), 7, dtype=torch.int64, device="cuda")
    tok, lp, _ = ops.sample_action_tokens(_full(np.repeat(row[None], D, 0)), WIN, do_sample=True, temperature=T,
                                          top_k=k, seed=5, counter=ctr)
    p = torch.softmax(torch.as_tensor(fx[f"{n}_scores"][1, 3]).double(), -1).numpy() * D
    counts = torch.bincount((tok[:, 0] - G.LO), minlength=256).cpu().numpy().astype(np.float64)
    assert counts[p == 0].sum() == 0
    keep = p >= 5
    e = np.append(p[keep], p[~keep].sum())
    c = np.append(counts[keep], counts[~keep].sum())
    if e[-1] < 5:
        e, c = e[:-1], c[:-1]
    assert stats.chisquare(c, e * c.sum() / e.sum()).pvalue > 1e-6


def test_counter_equals_host_offset_and_advances():
    ops = _ops()
    gen = torch.Generator(device="cuda").manual_seed(3)
    logits = torch.randn(96, 1, V, device="cuda", generator=gen) * 2
    hidden = (torch.randn(96, 128, device="cuda", generator=gen)).to(torch.bfloat16)
    w = (torch.randn(V, 128, device="cuda", generator=gen) * 0.2).to(torch.bfloat16)
    kw = dict(do_sample=True, temperature=0.8, top_k=50, seed=99)
    for c in (0, 12345, 1 << 62):
        ctr = torch.full((1,), c, dtype=torch.int64, device="cuda")
        a = ops.sample_action_tokens(logits, WIN, counter=ctr, **kw)
        b = ops.sample_action_tokens(logits, WIN, offset=c, **kw)
        assert int(ctr) == c + 1
        assert torch.equal(a[0], b[0]) and torch.equal(_bits(a[1]), _bits(b[1]))
        f1 = ops.linear_sample_action_tokens(hidden, w, WIN, counter=ctr, **kw)
        f2 = ops.linear_sample_action_tokens(hidden, w, WIN, offset=c + 1, **kw)
        assert int(ctr) == c + 2
        assert torch.equal(f1[0], f2[0]) and torch.equal(_bits(f1[1]), _bits(f2[1]))
        # a step call writes the dense call's outputs into its column; the fused [bsz, H] step tiles the rows as the
        # dense [N, H] call does
        out = _buffers(96, bins=False)
        for j in (0, 4, 6):
            ops.sample_action_tokens(logits, WIN, offset=c, out=out, column=j, **kw)
            assert torch.equal(out[0][:, j], b[0][:, 0]) and torch.equal(_bits(out[1][:, j]), _bits(b[1][:, 0]))
            ops.linear_sample_action_tokens(hidden, w, WIN, offset=c + 1, out=out, column=j, **kw)
            assert torch.equal(out[0][:, j], f2[0]) and torch.equal(_bits(out[1][:, j]), _bits(f2[1]))
    # the plain path stays as it was: the OFT [bsz, 56] call through the counter equals the offset call
    x = torch.randn(4, 56, V, device="cuda", generator=gen)
    ctr = torch.full((1,), 5, dtype=torch.int64, device="cuda")
    bins = ops.ActionBins(32000, np.linspace(-1, 1, 255), np.zeros(7), np.ones(7))
    a = ops.sample_action_tokens(x, WIN, counter=ctr, bins=bins, **kw)
    b = ops.sample_action_tokens(x, WIN, offset=5, bins=bins, **kw)
    for u, v in zip(a, b):
        assert torch.equal(_bits(u), _bits(v))


def _decode(ops, h0, w, E, M, bins, ctr, out):
    """A 7-step decode: the fused step, then a stand-in backbone step (embedding[token] @ M) for the next hidden."""
    h = h0
    for j in range(A):
        ops.linear_sample_action_tokens(h, w, WIN, do_sample=True, temperature=1.0, top_k=50, seed=11, counter=ctr,
                                        bins=bins, out=out, column=j)
        h = torch.tanh(E[out[0][:, j]].float() @ M).to(torch.bfloat16)
    return out


def test_seven_step_decode_in_one_cuda_graph():
    ops = _ops()
    gen = torch.Generator(device="cuda").manual_seed(8)
    B, H = 64, 256
    w = (torch.randn(V, H, device="cuda", generator=gen) * 0.2).to(torch.bfloat16)
    E = torch.randn(V, H, device="cuda", generator=gen).to(torch.bfloat16)
    M = torch.randn(H, H, device="cuda", generator=gen) / H ** 0.5 * 3
    h0 = torch.randn(B, H, device="cuda", generator=gen).to(torch.bfloat16)
    bins = ops.ActionBins(32000, np.linspace(-1, 1, 255), np.linspace(-1, 0, 7), np.linspace(0.5, 2, 7))
    ctr = torch.full((1,), 100, dtype=torch.int64, device="cuda")
    out = _buffers(B)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):  # warm-up: the bins tables reach the device, the allocator and cuBLAS settle
        _decode(ops, h0, w, E, M, bins, ctr, out)
    torch.cuda.current_stream().wait_stream(s)
    ctr.fill_(100)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        torch.cuda.set_sync_debug_mode("error")
        try:
            _decode(ops, h0, w, E, M, bins, ctr, out)
        finally:
            torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()
    assert int(ctr) == 100  # capture runs nothing
    torch.cuda.set_sync_debug_mode("error")
    try:
        graph.replay()
        r1 = [t.clone() for t in out]
        graph.replay()
        r2 = [t.clone() for t in out]
        ctr_e = torch.full((1,), 100, dtype=torch.int64, device="cuda")
        eager = _decode(ops, h0, w, E, M, bins, ctr_e, _buffers(B))
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert int(ctr) == 114 and int(ctr_e) == 107
    for u, v in zip(r1, eager):
        assert torch.equal(_bits(u), _bits(v))
    assert not torch.equal(r1[0], r2[0])
    assert ((r1[0] >= G.LO) & (r1[0] < G.HI)).all() and ((r2[0] >= G.LO) & (r2[0] < G.HI)).all()


def test_oft_call_in_a_cuda_graph():
    ops = _ops()
    gen = torch.Generator(device="cuda").manual_seed(4)
    bsz, H = 8, 256
    hidden = torch.randn(bsz, 58, H, device="cuda", generator=gen).to(torch.bfloat16)
    h = hidden[:, 1:-1]  # [bsz, 56, H] read in place
    w = (torch.randn(V, H, device="cuda", generator=gen) * 0.2).to(torch.bfloat16)
    bins = ops.ActionBins(32000, np.linspace(-1, 1, 255), np.zeros(7), np.ones(7))
    ctr = torch.full((1,), 40, dtype=torch.int64, device="cuda")
    kw = dict(do_sample=True, top_k=50, seed=2, bins=bins)
    ops.linear_sample_action_tokens(h, w, WIN, counter=ctr, **kw)  # warm-up
    ctr.fill_(40)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        res = ops.linear_sample_action_tokens(h, w, WIN, counter=ctr, **kw)
    torch.cuda.set_sync_debug_mode("error")
    try:
        graph.replay()
        r1 = [t.clone() for t in res]
        graph.replay()
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert int(ctr) == 42
    want = ops.linear_sample_action_tokens(h, w, WIN, offset=40, **kw)
    for u, v in zip(r1, want):
        assert torch.equal(_bits(u), _bits(v))
    assert r1[0].shape == (bsz, 56) and not torch.equal(r1[0], res[0])


def test_rollout_geometry_against_fp64():
    """B = 256, H = 4096, V = 32064, 7 steps at the training (T = 1, k = 50) and greedy settings."""
    ops = _ops()
    gen = torch.Generator(device="cuda").manual_seed(6)
    B, H = 256, 4096
    w = (torch.randn(V, H, device="cuda", generator=gen) * 0.05).to(torch.bfloat16)
    hs = (torch.randn(A, B, H, device="cuda", generator=gen) * 0.5).to(torch.bfloat16)
    ctr = torch.zeros(1, dtype=torch.int64, device="cuda")
    samp, greedy = _buffers(B, bins=False), _buffers(B, bins=False)
    for j in range(A):
        ops.linear_sample_action_tokens(hs[j], w, WIN, do_sample=True, top_k=50, seed=1, counter=ctr, out=samp,
                                        column=j)
        ops.linear_sample_action_tokens(hs[j], w, WIN, do_sample=False, seed=1, counter=ctr, out=greedy, column=j)
    assert int(ctr) == 2 * A
    z = torch.einsum("jbh,vh->bjv", hs.double(), w[G.LO:G.HI].double())  # [B, 7, 256]
    lp_s = O.window_logprobs(z, 0, 256, True, 1.0, 50).gather(-1, samp[0][..., None] - G.LO)[..., 0]
    fin = torch.isfinite(lp_s)
    assert fin.float().mean() > 0.999  # a near-tie at the 50th value can differ between fp32 and fp64
    torch.testing.assert_close(samp[1].double()[fin], lp_s[fin], rtol=1e-4, atol=1e-4)
    top2 = z.topk(2, -1).values
    clear = (top2[..., 0] - top2[..., 1]) > 1e-3
    assert clear.float().mean() > 0.99
    assert torch.equal(greedy[0][clear], z.argmax(-1)[clear] + G.LO)
    lp_g = O.window_logprobs(z, 0, 256, False).gather(-1, greedy[0][..., None] - G.LO)[..., 0]
    torch.testing.assert_close(greedy[1].double(), lp_g, rtol=1e-4, atol=1e-4)
