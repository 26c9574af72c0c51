"""Top-k filtered log-probabilities fused into the LM head (csrc/lmhead_topk.cu, ops.linear_logprobs_entropy(...,
top_k=k)): agreement with the logits-level op on the fp32 X.W^T and with fp64 at OpenVLA's vocabulary, bit identity
across forced row blocks, the k = 1 cases (exactly zero dX / dW, a two-way tie of identical W rows), the 3-D slice in
place with a frozen weight, repeat-call bits and peak memory against the materialised chain."""
from __future__ import annotations

import math

import pytest
import torch

import topk_oracle as O

pytestmark = pytest.mark.gpu

V = 32064
WIN = (32000 - 256, 32000)


def _ops():
    from rlinf_b200 import ops

    return ops


def _inputs(N, H, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(N, H, generator=g, device="cuda").to(torch.bfloat16)
    w = (torch.randn(V, H, generator=g, device="cuda") * H ** -0.5)
    w[WIN[0]:WIN[1]] *= 1.5  # window columns reach the top-k set in some rows, not in others
    w = w.to(torch.bfloat16)
    tgt = torch.randint(WIN[0], WIN[1], (N,), generator=g, device="cuda")
    return x, w, tgt


def _separated(z, k, gap=1e-4):
    """rows whose k-th and (k+1)-th largest logits are more than gap apart: the kept set does not depend on rounding"""
    v = torch.topk(z, k + 1, dim=-1).values
    return (v[:, k - 1] - v[:, k]) > gap


@pytest.mark.parametrize("N,H", [(333, 1536), (2048, 4096)])
@pytest.mark.parametrize("k", [1, 50])
def test_fused_against_logits_level_and_fp64(N, H, k):
    ops = _ops()
    x, w, tgt = _inputs(N, H, seed=N + k)
    xg, wg = x.clone().requires_grad_(True), w.clone().requires_grad_(True)
    lp, ent = ops.linear_logprobs_entropy(xg, wg, tgt, 1.6, WIN, top_k=k)
    z32 = (x.float() @ w.float().T).requires_grad_(True)
    lp2, ent2 = ops.logprobs_entropy_from_logits(z32, tgt, 1.6, WIN, top_k=k)
    z64 = x.double() @ w.double().T
    o = O.topk_logprobs_entropy(z64, tgt, 1.6, WIN, k)
    ok = _separated(z64, k)
    assert ok.float().mean() > 0.9
    for a in (lp.detach(), lp2.detach()):  # identical kept sets: the same NaN and -inf rows
        assert torch.equal(torch.isnan(a)[ok], torch.isnan(o["lp"])[ok])
        assert torch.equal(torch.isneginf(a)[ok], torch.isneginf(o["lp"])[ok])
    fin = ok & torch.isfinite(o["lp"])
    assert int(fin.sum()) > 0 and int(torch.isnan(o["lp"]).sum()) > 0
    torch.testing.assert_close(lp.detach()[fin].double(), o["lp"][fin], rtol=2e-3, atol=2e-3)
    torch.testing.assert_close(ent.detach()[ok].double(), o["ent"][ok], rtol=2e-3, atol=2e-3)
    torch.testing.assert_close(lp.detach()[fin], lp2.detach()[fin], rtol=1e-4, atol=1e-4)
    # gradients against the logits-level op's, chained through the matmul in fp32
    g = torch.Generator(device="cuda").manual_seed(5)
    g_lp, g_h = torch.randn(N, device="cuda", generator=g), torch.randn(N, device="cuda", generator=g)
    g_lp = torch.where(torch.isfinite(lp.detach()), g_lp, 0.0)
    (lp * g_lp).sum().add_((ent * g_h).sum()).backward()
    (dz,) = torch.autograd.grad((lp2 * g_lp).sum() + (ent2 * g_h).sum(), z32)
    dz = torch.where(ok.unsqueeze(-1), dz, 0.0)
    rows = ok.nonzero()[:, 0]
    dx_ref = dz[rows] @ w.float()
    torch.testing.assert_close(xg.grad[rows].float(), dx_ref, rtol=3e-2, atol=3e-3)
    if bool(ok.all()):
        torch.testing.assert_close(wg.grad.float(), dz.T @ x.float(), rtol=3e-2, atol=3e-3)


def test_row_blocks_are_bit_identical(monkeypatch):
    ops = _ops()
    x, w, tgt = _inputs(3 * 128 + 77, 1024, seed=3)

    def run():
        xg, wg = x.clone().requires_grad_(True), w.clone().requires_grad_(True)
        lp, ent = ops.linear_logprobs_entropy(xg, wg, tgt, 1.3, WIN, top_k=50)
        (torch.nan_to_num(lp, nan=0.0, neginf=0.0).sum() + ent.sum()).backward()
        return lp.detach(), ent.detach(), xg.grad, wg.grad

    one = run()
    monkeypatch.setattr(ops, "LMHEAD_TOPK_ROW_BLOCK", 128)  # four blocks of one row tile
    four = run()
    for a, b in zip(one, four):
        assert torch.equal(torch.nan_to_num(a, nan=7.0), torch.nan_to_num(b, nan=7.0))


@pytest.mark.parametrize("tie", [False, True])
def test_k1_argmax_target_and_two_way_tie(tie):
    ops = _ops()
    N, H, c = 256, 512, WIN[0] + 9
    x, w, _ = _inputs(N, H, seed=4)
    x[:, :64] = 1.0
    w[c, :64] = 1.0  # logit ~64 at column c, far above every other
    if tie:
        w[c + 100] = w[c]  # an identical row: the same accumulator bits, so both are kept
    tgt = torch.full((N,), c, device="cuda")
    xg, wg = x.clone().requires_grad_(True), w.clone().requires_grad_(True)
    lp, ent = ops.linear_logprobs_entropy(xg, wg, tgt, 1.0, WIN, top_k=1)
    if tie:
        want = torch.full_like(lp, -math.log(2.0))
        torch.testing.assert_close(lp.detach(), want, rtol=2 ** -22, atol=0)
        torch.testing.assert_close(ent.detach(), -want, rtol=2 ** -22, atol=0)
    else:
        assert (lp == 0).all() and (ent == 0).all()
        (lp * torch.randn_like(lp) + ent * torch.randn_like(ent)).sum().backward()
        assert (xg.grad == 0).all() and (wg.grad == 0).all()  # the DZ mask holds exactly the forward's selection


def test_3d_slice_in_place_frozen_weight_and_repeat_bits():
    ops = _ops()
    bsz, A, H = 96, 7, 1024
    x, w, _ = _inputs(bsz * (A + 2), H, seed=6)
    hid = x.view(bsz, A + 2, H).clone().requires_grad_(True)
    tgt = torch.randint(WIN[0], WIN[1], (bsz, A), device="cuda")
    outs = []
    for _ in range(2):
        hid.grad = None
        lp, ent = ops.linear_logprobs_entropy(hid[:, 1:A + 1], w, tgt, 1.6, WIN, top_k=50)
        (torch.nan_to_num(lp, nan=0.0, neginf=0.0).sum() + ent.sum()).backward()
        outs.append((lp.detach(), ent.detach(), hid.grad.clone()))
    for a, b in zip(*outs):
        assert torch.equal(torch.nan_to_num(a, nan=7.0), torch.nan_to_num(b, nan=7.0))
    flat = hid.detach()[:, 1:A + 1].reshape(-1, H)
    lp2, ent2 = ops.linear_logprobs_entropy(flat, w, tgt.reshape(-1), 1.6, WIN, top_k=50)
    assert torch.equal(torch.nan_to_num(outs[0][0].reshape(-1), nan=7.0), torch.nan_to_num(lp2, nan=7.0))
    g = outs[0][2]
    assert (g[:, 0] == 0).all() and (g[:, A + 1] == 0).all()


def test_peak_memory_below_materialised_chain():
    ops = _ops()
    x, w, tgt = _inputs(8192, 4096, seed=8)

    def peak(fn):
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        fn()
        torch.cuda.synchronize()
        return torch.cuda.max_memory_allocated() - base

    def fused():
        xg, wg = x.clone().requires_grad_(True), w.clone().requires_grad_(True)
        lp, ent = ops.linear_logprobs_entropy(xg, wg, tgt, 1.0, WIN, top_k=50)
        (torch.nan_to_num(lp, nan=0.0, neginf=0.0).sum() + ent.sum()).backward()

    def materialised():
        xg, wg = x.clone().requires_grad_(True), w.clone().requires_grad_(True)
        lp, ent = ops.logprobs_entropy_from_logits(xg @ wg.T, tgt, 1.0, WIN, top_k=50)
        (torch.nan_to_num(lp, nan=0.0, neginf=0.0).sum() + ent.sum()).backward()

    assert peak(fused) < peak(materialised)
