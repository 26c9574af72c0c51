"""Top-k filtered log-probabilities and entropies from the logits (csrc/topk.cu, ops.logprobs_entropy_from_logits(...,
top_k=k)): the reference fixture (tests/golden/golden_topk.npz) through the in-place [:, -7C-1:-1] slice, the fp64
oracle (tests/topk_oracle.py) at OpenVLA's vocabulary in fp32 and bf16, bit identity with the unfiltered op when top_k
does not filter, the k = 1 cases and repeat-call bit identity."""
from __future__ import annotations

import math
import os
import sys

import numpy as np
import pytest
import torch

import topk_oracle as O

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
import make_golden_topk as G  # noqa: E402

pytestmark = pytest.mark.gpu

V_VLA = 32064
WIN_VLA = (32000 - 256, 32000)
KS = (1, 50, 256, 4096, V_VLA - 1)


def _ops():
    from rlinf_b200 import ops

    return ops


@pytest.fixture(scope="module")
def fx():
    return dict(np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "golden_topk.npz")))


@pytest.mark.parametrize("C,T,k", [(C, T, k) for C in G.CHUNKS for T, k in G.CASES])
def test_fixture_through_the_inplace_slice(fx, C, T, k):
    ops = _ops()
    full = torch.from_numpy(fx[f"c{C}_logits"]).cuda().requires_grad_(True)
    R = G.ADIM * C
    S = full.shape[1]
    tgt = torch.from_numpy(fx[f"c{C}_target"]).cuda()
    n = G.case_name(C, T, k)
    lp, ent = ops.logprobs_entropy_from_logits(full[:, S - R - 1:-1], tgt, T, (G.LO, G.HI), top_k=k)
    want_lp, want_ent = fx[f"{n}_logprob"], fx[f"{n}_entropy"]
    got_lp, got_ent = lp.detach().cpu().numpy(), ent.detach().cpu().numpy()
    assert np.array_equal(np.isnan(got_lp), np.isnan(want_lp))
    assert np.array_equal(np.isneginf(got_lp), np.isneginf(want_lp))
    fin = np.isfinite(want_lp)
    np.testing.assert_allclose(got_lp[fin], want_lp[fin], rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(got_ent, want_ent, rtol=1e-5, atol=1e-5)
    assert np.signbit(got_ent[np.isnan(got_lp)]).all()  # -0.0 on rows with no kept column, as the reference
    # the log-prob-only gradient against the reference's autograd
    g_lp = torch.from_numpy(fx[f"c{C}_g_lp"]).cuda()
    (d,) = torch.autograd.grad(lp, full, grad_outputs=g_lp, retain_graph=True)
    d = d.cpu()
    assert (d[:, :S - R - 1] == 0).all() and (d[:, S - 1:] == 0).all()
    want = fx[f"{n}_grad_lp"]
    np.testing.assert_allclose(d[:, S - R - 1:-1].numpy(), want, rtol=1e-4, atol=1e-6)
    assert np.array_equal(d[:, S - R - 1:-1].numpy() == 0, want == 0)
    # the combined gradient against the oracle's closed form (the reference's is NaN, DESIGN §2)
    g_h = torch.from_numpy(fx[f"c{C}_g_h"]).cuda()
    (d2,) = torch.autograd.grad((lp, ent), full, grad_outputs=(g_lp, g_h))
    x = torch.from_numpy(fx[f"c{C}_logits"])[:, S - R - 1:-1]
    o = O.topk_logprobs_entropy(x, tgt.cpu(), T, (G.LO, G.HI), k, g_lp=g_lp.cpu(), g_h=g_h.cpu())
    got = d2[:, S - R - 1:-1].cpu().double()
    torch.testing.assert_close(got, o["grad"], rtol=1e-4, atol=1e-6)
    assert torch.equal(got != 0, o["grad"] != 0)


def _vla_logits(dtype, seed=0, bsz=288, A=7):
    """[bsz, A + 2, V] logits (the OpenVLA slice [:, -A-1:-1] holds bsz * A = 2016 rows), action bins lifted so that
    rows with and without kept columns both occur at small k."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(bsz, A + 2, V_VLA, device="cuda", generator=g) * 2.5
    x[..., WIN_VLA[0]:WIN_VLA[1]] += 2.0
    x = x.to(dtype)
    tgt = torch.randint(WIN_VLA[0], WIN_VLA[1], (bsz, A), device="cuda", generator=g)
    return x, tgt


@pytest.mark.parametrize("dtype,T", [(torch.float32, 1.0), (torch.float32, 1.6), (torch.bfloat16, 1.0)])
@pytest.mark.parametrize("k", KS)
def test_openvla_scale_against_fp64(dtype, T, k):
    ops = _ops()
    full, tgt = _vla_logits(dtype, seed=k)
    full.requires_grad_(True)
    A = tgt.shape[1]
    sl = full[:, 1:A + 1]  # = full[:, -A-1:-1]
    lp, ent = ops.logprobs_entropy_from_logits(sl, tgt, T, WIN_VLA, top_k=k)
    g = torch.Generator(device="cuda").manual_seed(99)
    g_lp = torch.randn(tgt.shape, device="cuda", generator=g)
    g_h = torch.randn(tgt.shape, device="cuda", generator=g)
    (d,) = torch.autograd.grad((lp, ent), full, grad_outputs=(g_lp, g_h))
    x = sl.detach()
    o = O.topk_logprobs_entropy(x, tgt, T, WIN_VLA, k, g_lp=g_lp, g_h=g_h)
    got_lp, got_ent = lp.detach().double(), ent.detach().double()
    assert torch.equal(torch.isnan(got_lp), torch.isnan(o["lp"]))
    assert torch.equal(torch.isneginf(got_lp), torch.isneginf(o["lp"]))
    fin = torch.isfinite(o["lp"])
    torch.testing.assert_close(got_lp[fin], o["lp"][fin], rtol=1e-4, atol=1e-5)
    torch.testing.assert_close(got_ent, o["ent"], rtol=1e-4, atol=1e-5)
    dg = d[:, 1:A + 1].double()
    assert (d[:, 0] == 0).all() and (d[:, A + 1] == 0).all()
    # identical kept sets: the gradient vanishes off the kept set, and on it only where the closed form is 0 (k = 1
    # with the target on the one kept column)
    assert torch.equal(dg != 0, o["grad"] != 0) and not ((dg != 0) & ~o["kept"]).any()
    tol = 1e-4 if dtype == torch.float32 else 8e-3  # bf16 gradient: one rounding of each element
    torch.testing.assert_close(dg, o["grad"], rtol=tol, atol=1e-6)
    if k == 1:
        assert 0 < int(torch.isnan(got_lp).sum()) < got_lp.numel()  # rows with and without a kept column


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_no_filter_is_bit_identical(dtype):
    ops = _ops()
    full, tgt = _vla_logits(dtype, seed=5, bsz=64)
    g = torch.Generator(device="cuda").manual_seed(1)
    g_lp, g_h = torch.randn(tgt.shape, device="cuda", generator=g), torch.randn(tgt.shape, device="cuda", generator=g)

    def run(**kw):
        x = full.clone().requires_grad_(True)
        lp, ent = ops.logprobs_entropy_from_logits(x[:, 1:8], tgt, 1.3, WIN_VLA, **kw)
        (d,) = torch.autograd.grad((lp, ent), x, grad_outputs=(g_lp, g_h))
        return lp, ent, d

    base = run()
    for k in (0, -1, V_VLA, V_VLA + 7):
        got = run(top_k=k)
        for a, b in zip(got, base):
            assert torch.equal(a.view(torch.int8 if a.dtype == torch.bfloat16 else torch.int32),
                               b.view(torch.int8 if b.dtype == torch.bfloat16 else torch.int32)), k


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_k1_target_is_argmax(dtype):
    ops = _ops()
    full, _ = _vla_logits(torch.float32, seed=7, bsz=32)
    full[..., WIN_VLA[0] + 17] = 40.0  # the row maximum, inside the window
    full = full.to(dtype).requires_grad_(True)
    tgt = torch.full((32, 7), WIN_VLA[0] + 17, device="cuda")
    lp, ent = ops.logprobs_entropy_from_logits(full[:, 1:8], tgt, 1.0, WIN_VLA, top_k=1)
    assert (lp == 0).all() and (ent == 0).all()
    (d,) = torch.autograd.grad((lp, ent), full, grad_outputs=(torch.randn_like(lp), torch.randn_like(ent)))
    assert (d == 0).all()


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_k1_two_way_tie(dtype):
    ops = _ops()
    full, _ = _vla_logits(torch.float32, seed=8, bsz=32)
    full[..., WIN_VLA[0] + 3] = 40.0
    full[..., WIN_VLA[0] + 200] = 40.0
    full = full.to(dtype)
    tgt = torch.full((32, 7), WIN_VLA[0] + 200, device="cuda")
    lp, ent = ops.logprobs_entropy_from_logits(full[:, 1:8], tgt, 1.0, WIN_VLA, top_k=1)
    want = torch.tensor(-math.log(2.0), dtype=torch.float32)
    torch.testing.assert_close(lp.cpu(), want.expand(lp.shape), rtol=2 ** -22, atol=0)
    torch.testing.assert_close(ent.cpu(), (-want).expand(ent.shape), rtol=2 ** -22, atol=0)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_repeat_calls_same_bits(dtype):
    ops = _ops()
    full, tgt = _vla_logits(dtype, seed=11, bsz=128)
    g_lp = torch.randn(tgt.shape, device="cuda")
    g_h = torch.randn(tgt.shape, device="cuda")
    outs = []
    for _ in range(2):
        x = full.clone().requires_grad_(True)
        lp, ent = ops.logprobs_entropy_from_logits(x[:, 1:8], tgt, 1.6, WIN_VLA, top_k=50)
        (d,) = torch.autograd.grad((lp, ent), x, grad_outputs=(g_lp, g_h))
        outs.append((lp, ent, d))
    for a, b in zip(*outs):
        assert torch.equal(torch.nan_to_num(a, nan=7.0), torch.nan_to_num(b, nan=7.0))
