"""The OpenVLA value head on the GPU (csrc/vla_value_head.cu through ops.vla_value_head): the reference fixture, forward
and backward against fp64 next to the eager bf16 nn.Sequential, batch invariance, backward determinism, skipped
gradients, no host sync, CUDA-graph capture, launch counts, and the chain into the embodied actor-critic PPO loss."""
from __future__ import annotations

import os
import re
import sys

import numpy as np
import pytest
import torch

import vla_value_head_oracle as OR

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
sys.path.insert(0, os.path.dirname(HERE))
import make_golden_vla_value_head as G  # noqa: E402

pytestmark = pytest.mark.gpu

DEV = "cuda"
NAMES = ("v", "dx", "dw0", "db0", "dw1", "db1", "dw2")
KERNELS = re.compile(r"(l0_fwd_kernel|tail_fwd_kernel|tail_bwd_kernel|::gemm_kernel<|small_grads_kernel)")


def make(N, H, O, seed, dev=DEV):
    """bf16 x [N, H], parameters (w0, b0, w1, b1, w2) and gv [N, O], at the scales of make_golden_vla_value_head."""
    g = torch.Generator().manual_seed(seed)

    def r(*shape, std=1.0):
        return (torch.randn(*shape, generator=g) * std).to(torch.bfloat16).to(dev)

    params = [r(512, H, std=(2.0 / 512) ** 0.5), r(512, std=0.1), r(128, 512, std=(2.0 / 128) ** 0.5),
              r(128, std=0.1), r(O, 128, std=0.02)]
    return r(N, H), params, r(N, O)


def run_op(x, params, gv, x_grad=True, p_grad=(True,) * 5):
    from rlinf_b200 import ops

    x = x.detach().requires_grad_(x_grad)
    ps = [p.detach().requires_grad_(q) for p, q in zip(params, p_grad)]
    v = ops.vla_value_head(x, *ps)
    wrt = [t for t in [x] + ps if t.requires_grad]
    grads = iter(torch.autograd.grad(v, wrt, gv)) if wrt else iter(())
    out = {"v": v.detach()}
    for name, t in zip(NAMES[1:], [x] + ps):
        out[name] = next(grads) if t.requires_grad else None
    return out


def run_eager(x, params, gv):
    H, O = x.shape[1], params[4].shape[0]
    seq = torch.nn.Sequential(torch.nn.Linear(H, 512), torch.nn.GELU(), torch.nn.Linear(512, 128), torch.nn.GELU(),
                              torch.nn.Linear(128, O, bias=False)).to(DEV, torch.bfloat16)
    with torch.no_grad():
        for p, q in zip(seq.parameters(), params):
            p.copy_(q)
    x = x.detach().clone().requires_grad_(True)
    v = seq(x)
    grads = torch.autograd.grad(v, [x] + list(seq.parameters()), gv)
    return dict(zip(NAMES, [v.detach()] + list(grads)))


def run_fp64(x, params, gv, bf16=False):
    v, saved = OR.forward(x, *params, bf16=bf16)
    out = OR.backward(x, params[0], params[2], params[4], saved, gv, bf16=bf16)
    out["v"] = v
    return out


def errors(got, ref):
    d = got.double() - ref
    return d.abs().max().item(), d.pow(2).mean().sqrt().item()


@pytest.mark.parametrize("H,O", [(H, O) for H in G.HS for O in G.OS])
def test_fixture_cases(H, O):
    """The fixture's bf16 module outputs, within one bf16 rounding of the largest element (the CPU module's fp32 sums
    run in another order; a flipped rounding of an intermediate moves an output by at most a few of its ulps)."""
    f = np.load(G.OUT)
    inp = {k: v.to(torch.bfloat16).to(DEV) for k, v in G.make_inputs(H, O).items()}
    got = run_op(inp["x"], [inp[k] for k in ("w0", "b0", "w1", "b1", "w2")], inp["gv"])
    got["dw0"], got["dw1"] = got["dw0"][G.W0_ROWS], got["dw1"][G.W1_ROWS]
    for k in NAMES:
        ref = G.from_bits(f[f"{G.case_name(H, O, 'bf16')}_{k}"]).double().to(DEV)
        mx, rms = errors(got[k], ref)
        assert mx <= 2 ** -6 * ref.abs().max().item() and rms <= 2 ** -8 * ref.pow(2).mean().sqrt().item(), (k, mx, rms)


@pytest.mark.parametrize("seed", [0, 1, 2])
@pytest.mark.parametrize("N", [0, 1, 40, 127, 1024, 4096])
@pytest.mark.parametrize("O", [1, 8, 25])
def test_against_fp64_no_worse_than_eager(O, N, seed):
    """Max-abs and RMS error against the exact fp64 result, per output, no worse than the eager bf16 nn.Sequential's:
    ours <= 1.25 x eager's plus one bf16 rounding (2^-8) of the largest (max-abs) or RMS (RMS) exact element, the slack
    for a single rounding falling the other way."""
    x, params, gv = make(N, 4096, O, 100 * seed + O)
    got = run_op(x, params, gv)
    if N == 0:
        assert got["v"].shape == (0, O) and got["dx"].shape == (0, 4096)
        assert all(int(got[k].count_nonzero()) == 0 for k in NAMES[2:])
        return
    eager = run_eager(x, params, gv)
    exact = run_fp64(x, params, gv)
    for k in NAMES:
        assert got[k].dtype == torch.bfloat16 and got[k].shape == exact[k].shape, k
        mo, ro = errors(got[k], exact[k])
        me, re_ = errors(eager[k], exact[k])
        scale_m, scale_r = exact[k].abs().max().item(), exact[k].pow(2).mean().sqrt().item()
        assert mo <= 1.25 * me + 2 ** -8 * scale_m, (k, mo, me, scale_m)
        assert ro <= 1.25 * re_ + 2 ** -8 * scale_r, (k, ro, re_, scale_r)


def test_batch_invariance_and_in_place_row():
    """A row's values are the same bits in a 4096-row batch, in random subsets, in a permutation, alone, and read in
    place from a [B, S, H] tensor at position -act*C - 1 whose other positions are all NaN."""
    from rlinf_b200 import ops

    N, H, O, act, C = 4096, 4096, 8, 7, 8
    x, params, _ = make(N, H, O, 7)
    with torch.no_grad():
        full = ops.vla_value_head(x, *params)
        assert torch.isfinite(full.float()).all()
        gen = torch.Generator(device="cpu").manual_seed(3)
        for n in (1, 2, 40, 127, 1000, 4095):
            idx = torch.randperm(N, generator=gen)[:n].to(DEV)
            assert torch.equal(ops.vla_value_head(x[idx], *params), full[idx]), n
        perm = torch.randperm(N, generator=gen).to(DEV)
        assert torch.equal(ops.vla_value_head(x[perm], *params), full[perm])
        for i in (0, 1, 63, 64, 2047, N - 1):
            assert torch.equal(ops.vla_value_head(x[i:i + 1], *params), full[i:i + 1]), i
        S = act * C + 2
        hs = torch.full((N, S, H), float("nan"), dtype=torch.bfloat16, device=DEV)
        p = -act * C - 1
        hs[:, p] = x
        row = hs[:, p]
        assert row.stride(0) == S * H
        assert torch.equal(ops.vla_value_head(row, *params), full)


def test_backward_deterministic():
    x, params, gv = make(1024, 4096, 25, 11)
    a, b = run_op(x, params, gv), run_op(x, params, gv)
    for k in NAMES:
        assert torch.equal(a[k], b[k]), k


def test_skipped_gradients_match_the_full_backward():
    x, params, gv = make(127, 4096, 8, 13)
    full = run_op(x, params, gv)
    cases = [(False, (True,) * 5), (True, (False,) * 5), (True, (False, False, True, True, True)),
             (False, (True, True, False, False, False)), (False, (False, False, False, False, True))]
    for xg, pg in cases:
        got = run_op(x, params, gv, x_grad=xg, p_grad=pg)
        assert torch.equal(got["v"], full["v"])
        for k, need in zip(NAMES[1:], (xg,) + pg):
            if need:
                assert torch.equal(got[k], full[k]), (k, xg, pg)
            else:
                assert got[k] is None, k


def test_no_host_sync():
    from rlinf_b200 import ops

    x, params, gv = make(40, 4096, 8, 17)
    xs = x.clone().requires_grad_(True)
    ps = [p.clone().requires_grad_(True) for p in params]
    ops.vla_value_head(x, *params)  # load the library outside the checked region
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        with torch.no_grad():
            ops.vla_value_head(x, *params)
        v = ops.vla_value_head(xs, *ps)
        torch.autograd.grad(v, [xs] + ps, gv)
    finally:
        torch.cuda.set_sync_debug_mode(0)


def test_cuda_graph_capture():
    from rlinf_b200 import ops

    x, params, gv = make(128, 4096, 8, 19)
    xs = x.clone().requires_grad_(True)
    ps = [p.clone().requires_grad_(True) for p in params]

    def fwd():
        with torch.no_grad():
            return ops.vla_value_head(x, *params)

    def fwd_bwd():
        v = ops.vla_value_head(xs, *ps)
        return (v.detach(),) + torch.autograd.grad(v, [xs] + ps, gv)

    want_f, want_fb = fwd(), fwd_bwd()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for _ in range(2):
            fwd(), fwd_bwd()
    torch.cuda.current_stream().wait_stream(s)
    g1, g2 = torch.cuda.CUDAGraph(), torch.cuda.CUDAGraph()
    with torch.cuda.graph(g1):
        out_f = fwd()
    with torch.cuda.graph(g2):
        out_fb = fwd_bwd()
    g1.replay()
    g2.replay()
    torch.cuda.synchronize()
    assert torch.equal(out_f, want_f)
    for a, b in zip(out_fb, want_fb):
        assert torch.equal(a, b)


def _count_kernels(fn):
    from torch.profiler import ProfilerActivity, profile

    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    return sum(1 for n in names if KERNELS.search(n)), names


def test_launch_counts():
    from rlinf_b200 import ops

    x, params, gv = make(1024, 4096, 25, 23)
    xs = x.clone().requires_grad_(True)
    ps = [p.clone().requires_grad_(True) for p in params]
    with torch.no_grad():
        nf, names = _count_kernels(lambda: ops.vla_value_head(x, *params))
    assert nf == 2 and len(names) == 2, names
    v = ops.vla_value_head(xs, *ps)
    nb, names = _count_kernels(lambda: torch.autograd.grad(v, [xs] + ps, gv, retain_graph=True))
    assert nb == 4 and len([n for n in names if "Memcpy" not in n and "Memset" not in n]) == 4, names


def test_chain_into_actor_critic_loss():
    """values [B, C] bf16 straight from the head into the embodied actor_critic PPO loss, then backward; against the
    same chain in fp64 torch (the fp64 head without roundings and the project's loss oracle)."""
    import rlinf_b200.algorithms as A
    from oracle import rl_oracle as RO
    from rlinf_b200 import ops

    B, C, act, H = 40, 8, 7, 4096
    x, params, _ = make(B, H, C, 29)
    g = torch.Generator().manual_seed(31)

    def r(*shape, std=1.0, mean=0.0):
        return (torch.randn(*shape, generator=g, dtype=torch.float64) * std + mean).to(DEV)

    lp = r(B, C * act, std=0.1, mean=-1.0)
    batch = dict(old_logprobs=lp + r(B, C * act, std=0.05), advantages=r(B, C), returns=r(B, C, std=0.2),
                 prev_values=r(B, C, std=0.2))
    hp = dict(clip_ratio_low=0.2, clip_ratio_high=0.28, value_clip=0.2, huber_delta=10.0)

    xs = x.clone().requires_grad_(True)
    ps = [p.clone().requires_grad_(True) for p in params]
    lps = lp.float().requires_grad_(True)
    values = ops.vla_value_head(xs, *ps)
    assert values.dtype == torch.bfloat16 and values.shape == (B, C)
    loss, _ = A.policy_loss(task_type="embodied", loss_type="actor_critic", logprob_type="action_level",
                            reward_type="action_level", single_action_dim=act, logprobs=lps, values=values,
                            **{k: v.float() for k, v in batch.items()}, **hp)
    loss.backward()

    x64 = x.double().requires_grad_(True)
    p64 = [p.double().requires_grad_(True) for p in params]
    h = torch.nn.functional.gelu(x64 @ p64[0].T + p64[1])
    h = torch.nn.functional.gelu(h @ p64[2].T + p64[3])
    v64 = h @ p64[4].T
    lp64 = lp.clone().requires_grad_(True)
    loss64, _ = RO.policy_loss_embodied("actor_critic", lp64, batch["old_logprobs"], batch["advantages"],
                                        "action_level", act, values=v64, prev_values=batch["prev_values"],
                                        returns=batch["returns"], reward_type="action_level", **hp)
    loss64.backward()
    assert abs(loss.item() - loss64.item()) <= 1e-2 * abs(loss64.item()) + 1e-4
    for got, want, name in [(lps.grad, lp64.grad, "logprobs"), (xs.grad, x64.grad, "dx")] + [
            (p.grad, q.grad, f"param{i}") for i, (p, q) in enumerate(zip(ps, p64))]:
        d = (got.double() - want).abs().max().item()
        assert d <= 0.05 * want.abs().max().item() + 1e-6, (name, d, want.abs().max().item())
