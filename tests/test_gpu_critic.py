"""The reasoning PPO critic on the GPU: ops.megatron_response_values (the value head on the response rows of Megatron
packed batches under TP / SP / CP) and reasoning_critic_loss (the token-level critic loss).

tp x cp grids are emulated on one device by running the op's per-rank stages rank by rank, each collective replaced by
a concatenation.  Checked: values against fp64 on the same bf16 operands and bit-identical on every rank and across
repeat calls; dX bit-identical to bf16(bf16(g) w) on the rank's own response rows and exactly zero elsewhere; dW
against fp64 and the per-rank shares against the (1, 1) run; the public op on every rank with its peers' buffers
served from the emulation; the loss and metrics against the fp64 oracle (tests/critic_oracle.py), deterministic, under
CUDA-graph replay, without host sync and at a stated launch count; the reference fixture per rank; the composition
values -> GAE -> loss -> backward against plain torch in fp64; and a 2-rank NCCL case skipped below 2 GPUs."""
from __future__ import annotations

import json
import os
import socket
import subprocess
import sys
import warnings

import numpy as np
import pytest
import torch

import critic_oracle as CO
import response_rows_mp_oracle as O
from rlinf_b200 import _lib, ops
from rlinf_b200 import response_rows as RR
from rlinf_b200.algorithms import calculate_adv_and_returns, reasoning_critic_loss

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
GRIDS = [(1, 1), (2, 1), (4, 1), (8, 1), (1, 2), (2, 2), (2, 4)]
BF16_HALF_ULP = 2.0 ** -8  # one bf16 rounding, relative


def _batch(tp, cp, shape="small", sparse=False):
    """Packed lengths padded as preprocess_packed_seqs pads them.  small: an empty response, a full one and prediction
    rows that straddle CP chunks and TP shards (L 48).  sparse: one-token responses at the end of 64-token sequences,
    so every CP rank but the first holds no prediction row.  big: 8 sequences of 1,536 rows, T = 12,288 (the config's
    max_tokens_per_mbs) with R / T = 0.70."""
    if shape == "big":
        p, r = torch.full((8,), 460), torch.full((8,), 1076)
        r[3], p[3] = 1000, 536
    elif sparse:
        p, r = torch.tensor([63, 40, 63]), torch.tensor([1, 0, 1])
    else:
        p, r = torch.tensor([7, 30, 3, 12, 1, 20]), torch.tensor([48, 0, 29, 17, 40, 5])
    n = p + r
    align = 2 * cp * tp if cp > 1 else tp
    N = n + (align - n % align) % align
    cu = torch.cat([torch.zeros(1, dtype=torch.int64), torch.cumsum(N, 0)])
    return cu, n, r, int(r.max()) if shape == "big" else 48


def _setup(tp, cp, sp, H, shape="small", sparse=False, seed=0):
    cu, n, r, L = _batch(tp, cp, shape, sparse)
    g = torch.Generator(device="cuda").manual_seed(seed)
    seqs = [torch.randn(int(cu[b + 1] - cu[b]), H, generator=g, device="cuda").to(torch.bfloat16)
            for b in range(len(n))]
    T_c = int(cu[-1]) // cp
    streams = [O.local_stream(seqs, cu, n, cp, c, T_c) for c in range(cp)]
    w = (torch.randn(1, H, generator=g, device="cuda") * (2.0 / H ** 0.5)).to(torch.bfloat16)
    plan = RR.megatron_parallel(cu, n, r, response_len=L, tp_size=tp, cp_size=cp, sequence_parallel=sp)
    return dict(cu=cu, n=n, r=r, L=L, T_c=T_c, seqs=seqs, streams=streams, w=w, plan=plan, tp=tp, cp=cp, sp=sp)


def _shards(s):
    tp, cp, sp, T_c = s["tp"], s["cp"], s["sp"], s["T_c"]
    Ts = T_c // tp if sp else T_c
    return Ts, [[s["streams"][c][k * Ts:(k + 1) * Ts] if sp else s["streams"][c] for k in range(tp)]
                for c in range(cp)]


def _emulate(s, g=None):
    """Every rank's forward (and, given the output gradient g, backward) through the op's stages."""
    tp, cp, sp, plan = s["tp"], s["cp"], s["sp"], s["plan"]
    Ts, hid = _shards(s)
    shape = (plan.bsz, plan.response_len)
    tg = torch.zeros(shape, dtype=torch.int64, device="cuda")
    idx = [[plan.index(tg, Ts, k, c) for k in range(tp)] for c in range(cp)]
    res = {"idx": idx, "tp_bufs": [], "vals": []}
    for c in range(cp):
        per_k = [ops.mp_value_head(hid[c][k], s["w"], idx[c][k]) for k in range(tp)]
        res["tp_bufs"].append(per_k)
        vs = [ops.mp_value_unpad(torch.stack(per_k), idx[c][k]) for k in range(tp)] if sp else per_k
        for k in range(1, tp):
            assert torch.equal(vs[k], vs[0])
        res["vals"].append(ops.mp_values(vs[0], None, idx[c][0]))
    allv = torch.stack(res["vals"])
    res["out"] = [[ops.mp_to_cells(allv, idx[c][k], shape, False)[0] for k in range(tp)] for c in range(cp)]
    if g is not None:
        res["dx"] = [[None] * tp for _ in range(cp)]
        res["dw"] = [[None] * tp for _ in range(cp)]
        for c in range(cp):
            for k in range(tp):
                grad, _ = ops.mp_cell_grads(g, None, idx[c][k])
                res["dx"][c][k], res["dw"][c][k] = ops.mp_value_head_backward(grad, hid[c][k], s["w"], idx[c][k])
    return res


def _fp64_values(s):
    """[bsz, L] fp64 values on the same bf16 operands, zeros past r_b."""
    L = s["L"]
    out = torch.zeros(len(s["n"]), L, dtype=torch.float64, device="cuda")
    wd = s["w"].double()[0]
    for b in range(len(s["n"])):
        rb = int(s["r"][b])
        if rb:
            p0 = int(s["n"][b]) - rb - 1
            out[b, :rb] = s["seqs"][b][p0:p0 + rb].double() @ wd
    return out


def _own_rows(s, c, k):
    """[(local row in rank (c, k)'s shard, b, j)] of the prediction rows whose gradient the rank computes."""
    Ts, _ = _shards(s)
    rows = O.prediction_rows(s["cu"], s["n"], s["r"], s["cp"])[c]
    if not s["sp"]:
        return rows
    return [(t - k * Ts, b, j) for t, b, j in rows if k * Ts <= t < (k + 1) * Ts]


def _check_values(s, e):
    v0 = e["out"][0][0]
    for c in range(s["cp"]):
        for k in range(s["tp"]):
            assert torch.equal(e["out"][c][k], v0), (c, k)
    ref = _fp64_values(s)
    err = (v0.double() - ref).abs()
    assert bool((err <= BF16_HALF_ULP * ref.abs() * 1.001 + 1e-6).all()), float(err.max())
    assert torch.equal(v0, v0.bfloat16().float())  # one rounding to bf16
    valid = torch.arange(s["L"], device="cuda")[None] < s["r"].cuda()[:, None]
    assert not v0[~valid].any()
    return v0


def _check_grads(s, e, g):
    H = s["w"].shape[1]
    Ts, hid = _shards(s)
    wf = s["w"].float()[0]
    gb = g.bfloat16().float()
    tot = torch.zeros(H, dtype=torch.float64, device="cuda")
    tot_abs = torch.zeros(H, dtype=torch.float64, device="cuda")
    for c in range(s["cp"]):
        for k in range(s["tp"]):
            own = _own_rows(s, c, k)
            want = torch.zeros(Ts, H, dtype=torch.bfloat16, device="cuda")
            dw64 = torch.zeros(H, dtype=torch.float64, device="cuda")
            mag = torch.zeros(H, dtype=torch.float64, device="cuda")
            if own:
                t = torch.tensor([x[0] for x in own], device="cuda")
                bj = (torch.tensor([x[1] for x in own], device="cuda"), torch.tensor([x[2] for x in own], device="cuda"))
                want[t] = (gb[bj][:, None] * wf[None]).bfloat16()
                terms = gb[bj].double()[:, None] * hid[c][k][t].double()
                dw64, mag = terms.sum(0), terms.abs().sum(0)
            assert torch.equal(e["dx"][c][k], want), (c, k)
            dw = e["dw"][c][k].double()[0]
            assert bool(((dw - dw64).abs() <= 2 * BF16_HALF_ULP * dw64.abs() + 1e-5 * mag + 1e-30).all()), (c, k)
            if not s["sp"] and k > 0:
                assert torch.equal(e["dw"][c][k], e["dw"][c][0])
            if s["sp"] or k == 0:
                tot += dw
                tot_abs += dw.abs() + mag * 1e-5
    return tot, tot_abs


def _grad(s, seed=7):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(len(s["n"]), s["L"], generator=g, device="cuda")


@pytest.mark.parametrize("H", [64, 1536])
@pytest.mark.parametrize("tp, cp, sp", [(tp, cp, sp) for tp, cp in GRIDS for sp in (True, False) if tp > 1 or not sp])
def test_emulated_grid(tp, cp, sp, H):
    s = _setup(tp, cp, sp, H)
    g = _grad(s)
    e = _emulate(s, g)
    v = _check_values(s, e)
    dw, dw_abs = _check_grads(s, e, g)
    # the per-rank dW shares add up to the (1, 1) run's dW: within one bf16 rounding of each share and of the total
    s1 = _setup(1, 1, False, H)
    e1 = _emulate(s1, g)
    assert torch.equal(e1["out"][0][0], v)
    d1 = e1["dw"][0][0].double()[0]
    assert bool(((dw - d1).abs() <= 1.01 * BF16_HALF_ULP * (dw_abs + d1.abs()) + 1e-30).all())
    # repeat calls: the same bits
    e2 = _emulate(s, g)
    for c in range(cp):
        for k in range(tp):
            assert torch.equal(e2["out"][c][k], e["out"][c][k])
            assert torch.equal(e2["dx"][c][k], e["dx"][c][k]) and torch.equal(e2["dw"][c][k], e["dw"][c][k])


@pytest.mark.parametrize("H", [1536, 3584])
@pytest.mark.parametrize("tp, cp, sp", [(1, 1, False), (2, 1, True), (2, 2, True), (1, 2, False)])
def test_emulated_grid_micro_batch(tp, cp, sp, H):
    """A packed micro-batch of T = 12,288 rows with R / T = 0.70 at the critic's hidden sizes."""
    s = _setup(tp, cp, sp, H, shape="big")
    assert int(s["cu"][-1]) == 12288
    g = _grad(s)
    e = _emulate(s, g)
    _check_values(s, e)
    _check_grads(s, e, g)


@pytest.mark.parametrize("sp", [True, False])
@pytest.mark.parametrize("tp, cp", [(1, 2), (2, 2), (2, 4)])
def test_emulated_grid_with_empty_cp_ranks(tp, cp, sp):
    """CP ranks 1.. hold no prediction row: the same values, zero dX and zero dW there."""
    s = _setup(tp, cp, sp, 64, sparse=True)
    assert [sum(x) if sp else x[0] for x in s["plan"].counts(s["T_c"])][1:] == [0] * (cp - 1)
    g = _grad(s)
    e = _emulate(s, g)
    _check_values(s, e)
    _check_grads(s, e, g)
    for c in range(1, cp):
        for k in range(tp):
            assert not e["dx"][c][k].any() and not e["dw"][c][k].any()


class _PeerDist:
    """torch.distributed stand-in for rank (c, k) of an emulated grid: each collective records its traffic and returns
    what the other ranks' stages put in, with this rank's own buffer in its slot."""

    def __init__(self, e, c, k):
        self.e, self.c, self.k, self.calls = e, c, k, []

    def is_available(self):
        return True

    def is_initialized(self):
        return True

    def get_world_size(self, group=None):
        return group[0]

    def get_rank(self, group=None):
        return group[1]

    def all_gather_into_tensor(self, out, inp, group=None):
        kind = group[2]
        self.calls.append(("all_gather", kind, inp.numel() * inp.element_size() * group[0], inp.dtype))
        peers, me = (list(self.e["vals"]), self.c) if kind == "cp" else (list(self.e["tp_bufs"][self.c]), self.k)
        assert torch.equal(peers[me], inp)
        peers[me] = inp
        out.copy_(torch.stack(peers))

    def all_reduce(self, *a, **kw):
        raise AssertionError("the value head makes no all-reduce")

    def reduce_scatter_tensor(self, *a, **kw):
        raise AssertionError("the value head makes no reduce-scatter")


def _peer_run(monkeypatch, s, e, c, k, g):
    import torch.distributed as dist

    fake = _PeerDist(e, c, k)
    for name in ("is_available", "is_initialized", "get_world_size", "get_rank", "all_gather_into_tensor",
                 "all_reduce", "reduce_scatter_tensor"):
        monkeypatch.setattr(dist, name, getattr(fake, name))
    _, hid = _shards(s)
    x = hid[c][k][:, None].clone().requires_grad_(True)
    w = s["w"].clone().requires_grad_(True)
    v = ops.megatron_response_values(x, w, s["plan"], tp_group=(s["tp"], k, "tp"), cp_group=(s["cp"], c, "cp"))
    n_fwd = len(fake.calls)
    (v * g).sum().backward()
    monkeypatch.undo()
    return v, x.grad[:, 0], w.grad, fake.calls, n_fwd


@pytest.mark.parametrize("tp, cp, sp, sparse", [(2, 2, True, False), (2, 2, False, False), (4, 1, True, False),
                                                (2, 1, False, False), (1, 2, False, False), (2, 2, True, True),
                                                (2, 4, True, True), (1, 2, False, True)])
def test_op_on_every_rank_matches_emulation(monkeypatch, tp, cp, sp, sparse):
    """The public op on every rank, its peers' buffers served from the emulation: values, dX and dW bit-identical to
    the emulation; collectives: under SP one [Rmax_k] fp32 all-gather over TP, one [Rmax_c, 2] fp32 all-gather over CP,
    none in the backward; ranks without rows take part in every one."""
    s = _setup(tp, cp, sp, 128, sparse=sparse)
    g = _grad(s)
    e = _emulate(s, g)
    for c in range(cp):
        for k in range(tp):
            v, dx, dw, calls, nf = _peer_run(monkeypatch, s, e, c, k, g)
            assert torch.equal(v, e["out"][c][k]), (c, k)
            assert torch.equal(dx, e["dx"][c][k]) and torch.equal(dw, e["dw"][c][k]), (c, k)
            ix = e["idx"][c][k]
            want = [("all_gather", "tp", tp * ix.Rmax_k * 4, torch.float32)] if sp and tp > 1 else []
            want += [("all_gather", "cp", cp * ix.Rmax_c * 8, torch.float32)] if cp > 1 else []
            assert calls[:nf] == want and calls[nf:] == []


def test_one_rank_op_frozen_inputs_and_no_rows():
    s = _setup(1, 1, False, 256)
    x = s["streams"][0]
    v = ops.megatron_response_values(x[:, None], s["w"], s["plan"])
    assert not v.requires_grad
    xx = x.clone().requires_grad_(True)
    v2 = ops.megatron_response_values(xx, s["w"], s["plan"])
    (v2 * _grad(s)).sum().backward()
    assert torch.equal(v, v2.detach()) and xx.grad is not None
    plan0 = RR.megatron_parallel(s["cu"], s["n"], torch.zeros_like(s["r"]), response_len=s["L"])
    z = ops.megatron_response_values(xx, s["w"], plan0)
    assert not z.any() and tuple(z.shape) == (len(s["n"]), s["L"])


def _count_syncs(fn):
    with warnings.catch_warnings(record=True) as rec:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            out = fn()
        finally:
            torch.cuda.set_sync_debug_mode("default")
    return out, sum("called a synchronizing CUDA operation" in str(w.message) for w in rec)


def test_values_host_syncs():
    s = _setup(1, 1, False, 256)
    x = s["streams"][0].clone().requires_grad_(True)
    torch.cuda.synchronize()
    v, fwd = _count_syncs(lambda: ops.megatron_response_values(x, s["w"], s["plan"]))
    _, bwd = _count_syncs(lambda: v.sum().backward())
    assert fwd == 0 and bwd == 0
    d = RR.megatron_parallel(*(t.cuda() for t in (s["cu"], s["n"], s["r"])), response_len=s["L"])
    v2, fwd = _count_syncs(lambda: ops.megatron_response_values(x.detach(), s["w"], d))
    assert fwd == 1 and torch.equal(v2, v.detach())


# ----------------------------------------------------------------------------------------------------------------
# the loss
# ----------------------------------------------------------------------------------------------------------------
def _loss_inputs(bsz, L, seed=0, scale=1.0, empty_rows=(), all_masked=False):
    g = torch.Generator().manual_seed(seed)
    v = torch.randn(bsz, L, generator=g) * scale
    ret = v + torch.randn(bsz, L, generator=g) * scale
    prev = v + torch.randn(bsz, L, generator=g) * 0.5 * scale
    r = torch.randint(0, L + 1, (bsz,), generator=g)
    mask = torch.arange(L)[None] < r[:, None]
    mask[list(empty_rows)] = False
    if all_masked:
        mask[:] = False
    return v, ret, prev, mask


def _check_loss(v, ret, prev, mask, value_clip, huber_delta):
    vc = v.cuda().requires_grad_(True)
    loss, metrics = reasoning_critic_loss(vc, ret.cuda(), prev.cuda(), mask.cuda(), value_clip=value_clip,
                                          huber_delta=huber_delta)
    loss.backward()
    assert list(metrics) == list(CO.KEYS) and all(m.dim() == 0 and m.is_cuda for m in metrics.values())
    ol, om, og = CO.critic_loss(v, ret, prev, mask, value_clip, huber_delta)
    torch.testing.assert_close(loss.double().cpu(), ol, rtol=1e-5, atol=1e-7)
    for k in CO.KEYS:
        torch.testing.assert_close(metrics[k].double().cpu(), om[k], rtol=1e-5, atol=1e-6, msg=k)
    bsz, L = v.shape
    assert round(float(metrics["critic/value_clip_ratio"]) * bsz * L) == CO.clip_count(v, prev, value_clip)
    torch.testing.assert_close(vc.grad.cpu(), og, rtol=1e-5, atol=1e-9)
    return loss, metrics, vc.grad


@pytest.mark.parametrize("bsz, L", [(1, 1), (6, 48), (64, 1076), (8, 5000), (3, 1025)])
def test_loss_matches_oracle(bsz, L):
    _check_loss(*_loss_inputs(bsz, L, seed=bsz + L, empty_rows=(0,)), value_clip=0.5, huber_delta=10000.0)


@pytest.mark.parametrize("delta", [0.3, 1.0])
def test_loss_linear_huber_branch(delta):
    v, ret, prev, mask = _loss_inputs(16, 300, seed=3, scale=2.0)
    e = (ret - v)[mask].abs()
    assert bool((e > delta).any()) and bool((e < delta).any())
    _check_loss(v, ret, prev, mask, value_clip=0.2, huber_delta=delta)


def test_loss_all_masked_is_zero():
    loss, metrics, grad = _check_loss(*_loss_inputs(4, 64, seed=5, all_masked=True), value_clip=0.5,
                                      huber_delta=10000.0)
    assert float(loss) == 0.0 and float(metrics["__sum__/_critic_explained_variance/count"]) == 0.0
    assert float(metrics["critic/value_clip_ratio"]) > 0 and not grad.any()


def test_loss_reads_strided_slices():
    """values = output[:, -L-1:-1], as Megatron's loss_func slices it, is read in place."""
    v, ret, prev, mask = _loss_inputs(6, 40, seed=8)
    full = torch.randn(6, 60).cuda()
    full[:, -41:-1] = v.cuda()
    full.requires_grad_(True)
    loss, _ = reasoning_critic_loss(full[:, -41:-1], ret.cuda(), prev.cuda(), mask.cuda(), value_clip=0.5)
    loss.backward()
    ol, _, og = CO.critic_loss(v, ret, prev, mask, 0.5, 10000.0)
    torch.testing.assert_close(loss.double().cpu(), ol, rtol=1e-5, atol=1e-7)
    assert not full.grad[:, :19].any() and not full.grad[:, -1].any()
    torch.testing.assert_close(full.grad[:, -41:-1].cpu(), og, rtol=1e-5, atol=1e-9)


def test_loss_deterministic_graph_replay_no_sync_and_launch_count():
    """Four library launches in the forward and one gradient scaling in the backward; no host sync; the same bits on
    repeat calls and under CUDA-graph replay."""
    v, ret, prev, mask = (t.cuda() for t in _loss_inputs(64, 2048, seed=11, empty_rows=(3,)))
    vv = v.clone().requires_grad_(True)

    def step():
        vv.grad = None
        loss, metrics = reasoning_critic_loss(vv, ret, prev, mask, value_clip=0.5)
        (loss * 0.25).backward()
        return loss.detach().clone(), torch.stack(list(metrics.values())).clone(), vv.grad.clone()

    runs = [step() for _ in range(2)]
    for a, b in zip(*runs):
        assert torch.equal(a, b)
    torch.cuda.synchronize()
    n0 = _lib.load().rb200_launch_count()
    torch.cuda.set_sync_debug_mode("error")
    try:
        step()
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert _lib.load().rb200_launch_count() - n0 == 5
    st = torch.cuda.Stream()
    st.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(st):
        step()
    torch.cuda.current_stream().wait_stream(st)
    graph = torch.cuda.CUDAGraph()
    vv.grad = None
    with torch.cuda.graph(graph):
        loss, metrics = reasoning_critic_loss(vv, ret, prev, mask, value_clip=0.5)
        (loss * 0.25).backward()
        out = (loss.detach(), torch.stack(list(metrics.values())), vv.grad)
    graph.replay()
    torch.cuda.synchronize()
    for a, b in zip(runs[0], out):
        assert torch.equal(a, b)


def test_loss_argument_errors():
    v, ret, prev, mask = (t.cuda() for t in _loss_inputs(2, 8))
    with pytest.raises(ValueError, match="returns has shape"):
        reasoning_critic_loss(v, ret[:, :4], prev, mask, value_clip=0.5)
    with pytest.raises(ValueError, match="must be torch.float32"):
        reasoning_critic_loss(v, ret.double(), prev, mask, value_clip=0.5)
    with pytest.raises(ValueError, match="loss_mask must be bool or uint8"):
        reasoning_critic_loss(v, ret, prev, mask.float(), value_clip=0.5)
    with pytest.raises(ValueError, match=r"\[bsz, L\]"):
        reasoning_critic_loss(v[0], ret[0], prev[0], mask[0], value_clip=0.5)


# ----------------------------------------------------------------------------------------------------------------
# composition: values -> GAE -> loss -> backward, against plain torch in fp64
# ----------------------------------------------------------------------------------------------------------------
def test_composition_values_gae_loss_backward():
    """Inference values -> calculate_adv_and_returns(gae) -> reasoning_critic_loss -> backward, against the same chain
    in plain torch and fp64 on the same bf16 operands, returns and previous values."""
    s1 = _setup(1, 1, False, 256)
    x1 = s1["streams"][0][:, None].clone().requires_grad_(True)
    w1 = s1["w"].clone().requires_grad_(True)
    bsz, L = len(s1["n"]), s1["L"]
    mask = (torch.arange(L)[None] < s1["r"][:, None]).cuda()
    rewards = torch.linspace(-1, 1, bsz, device="cuda")
    with torch.no_grad():
        old = ops.megatron_response_values(x1.detach(), w1, s1["plan"])
    res = calculate_adv_and_returns(task_type="reasoning", adv_type="gae", rewards=rewards, loss_mask=mask,
                                    values=old, gamma=1.0, gae_lambda=0.95, normalize_advantages=False)
    returns = res[1] if isinstance(res, tuple) else res["returns"]
    v = ops.megatron_response_values(x1, w1, s1["plan"])
    loss, _ = reasoning_critic_loss(v, returns, old, mask, value_clip=0.5)
    loss.backward()
    # plain torch, fp64, on the same bf16 operands
    xd = s1["streams"][0].double().requires_grad_(True)
    wd = s1["w"].double().requires_grad_(True)
    vals = torch.zeros(bsz, L, dtype=torch.float64, device="cuda")
    for b in range(bsz):
        rb = int(s1["r"][b])
        a = int(s1["cu"][b]) + int(s1["n"][b]) - rb - 1
        if rb:
            vals[b, :rb] = (xd[a:a + rb] @ wd[0])
    ret64, prev64 = returns.double(), old.double()
    vpc = prev64 + (vals - prev64).clamp(-0.5, 0.5)
    vl = torch.max(CO.huber(ret64 - vals, 1e4), CO.huber(ret64 - vpc, 1e4))
    loss64 = (vl * mask).sum() / mask.sum()
    loss64.backward()
    torch.testing.assert_close(loss.double(), loss64.detach(), rtol=2e-2, atol=1e-3)
    torch.testing.assert_close(w1.grad.double(), wd.grad, rtol=2e-2, atol=2e-2 * float(wd.grad.abs().max()))
    torch.testing.assert_close(x1.grad[:, 0].double(), xd.grad, rtol=2e-2, atol=2e-2 * float(xd.grad.abs().max()))
    assert torch.equal(x1.grad[:, 0].ne(0).any(-1), xd.grad.ne(0).any(-1))


# ----------------------------------------------------------------------------------------------------------------
# the reference fixture
# ----------------------------------------------------------------------------------------------------------------
GOLDEN = os.path.join(HERE, "golden", "golden_critic.npz")


@pytest.mark.skipif(not os.path.exists(GOLDEN), reason="fixture not generated")
def test_reference_fixture_per_rank():
    """The reference's inference values, training loss, metrics and gradients per rank of each fixture grid: the op's
    stages on the fixture's hidden shards and value weight (bf16-exact) reproduce them within the tolerances above."""
    gz = {k: torch.from_numpy(v) for k, v in np.load(GOLDEN).items()}
    for key in sorted(k[:-len("_meta")] for k in gz if k.endswith("_meta")):
        tp, cp, sp, L, bsz, T_c = (int(x) for x in gz[f"{key}_meta"][:6])
        value_clip, delta = (float(x) for x in gz[f"{key}_hyper"])
        plan = RR.megatron_parallel(gz[f"{key}_cu"], gz[f"{key}_n"], gz[f"{key}_r"], response_len=L, tp_size=tp,
                                    cp_size=cp, sequence_parallel=bool(sp))
        Ts = T_c // tp if sp else T_c
        w = gz["w"].cuda().to(torch.bfloat16)
        streams = []
        for c in range(cp):
            parts = [gz[f"{key}_c{c}_k{k}_hidden"] for k in range(tp)]
            streams.append((torch.cat(parts) if sp else parts[0]).cuda().to(torch.bfloat16))
        s = dict(tp=tp, cp=cp, sp=bool(sp), T_c=T_c, streams=streams, w=w, plan=plan)
        e = _emulate(s)
        v = e["out"][0][0]
        ref_v = gz[f"{key}_infer_values"].cuda()
        # a bf16 Linear + .float() on the same operands: both within one bf16 rounding of the exact value
        assert bool(((v - ref_v).abs() <= 2 * BF16_HALF_ULP * ref_v.abs()).all()), key
        ret, prev = gz[f"{key}_returns"].cuda(), gz[f"{key}_prev_values"].cuda()
        mask = gz[f"{key}_mask"].cuda().bool()
        vv = v.clone().requires_grad_(True)
        loss, metrics = reasoning_critic_loss(vv, ret, prev, mask, value_clip=value_clip, huber_delta=delta)
        loss.backward()
        ref_m = gz[f"{key}_metrics"]
        torch.testing.assert_close(loss.cpu(), gz[f"{key}_loss"], rtol=1e-5, atol=1e-6)
        for i, k in enumerate(CO.KEYS):
            if k == "critic/value_clip_ratio":  # the one deviation: the reference's cells past r_b (DESIGN.md §2)
                continue
            torch.testing.assert_close(metrics[k].cpu(), ref_m[i], rtol=1e-5, atol=1e-5, msg=(key, k))
        e = _emulate(s, vv.grad)
        for c in range(cp):
            for k in range(tp):
                rg = gz[f"{key}_c{c}_k{k}_grad"].cuda().reshape(Ts, -1).float()
                got = e["dx"][c][k].float()
                assert torch.equal(got.ne(0).any(-1), rg.ne(0).any(-1)), (key, c, k)
                torch.testing.assert_close(got, rg, rtol=2 * BF16_HALF_ULP, atol=1e-6 * float(rg.abs().max()) + 1e-30)
                rw = gz[f"{key}_c{c}_k{k}_wgrad"].cuda().float()
                torch.testing.assert_close(e["dw"][c][k].float(), rw, rtol=4 * BF16_HALF_ULP,
                                           atol=1e-3 * float(rw.abs().max()) + 1e-30)


# ----------------------------------------------------------------------------------------------------------------
# NCCL
# ----------------------------------------------------------------------------------------------------------------
def _free_port():
    with socket.socket() as so:
        so.bind(("127.0.0.1", 0))
        return so.getsockname()[1]


@pytest.mark.parametrize("tp, cp, sp", [(2, 1, True), (1, 2, False)])
def test_nccl_matches_emulation(tmp_path, tp, cp, sp):
    world = tp * cp
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    out = tmp_path / "out.json"
    env = dict(os.environ, RB200_DIST_OUT=str(out), RB200_GRID=f"{tp},{cp},{int(sp)}")
    cmd = [sys.executable, "-m", "torch.distributed.run", f"--nproc_per_node={world}",
           f"--master_port={_free_port()}", os.path.join(HERE, "dist_critic_worker.py")]
    proc = subprocess.run(cmd, env=env, capture_output=True, text=True, timeout=600)
    assert proc.returncode == 0, proc.stdout[-4000:] + proc.stderr[-4000:]
    res = json.loads(out.read_text())
    assert res["ok"], res
