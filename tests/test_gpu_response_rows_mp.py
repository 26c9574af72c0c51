"""ops.megatron_response_logprobs_entropy on the GPU: tp x cp grids emulated on one device by running the op's
per-rank stages rank by rank (each collective replaced by a concatenation or a sum), checked against the plan oracle
(tests/response_rows_mp_oracle.py), the existing vocabulary-parallel ops on rows gathered by torch indexing, fp64 on
the full logits and the reference fixture; the public op on every rank with its peers' buffers served from the
emulation (a torch.distributed stand-in), composed with reasoning_actor_loss and counted against the collective budget;
the one-rank op, repeat calls, host syncs, and 2- / 4-rank NCCL runs that are skipped on fewer GPUs."""
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

import response_rows_mp_oracle as O
from rlinf_b200 import ops
from rlinf_b200 import response_rows as RR

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
TEMP = 0.7
GRIDS = [(2, 1), (4, 1), (8, 1), (1, 2), (2, 2), (2, 4)]


def _batch(tp, cp, L=48, seed=0, fixed=None, sparse=False):
    """Packed lengths as preprocess_packed_seqs pads them (multiples of 2 cp tp, or tp with cp 1), with an empty
    response, a full one and prediction rows that straddle the CP chunk boundaries.  sparse: one-token responses at
    the end of 64-token sequences, whose prediction rows all lie in the last chunk (CP rank 0's) for cp <= 4, so every
    other CP rank holds none."""
    g = torch.Generator().manual_seed(seed)
    p = torch.tensor([63, 40, 63] if sparse else [7, 30, 3, 12, 1, 20])
    r = torch.tensor([1, 0, 1] if sparse else [L, 0, 29, 17, 40, 5])
    n = p + r
    align = 2 * cp * tp if cp > 1 else tp
    N = n + (align - n % align) % align
    cu = torch.cat([torch.zeros(1, dtype=torch.int64), torch.cumsum(N, 0)])
    T_c = int(cu[-1]) // cp if fixed is None else fixed // cp
    responses = torch.randint(0, 1 << 30, (len(n), L), generator=g)
    return cu, n, r, responses, T_c


def _weights(H, V, dev="cuda", seed=1):
    g = torch.Generator(device=dev).manual_seed(seed)
    w = (torch.randn(V, H, generator=g, device=dev) * (2.0 / H ** 0.5)).to(torch.bfloat16)
    return w


def _emulate(plan, streams, w, responses, tp, cp, sp, g_lp, g_ent, backward=True):
    """Every rank's forward (and backward) through the op's stages.  streams[c] = CP rank c's [T_c, H] rows."""
    H, Vs = w.shape[1], w.shape[0] // tp
    shards = [w[k * Vs:(k + 1) * Vs] for k in range(tp)]
    T_c = streams[0].shape[0]
    Ts = T_c // tp if sp else T_c
    hid = [[streams[c][k * Ts:(k + 1) * Ts] if sp else streams[c] for k in range(tp)] for c in range(cp)]
    idx = [[plan.index(responses, Ts, k, c) for k in range(tp)] for c in range(cp)]
    # per rank (c, k) what it puts into each collective: "rows" (SP row all-gather), "rec" (record all-gather),
    # "vals" (CP all-gather, per c), "grad_send" (SP reduce-scatter) or "part" (fp32 all-reduce)
    res = {"idx": idx, "hc": [], "lse": [], "ent": [], "vals": [], "rows": [], "rec": [], "grad_send": [],
           "part": []}
    for c in range(cp):
        if sp:
            res["rows"].append([ops.mp_pack(hid[c][k], idx[c][k]) for k in range(tp)])
            gathered = torch.stack(res["rows"][c])
            hcs = [ops.mp_unpad(gathered, idx[c][k]) for k in range(tp)]
        else:
            hcs = [ops.mp_pack(hid[c][k], idx[c][k]) for k in range(tp)]
        for k in range(1, tp):
            assert torch.equal(hcs[k], hcs[0])
        hc, tg = hcs[0], idx[c][0].targets
        if idx[c][0].R:
            res["rec"].append([ops.lmhead_vp_partials(hc, shards[k], tg, k, tp, TEMP) for k in range(tp)])
            lp, ent, lse = ops.vp_combine(torch.stack(res["rec"][c]), tg, Vs)
        else:
            res["rec"].append([torch.zeros(0, 4, device="cuda")] * tp)
            lp = ent = lse = torch.zeros(0, device="cuda")
        res["hc"].append(hc)
        res["lse"].append(lse)
        res["ent"].append(ent)
        res["vals"].append(ops.mp_values(lp, ent, idx[c][0]))
    allv = torch.stack(res["vals"])
    shape = (plan.bsz, plan.response_len)
    outs = [[ops.mp_to_cells(allv, idx[c][k], shape) for k in range(tp)] for c in range(cp)]
    res["out"] = outs
    if not backward:
        return res
    dx = [[None] * tp for _ in range(cp)]
    dw = [[None] * tp for _ in range(cp)]
    for c in range(cp):
        ix = idx[c]
        if ix[0].R == 0:
            for k in range(tp):
                dx[c][k] = torch.zeros_like(hid[c][k])
                dw[c][k] = torch.zeros_like(shards[k])
            empty = torch.zeros(0, H, device="cuda")
            res["grad_send"].append([ops.mp_pack_grad(empty, ix[k]) for k in range(tp)] if sp else None)
            res["part"].append([empty] * tp)
            continue
        parts = []
        for k in range(tp):
            glp, gh = ops.mp_cell_grads(g_lp, g_ent, ix[k])
            d32, dw[c][k] = ops.lmhead_vp_backward(res["hc"][c], shards[k], ix[k].targets, k, tp, res["lse"][c],
                                                   res["ent"][c], glp, gh, TEMP)
            parts.append(d32)
        sends = None
        if sp:
            sends = [ops.mp_pack_grad(parts[k], ix[k]) for k in range(tp)]  # [tp, Rmax_k, H] bf16 each
            for k in range(tp):
                buf = ops.mp_grad_buffer(ix[k], H)
                buf[:-1] = torch.stack([s[k].float() for s in sends]).sum(0).to(torch.bfloat16)
                dx[c][k] = ops.mp_unpack_grad(buf, ix[k])
        else:
            tot = torch.stack(parts).sum(0)
            for k in range(tp):
                dx[c][k] = ops.mp_pack_grad(tot, ix[k])
        res["grad_send"].append(sends)
        res["part"].append(parts)
    res["dx"], res["dw"] = dx, dw
    return res


def _setup(tp, cp, sp, H, V, seed=0, device_lengths=False, fixed=None, sparse=False):
    cu, n, r, responses, T_c = _batch(tp, cp, seed=seed, fixed=fixed, sparse=sparse)
    responses = responses % V
    g = torch.Generator(device="cuda").manual_seed(seed + 5)
    seqs = [torch.randn(int(cu[b + 1] - cu[b]), H, generator=g, device="cuda").to(torch.bfloat16)
            for b in range(len(n))]
    streams = [O.local_stream(seqs, cu, n, cp, c, T_c) for c in range(cp)]
    lens = (cu, n, r) if not device_lengths else tuple(t.cuda() for t in (cu, n, r))
    plan = RR.megatron_parallel(*lens, response_len=responses.shape[1], tp_size=tp, cp_size=cp, sequence_parallel=sp)
    return dict(cu=cu, n=n, r=r, responses=responses.cuda(), T_c=T_c, seqs=seqs, streams=streams, plan=plan)


def _fp64(s, w, g_lp, g_ent):
    """Log-probs, entropies and their gradients w.r.t. every position's hidden state, fp64 on the full logits."""
    L = s["responses"].shape[1]
    rows, tg, cells = [], [], []
    for b in range(len(s["n"])):
        for j in range(int(s["r"][b])):
            rows.append((b, int(s["n"][b] - s["r"][b]) - 1 + j))
            tg.append(int(s["responses"][b, j]))
            cells.append(b * L + j)
    h = torch.stack([s["seqs"][b][p] for b, p in rows]).double().requires_grad_(True)
    wd = w.double().requires_grad_(True)
    logp = torch.log_softmax((h @ wd.T) / TEMP, -1)
    lp = logp.gather(1, torch.tensor(tg, device="cuda")[:, None])[:, 0]
    ent = -(logp.exp() * logp).sum(-1)
    ci = torch.tensor(cells, device="cuda")
    ((lp * g_lp.reshape(-1)[ci].double()).sum() + (ent * g_ent.reshape(-1)[ci].double()).sum()).backward()
    full_lp = torch.zeros(g_lp.numel(), dtype=torch.float64, device="cuda")
    full_ent = torch.zeros_like(full_lp)
    full_lp[ci], full_ent[ci] = lp.detach(), ent.detach()
    return rows, full_lp.view(g_lp.shape), full_ent.view(g_lp.shape), h.grad, wd.grad


@pytest.mark.parametrize("H, V", [(64, 4096), (1536, 151936)])
@pytest.mark.parametrize("sp", [True, False])
@pytest.mark.parametrize("tp, cp", GRIDS)
def test_emulated_grid(tp, cp, sp, H, V):
    _check_grid(tp, cp, sp, H, V, sparse=False)


@pytest.mark.parametrize("sp", [True, False])
@pytest.mark.parametrize("tp, cp", [(1, 2), (2, 2), (2, 4)])
def test_emulated_grid_with_empty_cp_ranks(tp, cp, sp):
    """CP ranks 1.. hold no prediction row (R_c = 0): they still produce the same outputs, zero dX and zero dW."""
    _check_grid(tp, cp, sp, 64, 4096, sparse=True)


def _check_grid(tp, cp, sp, H, V, sparse):
    s = _setup(tp, cp, sp, H, V, sparse=sparse)
    if sparse:
        assert [sum(x) if sp else x[0] for x in s["plan"].counts(s["T_c"])][1:] == [0] * (cp - 1)
    w = _weights(H, V)
    L = s["responses"].shape[1]
    g = torch.Generator(device="cuda").manual_seed(9)
    g_lp = torch.randn(len(s["n"]), L, generator=g, device="cuda")
    g_ent = torch.randn(len(s["n"]), L, generator=g, device="cuda")
    e = _emulate(s["plan"], s["streams"], w, s["responses"], tp, cp, sp, g_lp, g_ent)
    Vs = V // tp
    # the plan kernel's maps are the oracle's
    for c in range(cp):
        for k in range(tp):
            ix = e["idx"][c][k]
            m = O.rank_maps(s["cu"], s["n"], s["r"], s["responses"].tolist(), L, tp, cp, sp, s["T_c"], k, c)
            assert (ix.R, ix.Rmax_k, ix.Rmax_c, ix.counts) == (m["R"], m["Rmax_k"], m["Rmax_c"], m["counts"])
            assert ix.counts == s["plan"].counts(s["T_c"])
            for name in ("rows", "targets", "cells", "unpad", "cell_map", "hidden_map") + (
                    ("send", "slot_map") if sp else ()):
                assert getattr(ix, name).tolist() == m[name], name
    # the same bits on every rank
    lp0, ent0 = e["out"][0][0]
    for c in range(cp):
        for k in range(tp):
            assert torch.equal(e["out"][c][k][0], lp0) and torch.equal(e["out"][c][k][1], ent0)
    # bit-identical to the existing VP ops on the compact rows gathered by torch indexing
    shards = [w[k * Vs:(k + 1) * Vs] for k in range(tp)]
    exp_lp = torch.zeros(len(s["n"]) * L, device="cuda")
    exp_ent = torch.zeros_like(exp_lp)
    for c in range(cp):
        m = O.rank_maps(s["cu"], s["n"], s["r"], s["responses"].tolist(), L, tp, cp, sp, s["T_c"], 0, c)
        if not m["R"]:
            continue
        hc = s["streams"][c][torch.tensor(m["rows"], device="cuda")]
        tg = torch.tensor(m["targets"], device="cuda")
        rec = torch.stack([ops.lmhead_vp_partials(hc, shards[k], tg, k, tp, TEMP) for k in range(tp)])
        lp, ent, _ = ops.vp_combine(rec, tg, Vs)
        ci = torch.tensor(m["cells"], device="cuda")
        exp_lp[ci], exp_ent[ci] = lp, ent
    assert torch.equal(lp0, exp_lp.view_as(lp0)) and torch.equal(ent0, exp_ent.view_as(ent0))
    # fp64 on the full logits
    rows, f_lp, f_ent, f_dh, f_dw = _fp64(s, w, g_lp, g_ent)
    torch.testing.assert_close(lp0.double(), f_lp, rtol=1e-4, atol=2e-3)
    torch.testing.assert_close(ent0.double(), f_ent, rtol=1e-4, atol=2e-3)
    # dX: each rank's shard holds its rows of the fp64 gradient, zeros elsewhere
    own = O.owner(s["cu"], s["n"], cp)
    T_c = s["T_c"]
    Ts = T_c // tp if sp else T_c
    want = [torch.zeros(T_c, H, dtype=torch.float64, device="cuda") for _ in range(cp)]
    for i, (b, p) in enumerate(rows):
        c, t = own[b, p]
        want[c][t] = f_dh[i]
    scale = f_dh.abs().max()
    for c in range(cp):
        for k in range(tp):
            got = e["dx"][c][k].double()
            ref = want[c][k * Ts:(k + 1) * Ts] if sp else want[c]
            assert not got[(ref == 0).all(-1)].any()
            torch.testing.assert_close(got, ref, rtol=0.02, atol=0.02 * float(scale))
    # dW_shard summed over the CP ranks (each holds its rows' share)
    for k in range(tp):
        dwk = sum(e["dw"][c][k].double() for c in range(cp))
        torch.testing.assert_close(dwk, f_dw[k * Vs:(k + 1) * Vs], rtol=0.02, atol=0.02 * float(f_dw.abs().max()))


@pytest.mark.parametrize("tp, cp", [(2, 2), (1, 2), (4, 1)])
def test_summed_gradients_match_cp1(tp, cp):
    """The same batch at cp = 1: per-position dX (summed over the CP ranks) and dW agree within bf16 rounding."""
    H, V = 256, 8192
    w = _weights(H, V)
    s = _setup(tp, cp, True, H, V)
    L = s["responses"].shape[1]
    g = torch.Generator(device="cuda").manual_seed(3)
    g_lp, g_ent = (torch.randn(len(s["n"]), L, generator=g, device="cuda") for _ in range(2))
    e = _emulate(s["plan"], s["streams"], w, s["responses"], tp, cp, True, g_lp, g_ent)
    cu1 = s["cu"]
    streams1 = [O.local_stream(s["seqs"], cu1, s["n"], 1, 0, int(cu1[-1]))]
    plan1 = RR.megatron_parallel(cu1, s["n"], s["r"], response_len=L, tp_size=1, cp_size=1)
    e1 = _emulate(plan1, streams1, w, s["responses"], 1, 1, False, g_lp, g_ent)
    torch.testing.assert_close(e["out"][0][0][0], e1["out"][0][0][0], rtol=1e-5, atol=1e-4)
    own = O.owner(cu1, s["n"], cp)
    Ts = s["T_c"] // tp
    for (b, pos), (c, t) in own.items():
        k = t // Ts
        a = e["dx"][c][k][t - k * Ts].float()
        ref = e1["dx"][0][0][int(cu1[b]) + pos].float()
        torch.testing.assert_close(a, ref, rtol=0.02, atol=2e-3)
    Vs = V // tp
    dw = torch.cat([sum(e["dw"][c][k].float() for c in range(cp)) for k in range(tp)])
    torch.testing.assert_close(dw, e1["dw"][0][0].float(), rtol=0.02, atol=2e-3)


def test_one_rank_op_matches_megatron_thd_and_stages():
    """tp = cp = 1 through the public op (no torch.distributed): the same rows, targets and cells as megatron_thd, the
    same bits as response_logprobs_entropy on the full stream, and dX zero off the response rows."""
    H, V = 512, 32064
    s = _setup(1, 1, False, H, V)
    w = _weights(H, V)
    L = s["responses"].shape[1]
    x = s["streams"][0]
    thd = RR.megatron_thd(s["cu"], s["n"], s["r"], response_len=L)
    # the token stream megatron_thd reads targets from: responses placed after each prediction row
    tok = torch.zeros(x.shape[0], dtype=torch.int64, device="cuda")
    for b in range(len(s["n"])):
        a = int(s["cu"][b] + s["n"][b] - s["r"][b])
        tok[a:a + int(s["r"][b])] = s["responses"][b, :int(s["r"][b])]
    it = thd.index(tok, x.shape[0])
    im = s["plan"].index(s["responses"], x.shape[0], 0, 0)
    assert torch.equal(it.rows, im.rows) and torch.equal(it.targets, im.targets)
    assert torch.equal(it.cell_map, im.cell_map) and torch.equal(it.cells[1:], im.cells)
    assert torch.equal(it.hidden_map, im.hidden_map)
    xx = x.clone().requires_grad_(True)
    ww = w.clone().requires_grad_(True)
    lp, ent = ops.megatron_response_logprobs_entropy(xx[:, None], ww, s["responses"], s["plan"], temperature=TEMP)
    xr = x.clone().requires_grad_(True)
    wr = w.clone().requires_grad_(True)
    rlp, rent = ops.response_logprobs_entropy(xr, wr, tok, thd, temperature=TEMP)
    assert torch.equal(lp, rlp) and torch.equal(ent, rent)
    g = torch.Generator(device="cuda").manual_seed(2)
    glp, gh = (torch.randn(lp.shape, generator=g, device="cuda") for _ in range(2))
    (lp * glp + ent * gh).sum().backward()
    (rlp * glp + rent * gh).sum().backward()
    torch.testing.assert_close(ww.grad.float(), wr.grad.float(), rtol=1e-2, atol=1e-3)
    torch.testing.assert_close(xx.grad.float(), xr.grad.float(), rtol=1e-2, atol=1e-3)
    assert torch.equal(xx.grad.ne(0).any(-1), xr.grad.ne(0).any(-1))
    # repeat calls: the same bits
    lp2, ent2 = ops.megatron_response_logprobs_entropy(x, w, s["responses"], s["plan"], temperature=TEMP)
    assert torch.equal(lp2, lp) and torch.equal(ent2, ent)


def test_device_lengths_match_host_lengths():
    for tp, cp, sp in ((2, 2, True), (4, 1, True), (2, 1, False)):
        s = _setup(tp, cp, sp, 64, 4096)
        d = _setup(tp, cp, sp, 64, 4096, device_lengths=True)
        assert d["plan"].on_device and not s["plan"].on_device
        Ts = s["T_c"] // tp if sp else s["T_c"]
        for c in range(cp):
            for k in range(tp):
                a, b = s["plan"].index(s["responses"], Ts, k, c), d["plan"].index(d["responses"], Ts, k, c)
                assert (a.R, a.Rmax_k, a.Rmax_c, a.counts) == (b.R, b.Rmax_k, b.Rmax_c, b.counts)
                for name in ("rows", "targets", "cells", "unpad", "cell_map", "hidden_map"):
                    assert torch.equal(getattr(a, name), getattr(b, name)), name


def test_device_length_errors_and_fixed_padding():
    cu, n, r = torch.tensor([0, 8, 16]), torch.tensor([8, 5]), torch.tensor([2, 1])
    plan = RR.megatron_parallel(cu.cuda(), n.cuda(), r.cuda(), response_len=4, tp_size=2, cp_size=2,
                                sequence_parallel=True)
    resp = torch.zeros(2, 4, dtype=torch.int64, device="cuda")
    with pytest.raises(ValueError, match="too few rows"):
        plan.index(resp, 1, 0, 0)  # T_c = 2 < 16 / 2
    bad = RR.megatron_parallel(torch.tensor([0, 6, 16]).cuda(), n.cuda(), r.cuda(), response_len=4, cp_size=2)
    with pytest.raises(ValueError, match="multiple of 2"):
        bad.index(resp, 8, 0, 0)
    # padding_seqlen: the CP-local stream is longer than cu[-1] / cp; the extra rows are nobody's
    s = _setup(2, 2, True, 64, 4096, fixed=4 * 128)
    ix = s["plan"].index(s["responses"], s["T_c"] // 2, 1, 1)
    m = O.rank_maps(s["cu"], s["n"], s["r"], s["responses"].tolist(), 48, 2, 2, True, s["T_c"], 1, 1)
    assert ix.hidden_map.tolist() == m["hidden_map"] and ix.send.tolist() == m["send"]


def _count_syncs(fn):
    with warnings.catch_warnings(record=True) as rec:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            out = fn()
        finally:
            torch.cuda.set_sync_debug_mode("default")
    return out, sum("called a synchronizing CUDA operation" in str(w.message) for w in rec)


def test_no_host_sync_with_host_lengths():
    s = _setup(1, 1, False, 256, 8192)
    w = _weights(256, 8192)
    x = s["streams"][0].clone().requires_grad_(True)
    resp = s["responses"]
    torch.cuda.synchronize()
    (lp, ent), fwd = _count_syncs(lambda: ops.megatron_response_logprobs_entropy(x, w, resp, s["plan"]))
    _, bwd = _count_syncs(lambda: (lp.sum() + ent.sum()).backward())
    assert fwd == 0 and bwd == 0
    d = _setup(1, 1, False, 256, 8192, device_lengths=True)
    _, fwd = _count_syncs(lambda: ops.megatron_response_logprobs_entropy(x.detach(), w, resp, d["plan"]))
    assert fwd == 1


class _PeerDist:
    """torch.distributed stand-in for rank (c, k) of a grid emulated by _emulate: each collective records its traffic
    and returns what the other ranks' stages put in, with this rank's own buffer in its slot, reduced in the
    emulation's order - so the op's own wiring of the collectives must reproduce the emulation's bits."""

    def __init__(self, e, c, k, tp, cp):
        self.e, self.c, self.k, self.tp, self.cp, self.calls = e, c, k, tp, cp, []

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
        if kind == "cp":
            peers, me = list(self.e["vals"]), self.c
        else:
            peers, me = list(self.e["rows" if inp.dtype == torch.bfloat16 else "rec"][self.c]), self.k
        assert torch.equal(peers[me], inp)  # the op's own buffer is what the stages give
        peers[me] = inp
        out.copy_(torch.stack(peers))

    def reduce_scatter_tensor(self, out, inp, group=None):
        self.calls.append(("reduce_scatter", group[2], inp.numel() * inp.element_size(), inp.dtype))
        sends = list(self.e["grad_send"][self.c])
        sends[self.k] = inp.view(sends[self.k].shape)
        out.copy_(torch.stack([x[self.k].float() for x in sends]).sum(0).to(torch.bfloat16))

    def all_reduce(self, t, group=None):
        self.calls.append(("all_reduce", group[2], t.numel() * t.element_size(), t.dtype))
        parts = list(self.e["part"][self.c])
        parts[self.k] = t.clone()
        t.copy_(torch.stack(parts).sum(0))


def _peer_run(monkeypatch, s, w, e, tp, cp, sp, c, k, loss_fn=None, g_lp=None, g_ent=None):
    """The public op as rank (c, k), its peers served from the emulation: (lp, ent, dX, dW_shard, calls, n_fwd)."""
    import torch.distributed as dist

    fake = _PeerDist(e, c, k, tp, cp)
    for name in ("is_available", "is_initialized", "get_world_size", "get_rank", "all_gather_into_tensor",
                 "reduce_scatter_tensor", "all_reduce"):
        monkeypatch.setattr(dist, name, getattr(fake, name))
    Vs = w.shape[0] // tp
    Ts = s["T_c"] // tp if sp else s["T_c"]
    x = (s["streams"][c][k * Ts:(k + 1) * Ts] if sp else s["streams"][c])[:, None].clone().requires_grad_(True)
    ws = w[k * Vs:(k + 1) * Vs].clone().requires_grad_(True)
    lp, ent = ops.megatron_response_logprobs_entropy(x, ws, s["responses"], s["plan"], temperature=TEMP,
                                                     tp_group=(tp, k, "tp"), cp_group=(cp, c, "cp"))
    n_fwd = len(fake.calls)
    loss = loss_fn(lp, ent) if loss_fn is not None else (lp * g_lp + ent * g_ent).sum()
    loss.backward()
    monkeypatch.undo()
    return lp, ent, loss, x.grad[:, 0], ws.grad, fake.calls, n_fwd


WIRING = [(2, 2, True, False), (2, 2, False, False), (4, 1, True, False), (2, 1, False, False), (1, 2, False, False),
          (2, 2, True, True), (2, 4, True, True), (1, 2, False, True)]


@pytest.mark.parametrize("tp, cp, sp, sparse", WIRING)
def test_op_on_every_rank_matches_emulation(monkeypatch, tp, cp, sp, sparse):
    """The public op on every rank of the grid (its SP row all-gather, unpad, record all-gather, CP value all-gather
    and bf16 reduce-scatter or fp32 all-reduce, with the other ranks' buffers served from the emulation): log-probs,
    entropies, dX shard and d_weight_shard bit-identical to the emulation, CP ranks without rows included."""
    H, V = 128, 4096
    s = _setup(tp, cp, sp, H, V, sparse=sparse)
    w = _weights(H, V)
    L = s["responses"].shape[1]
    g = torch.Generator(device="cuda").manual_seed(4)
    g_lp, g_ent = (torch.randn(len(s["n"]), L, generator=g, device="cuda") for _ in range(2))
    e = _emulate(s["plan"], s["streams"], w, s["responses"], tp, cp, sp, g_lp, g_ent)
    for c in range(cp):
        for k in range(tp):
            lp, ent, _, dx, dw, _, _ = _peer_run(monkeypatch, s, w, e, tp, cp, sp, c, k, g_lp=g_lp, g_ent=g_ent)
            assert torch.equal(lp, e["out"][c][k][0]) and torch.equal(ent, e["out"][c][k][1]), (c, k)
            assert torch.equal(dx, e["dx"][c][k]) and torch.equal(dw, e["dw"][c][k]), (c, k)


@pytest.mark.parametrize("agg", ["token-mean", "seq-mean-token-sum"])
@pytest.mark.parametrize("tp, cp, sp, sparse", [(2, 2, True, False), (1, 2, False, False), (2, 2, True, True)])
def test_composition_with_reasoning_actor_loss(monkeypatch, tp, cp, sp, sparse, agg):
    """reasoning_actor_loss on each rank's outputs (Megatron's loss_func order): the same loss bits on every rank, and
    each rank's gradients those of the emulation driven by the loss's own output gradients."""
    from rlinf_b200.algorithms import reasoning_actor_loss

    H, V = 128, 4096
    s = _setup(tp, cp, sp, H, V, sparse=sparse)
    w = _weights(H, V)
    bsz, L = s["responses"].shape
    gen = torch.Generator().manual_seed(3)
    f = lambda sc=1.0: (torch.randn(bsz, L, generator=gen) * sc).cuda()  # noqa: E731
    old, adv, ref = f(0.5) - 3, f(), f(0.5) - 3
    mask = (torch.arange(L)[None] < s["r"][:, None]).cuda()

    def loss_fn(lp, ent):
        return reasoning_actor_loss(lp, adv, mask, old_logprobs=old, ref_logprobs=ref, entropy=ent,
                                    loss_agg_func=agg, entropy_bonus=0.01, kl_beta=0.05,
                                    kl_penalty_type="low_var_kl", kl_order="megatron")[0]

    e0 = _emulate(s["plan"], s["streams"], w, s["responses"], tp, cp, sp, None, None, backward=False)
    lp0 = e0["out"][0][0][0].clone().requires_grad_(True)
    ent0 = e0["out"][0][0][1].clone().requires_grad_(True)
    loss0 = loss_fn(lp0, ent0)
    loss0.backward()
    e = _emulate(s["plan"], s["streams"], w, s["responses"], tp, cp, sp, lp0.grad, ent0.grad)
    for c in range(cp):
        for k in range(tp):
            _, _, loss, dx, dw, _, _ = _peer_run(monkeypatch, s, w, e, tp, cp, sp, c, k, loss_fn=loss_fn)
            assert torch.equal(loss, loss0), (c, k)
            assert torch.equal(dx, e["dx"][c][k]) and torch.equal(dw, e["dw"][c][k]), (c, k)


@pytest.mark.parametrize("tp, cp, sp, sparse", [(2, 2, True, False), (4, 1, True, False), (2, 1, False, False),
                                                (1, 2, False, False), (2, 2, True, True), (2, 2, False, True)])
def test_collective_budget(monkeypatch, tp, cp, sp, sparse):
    """Forward: under SP one bf16 all-gather of tp * Rmax_k * H * 2 bytes over TP, the [R_c, 4] record all-gather,
    one [Rmax_c, 2] fp32 all-gather over CP; backward: one bf16 reduce-scatter over TP (SP) or one fp32 all-reduce of
    R_c * H * 4 bytes (no SP), nothing over CP.  The last CP rank is checked; with sparse lengths it has no row and
    still makes every collective."""
    H, V = 128, 4096
    s = _setup(tp, cp, sp, H, V, sparse=sparse)
    w = _weights(H, V)
    L = s["responses"].shape[1]
    ones = torch.ones(len(s["n"]), L, device="cuda")
    e = _emulate(s["plan"], s["streams"], w, s["responses"], tp, cp, sp, ones, ones)
    k, c = tp - 1, cp - 1
    _, _, _, _, _, calls, nf = _peer_run(monkeypatch, s, w, e, tp, cp, sp, c, k, g_lp=ones, g_ent=ones)
    ix = e["idx"][c][k]
    assert (ix.R == 0) == sparse
    want = ([("all_gather", "tp", tp * ix.Rmax_k * H * 2, torch.bfloat16)] if sp and tp > 1 else [])
    want += [("all_gather", "tp", tp * ix.R * 16, torch.float32)] if tp > 1 else []
    want += [("all_gather", "cp", cp * ix.Rmax_c * 8, torch.float32)] if cp > 1 else []
    assert calls[:nf] == want
    if tp > 1:
        bwd = [("reduce_scatter", "tp", tp * ix.Rmax_k * H * 2, torch.bfloat16)] if sp else [
            ("all_reduce", "tp", ix.R * H * 4, torch.float32)]
    else:
        bwd = []
    assert calls[nf:] == bwd


def _free_port():
    with socket.socket() as so:
        so.bind(("127.0.0.1", 0))
        return so.getsockname()[1]


@pytest.mark.parametrize("tp, cp, sp, sparse", [(2, 1, True, False), (1, 2, False, False), (2, 2, True, False),
                                                (1, 2, False, True), (2, 2, True, True)])
def test_nccl_matches_emulation(tmp_path, tp, cp, sp, sparse):
    world = tp * cp
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs {world} GPUs")
    out = tmp_path / "out.json"
    env = dict(os.environ, RB200_DIST_OUT=str(out), RB200_GRID=f"{tp},{cp},{int(sp)},{int(sparse)}")
    cmd = [sys.executable, "-m", "torch.distributed.run", f"--nproc_per_node={world}",
           f"--master_port={_free_port()}", os.path.join(HERE, "dist_response_rows_mp_worker.py")]
    proc = subprocess.run(cmd, env=env, capture_output=True, text=True, timeout=600)
    assert proc.returncode == 0, proc.stdout[-4000:] + proc.stderr[-4000:]
    res = json.loads(out.read_text())
    assert res["ok"], res


GOLDEN = os.path.join(HERE, "golden", "golden_response_rows_mp.npz")


@pytest.mark.skipif(not os.path.exists(GOLDEN), reason="fixture not generated")
def test_reference_fixture_semantics_per_rank():
    """The reference's forward and log-prob gradient, per rank of each fixture grid (ranks without rows included): the
    op's stages on the fixture's hidden shards (bf16-exact) give the reference's training and inference log-probs and,
    for every rank, a dX shard that is zero exactly where the reference's is."""
    gz = {k: torch.from_numpy(v) for k, v in np.load(GOLDEN).items()}
    for key in sorted(k[:-len("_meta")] for k in gz if k.endswith("_meta")):
        tp, cp, sp, L, bsz, T_c, V = (int(x) for x in gz[f"{key}_meta"])
        W = gz["W"].cuda().to(torch.bfloat16)
        plan = RR.megatron_parallel(gz[f"{key}_cu"], gz[f"{key}_n"], gz[f"{key}_r"], response_len=L, tp_size=tp,
                                    cp_size=cp, sequence_parallel=bool(sp))
        resp = gz[f"{key}_responses"].cuda()
        Ts = T_c // tp if sp else T_c
        streams = []
        for c in range(cp):
            parts = [gz[f"{key}_c{c}_k{k}_hidden"] for k in range(tp)]
            streams.append((torch.cat(parts) if sp else parts[0]).cuda().to(torch.bfloat16))
        g_lp = gz[f"{key}_g"].cuda()
        e = _emulate(plan, streams, W, resp, tp, cp, bool(sp), g_lp, torch.zeros_like(g_lp))
        lp = e["out"][0][0][0]
        ref = gz[f"{key}_logprobs"].cuda()
        valid = torch.arange(L, device="cuda")[None] < gz[f"{key}_r"].cuda()[:, None]
        torch.testing.assert_close(lp[valid], ref[valid], rtol=1e-3, atol=2e-2)
        # the inference path's output, zeros past r_b included
        torch.testing.assert_close(lp, gz[f"{key}_infer_logprobs"].cuda(), rtol=1e-3, atol=2e-2)
        assert not lp[~valid].any()
        for c in range(cp):
            for k in range(tp):
                rg = gz[f"{key}_c{c}_k{k}_grad"].cuda().reshape(Ts, -1)
                got = e["dx"][c][k].float()
                assert torch.equal((got != 0).any(-1), (rg != 0).any(-1)), (key, c, k)
                torch.testing.assert_close(got, rg, rtol=0.05, atol=0.05 * float(rg.abs().max()) + 1e-6)
