"""ops.response_logprobs_entropy on the GPU: the LM head on the response rows of padded, FSDP-packed and Megatron THD
batches only.  Bit-identity with linear_logprobs_entropy on the rows gathered by torch indexing (log-probs, entropies,
dW, dX on response rows and exact zeros elsewhere), agreement with fp64 on the full logits, the reference fixture's
semantics, vocabulary parallelism, composition with reasoning_actor_loss, invariance of the loss to the masked
columns, repeatability, host syncs, launches and peak memory."""
from __future__ import annotations

import itertools
import json
import os
import warnings

import numpy as np
import pytest
import torch

import response_rows_oracle as O
from rlinf_b200 import _lib, ops
from rlinf_b200 import response_rows as RR
from rlinf_b200.algorithms import reasoning_actor_loss

pytestmark = pytest.mark.gpu
V_BIG = 151936
HERE = os.path.dirname(os.path.abspath(__file__))


def make_batch(layout, H, V, seed=0, bsz=5, L=48, device_lengths=False):
    """(plan, hidden, tokens, a, r, shift) of a seeded batch: one empty response and one of full length."""
    g = torch.Generator().manual_seed(seed)
    r = torch.randint(1, L, (bsz,), generator=g)
    r[1], r[-1] = 0, L
    p = torch.randint(1, 24, (bsz,), generator=g)
    if layout == "padded":
        S = 24 + L
        plan = RR.padded(bsz, S, L, r.cuda() if device_lengths else r)
        a, shape, shift = O.first_rows("padded", r, S=S, L=L), (bsz, S), 0
    elif layout == "fsdp_packed":
        T = int((p + r).sum()) + 5  # eos-padded to a fixed length
        plan = RR.fsdp_packed(p.cuda() if device_lengths else p, r, 24, response_len=L)
        a, shape, shift = O.first_rows("fsdp_packed", r, prompt_lengths=p), (1, T), 1
    else:
        n = p + r
        cu = torch.zeros(bsz + 1, dtype=torch.int64)
        cu[1:] = torch.cumsum(n + n % 2, 0)  # aligned to TP 2
        T = int(cu[-1]) + 6
        plan = RR.megatron_thd(cu.cuda() if device_lengths else cu, n, r, response_len=L)
        a, shape, shift = O.first_rows("megatron_thd", r, cu_seqlens_padded=cu, seq_lengths=n), (T, 1), 0
    x = (torch.randn(*shape, H, generator=g) * 2).to(torch.bfloat16).cuda()
    tok = torch.randint(0, V, shape, generator=g).cuda()
    return plan, x, tok, a, r, shift


def weight(V, H, seed=1):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(V, H, generator=g) * (2.0 / H ** 0.5)).to(torch.bfloat16).cuda()


def upstream(bsz, L, seed=2):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(bsz, L, generator=g).cuda(), torch.randn(bsz, L, generator=g).cuda()


def torch_route(x, w, tok, a, r, shift, L, temperature, want_ent, need_x, need_w, glp, gh):
    """linear_logprobs_entropy on the response rows gathered by torch indexing, cells by torch indexing."""
    H = x.shape[-1]
    x2 = x.reshape(-1, H)
    rows, targets = O.rows_and_targets(a, r, tok.reshape(-1).cpu(), shift)
    hc = x2[torch.tensor(rows, device="cuda")].detach().requires_grad_(need_x)
    ww = w.detach().clone().requires_grad_(need_w)
    lp, ent = ops.linear_logprobs_entropy(hc, ww, torch.tensor(targets, device="cuda"), temperature,
                                          compute_entropy=want_ent)
    lpc, entc = torch.zeros(len(a), L, device="cuda"), torch.zeros(len(a), L, device="cuda")
    o = 0
    for b, rb in enumerate(r.tolist()):
        if rb:
            lpc[b, :rb] = lp[o:o + rb]
            if want_ent:
                entc[b, :rb] = ent[o + shift:o + shift + rb]
            o += rb + shift
    loss = (lpc * glp).sum() + ((entc * gh).sum() if want_ent else 0)
    dx = dw = None
    if need_x or need_w:
        loss.backward()
    if need_x:
        dx = torch.zeros_like(x2)
        dx[torch.tensor(rows, device="cuda")] = hc.grad
    if need_w:
        dw = ww.grad
    return lpc, (entc if want_ent else None), dx, dw


def op_route(x, w, tok, plan, temperature, want_ent, need_x, need_w, glp, gh, group=None):
    xx = x.detach().clone().requires_grad_(need_x)
    ww = w.detach().clone().requires_grad_(need_w)
    lp, ent = ops.response_logprobs_entropy(xx, ww, tok, plan, temperature=temperature, compute_entropy=want_ent,
                                            group=group)
    if need_x or need_w:
        ((lp * glp).sum() + ((ent * gh).sum() if want_ent else 0)).backward()
    return lp, ent, (xx.grad.reshape(-1, x.shape[-1]) if need_x else None), (ww.grad if need_w else None)


LAYOUTS = ["padded", "fsdp_packed", "megatron_thd"]
MODES = [(True, True, True), (False, True, True), (True, False, True), (True, True, False)]  # ent, need_x, need_w


@pytest.mark.parametrize("layout", LAYOUTS)
@pytest.mark.parametrize("H", [64, 1536])
@pytest.mark.parametrize("mode", MODES, ids=["all", "no_entropy", "hidden_frozen", "weight_frozen"])
def test_bit_identical_to_torch_gathered_rows(layout, H, mode):
    want_ent, need_x, need_w = mode
    plan, x, tok, a, r, shift = make_batch(layout, H, V_BIG)
    w = weight(V_BIG, H)
    glp, gh = upstream(plan.bsz, plan.response_len)
    got = op_route(x, w, tok, plan, 0.8, want_ent, need_x, need_w, glp, gh)
    want = torch_route(x, w, tok, a, r, shift, plan.response_len, 0.8, want_ent, need_x, need_w, glp, gh)
    assert torch.equal(got[0], want[0])
    assert (got[1] is None) == (not want_ent)
    if want_ent:
        assert torch.equal(got[1], want[1])
    if need_x:
        assert torch.equal(got[2], want[2])  # zero rows outside the responses included
        rows = O.rows_and_targets(a, r, tok.reshape(-1).cpu(), shift)[0]
        outside = torch.ones(got[2].shape[0], dtype=torch.bool)
        outside[rows] = False
        assert not got[2][outside.cuda()].any()
    if need_w:
        assert torch.equal(got[3], want[3])


@pytest.mark.parametrize("layout", LAYOUTS)
def test_device_lengths_match_host_lengths(layout):
    plan_h, x, tok, *_ = make_batch(layout, 64, 4096)
    plan_d = make_batch(layout, 64, 4096, device_lengths=True)[0]
    assert plan_d.on_device
    w = weight(4096, 64)
    glp, gh = upstream(plan_h.bsz, plan_h.response_len)
    a = op_route(x, w, tok, plan_h, 1.0, True, True, True, glp, gh)
    b = op_route(x, w, tok, plan_d, 1.0, True, True, True, glp, gh)
    for u, v in zip(a, b):
        assert torch.equal(u, v)


def test_device_length_errors_come_back_from_the_plan_kernel():
    x = torch.zeros(1, 40, 64, dtype=torch.bfloat16, device="cuda")
    tok = torch.zeros(1, 40, dtype=torch.int64, device="cuda")
    w = weight(1024, 64)
    bad = [RR.fsdp_packed(torch.tensor([3, 0], device="cuda"), torch.tensor([2, 2], device="cuda"), 6, response_len=4),
           RR.fsdp_packed(torch.tensor([3, 2], device="cuda"), torch.tensor([5, 2], device="cuda"), 6, response_len=4),
           RR.fsdp_packed(torch.tensor([33, 2], device="cuda"), torch.tensor([4, 4], device="cuda"), 33,
                          response_len=4),
           RR.megatron_thd(torch.tensor([0, 4, 8], device="cuda"), torch.tensor([6, 3], device="cuda"),
                           torch.tensor([2, 1], device="cuda"), response_len=4)]
    for plan, msg in zip(bad, ["no prompt token", "response_len", r"outside \[0, T\)", "overlap"]):
        with pytest.raises(ValueError, match=msg):
            ops.response_logprobs_entropy(x, w, tok, plan)


@pytest.mark.parametrize("layout", LAYOUTS)
def test_plan_kernel_maps_match_oracle(layout):
    plan, x, tok, a, r, shift = make_batch(layout, 64, 4096)
    T = tok.numel()
    idx = plan.index(tok.reshape(-1), T)
    rows, targets = O.rows_and_targets(a, r, tok.reshape(-1).cpu(), shift)
    assert idx.R == len(rows) == plan.num_rows
    assert idx.rows.tolist() == rows and idx.targets.tolist() == targets
    hm = [-1] * T
    for c, row in enumerate(rows):
        hm[row] = c
    assert idx.hidden_map.tolist() == hm


@pytest.mark.parametrize("layout", LAYOUTS)
def test_vs_fp64_full_logits(layout):
    H, temp = 64, 0.8
    plan, x, tok, a, r, shift = make_batch(layout, H, V_BIG)
    w = weight(V_BIG, H)
    lp, ent = ops.response_logprobs_entropy(x, w, tok, plan, temperature=temp)
    z = (x.reshape(-1, H).double() @ w.double().T) / temp
    logp = torch.log_softmax(z, -1)
    t = tok.reshape(-1)
    nxt = torch.cat([t[1:], t[-1:]])
    lp_rows = logp.gather(1, nxt[:, None])[:, 0].cpu()
    ent_rows = -(logp.exp() * logp).sum(-1).cpu()
    L = plan.response_len
    torch.testing.assert_close(lp.cpu().double(), O.to_cells(lp_rows, a, r, L), rtol=1e-4, atol=1e-4)
    torch.testing.assert_close(ent.cpu().double(), O.to_cells(ent_rows, a, r, L, shift), rtol=1e-4, atol=1e-4)


def test_reference_fixture_semantics():
    """The fixture's response columns at its tiny shapes: the FSDP-packed entropy one row later, zeros past r_b."""
    gz = {k: torch.from_numpy(v) for k, v in np.load(os.path.join(HERE, "golden", "golden_response_rows.npz")).items()}
    V, H, MP, L, S, PAD = (int(v) for v in gz["meta"])
    r, p, temp = gz["response_lengths"], gz["prompt_lengths"], float(gz["temperature"])
    w = gz["W"].to(torch.bfloat16).cuda()
    cases = {"fsdp_padded": RR.padded(len(r), S, L, r), "fsdp_packed_var": RR.fsdp_packed(p, r, MP, response_len=L),
             "megatron_tp1_var_train": RR.megatron_thd(gz["megatron_tp1_var_train_cu"], gz["seq_lengths"], r,
                                                       response_len=L)}
    valid = torch.arange(L)[None] < r[:, None]
    for case, plan in cases.items():
        h = gz[f"{case}_hidden"].to(torch.bfloat16)
        lp, ent = ops.response_logprobs_entropy(h.cuda(), w, gz[f"{case}_tokens"].cuda(), plan, temperature=temp)
        lp, ent = lp.cpu(), ent.cpu()
        ref_lp = gz[f"{case}_logprobs"]
        ref_ent = gz[f"{case}_entropy"]
        torch.testing.assert_close(lp[valid], ref_lp[valid], rtol=0.05, atol=0.05, msg=case)  # bf16 inputs
        torch.testing.assert_close(ent[valid], ref_ent[valid], rtol=0.05, atol=0.05, msg=case)
        assert not lp[~valid].any() and not ent[~valid].any()
    # the one-column entropy offset is visible at this precision
    h = gz["fsdp_packed_var_hidden"].to(torch.bfloat16).cuda()
    _, ent = ops.response_logprobs_entropy(h, w, gz["fsdp_packed_var_tokens"].cuda(), cases["fsdp_packed_var"],
                                           temperature=temp)
    z = (h.reshape(-1, H).double() @ w.double().T) / temp
    logp = torch.log_softmax(z, -1)
    ent_rows = -(logp.exp() * logp).sum(-1).cpu()
    a = O.first_rows("fsdp_packed", r, prompt_lengths=p)
    torch.testing.assert_close(ent.cpu().double(), O.to_cells(ent_rows, a, r, L, 1), rtol=1e-4, atol=1e-4)
    assert (ent.cpu().double() - O.to_cells(ent_rows, a, r, L, 0))[valid].abs().max() > 0.1


@pytest.mark.parametrize("P", [2, 4])
def test_vocab_parallel_emulated(P):
    """P ranks emulated on one device over the plan's rows: bit-identical to the vocabulary-parallel ops on the rows
    gathered by torch indexing, and equal to the one-rank op within fp32 merge-order rounding."""
    H, temp = 1536, 0.8
    plan, x, tok, a, r, shift = make_batch("megatron_thd", H, V_BIG)
    w = weight(V_BIG, H)
    T = tok.numel()
    idx = plan.index(tok.reshape(-1), T)
    Vs = V_BIG // P
    hc = x.reshape(T, H)[idx.rows]
    rows, targets = O.rows_and_targets(a, r, tok.reshape(-1).cpu(), shift)
    assert torch.equal(hc, x.reshape(T, H)[torch.tensor(rows, device="cuda")])
    rec = torch.stack([ops.lmhead_vp_partials(ops.gather_rows(x.reshape(T, H), idx.rows), w[k * Vs:(k + 1) * Vs],
                                              idx.targets, k, P, temp) for k in range(P)])
    rec_t = torch.stack([ops.lmhead_vp_partials(hc, w[k * Vs:(k + 1) * Vs], torch.tensor(targets, device="cuda"), k, P,
                                                temp) for k in range(P)])
    assert torch.equal(rec, rec_t)
    elp, eent, _ = ops.vp_combine(rec, idx.targets, Vs)
    lp1, ent1 = ops.response_logprobs_entropy(x, w, tok, plan, temperature=temp)
    z = torch.zeros(1, device="cuda")
    lp = torch.cat([elp, z])[idx.cell_map].view(lp1.shape)
    ent = torch.cat([eent, z])[idx.cell_map].view(lp1.shape)
    torch.testing.assert_close(lp, lp1, rtol=1e-5, atol=1e-5)
    torch.testing.assert_close(ent, ent1, rtol=1e-5, atol=1e-5)


def test_two_rank_nccl_matches_emulation(tmp_path):
    import socket
    import subprocess
    import sys

    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    outp = tmp_path / "rr.json"
    env = dict(os.environ, RB200_DIST_OUT=str(outp))
    worker = os.path.join(HERE, "dist_response_rows_worker.py")
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2",
                        "--master-addr", "127.0.0.1", "--master-port", str(port), worker], env=env, capture_output=True,
                       text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    res = json.loads(outp.read_text())
    assert res["ok"], res


LOSS_OPTS = list(itertools.product(["token-mean", "seq-mean-token-sum", "seq-mean-token-mean"], ["fsdp", "megatron"],
                                   [False, True], [False, True]))


def _loss_inputs(bsz, L, seed=3):
    g = torch.Generator().manual_seed(seed)
    f = lambda s=1.0: (torch.randn(bsz, L, generator=g) * s).cuda()  # noqa: E731
    return dict(old_logprobs=f(0.5) - 3, advantages=f(), ref_logprobs=f(0.5) - 3, rollout_logprobs=f(0.5) - 3)


def _loss(lp, ent, mask, ins, agg, order, rtkl, isfix):
    kw = dict(advantages=ins["advantages"], loss_mask=mask, entropy=ent, ref_logprobs=ins["ref_logprobs"],
              loss_agg_func=agg, entropy_bonus=0.01, kl_beta=0.05, kl_penalty_type="low_var_kl", kl_order=order,
              clip_ratio_c=3.0)
    if rtkl or isfix:
        kw.update(rollout_logprobs=ins["rollout_logprobs"], recomputed_logprobs=ins["old_logprobs"],
                  importance_sampling_fix=isfix, importance_sampling_clip=2.0 if isfix else None)
    else:
        kw.update(old_logprobs=ins["old_logprobs"])
    return reasoning_actor_loss(lp, **kw)


@pytest.mark.parametrize("layout", LAYOUTS)
def test_composition_with_reasoning_actor_loss(layout):
    H = 1536
    plan, x, tok, a, r, shift = make_batch(layout, H, V_BIG)
    w = weight(V_BIG, H)
    L = plan.response_len
    mask = (torch.arange(L)[None] < r[:, None]).cuda()
    ins = _loss_inputs(plan.bsz, L)
    grads = []
    for route in ("op", "torch"):
        xx, ww = x.detach().clone().requires_grad_(True), w.detach().clone().requires_grad_(True)
        if route == "op":
            lp, ent = ops.response_logprobs_entropy(xx, ww, tok, plan, temperature=0.9)
        else:
            rows, targets = O.rows_and_targets(a, r, tok.reshape(-1).cpu(), shift)
            ri = torch.tensor(rows, device="cuda")
            clp, cent = ops.linear_logprobs_entropy(xx.reshape(-1, H)[ri], ww, torch.tensor(targets, device="cuda"),
                                                    0.9)
            z = torch.zeros(1, device="cuda")
            cm = torch.tensor([[sum(int(v) + shift for v in r[:b] if int(v) > 0) + j if j < int(r[b]) else -1
                                for j in range(L)] for b in range(plan.bsz)], device="cuda")
            lp = torch.cat([clp, z])[cm]
            ent = torch.cat([cent, z])[shift:][cm]
        loss, _ = _loss(lp, ent, mask, ins, "token-mean", "fsdp", False, False)
        loss.backward()
        grads.append((loss.detach(), xx.grad, ww.grad))
    for u, v in zip(*grads):
        assert torch.equal(u, v)


@pytest.mark.parametrize("agg, order, rtkl, isfix", LOSS_OPTS)
def test_loss_invariant_to_masked_columns(agg, order, rtkl, isfix):
    """Zeros (this op) or the reference's values (log p(pad), the last token's values) at j >= r_b: the same loss,
    gradients and metrics, bit for bit.  Every row has a response token: an empty row makes seq-mean-token-mean NaN
    whatever its columns hold (the reference's quirk, kept)."""
    bsz, L = 6, 64
    g = torch.Generator().manual_seed(4)
    r = torch.tensor([10, 2, 64, 33, 1, 50])
    mask = (torch.arange(L)[None] < r[:, None]).cuda()
    lp0 = (torch.randn(bsz, L, generator=g) * 0.5 - 3).cuda() * mask
    ent0 = torch.rand(bsz, L, generator=g).cuda() * mask
    junk_lp = (torch.randn(bsz, L, generator=g) * 5 - 9).cuda()
    junk_ent = (torch.rand(bsz, L, generator=g) * 4).cuda()
    ins = _loss_inputs(bsz, L)
    outs = []
    for lp, ent in ((lp0, ent0), (torch.where(mask, lp0, junk_lp), torch.where(mask, ent0, junk_ent))):
        lp, ent = lp.clone().requires_grad_(True), ent.clone().requires_grad_(True)
        loss, metrics = _loss(lp, ent, mask, ins, agg, order, rtkl, isfix)
        loss.backward()
        outs.append([loss.detach(), lp.grad, ent.grad] + [metrics[k] for k in sorted(metrics)])
    for u, v in zip(*outs):
        torch.testing.assert_close(u, v, rtol=0, atol=0, equal_nan=True)


def test_repeat_calls_same_bits():
    plan, x, tok, *_ = make_batch("fsdp_packed", 1536, V_BIG)
    w = weight(V_BIG, 1536)
    glp, gh = upstream(plan.bsz, plan.response_len)
    a = op_route(x, w, tok, plan, 0.7, True, True, True, glp, gh)
    b = op_route(x, w, tok, plan, 0.7, True, True, True, glp, gh)
    for u, v in zip(a, b):
        assert torch.equal(u, v)


def _count_syncs(fn):
    with warnings.catch_warnings(record=True) as rec:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            out = fn()
        finally:
            torch.cuda.set_sync_debug_mode("default")
    return out, sum("called a synchronizing CUDA operation" in str(w.message) for w in rec)


@pytest.mark.parametrize("device_lengths", [False, True])
def test_host_syncs_and_launches(device_lengths):
    H, V = 1536, V_BIG
    plan, x, tok, *_ = make_batch("megatron_thd", H, V, device_lengths=device_lengths)
    w = weight(V, H)
    glp, gh = upstream(plan.bsz, plan.response_len)
    xx, ww = x.clone().requires_grad_(True), w.clone().requires_grad_(True)
    ops.response_logprobs_entropy(xx, ww, tok, plan)  # warm-up
    torch.cuda.synchronize()
    lib = _lib.load()
    n0 = lib.rb200_launch_count()
    (lp, ent), fwd_syncs = _count_syncs(lambda: ops.response_logprobs_entropy(xx, ww, tok, plan))
    n_fwd = lib.rb200_launch_count() - n0
    _, bwd_syncs = _count_syncs(lambda: ((lp * glp).sum() + (ent * gh).sum()).backward())
    n_bwd = lib.rb200_launch_count() - n0 - n_fwd
    assert fwd_syncs == (1 if device_lengths else 0)
    assert bwd_syncs == 0
    # the fused op alone on the same R rows
    idx = plan.index(tok.reshape(-1), tok.numel())
    hc = x.reshape(-1, H)[idx.rows].requires_grad_(True)
    n1 = lib.rb200_launch_count()
    clp, cent = ops.linear_logprobs_entropy(hc, ww.detach().requires_grad_(True), idx.targets)
    n_lin_fwd = lib.rb200_launch_count() - n1
    (clp.sum() + cent.sum()).backward()
    n_lin_bwd = lib.rb200_launch_count() - n1 - n_lin_fwd
    # forward: plan + hidden gather + 2 cell gathers; backward: 2 cell gathers + the dX scatter
    assert n_fwd == n_lin_fwd + 4, (n_fwd, n_lin_fwd)
    assert n_bwd == n_lin_bwd + 3, (n_bwd, n_lin_bwd)


def test_peak_memory_bound():
    H, V = 1536, V_BIG
    bsz, L = 8, 1536
    plan, x, tok, a, r, shift = make_batch("padded", H, V, bsz=bsz, L=L)
    w = weight(V, H)
    glp, gh = upstream(bsz, L)
    T = tok.numel()
    idx = plan.index(tok.reshape(-1), T)
    hc = x.reshape(T, H)[idx.rows].contiguous()
    tg = idx.targets.clone()
    del idx

    def peak(fn):
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        fn()
        torch.cuda.synchronize()
        return torch.cuda.max_memory_allocated() - base

    def lin():
        hh, ww = hc.detach().requires_grad_(True), w.detach().requires_grad_(True)
        lp, ent = ops.linear_logprobs_entropy(hh, ww, tg)
        (lp.sum() + ent.sum()).backward()

    def op():
        xx, ww = x.detach().requires_grad_(True), w.detach().requires_grad_(True)
        lp, ent = ops.response_logprobs_entropy(xx, ww, tok, plan)
        ((lp * glp).sum() + (ent * gh).sum()).backward()

    p_lin, p_op = peak(lin), peak(op)
    R = hc.shape[0]
    allowance = T * H * 2 + 8 * (2 * T + 3 * bsz * L + 4 * R) + (2 << 20)  # dX [T, H], the plan, allocator rounding
    assert p_op <= p_lin + allowance, (p_op, p_lin, allowance)
