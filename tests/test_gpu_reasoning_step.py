"""Reasoning step bookkeeping on the GPU: utils.distributed.compute_rollout_metrics(_dynamic), MegatronLossEpilogue,
valid_token_count and step_metrics.

Data-parallel ranks are emulated on one device: a torch.distributed stand-in serves each rank's peers' buffers (records
for the all-gather, packed metrics for the SUM all-reduce, added in rank order) and counts the collectives.  Checked:
the device against the torch oracle (tests/reasoning_step_oracle.py) bit for bit, per rank, on the fixture's batches
and hyper-parameters; against the reference fixture within one fp32 rounding where the reference's result depends on
its own summation order; against fp64 at bsz 512 x L 8,192 and 64 x 32,768; repeat calls bit-identical; no host sync
from the first micro-batch's epilogue to the step finish, nor in the rollout metrics before their one copy; one
collective per micro-batch and at most two for the rollout metrics; the composition with reasoning_actor_loss and
reasoning_critic_loss, whose scaled gradient is the scale times the unscaled one, bit for bit, and exactly zero under
early stop; and a 2-rank NCCL run, skipped below 2 GPUs."""
from __future__ import annotations

import json
import os
import socket
import subprocess
import sys

import numpy as np
import pytest
import torch

import reasoning_step_oracle as O
from rlinf_b200 import _lib, ops
from rlinf_b200.algorithms import (MegatronLossEpilogue, reasoning_actor_loss, reasoning_critic_loss, step_metrics,
                                   valid_token_count)
from rlinf_b200.utils import distributed as RD

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_golden_reasoning_step as G  # noqa: E402

pytestmark = pytest.mark.gpu
FIX = os.path.join(HERE, "golden", "golden_reasoning_step.npz")
DEV = torch.device("cuda")


def _same(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return a.shape == b.shape and bool(np.all((a == b) | (np.isnan(a) & np.isnan(b))))


def _close(a, b, ulps):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    tol = ulps * 2.0 ** -23 * np.maximum(np.abs(b), 1.0)
    return a.shape == b.shape and bool(np.all((np.abs(a - b) <= tol) | (np.isnan(a) & np.isnan(b))))


class _PeerDist:
    """torch.distributed stand-in for data-parallel rank `rank` of P (groups are (size, rank) tuples; None is the
    world of `world` ranks): all-gathers return every rank's buffer from `peers`, SUM all-reduces add the peers'
    buffers in rank order, every collective is recorded."""

    def __init__(self, rank, P, peers, world=None):
        self.rank, self.P, self.peers, self.world, self.calls = rank, P, peers, world or P, []

    def is_available(self):
        return True

    def is_initialized(self):
        return True

    def get_world_size(self, group=None):
        return self.world if group is None else group[0]

    def get_rank(self, group=None):
        return self.rank

    def all_gather_into_tensor(self, out, inp, group=None):
        self.calls.append(("all_gather", group is None, tuple(inp.shape)))
        bufs = list(self.peers(inp))
        assert torch.equal(bufs[self.rank].nan_to_num(), inp.nan_to_num())  # an all-masked record holds a NaN mean
        out.copy_(torch.stack(bufs).reshape(out.shape))

    def all_reduce(self, t, op=None, group=None):
        self.calls.append(("all_reduce", group is None, tuple(t.shape)))
        bufs = list(self.peers(t))
        acc = bufs[0].clone()
        for b in bufs[1:]:
            acc += b
        t.copy_(acc)


def _patch(monkeypatch, fake):
    import torch.distributed as dist

    for name in ("is_available", "is_initialized", "get_world_size", "get_rank", "all_gather_into_tensor",
                 "all_reduce"):
        monkeypatch.setattr(dist, name, getattr(fake, name))


def _to_dev(b):
    return {k: (v.to(DEV) if isinstance(v, torch.Tensor) else v) for k, v in b.items()}


def _records(batches, dynamic):
    out = []
    for b in batches:
        mask = b["response_mask"] if dynamic else b["response_mask"][:, -G.L:]
        out.append(ops.reasoning_rollout_record(b["advantages"], mask, b["prompt_lengths"], b["response_lengths"],
                                                b["rewards"], b["is_end"], values=None if dynamic else b.get("values"),
                                                idx_to_traj=b.get("idx_to_traj") if dynamic else None))
    return out


def _run_rollout(monkeypatch, batches, rank, dynamic=False, world=None, return_lengths=False):
    P = len(batches)
    recs = _records(batches, dynamic)

    def peers(t):
        if t.dtype == torch.float64:  # the records
            return recs
        if t.dtype == torch.float32:  # values_mean over the default group: every DP rank's, world // P times
            return [r[_lib.RR_VALUES_MEAN:_lib.RR_VALUES_MEAN + 1].float() for r in recs] * (world // P)
        nmax = t.shape[0]  # the padded lengths
        out = []
        for b in batches:
            x = torch.zeros((nmax, 2), dtype=torch.int64, device=DEV)
            x[:b["prompt_lengths"].numel(), 0] = b["prompt_lengths"]
            x[:b["prompt_lengths"].numel(), 1] = b["response_lengths"]
            out.append(x)
        return out

    fake = _PeerDist(rank, P, peers, world)
    _patch(monkeypatch, fake)
    fn = RD.compute_rollout_metrics_dynamic if dynamic else RD.compute_rollout_metrics
    try:
        res = fn(batches[rank], 12, G.L, data_parallel_group=(P, rank), return_lengths=return_lengths)
    finally:
        monkeypatch.undo()
    return res, fake.calls


@pytest.mark.parametrize("P", [2, 4])
@pytest.mark.parametrize("case", ["values", "novalues", "dynamic"])
def test_rollout_metrics_match_oracle_and_fixture_per_rank(monkeypatch, P, case):
    g = np.load(FIX)
    dynamic = case == "dynamic"
    host = [G.rollout_batch(case, r) for r in range(P)]
    batches = [_to_dev(b) for b in host]
    want = O.rollout_metrics(host, G.L, dynamic=dynamic)
    for r in range(P):
        (m, pl, dl), calls = _run_rollout(monkeypatch, batches, r, dynamic, return_lengths=True)
        assert list(m) == list(g[f"P{P}_r{r}_rollout_{case}_keys"])
        assert _same([m[k] for k in m], [want[k] for k in m]), (r, m, want)
        # the reference's per-rank reward sum is torch's fp32 sum, and its ranks are added in gloo's order
        assert _close([m[k] for k in m], g[f"P{P}_r{r}_rollout_{case}_vals"], P), r
        assert np.array_equal(dl.cpu().numpy(), g[f"P{P}_r{r}_rollout_{case}_dlens"])
        assert np.array_equal(pl.cpu().numpy(), g[f"P{P}_r{r}_rollout_{case}_plens"])
        assert pl.is_cuda == dynamic  # the reference returns CPU tensors, and device tensors in the dynamic variant
        assert [c[0] for c in calls] == ["all_gather", "all_gather"]
        _, calls = _run_rollout(monkeypatch, batches, r, dynamic)
        assert calls == [("all_gather", False, (_lib.RR_NUM,))]


def test_values_mean_over_a_larger_world_is_the_second_collective(monkeypatch):
    P = 2
    host = [G.rollout_batch("values", r) for r in range(P)]
    batches = [_to_dev(b) for b in host]
    want = O.rollout_metrics(host, G.L)
    (m, _, _), calls = _run_rollout(monkeypatch, batches, 0, world=2 * P)
    assert [c[:2] for c in calls] == [("all_gather", False), ("all_reduce", True)]
    assert _close(m["values_mean"], want["values_mean"], 2)
    assert {k: m[k] for k in m if k != "values_mean"} == {k: want[k] for k in want if k != "values_mean"}


@pytest.mark.parametrize("P", [2, 4])
def test_all_masked_rank_raises_the_reference_error_on_every_rank(monkeypatch, P):
    batches = [_to_dev(G.rollout_batch("empty", r)) for r in range(P)]
    for r in range(P):
        with pytest.raises(RuntimeError):
            _run_rollout(monkeypatch, batches, r)


@pytest.mark.parametrize("bsz, L", [(512, 8192), (64, 32768)])
def test_rollout_record_against_fp64(bsz, L):
    gen = torch.Generator(device=DEV).manual_seed(bsz)
    adv = torch.randn(bsz, L, device=DEV, generator=gen) * 2.0
    vals = torch.randn(bsz, L, device=DEV, generator=gen)
    rlen = torch.randint(1, L + 1, (bsz,), device=DEV, generator=gen)
    plen = torch.randint(1, 2048, (bsz,), device=DEV, generator=gen)
    full = torch.zeros(bsz, 2 * L, dtype=torch.bool, device=DEV)
    full[:, L:] = torch.arange(L, device=DEV)[None] < rlen[:, None]
    mask = full[:, -L:]
    rewards = torch.randn(bsz, device=DEV, generator=gen)
    is_end = torch.rand(bsz, device=DEV, generator=gen) < 0.5
    batch = {"advantages": adv, "response_mask": full, "prompt_lengths": plen, "response_lengths": rlen,
             "rewards": rewards, "is_end": is_end, "values": vals}
    m, pl, dl = RD.compute_rollout_metrics(batch, 2048, L)
    a64, v64 = adv.double()[mask], vals.double()[mask]
    n = bsz
    assert m["total_num_sequence"] == n
    assert m["prompt_length"] == float(np.float32(int(plen.sum()))) / n
    assert abs(m["advantages_mean"] - float(a64.mean())) <= 2e-6 * max(1.0, abs(float(a64.mean())))
    assert m["advantages_max"] == float(a64.max()) and m["advantages_min"] == float(a64.min())
    assert m["values_max"] == float(v64.max()) and m["values_min"] == float(v64.min())
    assert abs(m["values_mean"] - float(v64.mean())) <= 2.0 ** -22
    assert abs(m["reward_scores"] - float(rewards.double().mean())) <= 2.0 ** -22
    r64 = rlen.double()
    assert m["average_response_length"] == float(np.float32(np.float32(int(rlen.sum())) / np.float32(n)))
    assert abs(m["variance_of_response_length"] - float(r64.var())) <= 2.0 ** -23 * float(r64.var())
    assert m["max_of_response_length"] == float(rlen.max()) and m["min_of_response_length"] == float(rlen.min())
    assert torch.equal(dl, rlen.cpu()) and torch.equal(pl, plen.cpu())
    again = RD.compute_rollout_metrics(batch, 2048, L, return_lengths=False)[0]
    assert _same(list(again.values()), list(m.values()))  # repeat calls: the same bits


def test_rollout_metrics_make_no_host_sync_before_their_copy():
    b = _to_dev(G.rollout_batch("dynamic", 1))
    idx = torch.as_tensor(b["idx_to_traj"], device=DEV)
    b2 = _to_dev(G.rollout_batch("values", 1))
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        r1 = ops.reasoning_rollout_record(b["advantages"], b["response_mask"], b["prompt_lengths"],
                                          b["response_lengths"], b["rewards"], b["is_end"], idx_to_traj=idx)
        r2 = ops.reasoning_rollout_record(b2["advantages"], b2["response_mask"][:, -G.L:], b2["prompt_lengths"],
                                          b2["response_lengths"], b2["rewards"], b2["is_end"], values=b2["values"])
        m1 = ops.reasoning_rollout_finish(r1.view(1, -1))
        m2 = ops.reasoning_rollout_finish(torch.stack([r2, r2]))
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert m1.shape == (_lib.RM_NUM + 1,) and m2.shape == (_lib.RM_NUM + 2,)


# ---- loss_func epilogue --------------------------------------------------------------------------------------------

def _actor_step(monkeypatch, P, vts, capture=None):
    """Every rank's epilogue over the fixture's actor micro-batches.  Returns per rank [(scaled loss, metrics)] per
    micro-batch, the step dict and the collectives."""
    gvt = None
    if vts:
        tot = sum(float(G.actor_inputs(r, mb, P)[2].sum()) for r in range(P) for mb in range(G.N_MB))
        gvt = (torch.tensor(tot, dtype=torch.float32) / G.N_MB).to(DEV).reshape(1)
    out = []
    for r in range(P):
        _patch(monkeypatch, _PeerDist(r, P, None))  # the epilogue reads the data-parallel size when it is built
        ep = MegatronLossEpilogue("actor", num_microbatches=G.N_MB, data_parallel_group=(P, r),
                                  early_stop_imp_ratio=G.EARLY_STOP, global_valid_token=gvt)
        monkeypatch.undo()
        rows, calls = [], []
        for mb in range(G.N_MB):
            packs = []
            for q in range(P):  # every rank's packed buffer, from a throw-away epilogue
                vals, loss, mask = G.actor_inputs(q, mb, P)
                md = {k: vals[i].to(DEV) for i, k in enumerate(G.ACTOR_KEYS)}
                cap = _PeerDist(q, P, lambda t: None)
                cap.all_reduce = lambda t, op=None, group=None: packs.append(t.clone())
                _patch(monkeypatch, cap)
                tmp = MegatronLossEpilogue("actor", num_microbatches=G.N_MB, data_parallel_group=(P, q),
                                           early_stop_imp_ratio=G.EARLY_STOP, global_valid_token=gvt)
                tmp(loss.to(DEV), md, mask.to(DEV), mb)
                monkeypatch.undo()
            vals, loss, mask = G.actor_inputs(r, mb, P)
            md = {k: vals[i].to(DEV) for i, k in enumerate(G.ACTOR_KEYS)}
            fake = _PeerDist(r, P, lambda t: packs)
            _patch(monkeypatch, fake)
            scaled, m = ep(loss.to(DEV), md, mask.to(DEV), mb)
            monkeypatch.undo()
            rows.append((scaled, m))
            calls += fake.calls
        out.append((rows, step_metrics(ep), calls))
    return out


@pytest.mark.parametrize("P", [2, 4])
@pytest.mark.parametrize("case", list(G.ACTOR_CASES))
def test_actor_epilogue_matches_oracle_and_fixture_per_rank(monkeypatch, P, case):
    g = np.load(FIX)
    res = _actor_step(monkeypatch, P, G.ACTOR_CASES[case])
    gvt = None
    if G.ACTOR_CASES[case]:
        gvt = np.float32(torch.tensor(sum(float(G.actor_inputs(r, mb, P)[2].sum()) for r in range(P)
                                          for mb in range(G.N_MB)), dtype=torch.float32) / G.N_MB)
    final = G.ACTOR_KEYS.index("actor/final_loss")
    oracle_rows = [[] for _ in range(P)]
    for mb in range(G.N_MB):
        per = [(G.actor_inputs(q, mb, P)[0].numpy(), np.float32(G.actor_inputs(q, mb, P)[1]),
                int(G.actor_inputs(q, mb, P)[2].sum())) for q in range(P)]
        want = O.epilogue(per, final, G.ACTOR_KEYS.index("actor/ratio"), 0, G.EARLY_STOP, gvt, G.N_MB)
        for r in range(P):
            scaled, m = res[r][0][mb]
            got = [float(m[k]) for k in G.ACTOR_KEYS]
            assert float(scaled) == float(want[r][1]) and _same(got, want[r][2]), (r, mb)
            assert _close(float(scaled), g[f"P{P}_r{r}_actor_{case}_mb{mb}_loss"], 0)
            assert _close(got, g[f"P{P}_r{r}_actor_{case}_mb{mb}_metrics"], P - 1), (r, mb)
            oracle_rows[r].append(want[r][2])
    for r in range(P):
        rows, step, calls = res[r]
        assert list(step) == list(g[f"P{P}_r{r}_actor_{case}_step_keys"])
        assert _same(list(step.values()), O.step_finish(oracle_rows[r]))
        assert _close(list(step.values()), g[f"P{P}_r{r}_actor_{case}_step_vals"], P - 1)
        assert calls == [("all_reduce", False, (len(G.ACTOR_KEYS) + 1,))] * G.N_MB  # one collective per micro-batch


@pytest.mark.parametrize("P", [2, 4])
@pytest.mark.parametrize("case", G.CRITIC_CASES)
def test_critic_epilogue_and_explained_variance(monkeypatch, P, case):
    g = np.load(FIX)
    order = [k for k in G.CRITIC_KEYS if k not in G.EV] + list(G.EV)
    perm = [G.CRITIC_KEYS.index(k) for k in order]
    _patch(monkeypatch, _PeerDist(0, P, None))  # the epilogue reads the data-parallel size when it is built
    eps = [MegatronLossEpilogue("critic", num_microbatches=G.N_MB, data_parallel_group=(P, r)) for r in range(P)]
    monkeypatch.undo()
    rows = [[] for _ in range(P)]
    for mb in range(G.N_MB):
        ins = [G.critic_inputs(q, mb, case, P) for q in range(P)]
        packs = []
        for q, (vals, loss) in enumerate(ins):
            cap = _PeerDist(q, P, lambda t: None)
            cap.all_reduce = lambda t, op=None, group=None: packs.append(t.clone())
            _patch(monkeypatch, cap)
            tmp = MegatronLossEpilogue("critic", num_microbatches=G.N_MB, data_parallel_group=(P, q))
            tmp(loss.to(DEV), {k: vals[i].to(DEV) for i, k in enumerate(G.CRITIC_KEYS)}, None, mb)
            monkeypatch.undo()
        want = O.epilogue([(v.numpy()[perm], np.float32(l), None) for v, l in ins], order.index("critic/final_value_loss"),
                          None, len(G.EV))
        for r, (vals, loss) in enumerate(ins):
            fake = _PeerDist(r, P, lambda t: packs)
            _patch(monkeypatch, fake)
            scaled, m = eps[r](loss.to(DEV), {k: vals[i].to(DEV) for i, k in enumerate(G.CRITIC_KEYS)}, None, mb)
            monkeypatch.undo()
            assert torch.equal(scaled, loss.to(DEV))  # the critic's loss is not scaled
            assert list(m) == order and _same([float(m[k]) for k in order], want[r][2])
            assert _close([float(m[k]) for k in order], g[f"P{P}_r{r}_critic_{case}_mb{mb}_metrics"][perm], P - 1)
            rows[r].append(want[r][2])
    for r in range(P):
        step = step_metrics(eps[r])
        assert list(step) == list(g[f"P{P}_r{r}_critic_{case}_step_keys"])
        assert _same(list(step.values()), O.step_finish(rows[r], len(G.EV)))
        assert _close(list(step.values()), g[f"P{P}_r{r}_critic_{case}_step_vals"], P - 1)


def _loss_inputs(bsz=6, L=40, seed=3):
    gen = torch.Generator(device=DEV).manual_seed(seed)
    lp = -torch.rand(bsz, L, device=DEV, generator=gen) * 2
    old = lp + 0.05 * torch.randn(bsz, L, device=DEV, generator=gen)
    adv = torch.randn(bsz, L, device=DEV, generator=gen)
    mask = torch.rand(bsz, L, device=DEV, generator=gen) < 0.8
    return lp, old, adv, mask


@pytest.mark.parametrize("early_stop", [None, 0.5])
def test_composes_with_the_actor_loss_and_scales_the_gradient(early_stop):
    lp, old, adv, mask = _loss_inputs()
    gvt = valid_token_count(torch.cat([torch.zeros_like(mask), mask], 1), mask.shape[1]) * 1.5
    x0 = lp.clone().requires_grad_(True)
    loss0, _ = reasoning_actor_loss(x0, adv, mask, old_logprobs=old)
    loss0.backward()
    x = lp.clone().requires_grad_(True)
    loss, metrics = reasoning_actor_loss(x, adv, mask, old_logprobs=old)
    ep = MegatronLossEpilogue("actor", num_microbatches=2, early_stop_imp_ratio=early_stop, global_valid_token=gvt)
    scaled, m = ep(loss, metrics, mask, 0)
    scaled.backward()
    scale = torch.tensor(0.0 if early_stop is not None else float(
        np.float32(np.float32(np.float32(int(mask.sum())) / np.float32(float(gvt))) * 1) * 2), device=DEV)
    if early_stop is not None:
        assert float(m["actor/ratio"]) > early_stop
        assert torch.equal(x.grad, torch.zeros_like(x.grad)) and float(scaled) == 0.0
    else:
        assert torch.equal(scaled, loss * scale) and torch.equal(x.grad, x0.grad * scale)
        assert float(m["actor/final_loss"]) == float(loss * scale)


def test_composes_with_the_critic_loss_and_step_is_sync_free():
    gen = torch.Generator(device=DEV).manual_seed(5)
    v = torch.randn(4, 64, device=DEV, generator=gen)
    ret = torch.randn(4, 64, device=DEV, generator=gen)
    prev = v + 0.1 * torch.randn(4, 64, device=DEV, generator=gen)
    mask = torch.rand(4, 64, device=DEV, generator=gen) < 0.7
    lp, old, adv, amask = _loss_inputs()
    gvt = valid_token_count(amask, amask.shape[1])
    outs = []
    for attempt in range(2):
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            ec = MegatronLossEpilogue("critic", num_microbatches=2)
            ea = MegatronLossEpilogue("actor", num_microbatches=2, early_stop_imp_ratio=2.0, global_valid_token=gvt)
            for mb in range(2):
                vv = v.clone().requires_grad_(True)
                loss, md = reasoning_critic_loss(vv, ret, prev, mask, value_clip=0.2)
                scaled, _ = ec(loss, md, mask, mb)
                scaled.backward()
                x = lp.clone().requires_grad_(True)
                loss, md = reasoning_actor_loss(x, adv, amask, old_logprobs=old)
                scaled, _ = ea(loss, md, amask, mb)
                scaled.backward()
            fc = ops.step_metrics_finish(ec.step_acc, len(ec.keys[0]), len(ec.keys[1]))
            fa = ops.step_metrics_finish(ea.step_acc, len(ea.keys[0]), len(ea.keys[1]))
        finally:
            torch.cuda.set_sync_debug_mode(0)
        sc, sa = step_metrics(ec), step_metrics(ea)
        assert "critic/explained_variance" in sc and not any(k.startswith("__sum__") for k in sc)
        fc, fa = fc.cpu().numpy(), fa.cpu().numpy()
        assert _same(list(sc.values()), np.append(fc[:len(ec.keys[0])], fc[-1]))
        assert _same(list(sa.values()), fa[:len(ea.keys[0])])
        outs.append((sc, sa))
    assert outs[0] == outs[1]  # repeat steps give the same bits


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def test_nccl_two_ranks_match_emulation(tmp_path):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    out = tmp_path / "out.json"
    env = dict(os.environ, RB200_DIST_OUT=str(out))
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nproc_per_node=2", f"--master_port={_free_port()}",
           os.path.join(HERE, "dist_reasoning_step_worker.py")]
    proc = subprocess.run(cmd, env=env, capture_output=True, text=True, timeout=600)
    assert proc.returncode == 0, proc.stdout[-4000:] + proc.stderr[-4000:]
    assert json.loads(out.read_text())["ok"]
