"""Torch-on-CPU oracle of the reasoning step bookkeeping (csrc/reasoning_stats.cu), written as the device computes it:

  - rollout metrics: each rank's record (fp64 sums of the valid advantages and values, rounded to fp32 as the
    reference rounds its reduction vector; exact integer length sums), the records added in fp32 in rank order, the
    metrics formed in fp64;
  - the loss_func epilogue: the packed metrics SUM-reduced in rank order in fp32, / dp for the averaged keys, early
    stop on the averaged actor/ratio, the valid-token scale as a chain of fp32 operations;
  - the step finish: fp32 means over the micro-batches in index order and the explained variance in fp32.

With reference=True each rank's reward sum is torch's fp32 sum, as in the reference; the device adds the rewards in
fp64 and rounds once.  tests/test_reasoning_step_cpu.py checks that mode against the reference fixture
(tests/golden/golden_reasoning_step.npz): bit for bit at 2 ranks, where an fp32 sum of two terms has one result, and
within one fp32 rounding per added rank at 4 ranks, where gloo's all-reduce adds the ranks in an order of its own.
The GPU tests check the device against the default mode bit for bit."""
from __future__ import annotations

import math

import numpy as np
import torch

F32 = np.float32

ROLLOUT_KEYS = ("total_num_sequence", "prompt_length", "response_length", "average_response_length",
                "variance_of_response_length", "max_of_response_length", "min_of_response_length", "total_length",
                "reward_scores", "fraction_of_samples_properly_ended", "advantages_mean", "advantages_max",
                "advantages_min")
VALUE_KEYS = ("values_mean", "values_max", "values_min")
DYNAMIC_KEYS = ("total_num_sequence", "prompt_length", "response_length", "total_length", "max_prompt_length",
                "max_response_length", "max_total_length", "reward_scores_traj", "reward_scores_turn",
                "avg_turns_per_traj", "fraction_of_samples_properly_ended", "advantages_mean", "advantages_max",
                "advantages_min")


def record(batch, response_len, dynamic=False, reference=False):
    """One rank's record as a dict of Python numbers (None for the all-masked error)."""
    adv = batch["advantages"].double()
    mask = batch["response_mask"] if dynamic else batch["response_mask"][:, -response_len:]
    valid = adv[mask]
    if valid.numel() == 0:
        return None
    plen, rlen = batch["prompt_lengths"].long(), batch["response_lengths"].long()
    rewards = batch["rewards"].float().reshape(-1)
    r = {"sum_plen": F32(int(plen.sum())), "sum_rlen": F32(int(rlen.sum())),
         "sum_rewards": F32(float(rewards.sum() if reference else rewards.double().sum())), "sum_end": F32(int(torch.as_tensor(batch["is_end"]).sum())),
         "sum_adv": F32(float(valid.sum())), "num_seq": F32(plen.numel()), "n_valid": F32(valid.numel()),
         "adv_neg_min": -F32(float(valid.min())), "adv_max": F32(float(valid.max())),
         "max_plen": F32(int(plen.max())), "max_rlen": F32(int(rlen.max())), "max_total": F32(int((plen + rlen).max())),
         "rlen": [int(x) for x in rlen]}
    if "values" in batch and not dynamic:
        v = batch["values"].double()[mask]
        r.update(values_mean=F32(float(v.sum()) / v.numel()), val_neg_min=-F32(float(v.min())),
                 val_max=F32(float(v.max())))
    if dynamic:
        idx = [int(t) for t in batch["idx_to_traj"]]
        ntraj = max(idx) + 1
        s_traj = 0.0
        for t in range(ntraj):
            s, c = F32(0), 0
            for i, ti in enumerate(idx):
                if ti == t:
                    s = F32(s + F32(rewards[i].item()))
                    c += 1
            s_traj += float(F32(s / F32(max(c, 1))))
        r.update(sum_traj=F32(s_traj), num_traj=F32(ntraj))
    return r


def _fsum(xs):
    """fp32 sum in rank order."""
    s = F32(0)
    for x in xs:
        s = F32(s + F32(x))
    return s


def rollout_metrics(batches, response_len, dynamic=False, reference=False):
    """The metrics dict of compute_rollout_metrics(_dynamic) over the data-parallel ranks' batches, or the string
    "RuntimeError" when a rank has no valid token."""
    recs = [record(b, response_len, dynamic, reference) for b in batches]
    if any(r is None for r in recs):
        return "RuntimeError"
    S = {k: float(_fsum((r[k] for r in recs))) for k in ("sum_plen", "sum_rlen", "sum_rewards", "sum_end", "sum_adv",
                                                        "num_seq", "n_valid")}
    X = {k: float(max(r[k] for r in recs)) for k in ("adv_neg_min", "adv_max", "max_plen", "max_rlen", "max_total")}
    n = S["num_seq"]
    m = {"total_num_sequence": n, "prompt_length": S["sum_plen"] / n, "response_length": S["sum_rlen"] / n,
         "total_length": (S["sum_plen"] + S["sum_rlen"]) / n, "fraction_of_samples_properly_ended": S["sum_end"] / n,
         "advantages_mean": S["sum_adv"] / S["n_valid"], "advantages_max": X["adv_max"],
         "advantages_min": -X["adv_neg_min"]}
    if dynamic:
        st, nt = float(_fsum((r["sum_traj"] for r in recs))), float(_fsum((r["num_traj"] for r in recs)))
        m.update(max_prompt_length=int(X["max_plen"]), max_response_length=int(X["max_rlen"]),
                 max_total_length=int(X["max_total"]), reward_scores_traj=st / nt, reward_scores_turn=S["sum_rewards"] / n,
                 avg_turns_per_traj=n / nt)
        return {k: m[k] for k in DYNAMIC_KEYS}
    lens = [x for r in recs for x in r["rlen"]]
    cnt, s1, s2 = len(lens), sum(lens), sum(x * x for x in lens)
    m.update(average_response_length=float(F32(F32(s1) / F32(cnt))),
             variance_of_response_length=float(F32((cnt * s2 - s1 * s1) / (cnt * (cnt - 1.0)))) if cnt > 1 else math.nan,
             max_of_response_length=float(F32(max(lens))), min_of_response_length=float(F32(min(lens))),
             reward_scores=S["sum_rewards"] / n)
    keys = ROLLOUT_KEYS
    if "values_mean" in recs[0]:
        m.update(values_mean=float(F32(_fsum((r["values_mean"] for r in recs)) / F32(len(recs)))),
                 values_max=float(max(r["val_max"] for r in recs)), values_min=-float(max(r["val_neg_min"] for r in recs)))
        keys = keys + VALUE_KEYS
    return {k: m[k] for k in keys}


def epilogue(per_rank, final_slot, ratio_slot=None, n_sum=0, early_stop=None, gvt=None, num_microbatches=1):
    """One micro-batch's epilogue on every rank.  per_rank: list of (vals fp32 array in key order with the averaged
    keys first and n_sum SUM keys last, loss fp32, mask count or None).  Returns per rank (scale, scaled loss,
    reduced metrics as an fp32 array)."""
    P = len(per_rank)
    n = len(per_rank[0][0])
    n_avg = n - n_sum
    packs = []
    for vals, loss, msum in per_rank:
        s = F32(1)
        if gvt is not None:
            s = F32(F32(F32(F32(msum) / F32(gvt)) * F32(P)) * F32(num_microbatches))
        p = np.array(vals, dtype=F32).copy()
        p[final_slot] = F32(F32(loss) * s)
        packs.append((np.append(p, F32(F32(F32(loss) * F32(0)) * s)), s))
    tot = np.array([_fsum(p[k] for p, _ in packs) for k in range(n + 1)], dtype=F32)
    stop = early_stop is not None and ratio_slot is not None and F32(tot[ratio_slot] / F32(P)) > F32(early_stop)
    red = tot[:n].copy()
    if stop:
        red[final_slot] = tot[n]
    red[:n_avg] = (red[:n_avg] / F32(P)).astype(F32)
    out = []
    for (p, s), (vals, loss, _) in zip(packs, per_rank):
        scale = F32(0) if stop else s
        out.append((scale, F32(F32(loss) * scale), red))
    return out


def step_finish(rows, n_sum=0):
    """rows: [n_mb, n] fp32 reduced metrics.  -> fp32 array [n_avg (+ 1 explained variance when n_sum == 5)]."""
    rows = np.asarray(rows, dtype=F32)
    n_mb, n = rows.shape
    n_avg = n - n_sum
    acc = np.zeros(n, dtype=F32)
    for m in range(n_mb):
        acc = (acc + rows[m]).astype(F32)
    out = list((acc[:n_avg] / F32(n_mb)).astype(F32))
    if n_sum == 5:
        count, rs, rsq, es, esq = (F32(x) for x in acc[n_avg:])
        ev = F32(math.nan)
        if not count < 2:
            rc = F32(rsq - F32(F32(rs * rs) / count))
            if not np.isnan(rc) and rc != 0:
                ec = F32(esq - F32(F32(es * es) / count))
                if not np.isnan(ec):
                    ev = F32(F32(1) - F32(ec / rc))
        out.append(ev)
    return np.array(out, dtype=F32)
