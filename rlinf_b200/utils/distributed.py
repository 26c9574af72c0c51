"""rlinf/utils/distributed.py (SURVEY a24), CUDA-backed: the masked fp64 normalisations and the reasoning rollout
metrics.

`masked_normalization` (:866-939), `masked_stats` (:942-954), `normalize_from_stats` (:957-965).  The reference issues
three all-reduces (factor, sum, sum of squares); here the three fp64 statistics come out of ONE reduction kernel into
one 24-byte buffer that is all-reduced ONCE, and one elementwise kernel applies the normalisation.

`compute_rollout_metrics` (:186-306) and `compute_rollout_metrics_dynamic` (:34-183).  The reference makes two
all_gather_object calls, four all-reduces and about 15 .item() calls; here each rank writes one fp64 record on the
device, the data-parallel group all-gathers the records once, one kernel combines them in rank order, and the metrics
reach the host in one device-to-host copy.
"""
from __future__ import annotations

from typing import Optional

import torch
import torch.distributed as dist

from .. import _lib as L
from .. import ops


def masked_stats(x: torch.Tensor, mask: Optional[torch.Tensor] = None) -> torch.Tensor:
    """{count, sum, sum of squares} of the valid values, float64[3] on the device (distributed.py:942-954)."""
    return ops.masked_moments(x, mask)


def normalize_from_stats(x: torch.Tensor, stats: torch.Tensor) -> torch.Tensor:
    """(x - mean) * rsqrt(max(var, 0) + 1e-5) from (all-reduced) {count, sum, sumsq} (distributed.py:957-965)."""
    return ops.masked_normalize(x, stats, None, mode=1).view(x.shape)


@torch.no_grad()
def masked_normalization(x: torch.Tensor, mask: Optional[torch.Tensor] = None, dim=None, inplace: bool = False,
                         unbiased: bool = False, eps: float = 1e-5, high_precision: bool = True,
                         all_reduce: bool = True, group=None) -> torch.Tensor:
    """Advantage normalisation over the whole (data-parallel) batch (distributed.py:866-939).  Semantics kept: the
    input is multiplied by the mask BEFORE the statistics and the masked entries come out as (0 - mean)/(std + eps).
    `dim` other than None / all dimensions is not needed by any caller of the reference and is not implemented."""
    if dim is not None and tuple(sorted(d % x.dim() for d in (dim if isinstance(dim, (tuple, list)) else (dim,)))) != tuple(
            range(x.dim())):
        raise NotImplementedError("masked_normalization: only dim=None (all dimensions) is implemented")
    if not high_precision:
        raise NotImplementedError("masked_normalization: statistics are always accumulated in float64")
    if mask is not None and mask.shape != x.shape:
        raise AssertionError((tuple(mask.shape), tuple(x.shape), dim))
    stats = ops.masked_moments(x, mask)
    if mask is None:
        stats[0] = float(x.numel())
    if all_reduce and dist.is_available() and dist.is_initialized():
        dist.all_reduce(stats, op=dist.ReduceOp.SUM, group=group)
    out = ops.masked_normalize(x, stats, mask, mode=0, eps=eps, unbiased=unbiased).view(x.shape)
    if inplace and x.is_cuda and x.dtype == torch.float32:
        x.copy_(out)
        return x
    return out


_KEYS = ("total_num_sequence", "prompt_length", "response_length", "average_response_length",
         "variance_of_response_length", "max_of_response_length", "min_of_response_length", "total_length",
         "reward_scores", "fraction_of_samples_properly_ended", "advantages_mean", "advantages_max", "advantages_min")
_VALUE_KEYS = ("values_mean", "values_max", "values_min")
_DYNAMIC_KEYS = ("total_num_sequence", "prompt_length", "response_length", "total_length", "max_prompt_length",
                 "max_response_length", "max_total_length", "reward_scores_traj", "reward_scores_turn",
                 "avg_turns_per_traj", "fraction_of_samples_properly_ended", "advantages_mean", "advantages_max",
                 "advantages_min")
_INT_KEYS = ("max_prompt_length", "max_response_length", "max_total_length")


def _dist_on() -> bool:
    return dist.is_available() and dist.is_initialized()


def _rollout_metrics(rollout_batch, mask, data_parallel_group, idx_to_traj, return_lengths, lengths_on_cpu):
    values = rollout_batch["values"] if idx_to_traj is None and "values" in rollout_batch else None
    plen, rlen = rollout_batch["prompt_lengths"], rollout_batch["response_lengths"]
    rec = ops.reasoning_rollout_record(rollout_batch["advantages"], mask, plen, rlen, rollout_batch["rewards"],
                                       rollout_batch["is_end"], values=values, idx_to_traj=idx_to_traj)
    on = _dist_on()
    P = dist.get_world_size(data_parallel_group) if on else 1
    if P > 1:
        records = torch.empty((P, L.RR_NUM), dtype=torch.float64, device=rec.device)
        dist.all_gather_into_tensor(records, rec, group=data_parallel_group)
    else:
        records = rec.view(1, L.RR_NUM)
    world_sum, world = None, 0
    if values is not None and on and dist.get_world_size() != P:
        # values_mean is averaged over the default group, not the data-parallel group (distributed.py:275)
        world_sum = rec[L.RR_VALUES_MEAN:L.RR_VALUES_MEAN + 1].to(torch.float32)
        dist.all_reduce(world_sum, op=dist.ReduceOp.SUM)
        world = dist.get_world_size()
    host = ops.reasoning_rollout_finish(records, world_sum, world).cpu().tolist()  # the one device-to-host copy
    verdict = int(host[L.RM_VERDICT])
    if verdict & L.RV_EMPTY:
        raise RuntimeError("max(): Expected reduction dim to be specified for input.numel() == 0: a data-parallel rank "
                           "has no valid response token (response_mask is all False)")
    if verdict & L.RV_BAD_TRAJ:
        raise IndexError("idx_to_traj holds a negative trajectory index")
    keys = _DYNAMIC_KEYS if idx_to_traj is not None else _KEYS + (_VALUE_KEYS if values is not None else ())
    metrics = {k: (int(host[L.RM_SLOTS[k]]) if k in _INT_KEYS else host[L.RM_SLOTS[k]]) for k in keys}
    if not return_lengths:
        return metrics, None, None
    counts = [int(c) for c in host[L.RM_NUM:]]
    own = torch.stack([L.to_device(torch.as_tensor(plen).reshape(-1), rec.device, torch.int64),
                       L.to_device(torch.as_tensor(rlen).reshape(-1), rec.device, torch.int64)], dim=1)
    if P > 1:
        # one padded all-gather of [P, max num_seq, 2] lengths, asked for only when FLOPs are counted
        nmax = max(counts)
        send = torch.zeros((nmax, 2), dtype=torch.int64, device=rec.device)
        send[:own.shape[0]] = own
        gathered = torch.empty((P, nmax, 2), dtype=torch.int64, device=rec.device)
        dist.all_gather_into_tensor(gathered, send, group=data_parallel_group)
        lengths = torch.cat([gathered[r, :counts[r]] for r in range(P)])
    else:
        lengths = own
    if lengths_on_cpu:
        lengths = lengths.cpu()
    return metrics, lengths[:, 0].contiguous(), lengths[:, 1].contiguous()


def compute_rollout_metrics(rollout_batch: dict, max_prompt_len: int, response_len: int,
                            data_parallel_group=None, use_critic: bool = False, *, return_lengths: bool = True):
    """rlinf/utils/distributed.py:186-306 on the device.  Returns (metrics, total_prompt_lengths,
    total_decode_lengths): metrics are floats under the reference's keys (values_* when the batch has "values");
    the length tensors are every data-parallel rank's lengths in rank order, on the CPU, or None with
    return_lengths=False (the runner needs them only to count FLOPs).

    Collectives: one all-gather of the [P, RR_NUM] fp64 records over the data-parallel group, plus one one-float
    all-reduce over the default group when the batch has values and the default group is larger (values_mean is
    averaged there in the reference), plus the padded length all-gather when return_lengths.  One device-to-host copy
    before the metrics are formed.

    Kept from the reference: the SUM fields are rounded to fp32 before the reduction; values_mean is the mean of the
    ranks' fp32 masked means; the length statistics are those of the gathered lengths (from exact integer sums here).
    values_max / values_min are reduced over the data-parallel group, whose ranks hold the same batches as the rest of
    the default group.  A rank whose response mask is all False raises RuntimeError on every rank (the reference's
    torch.max raises on that rank only)."""
    mask = rollout_batch["response_mask"][:, -response_len:]
    return _rollout_metrics(rollout_batch, mask, data_parallel_group, None, return_lengths, True)


def compute_rollout_metrics_dynamic(rollout_batch: dict, max_prompt_len: int, response_len: int,
                                    data_parallel_group=None, use_critic: bool = False, *,
                                    return_lengths: bool = True):
    """rlinf/utils/distributed.py:34-183 on the device, for multi-turn batches: rollout_batch["idx_to_traj"] (a list
    or an int64 tensor) maps each turn to its trajectory; rewards are averaged per trajectory in turn order and the
    metrics are the reference's keys (reward_scores_traj, reward_scores_turn, avg_turns_per_traj, max_*_length...).
    The length tensors are returned on the device, as in the reference.  Collectives and error as
    compute_rollout_metrics, without the values all-reduce."""
    return _rollout_metrics(rollout_batch, rollout_batch["response_mask"], data_parallel_group,
                            rollout_batch["idx_to_traj"], return_lengths, False)
