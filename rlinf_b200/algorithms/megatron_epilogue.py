"""The Megatron reasoning workers' loss_func tail and step finish on the device, with no host sync.

MegatronActor's loss_func (rlinf/workers/actor/megatron_actor_worker.py:258-307) all-reduces actor/ratio for the
early-stop test, reads it on the host, reads the valid-token scale with .item() and averages every metric over data
parallel with one all-reduce per key; MegatronCritic's (megatron_critic_worker.py:104-121) makes one all-reduce per
metric, five of them for the explained-variance sums.  _process_fwd_bwd_outputs (megatron_worker.py:550-599) then
reads every key with .cpu().item().  Here:

    epilogue = MegatronLossEpilogue("actor", data_parallel_group=dp_group, early_stop_imp_ratio=...,
                                    num_microbatches=n_mb, global_valid_token=valid_token_count(...))
    ...in loss_func of micro-batch mb:
    loss, metrics = reasoning_actor_loss(...)
    loss, metrics = epilogue(loss, metrics, mask, mb)      # one data-parallel all-reduce, no host sync
    ...after forward_backward:
    train_metrics = step_metrics(epilogue)                 # one device-to-host copy

The scale (0 when the micro-batch is early-stopped, else mask_sum / global_valid_token * dp * num_microbatches with
the valid-token scale, else 1) stays on the device and multiplies the loss inside autograd, so the gradient carries it.
"""
from __future__ import annotations

import ctypes as C
from typing import Optional

import torch
import torch.distributed as dist

from .. import _lib as L
from .. import ops

EV_KEYS = tuple(f"__sum__/_critic_explained_variance/{k}"
                for k in ("count", "returns_sum", "returns_sq_sum", "errors_sum", "errors_sq_sum"))
EV_KEY = "critic/explained_variance"
_FINAL = {"actor": "actor/final_loss", "critic": "critic/final_value_loss"}


def _dist_on() -> bool:
    return dist.is_available() and dist.is_initialized()


def _dp_group(group):
    """group, or Megatron's data-parallel group when megatron.core is initialised, or the world."""
    if group is not None or not _dist_on():
        return group
    try:
        from megatron.core import parallel_state
    except ImportError:
        return None
    return parallel_state.get_data_parallel_group() if parallel_state.model_parallel_is_initialized() else None


def valid_token_count(response_mask: torch.Tensor, response_len: int, group=None) -> torch.Tensor:
    """_setup_valid_token_scale (megatron_worker.py:640-654): response_mask[:, -response_len:].to(float32).sum(),
    SUM-all-reduced over the data-parallel group, as a 0-dim fp32 device tensor.  One all-reduce, no host sync."""
    total = ops.mask_count_f32(response_mask[:, -response_len:])
    if _dist_on():
        dist.all_reduce(total, op=dist.ReduceOp.SUM, group=_dp_group(group))
    return total


class MegatronLossEpilogue:
    """The loss_func tail of MegatronActor (role "actor") or MegatronCritic (role "critic") for one training step of
    num_microbatches micro-batches.  Build it once per step; call it once per micro-batch with the loss, the metrics
    of reasoning_actor_loss / reasoning_critic_loss (0-dim fp32 device tensors under the worker's keys), the loss mask
    and the micro-batch index.

    Returns (scaled_loss, metrics): scaled_loss = loss * scale with the scale on the device (exactly the loss when
    neither early stop nor the valid-token scale applies), metrics the data-parallel-reduced 0-dim tensors: every key
    averaged over data parallel as Megatron's average_losses_across_data_parallel_group does (SUM, then / dp) but the
    explained-variance sums, which are SUM-reduced; the final loss key holds the scaled loss.  Early stop compares the
    averaged actor/ratio with early_stop_imp_ratio.  One SUM all-reduce per call, two launches (four with the
    valid-token scale), no host sync."""

    def __init__(self, role: str, *, num_microbatches: int, data_parallel_group=None,
                 early_stop_imp_ratio: Optional[float] = None, global_valid_token: Optional[torch.Tensor] = None):
        if role not in _FINAL:
            raise ValueError(f"MegatronLossEpilogue: role must be 'actor' or 'critic', got {role!r}")
        if role == "critic" and (early_stop_imp_ratio is not None or global_valid_token is not None):
            raise ValueError("MegatronLossEpilogue: the critic's loss_func has no early stop or valid-token scale")
        if int(num_microbatches) <= 0:
            raise ValueError(f"MegatronLossEpilogue: num_microbatches must be positive, got {num_microbatches}")
        if global_valid_token is not None and (not global_valid_token.is_cuda or global_valid_token.numel() != 1
                                               or global_valid_token.dtype != torch.float32):
            raise ValueError("MegatronLossEpilogue: global_valid_token must be a one-element fp32 CUDA tensor")
        self.role = role
        self.num_microbatches = int(num_microbatches)
        self.group = _dp_group(data_parallel_group)
        self.dp = dist.get_world_size(self.group) if _dist_on() else 1
        self.early_stop_imp_ratio = early_stop_imp_ratio
        self.global_valid_token = global_valid_token
        self.keys = None  # (averaged keys, SUM keys), fixed by the first call
        self.step_acc = None
        self.seen = set()

    def _layout(self, metrics: dict):
        final = _FINAL[self.role]
        avg = [k for k, v in metrics.items() if v is not None and k not in EV_KEYS]
        if final not in avg:
            avg.append(final)
        sums = [k for k in EV_KEYS if metrics.get(k) is not None]
        if len(avg) + len(sums) > L.EPI_MAX_KEYS:
            raise ValueError(f"MegatronLossEpilogue: at most {L.EPI_MAX_KEYS} metric keys")
        return avg, sums

    def __call__(self, loss: torch.Tensor, metrics: dict, mask: Optional[torch.Tensor], mb_index: int):
        avg, sums = self._layout(metrics)
        if self.keys is None:
            self.keys = (avg, sums)
            self.step_acc = torch.empty((self.num_microbatches, len(avg) + len(sums)), dtype=torch.float32,
                                        device=loss.device)
        elif (avg, sums) != self.keys:
            raise ValueError("MegatronLossEpilogue: every micro-batch of a step must report the same metric keys")
        if not 0 <= int(mb_index) < self.num_microbatches:
            raise ValueError(f"MegatronLossEpilogue: mb_index {mb_index} outside [0, {self.num_microbatches})")
        if not loss.is_cuda or loss.dtype != torch.float32 or loss.numel() != 1:
            raise ValueError("MegatronLossEpilogue: loss must be a one-element fp32 CUDA tensor")
        dev = loss.device
        final = _FINAL[self.role]
        n = len(avg) + len(sums)
        a = L.MbEpilogueArgs()
        a.n_avg, a.n_sum = len(avg), len(sums)
        a.final_slot = avg.index(final)
        a.ratio_slot = avg.index("actor/ratio") if "actor/ratio" in avg else -1
        keep = []
        for i, k in enumerate(avg + sums):
            if k == final:
                continue
            v = metrics[k]
            if not v.is_cuda or v.dtype != torch.float32 or v.numel() != 1:
                raise ValueError(f"MegatronLossEpilogue: metric {k} must be a one-element fp32 CUDA tensor")
            keep.append(v)
            a.src[i] = v.data_ptr()
        loss_d = loss.detach()
        a.loss = loss_d.data_ptr()
        gvt = self.global_valid_token
        if gvt is not None:
            if mask is None or mask.dim() != 2:
                raise ValueError("MegatronLossEpilogue: the valid-token scale needs the [bsz, L] loss mask")
            m = ops._cells(L.as_u8(mask), "mask", tuple(mask.shape), dev, torch.uint8)
            keep.append(m)
            a.mask, a.mask_stride, a.bsz, a.L = m.data_ptr(), m.stride(0), m.shape[0], m.shape[1]
            a.global_valid_token = gvt.data_ptr()
            wsb = L.load().rb200_token_loss_workspace_bytes(m.shape[0], m.shape[1])
            if wsb < 0:
                raise ValueError(f"MegatronLossEpilogue: unsupported mask shape {tuple(m.shape)} (bsz <= 65535)")
        else:
            wsb = L.EPI_WS_MIN
        ws = torch.empty(wsb, dtype=torch.uint8, device=dev)
        pack = torch.empty(n + 1, dtype=torch.float32, device=dev)
        scale = torch.empty(1, dtype=torch.float32, device=dev)
        out = torch.empty(n, dtype=torch.float32, device=dev)
        a.dp, a.num_microbatches, a.n_mb, a.mb = self.dp, self.num_microbatches, self.num_microbatches, int(mb_index)
        a.has_early_stop = int(self.early_stop_imp_ratio is not None)
        a.early_stop_imp_ratio = float(self.early_stop_imp_ratio or 0.0)
        a.workspace, a.workspace_bytes = ws.data_ptr(), wsb
        a.pack, a.scale, a.metrics, a.step_acc = pack.data_ptr(), scale.data_ptr(), out.data_ptr(), \
            self.step_acc.data_ptr()
        ops.mb_epilogue_pack(a, dev)
        if _dist_on():
            dist.all_reduce(pack, op=dist.ReduceOp.SUM, group=self.group)
        ops.mb_epilogue_apply(a, dev)
        self.seen.add(int(mb_index))
        scaled = loss * scale.reshape(loss.shape)
        return scaled, {k: out[i] for i, k in enumerate(avg + sums)}


def step_metrics(epilogue: MegatronLossEpilogue) -> dict:
    """_process_fwd_bwd_outputs (megatron_worker.py:550-599) for a training step: each averaged key's mean over the
    micro-batches as a float, and critic/explained_variance from the summed explained-variance statistics when the
    step reported them.  One launch and one device-to-host copy."""
    if epilogue.keys is None:
        return {}
    missing = sorted(set(range(epilogue.num_microbatches)) - epilogue.seen)
    if missing:
        raise ValueError(f"step_metrics: micro-batches {missing} were not recorded")
    avg, sums = epilogue.keys
    host = ops.step_metrics_finish(epilogue.step_acc, len(avg), len(sums)).cpu().tolist()
    out = {k: host[i] for i, k in enumerate(avg)}
    if len(sums) == len(EV_KEYS):
        out[EV_KEY] = host[len(avg) + len(sums)]
    return out
