"""Response-rows plans: which rows of a reasoning batch's hidden states the actor loss reads.

A plan describes sequence b of a micro-batch by a_b, the row of its first response token in the flattened [T, H]
hidden states, and r_b, its response length (0 <= r_b <= response_len; an empty response has no rows and an all-zero
output row), plus one entropy alignment for the whole plan.  Response token j is predicted by row a_b - 1 + j and its
target is the token at a_b + j.  One constructor per batch layout of the reference's workers:

    padded(bsz, S, response_len, response_lengths)        FSDP without packing: [bsz, S], a_b = b S + S - L
    fsdp_packed(prompt_lengths, response_lengths, max_prompt_len, response_len=...)
                                                          FSDP's pack_fsdp_input: a_b = sum_{i<b} (p_i + r_i) + p_b
    megatron_thd(cu_seqlens_padded, seq_lengths, response_lengths, response_len=...)
                                                          Megatron's preprocess_packed_seqs (cp 1): a_b = cu[b] + n_b - r_b

fsdp_packed keeps the reference's entropy alignment: its packed branch takes the entropy of the row AT response token
j, one row after the row that predicts it, so each sequence needs r_b + 1 rows (DESIGN.md §2).

Lengths on the host are checked on the host when the plan is built (and against T when it is used), with no device
sync.  Lengths on the device are checked by the plan kernel, whose verdict comes back with R in one device-to-host
copy.  Violations raise ValueError.  `index()` runs the plan kernel (csrc/response_rows.cu) and returns the index maps
that ops.response_logprobs_entropy gathers with.
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Optional

import torch

from . import _lib as L

PADDED, FSDP_PACKED, MEGATRON_THD = 0, 1, 2
MAX_BSZ = 8192

# RB200_RR_* bits of the plan kernel's status word, in the order they are reported
_ERRORS = {
    1: "a response length lies outside [0, response_len]",
    2: "a sequence has no prompt token, so the row before its first response token is not its own",
    4: "a sequence's rows lie outside [0, T)",
    8: "sequences overlap or are not in ascending order",
    16: "a prompt length exceeds max_prompt_len",
    32: "more response rows than the plan's capacity",
}


def _error(bits: int, what: str) -> ValueError:
    msgs = [m for b, m in _ERRORS.items() if bits & b]
    return ValueError(f"{what}: " + "; ".join(msgs))


def _lengths(x, name: str) -> torch.Tensor:
    t = x if isinstance(x, torch.Tensor) else torch.as_tensor(x)
    if t.dim() != 1 or t.dtype.is_floating_point or t.dtype == torch.bool:
        raise ValueError(f"{name} must be a 1-D integer tensor or list, got {tuple(t.shape)} {t.dtype}")
    return t.to(torch.int64)


@dataclass(frozen=True)
class RowIndex:
    """Index maps of one plan on one batch (int64, device; -1 = the appended zero row)."""
    R: int
    rows: torch.Tensor        # [R] hidden row of each compact row
    targets: torch.Tensor     # [R] token at row + 1, -1 where the log-prob is not read
    cell_map: torch.Tensor    # [bsz * L] compact row of each response cell's log-prob
    hidden_map: torch.Tensor  # [T] compact row of each hidden row
    cells: torch.Tensor       # [R + 1] -1, then the response cell of each compact row's log-prob


@dataclass(frozen=True)
class ResponseRowPlan:
    layout: int
    bsz: int
    response_len: int
    entropy_shift: int
    param: int                      # S (padded), max_prompt_len (fsdp_packed), 0 (megatron_thd)
    len0: Optional[torch.Tensor]    # prompt lengths (fsdp_packed) / cu_seqlens_padded (megatron_thd)
    len1: Optional[torch.Tensor]    # valid tokens per sequence (megatron_thd)
    resp: torch.Tensor              # r_b
    first_rows: Optional[torch.Tensor] = None  # a_b, host plans only
    num_rows: Optional[int] = None             # R, host plans only
    end_row: Optional[int] = None              # one past the last row a sequence reads, host plans only

    @property
    def on_device(self) -> bool:
        return self.resp.is_cuda

    def index(self, tokens: torch.Tensor, T: int) -> RowIndex:
        """Run the plan kernel on token ids [T] (int64, device)."""
        what = "response_logprobs_entropy"
        if self.layout == PADDED and T != self.bsz * self.param:
            raise ValueError(f"{what}: a padded plan of {self.bsz} x {self.param} needs T = "
                             f"{self.bsz * self.param} rows, got {T}")
        dev = tokens.device
        if self.on_device:
            R = None
            cap = min(T, self.bsz * (self.response_len + self.entropy_shift))
            lens = [t.to(dev) if t is not None else None for t in (self.len0, self.len1, self.resp)]
        else:
            if self.end_row > T:
                raise _error(4, what)
            R = cap = self.num_rows
            host = [t for t in (self.len0, self.len1, self.resp) if t is not None]
            flat = torch.cat(host).to(dev, non_blocking=True)  # one copy, no host sync
            lens, off = [], 0
            for t in (self.len0, self.len1, self.resp):
                lens.append(None if t is None else flat[off:off + t.numel()])
                off += 0 if t is None else t.numel()
        rows = torch.empty(cap, dtype=torch.int64, device=dev)
        targets = torch.empty(cap, dtype=torch.int64, device=dev)
        cell_map = torch.empty(self.bsz * self.response_len, dtype=torch.int64, device=dev)
        hidden_map = torch.empty(T, dtype=torch.int64, device=dev)
        cells = torch.empty(cap + 1, dtype=torch.int64, device=dev)
        status = torch.empty(2, dtype=torch.int64, device=dev)
        L.check(L.load().rb200_response_rows_plan(self.layout, L.ptr(lens[0]), L.ptr(lens[1]), L.ptr(lens[2]),
                                                  self.bsz, self.param, self.response_len, T, self.entropy_shift,
                                                  L.ptr(tokens), cap, L.ptr(rows), L.ptr(targets), L.ptr(cell_map),
                                                  L.ptr(hidden_map), L.ptr(cells), L.ptr(status), L.stream_ptr(dev)),
                "response_rows_plan")
        if R is None:
            R, bits = status.tolist()  # the forward's one device-to-host copy
            if bits:
                raise _error(bits, what)
        return RowIndex(R, rows[:R], targets[:R], cell_map, hidden_map, cells[:R + 1])


def _host_plan(layout, bsz, L_resp, shift, param, len0, len1, resp, starts, firsts, what):
    """Check a host plan as the plan kernel does and fill in a_b, R and the end row."""
    bits = 0
    if bool(((resp < 0) | (resp > L_resp)).any()):
        bits |= 1
    if bool((firsts - starts < 1).any()):
        bits |= 2
    if bool((starts < 0).any()):
        bits |= 4
    ends = firsts + resp
    if bsz > 1 and bool((starts[1:] < ends[:-1]).any()):
        bits |= 8
    if layout == MEGATRON_THD and bool((starts + len1 > len0[1:]).any()):
        bits |= 8
    if layout == FSDP_PACKED and bool((len0 > param).any()):
        bits |= 16
    if bits:
        raise _error(bits, what)
    R = int(torch.where(resp > 0, resp + shift, torch.zeros_like(resp)).sum())
    return ResponseRowPlan(layout, bsz, L_resp, shift, param, len0, len1, resp, firsts, R, int(ends.max()))


def _check_common(bsz: int, response_len: int, what: str):
    if not 0 < bsz <= MAX_BSZ:
        raise ValueError(f"{what}: needs 1 <= bsz <= {MAX_BSZ}, got {bsz}")
    if response_len <= 0:
        raise ValueError(f"{what}: response_len must be positive, got {response_len}")


def padded(bsz: int, S: int, response_len: int, response_lengths) -> ResponseRowPlan:
    """FSDP's forward_batch without packing: hidden [bsz, S, H] of prompts left-padded to S - response_len and
    responses right-padded to response_len; the reference computes `logits[:, -L-1:-1]`."""
    what = "response_rows.padded"
    bsz, S, response_len = int(bsz), int(S), int(response_len)
    _check_common(bsz, response_len, what)
    if S - response_len < 1:
        raise _error(2, what)
    resp = _lengths(response_lengths, "response_lengths")
    if resp.numel() != bsz:
        raise ValueError(f"{what}: {resp.numel()} response lengths for bsz {bsz}")
    if resp.is_cuda:
        return ResponseRowPlan(PADDED, bsz, response_len, 0, S, None, None, resp)
    starts = torch.arange(bsz, dtype=torch.int64) * S
    return _host_plan(PADDED, bsz, response_len, 0, S, None, None, resp, starts, starts + S - response_len, what)


def fsdp_packed(prompt_lengths, response_lengths, max_prompt_len: int, *, response_len: int) -> ResponseRowPlan:
    """FSDP's forward_batch with enable_dynamic_batch_size / variable_seq_lengths: prepare_pack_fsdp +
    pack_fsdp_input concatenate each sequence's p_b prompt and r_b response tokens into one [1, T] stream.
    response_len is the width of the unpacked output (max_seq_len_unpack - max_prompt_len in the reference)."""
    what = "response_rows.fsdp_packed"
    p = _lengths(prompt_lengths, "prompt_lengths")
    resp = _lengths(response_lengths, "response_lengths")
    bsz, response_len = p.numel(), int(response_len)
    _check_common(bsz, response_len, what)
    if resp.numel() != bsz:
        raise ValueError(f"{what}: {bsz} prompt lengths and {resp.numel()} response lengths")
    if p.is_cuda or resp.is_cuda:
        dev = p.device if p.is_cuda else resp.device
        return ResponseRowPlan(FSDP_PACKED, bsz, response_len, 1, int(max_prompt_len), p.to(dev), None, resp.to(dev))
    span = p + resp
    starts = torch.cumsum(span, 0) - span
    return _host_plan(FSDP_PACKED, bsz, response_len, 1, int(max_prompt_len), p, None, resp, starts, starts + p, what)


def megatron_thd(cu_seqlens_padded, seq_lengths, response_lengths, *, response_len: int,
                 cp_size: int = 1) -> ResponseRowPlan:
    """Megatron's custom_forward with pack_seqs: preprocess_packed_seqs puts sequence b's n_b valid tokens
    (= attention_mask[b].sum()) at cu_seqlens_padded[b]; the loss reads `[:, -L-1:-1]` of the unpacked output."""
    what = "response_rows.megatron_thd"
    if int(cp_size) != 1:
        raise ValueError(f"{what}: context parallelism (cp_size {cp_size}) is not supported")
    cu = _lengths(cu_seqlens_padded, "cu_seqlens_padded")
    n = _lengths(seq_lengths, "seq_lengths")
    resp = _lengths(response_lengths, "response_lengths")
    bsz, response_len = n.numel(), int(response_len)
    _check_common(bsz, response_len, what)
    if cu.numel() != bsz + 1 or resp.numel() != bsz:
        raise ValueError(f"{what}: needs bsz + 1 = {bsz + 1} cu_seqlens_padded and {bsz} response lengths, got "
                         f"{cu.numel()} and {resp.numel()}")
    if cu.is_cuda or n.is_cuda or resp.is_cuda:
        dev = next(t.device for t in (cu, n, resp) if t.is_cuda)
        return ResponseRowPlan(MEGATRON_THD, bsz, response_len, 0, 0, cu.to(dev), n.to(dev), resp.to(dev))
    starts = cu[:-1]
    return _host_plan(MEGATRON_THD, bsz, response_len, 0, 0, cu, n, resp, starts, starts + n - resp, what)
