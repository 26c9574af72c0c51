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

megatron_parallel(...) is the Megatron THD layout under sequence and context parallelism, for
ops.megatron_response_logprobs_entropy: each rank holds a shard of the packed stream (csrc/response_rows_mp.cu).
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
    64: "the hidden shard has too few rows for the packed stream (T_c < cu_seqlens_padded[-1] / cp_size), or T_c is "
        "not divisible by tp_size",
    128: "a padded sequence length (or cu_seqlens_padded[0]) is not a multiple of 2 * cp_size",
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


# ---------------------------------------------------------------------------------------------------------------
# Megatron THD under sequence (SP) and context (CP) parallelism
# ---------------------------------------------------------------------------------------------------------------
MP_MAX_RANKS = 64


@dataclass(frozen=True)
class MPIndex:
    """Index maps of a megatron_parallel plan for rank (tp_rank k, cp_rank c) (int64, device; -1 = pad / zero row).
    R is R_c, the prediction rows CP rank c holds; counts[c][k] the rows TP shard k of CP rank c holds (SP), or R_c in
    every k without SP.  Rmax_k / Rmax_c are the padded row counts of the TP row all-gather and the CP value
    all-gather (at least 1, so every collective has a buffer)."""
    tp: int
    cp: int
    k: int
    c: int
    sp: bool
    T_c: int
    R: int
    Rmax_k: int
    Rmax_c: int
    counts: tuple
    rows: torch.Tensor        # [R] CP-local row of each compact row
    targets: torch.Tensor     # [R] responses[b, j]
    cells: torch.Tensor       # [R] response cell b * L + j of each compact row
    unpad: torch.Tensor       # [R] row of the TP-gathered [tp * Rmax_k] buffer (SP), identity without
    send: Optional[torch.Tensor]      # [Rmax_k] rows of the hidden shard to all-gather (SP), -1 = pad
    slot_map: Optional[torch.Tensor]  # [tp * Rmax_k] compact row of each reduce-scatter slot (SP), -1 = pad
    cell_map: torch.Tensor    # [bsz * L] row of the CP-gathered [cp * Rmax_c] values, -1 past r_b
    hidden_map: torch.Tensor  # [T_c / tp] slot of the reduce-scattered rows (SP) or [T_c] compact row (no SP)

    @property
    def shard_rows(self) -> int:
        return self.T_c // self.tp if self.sp else self.T_c


def _mp_runs(cu, n, resp, cp: int, c: int):
    """Per sequence, CP rank c's two runs of prediction rows: (tA, cA, tB, cB), CP-local rows (host tensors)."""
    N = cu[1:] - cu[:-1]
    p0 = n - resp - 1
    p1 = p0 + resp.clamp(min=0)
    if cp == 1:
        start, half, a0, a1 = cu[:-1], N, torch.zeros_like(N), N
        b0 = b1 = torch.zeros_like(N)
    else:
        start, half = cu[:-1] // cp, N // (2 * cp)
        a0 = half * c
        a1 = a0 + half
        b0 = N - half * (c + 1)
        b1 = b0 + half
    pA, pB = torch.maximum(p0, a0), torch.maximum(p0, b0)
    cA = (torch.minimum(p1, a1) - pA).clamp(min=0)
    cB = (torch.minimum(p1, b1) - pB).clamp(min=0)
    return start + pA - a0, cA, start + half + pB - b0, cB


def _overlap(t0, cnt, lo, hi) -> int:
    return int((torch.minimum(t0 + cnt, torch.full_like(t0, hi)) - t0.clamp(min=lo)).clamp(min=0).sum())


@dataclass(frozen=True)
class MegatronParallelPlan:
    bsz: int
    response_len: int
    tp_size: int
    cp_size: int
    sequence_parallel: bool
    cu: torch.Tensor
    n: torch.Tensor
    resp: torch.Tensor

    @property
    def on_device(self) -> bool:
        return self.resp.is_cuda

    def counts(self, T_c: int):
        """Rows of every rank (c, k) as nested tuples [cp][tp] (host plans; no device work)."""
        tp, cp, sp = self.tp_size, self.cp_size, self.sequence_parallel
        out = []
        for c in range(cp):
            tA, cA, tB, cB = _mp_runs(self.cu, self.n, self.resp, cp, c)
            if sp:
                Ts = T_c // tp
                out.append(tuple(_overlap(tA, cA, k * Ts, (k + 1) * Ts) + _overlap(tB, cB, k * Ts, (k + 1) * Ts)
                                 for k in range(tp)))
            else:
                out.append((int(cA.sum() + cB.sum()),) * tp)
        return tuple(out)

    def index(self, responses: torch.Tensor, shard_rows: int, tp_rank: int, cp_rank: int) -> MPIndex:
        """Run the plan kernel for rank (tp_rank, cp_rank) whose hidden shard has `shard_rows` rows; responses
        [bsz, response_len] int64 on the device."""
        what = "megatron_response_logprobs_entropy"
        tp, cp, sp = self.tp_size, self.cp_size, self.sequence_parallel
        if not (0 <= tp_rank < tp and 0 <= cp_rank < cp):
            raise ValueError(f"{what}: rank (tp {tp_rank}, cp {cp_rank}) outside the plan's tp {tp} x cp {cp} grid")
        T_c = shard_rows * tp if sp else shard_rows
        dev = responses.device
        if tuple(responses.shape) != (self.bsz, self.response_len):
            raise ValueError(f"{what}: responses must be [bsz, response_len] = [{self.bsz}, {self.response_len}], "
                             f"got {tuple(responses.shape)}")
        if self.on_device:
            counts = None
            cap_c = min(T_c, self.bsz * self.response_len)
            cap_k = min(T_c // tp, cap_c) if sp else 0
            lens = [t.to(dev) for t in (self.cu, self.n, self.resp)]
        else:
            if int(self.cu[-1]) // cp > T_c or T_c <= 0:
                raise _error(64, what)
            counts = self.counts(T_c)
            cap_c = sum(counts[cp_rank]) if sp else counts[cp_rank][0]
            cap_k = max(1, max(counts[cp_rank])) if sp else 0
            flat = torch.cat([self.cu, self.n, self.resp]).to(dev, non_blocking=True)  # one copy, no host sync
            b = self.bsz
            lens = [flat[:b + 1], flat[b + 1:2 * b + 1], flat[2 * b + 1:]]
        i64 = dict(dtype=torch.int64, device=dev)
        rows, targets, cells, unpad = (torch.empty(cap_c, **i64) for _ in range(4))
        send = torch.empty(cap_k, **i64) if sp else None
        slot_map = torch.empty(tp * cap_k, **i64) if sp else None
        cell_map = torch.empty(self.bsz * self.response_len, **i64)
        hidden_map = torch.empty(shard_rows, **i64)
        status = torch.empty(1 + cp * tp, **i64)
        L.check(L.load().rb200_response_rows_mp_plan(
            L.ptr(lens[0]), L.ptr(lens[1]), L.ptr(lens[2]), L.ptr(responses), self.bsz, self.response_len, T_c, tp,
            cp, int(sp), tp_rank, cp_rank, cap_c, cap_k, L.ptr(rows), L.ptr(send), L.ptr(unpad), L.ptr(slot_map),
            L.ptr(targets), L.ptr(cell_map), L.ptr(cells), L.ptr(hidden_map), L.ptr(status), L.stream_ptr(dev)),
            "response_rows_mp_plan")
        if counts is None:
            st = status.tolist()  # the forward's one device-to-host copy
            if st[0]:
                raise _error(st[0], what)
            counts = tuple(tuple(st[1 + c * tp:1 + (c + 1) * tp]) for c in range(cp))
        R = sum(counts[cp_rank]) if sp else counts[cp_rank][0]
        Rmax_c = max(1, max(sum(x) if sp else x[0] for x in counts))
        Rmax_k = max(1, max(counts[cp_rank])) if sp else R
        nk = Rmax_k if sp else 0
        return MPIndex(tp, cp, tp_rank, cp_rank, sp, T_c, R, Rmax_k, Rmax_c, counts, rows[:R], targets[:R],
                       cells[:R], unpad[:R], send[:nk] if sp else None, slot_map[:tp * nk] if sp else None,
                       cell_map, hidden_map)


def megatron_parallel(cu_seqlens_padded, seq_lengths, response_lengths, *, response_len: int, tp_size: int = 1,
                      cp_size: int = 1, sequence_parallel: bool = False) -> MegatronParallelPlan:
    """Megatron's custom_forward with pack_seqs under tensor (tp_size), sequence (sequence_parallel) and context
    (cp_size) parallelism, for ops.megatron_response_logprobs_entropy.  The lengths are megatron_thd's: the
    cu_seqlens_padded of preprocess_packed_seqs (padded lengths N_b, multiples of 2 * cp_size when cp_size > 1), n_b =
    attention_mask.sum(-1) and r_b, on the host or the device.  Ownership follows preprocess_packed_seqs: with cp_size 1
    sequence b sits at rows cu[b] + p of the packed stream; with cp_size > 1, half = N_b / (2 cp), CP rank c holds
    positions [half c, half (c + 1)) at its rows cu[b] / cp + ... and [N_b - half (c + 1), N_b - half c) at
    cu[b] / cp + half + ...; under sequence parallelism TP rank k holds rows [k T_c / tp, (k + 1) T_c / tp) of its CP
    rank's T_c rows.  Every rank must pass the same lengths: they are not compared across ranks (that would cost a
    collective), and lengths that disagree give wrong collective sizes."""
    what = "response_rows.megatron_parallel"
    tp, cp, sp = int(tp_size), int(cp_size), bool(sequence_parallel)
    if tp < 1 or cp < 1 or tp * cp > MP_MAX_RANKS:
        raise ValueError(f"{what}: needs tp_size, cp_size >= 1 and tp_size * cp_size <= {MP_MAX_RANKS}, got "
                         f"{tp} x {cp}")
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
        return MegatronParallelPlan(bsz, response_len, tp, cp, sp, cu.to(dev), n.to(dev), resp.to(dev))
    bits = 0
    if bool(((resp < 0) | (resp > response_len)).any()):
        bits |= 1
    if bool((n - resp < 1).any()):
        bits |= 2
    if int(cu[0]) < 0:
        bits |= 4
    if bool((cu[:-1] + n > cu[1:]).any()):
        bits |= 8
    if cp > 1 and (bool(((cu[1:] - cu[:-1]) % (2 * cp) != 0).any()) or int(cu[0]) % (2 * cp) != 0):
        bits |= 128
    if bits:
        raise _error(bits, what)
    return MegatronParallelPlan(bsz, response_len, tp, cp, sp, cu, n, resp)
