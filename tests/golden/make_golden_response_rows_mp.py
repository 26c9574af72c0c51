"""Response-rows fixtures under Megatron sequence and context parallelism: the reference's own code on the CPU, over
gloo processes laid out as Megatron's (TP fastest, rank = c * tp + k):
    python tests/golden/make_golden_response_rows_mp.py  ->  tests/golden/golden_response_rows_mp.npz

Executed as the reference wrote them (extracted from its source with `ast`, compiled in place; only numerical outputs
are stored): `MegatronActor.get_forward_step_func` around `MegatronModelManager.custom_forward`, with
`preprocess_packed_seqs` / `postprocess_packed_seqs` (rlinf/hybrid_engines/megatron/utils.py) and
`vocab_parallel_entropy_and_log_probs` (its `_VocabParallelEntropyAndCrossEntropy` over the TP group, with the
non-aliasing gradient helpers of make_golden_vp.py).  `parallel_state` is a stand-in with TP and CP subgroups.

The model is a stand-in: position p of a sequence gets hidden = bf16(E[id] + Pe[p]) (H 64; p from
preprocess_packed_seqs applied to the position ids), and the output layer is written from ColumnParallelLinear's
documented behaviour: under sequence parallelism the rank's hidden shard is all-gathered over TP in the forward and its
gradient reduce-scattered in the backward (gloo has no reduce-scatter: an all-reduce, then the rank's chunk); without
it the input is copied to every TP rank and its gradient all-reduced.  logits = hidden @ W_shard^T (V 512,
bf16-exact W).

Grids (tp, cp, SP): (2, 1, on), (1, 2, off), (2, 2, on); variable_seq_lengths on and off (padding_seqlen = S); the
training output and the inference output; two batches.  The main batch (keys ..._var / ..._fixed) has an empty
response, a full one and prediction rows that straddle CP chunk and TP shard boundaries.  The sparse batch (keys
..._var_empty / ..._fixed_empty) has one-token responses at the end of long sequences: every prediction row lies in
the last chunk, which CP rank 0 holds, so CP rank 1 of (1, 2) and (2, 2) has none, and in (2, 1) TP shard 0 holds only
a sequence without a response.  Stored per rank: the hidden shard, preprocess_packed_seqs of the position
ids + 1 (0 = padding: the ownership), and the gradient of sum(g * log_probs[:, -L-1:-1]) w.r.t. the shard (log-probs
only: the reference's entropy gradient is the known deviation, DESIGN.md §2; g is zero at j >= r_b, as under a loss
mask, because the reference's training output holds log p(pad) at column r_b).  Per case: the lengths, responses, g, the
training and inference log-probs [bsz, L] (identical on every rank)."""
from __future__ import annotations

import ast
import copy
import itertools
import os
import re
import sys
import tempfile
import types

import numpy as np
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from ref_loader import REFERENCE_ROOT  # noqa: E402
from make_golden_response_rows import extract, to_cfg  # noqa: E402

V, H, NPOS = 512, 64, 64
PAD = 3
TEMPERATURE = 0.7
BATCHES = {"": ([6, 3, 5, 2], [0, 8, 2, 6]), "_empty": ([9, 7, 7, 6], [0, 1, 1, 0])}  # (prompts, responses)
MAX_PROMPT, L = 10, 8
S = MAX_PROMPT + L
GRIDS = [(2, 1, True), (1, 2, False), (2, 2, True)]


def batch(prompts, responses):
    g = torch.Generator().manual_seed(17)
    bsz = len(prompts)
    ids = torch.full((bsz, S), PAD, dtype=torch.int64)
    mask = torch.zeros((bsz, S), dtype=torch.bool)
    for b, (p, r) in enumerate(zip(prompts, responses)):
        ids[b, MAX_PROMPT - p:MAX_PROMPT + r] = torch.randint(4, V, (p + r,), generator=g)
        mask[b, MAX_PROMPT - p:MAX_PROMPT + r] = True
    pos = (torch.cumsum(mask.long(), -1) - 1).clamp(min=0)
    resp_mask = mask.clone()
    resp_mask[:, :MAX_PROMPT] = False
    gl = torch.randn(bsz, L, generator=g)
    gl[torch.arange(L)[None] >= torch.tensor(responses)[:, None]] = 0  # as a loss mask does
    return ids, mask, pos, resp_mask, gl


def weights():
    g = torch.Generator().manual_seed(23)
    E = torch.randn(V, H, generator=g)
    Pe = 0.5 * torch.randn(NPOS, H, generator=g)
    W = (0.4 * torch.randn(V, H, generator=g)).bfloat16().float()
    return E, Pe, W


def _vp_class(tp_group):
    import make_golden_vp as VP

    src = open(os.path.join(REFERENCE_ROOT, "rlinf", "utils", "distributed.py")).read()
    node = next(n for n in ast.parse(src).body
                if isinstance(n, ast.ClassDef) and n.name == "_VocabParallelEntropyAndCrossEntropy")

    class parallel_state:  # noqa: N801 - Megatron's module name
        get_tensor_model_parallel_group = staticmethod(lambda: tp_group)
        get_tensor_model_parallel_rank = staticmethod(lambda: dist.get_rank(tp_group))
        get_tensor_model_parallel_world_size = staticmethod(lambda: dist.get_world_size(tp_group))

    class VocabUtility:
        @staticmethod
        def vocab_range_from_per_partition_vocab_size(per_partition, rank, world_size):
            return rank * per_partition, (rank + 1) * per_partition

    ce = types.ModuleType("megatron.core.tensor_parallel.cross_entropy")
    ce.VocabParallelCrossEntropy = VP._CEUtils
    for name in ("megatron", "megatron.core", "megatron.core.tensor_parallel"):
        sys.modules.setdefault(name, types.ModuleType(name))
    sys.modules["megatron.core.tensor_parallel.cross_entropy"] = ce
    ns = {"torch": torch, "parallel_state": parallel_state, "VocabUtility": VocabUtility}
    exec(compile(ast.Module(body=[node], type_ignores=[]), "distributed.py", "exec"), ns)
    return ns["_VocabParallelEntropyAndCrossEntropy"]


class _SPGather(torch.autograd.Function):
    """ColumnParallelLinear's sequence-parallel input: all-gather over TP forward, reduce-scatter backward."""

    @staticmethod
    def forward(ctx, x, group):
        ctx.group = group
        P = dist.get_world_size(group)
        out = [torch.empty_like(x) for _ in range(P)]
        dist.all_gather(out, x.contiguous(), group=group)
        return torch.cat(out)

    @staticmethod
    def backward(ctx, g):
        g = g.contiguous()
        dist.all_reduce(g, group=ctx.group)
        P, k = dist.get_world_size(ctx.group), dist.get_rank(ctx.group)
        n = g.shape[0] // P
        return g[k * n:(k + 1) * n], None


class _TPCopy(torch.autograd.Function):
    """ColumnParallelLinear's input without sequence parallelism: identity forward, all-reduce over TP backward."""

    @staticmethod
    def forward(ctx, x, group):
        ctx.group = group
        return x.view_as(x)

    @staticmethod
    def backward(ctx, g):
        g = g.contiguous()
        dist.all_reduce(g, group=ctx.group)
        return g, None


class Model:
    pre_process = post_process = True

    def __init__(self, E, Pe, W, tp, k, sp, tp_group, positions):
        self.E, self.Pe, self.W, self.tp, self.k, self.sp, self.g = E, Pe, W, tp, k, sp, tp_group
        self.positions, self.shard = positions, None

    def __call__(self, input_ids, attention_mask, position_ids, packed_seq_params, **kw):
        full = (self.E[input_ids[0]] + self.Pe[self.positions]).bfloat16().float()  # [T_c, H]
        Ts = full.shape[0] // self.tp if self.sp else full.shape[0]
        self.shard = (full[self.k * Ts:(self.k + 1) * Ts] if self.sp else full).clone().requires_grad_(True)
        x = _SPGather.apply(self.shard, self.g) if self.sp else _TPCopy.apply(self.shard, self.g)
        Vs = V // self.tp
        return (x @ self.W[self.k * Vs:(self.k + 1) * Vs].T)[None]


def _worker(rank, tp, cp, sp, init_file, out_dir):
    world = tp * cp
    dist.init_process_group("gloo", init_method=f"file://{init_file}", rank=rank, world_size=world)
    torch.set_num_threads(1)
    tp_groups = [dist.new_group([c * tp + k for k in range(tp)]) for c in range(cp)]
    cp_groups = [dist.new_group([c * tp + k for c in range(cp)]) for k in range(tp)]
    c, k = rank // tp, rank % tp
    tp_group, cp_group = tp_groups[c], cp_groups[k]

    class parallel_state:  # noqa: N801 - Megatron's module name
        get_tensor_model_parallel_world_size = staticmethod(lambda: tp)
        get_context_parallel_world_size = staticmethod(lambda: cp)
        get_context_parallel_rank = staticmethod(lambda: c)
        get_context_parallel_group = staticmethod(lambda: cp_group)

    PackedSeqParams = lambda **kw: types.SimpleNamespace(**kw)  # noqa: E731
    mutils = os.path.join(REFERENCE_ROOT, "rlinf/hybrid_engines/megatron/utils.py")
    dist_py = os.path.join(REFERENCE_ROOT, "rlinf/utils/distributed.py")
    manager = os.path.join(REFERENCE_ROOT, "rlinf/hybrid_engines/megatron/megatron_model_manager.py")
    actor = os.path.join(REFERENCE_ROOT, "rlinf/workers/actor/megatron_actor_worker.py")
    globs = {"torch": torch, "copy": copy, "parallel_state": parallel_state, "PackedSeqParams": PackedSeqParams,
             "Optional": None, "_VocabParallelEntropyAndCrossEntropy": _vp_class(tp_group),
             "unwrap_model": lambda m: m}
    extract(mutils, ["preprocess_packed_seqs", "postprocess_packed_seqs"], globs)
    extract(dist_py, ["vocab_parallel_entropy_and_log_probs"], globs)
    custom_forward = extract(manager, ["custom_forward"], globs, "MegatronModelManager")["custom_forward"]
    step = extract(actor, ["get_forward_step_func"], globs, "MegatronActor")["get_forward_step_func"]
    pre = globs["preprocess_packed_seqs"]

    E, Pe, W = weights()
    res = {}
    for (suffix, lens), var in itertools.product(BATCHES.items(), (True, False)):
        ids, mask, pos, resp_mask, gl = batch(*lens)
        padding = None if var else S
        positions = pre(pos, mask, padding_seqlen=padding)[0][0]
        own = pre((pos + 1) * mask, mask, padding_seqlen=padding)[0][0]
        key = f"tp{tp}_cp{cp}_sp{int(sp)}_{'var' if var else 'fixed'}{suffix}"
        for return_loss in (True, False):
            model = Model(E, Pe, W, tp, k, sp, tp_group, positions)
            self = types.SimpleNamespace(
                variable_seq_lengths=var, enable_dynamic_batch_size=False, encoder_seq_length=S, response_len=L,
                calculate_entropy=True, calculate_entropy_loss=True, return_loss=return_loss,
                custom_forward=custom_forward, transformer_config=types.SimpleNamespace(sequence_parallel=sp),
                cfg=to_cfg({"algorithm": {"sampling_params": {"temperature": TEMPERATURE}}}))
            fwd = step(self)
            b = {"input_ids": ids, "attention_mask": mask, "position_ids": pos, "response_mask": resp_mask}
            b = {kk: types.SimpleNamespace(cuda=lambda v=v: v) for kk, v in b.items()}
            output, _ = fwd(iter([b]), model)
            if not return_loss:
                res[f"{key}_infer_logprobs"] = output.detach().numpy()
                continue
            lp = output["log_probs"][:, -L - 1:-1]
            (lp * gl).sum().backward()
            _, psp = pre(ids, mask, padding_seqlen=padding)
            T_c = positions.shape[0]
            res[f"{key}_meta"] = np.array([tp, cp, int(sp), L, len(lens[0]), T_c, V])
            res[f"{key}_cu"] = psp.cu_seqlens_q_padded.long().numpy()
            res[f"{key}_logprobs"] = lp.detach().numpy()
            Ts = T_c // tp if sp else T_c
            sl = slice(k * Ts, (k + 1) * Ts) if sp else slice(0, T_c)
            res[f"{key}_c{c}_k{k}_hidden"] = model.shard.detach().numpy()
            res[f"{key}_c{c}_k{k}_positions"] = own[sl].numpy()
            res[f"{key}_c{c}_k{k}_grad"] = model.shard.grad.numpy()
    np.savez(os.path.join(out_dir, f"r{rank}.npz"), **res)
    dist.destroy_process_group()


def main():
    E, Pe, W = weights()
    out = {"W": W.numpy(), "temperature": np.array(TEMPERATURE)}
    for tp, cp, sp in GRIDS:
        with tempfile.TemporaryDirectory() as tmp:
            mp.spawn(_worker, args=(tp, cp, sp, os.path.join(tmp, "init"), tmp), nprocs=tp * cp, join=True)
            ranks = [dict(np.load(os.path.join(tmp, f"r{r}.npz"))) for r in range(tp * cp)]
        for r in ranks:
            for key, v in r.items():
                if key in out and not re.search(r"_c\d+_k\d+_", key):
                    assert np.array_equal(out[key], v, equal_nan=True), key  # the same on every rank
                out[key] = v
        for (suffix, lens), var in itertools.product(BATCHES.items(), ("var", "fixed")):
            ids, mask, _, _, gl = batch(*lens)
            key = f"tp{tp}_cp{cp}_sp{int(sp)}_{var}{suffix}"
            out[f"{key}_n"] = mask.sum(-1).numpy()
            out[f"{key}_r"] = np.array(lens[1])
            out[f"{key}_responses"] = ids[:, -L:].numpy()
            out[f"{key}_g"] = gl.numpy()
    path = os.path.join(HERE, "golden_response_rows_mp.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
