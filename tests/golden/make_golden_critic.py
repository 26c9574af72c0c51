"""Reasoning-critic fixtures: the reference's own critic code on the CPU, over gloo processes laid out as Megatron's
(TP fastest, rank = c * tp + k):
    python tests/golden/make_golden_critic.py  ->  tests/golden/golden_critic.npz

Executed as the reference wrote them (extracted from its source with `ast`, compiled in place, or imported unmodified
through ref_loader; only numerical outputs are stored): `MegatronCritic.get_forward_step_func` (its
forward_output_and_loss_func body, inference and training) around `MegatronModelManager.custom_forward`, with
`preprocess_packed_seqs` / `postprocess_packed_seqs`; the value head `LinearForLastLayer` (a bf16 nn.Linear(H, 1)
without bias, cast with .float()); `compute_ppo_critic_loss` and `compute_critic_explained_variance_stats`.
`parallel_state` is a stand-in with TP, CP and (one-rank) data-parallel subgroups, and
`tensor_parallel.gather_from_sequence_parallel_region(x, tensor_parallel_output_grad=False)` is written from Megatron's
documented behaviour: all-gather along the sequence dimension in the forward, the rank's own chunk of the gradient in
the backward.

The decoder is make_golden_response_rows_mp.py's stand-in (hidden = bf16(E[id] + Pe[p]), H 64), with its batches:
the main one (an empty response, a full one, prediction rows across CP chunks and TP shards) and the sparse one, in
which CP rank 1 of (1, 2) and (2, 2) holds no response row.  Grids (tp, cp, SP): (1, 1, off), (2, 1, on), (1, 2, off)
and (2, 2, on).  Hyper-parameters: value_clip 0.5 with huber_delta 10000 (the worker's), and on the main batch also
value_clip 0.2 with huber_delta 0.3, whose errors reach Huber's linear branch.

Stored per case: the lengths, the value weight, returns, prev_values and the response mask; the inference values
(vpreds * mask) and the training vpreds; the loss, the metrics in critic_oracle.KEYS order (before Megatron's
data-parallel average, a no-op at one data-parallel rank) and d loss / d vpreds; per rank the hidden shard, its
gradient and the value weight's gradient."""
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
sys.path.insert(0, os.path.dirname(HERE))
import ref_loader  # noqa: E402
from make_golden_response_rows import extract  # noqa: E402
from make_golden_response_rows_mp import BATCHES, H, L, batch, weights  # noqa: E402

GRIDS = [(1, 1, False), (2, 1, True), (1, 2, False), (2, 2, True)]
HYPER = {"": (0.5, 10000.0), "_huber": (0.2, 0.3)}  # suffix -> (value_clip, huber_delta)


def value_weight():
    g = torch.Generator().manual_seed(29)
    return (0.3 * torch.randn(1, H, generator=g)).bfloat16()


def targets(bsz, seed):
    g = torch.Generator().manual_seed(seed)
    returns = 0.8 * torch.randn(bsz, L, generator=g)
    prev = 0.5 * torch.randn(bsz, L, generator=g)
    return returns, prev


class _GatherFromSP(torch.autograd.Function):
    """gather_from_sequence_parallel_region(x, tensor_parallel_output_grad=False): all-gather dim 0 over TP; the
    backward takes the rank's own chunk of the gradient (no reduction)."""

    @staticmethod
    def forward(ctx, x, group):
        ctx.group = group
        P = dist.get_world_size(group)
        out = [torch.empty_like(x) for _ in range(P)]
        dist.all_gather(out, x.contiguous(), group=group)
        return torch.cat(out)

    @staticmethod
    def backward(ctx, g):
        P, k = dist.get_world_size(ctx.group), dist.get_rank(ctx.group)
        n = g.shape[0] // P
        return g[k * n:(k + 1) * n], None


def _value_head_class(tp_group):
    src = open(os.path.join(ref_loader.REFERENCE_ROOT, "rlinf/hybrid_engines/megatron/megatron_model_manager.py")).read()
    node = next(n for n in ast.parse(src).body if isinstance(n, ast.ClassDef) and n.name == "LinearForLastLayer")
    def gather_from_sequence_parallel_region(x, tensor_parallel_output_grad=True):
        assert not tensor_parallel_output_grad, "the critic's value head passes tensor_parallel_output_grad=False"
        return _GatherFromSP.apply(x, tp_group)

    tensor_parallel = types.SimpleNamespace(gather_from_sequence_parallel_region=gather_from_sequence_parallel_region)
    ns = {"torch": torch, "tensor_parallel": tensor_parallel}
    exec(compile(ast.Module(body=[node], type_ignores=[]), "megatron_model_manager.py", "exec"), ns)
    return ns["LinearForLastLayer"]


class Model:
    """GPTModel's last stage with the critic's output layer: decoder stand-in -> output_layer -> [b, s, 1]."""
    pre_process = post_process = True

    def __init__(self, E, Pe, head, tp, k, sp, positions):
        self.E, self.Pe, self.head, self.tp, self.k, self.sp = E, Pe, head, tp, k, sp
        self.positions, self.shard = positions, None

    def __call__(self, input_ids, attention_mask, position_ids, packed_seq_params, **kw):
        full = (self.E[input_ids[0]] + self.Pe[self.positions]).bfloat16()  # [T_c, H]
        Ts = full.shape[0] // self.tp if self.sp else full.shape[0]
        self.shard = (full[self.k * Ts:(self.k + 1) * Ts] if self.sp else full).clone().requires_grad_(True)
        logits, _ = self.head(self.shard[:, None])  # [s, b, 1], sequence-first
        return logits.transpose(0, 1).contiguous()


def _worker(rank, tp, cp, sp, init_file, out_dir):
    world = tp * cp
    dist.init_process_group("gloo", init_method=f"file://{init_file}", rank=rank, world_size=world)
    torch.set_num_threads(1)
    ref = ref_loader.load_reference()
    tp_groups = [dist.new_group([c * tp + k for k in range(tp)]) for c in range(cp)]
    cp_groups = [dist.new_group([c * tp + k for c in range(cp)]) for k in range(tp)]
    dp_groups = [dist.new_group([r]) for r in range(world)]
    c, k = rank // tp, rank % tp
    tp_group, cp_group = tp_groups[c], cp_groups[k]

    class parallel_state:  # noqa: N801 - Megatron's module name
        get_tensor_model_parallel_world_size = staticmethod(lambda: tp)
        get_context_parallel_world_size = staticmethod(lambda: cp)
        get_context_parallel_rank = staticmethod(lambda: c)
        get_context_parallel_group = staticmethod(lambda: cp_group)
        get_data_parallel_group = staticmethod(lambda: dp_groups[rank])

    PackedSeqParams = lambda **kw: types.SimpleNamespace(**kw)  # noqa: E731
    root = ref_loader.REFERENCE_ROOT
    globs = {"torch": torch, "copy": copy, "parallel_state": parallel_state, "PackedSeqParams": PackedSeqParams,
             "Optional": None, "unwrap_model": lambda m: m,
             "average_losses_across_data_parallel_group": lambda ls: torch.cat([x.clone().detach().view(1)
                                                                                 for x in ls]),
             "compute_ppo_critic_loss": ref.losses.compute_ppo_critic_loss,
             "CRITIC_EXPLAINED_VARIANCE_STAT_KEYS": ref.metric_utils.CRITIC_EXPLAINED_VARIANCE_STAT_KEYS}
    extract(os.path.join(root, "rlinf/hybrid_engines/megatron/utils.py"),
            ["preprocess_packed_seqs", "postprocess_packed_seqs"], globs)
    custom_forward = extract(os.path.join(root, "rlinf/hybrid_engines/megatron/megatron_model_manager.py"),
                             ["custom_forward"], globs, "MegatronModelManager")["custom_forward"]
    step = extract(os.path.join(root, "rlinf/workers/critic/megatron_critic_worker.py"), ["get_forward_step_func"],
                   globs, "MegatronCritic")["get_forward_step_func"]
    pre = globs["preprocess_packed_seqs"]
    head_cls = _value_head_class(tp_group)

    E, Pe, _ = weights()
    w = value_weight()
    res = {}
    for (suffix, lens), (hsuf, (value_clip, delta)) in itertools.product(BATCHES.items(), HYPER.items()):
        if hsuf and suffix:
            continue  # the linear-branch case on the main batch only
        ids, mask, pos, resp_mask, _ = batch(*lens)
        bsz = ids.shape[0]
        returns, prev = targets(bsz, 31 + len(suffix) + len(hsuf))
        positions = pre(pos, mask)[0][0]
        key = f"tp{tp}_cp{cp}_sp{int(sp)}{suffix}{hsuf}"
        for return_loss in (False, True):
            head = head_cls(H, 1, sequence_parallel=sp).to(torch.bfloat16)
            with torch.no_grad():
                head.weight.copy_(w)
            model = Model(E, Pe, head, tp, k, sp, positions)
            self = types.SimpleNamespace(response_len=L, return_loss=return_loss, custom_forward=custom_forward,
                                         transformer_config=types.SimpleNamespace(sequence_parallel=sp),
                                         value_clip=value_clip, loss_agg_func=None)
            fwd = step(self)
            b = {"input_ids": ids, "attention_mask": mask, "position_ids": pos, "response_mask": resp_mask,
                 "returns": returns, "values": prev}
            b = {kk: types.SimpleNamespace(cuda=lambda v=v: v) for kk, v in b.items()}
            output, loss_func = fwd(iter([b]), model)
            if not return_loss:
                res[f"{key}_infer_values"] = output.detach().float().numpy()
                continue
            output.retain_grad()
            if delta != 10000.0:  # the worker passes huber_delta=10000; the linear branch needs a smaller one
                loss, metrics = _loss_with_delta(ref, output, returns, prev, resp_mask, value_clip, delta)
            else:
                loss, metrics = loss_func(output)
            loss.backward()
            _, psp = pre(ids, mask)
            T_c = positions.shape[0]
            res[f"{key}_meta"] = np.array([tp, cp, int(sp), L, bsz, T_c])
            res[f"{key}_hyper"] = np.array([value_clip, delta])
            res[f"{key}_cu"] = psp.cu_seqlens_q_padded.long().numpy()
            res[f"{key}_train_values"] = output[:, -L - 1:-1, 0].detach().numpy()
            res[f"{key}_vgrad"] = output.grad[:, -L - 1:-1, 0].numpy()
            res[f"{key}_loss"] = loss.detach().numpy()
            keys = ("critic/value_loss", "critic/value_clip_ratio") + tuple(
                ref.metric_utils.CRITIC_EXPLAINED_VARIANCE_STAT_KEYS) + ("critic/final_value_loss",)
            res[f"{key}_metrics"] = np.array([float(metrics[kk].reshape(-1)[0]) for kk in keys], dtype=np.float32)
            res[f"{key}_c{c}_k{k}_hidden"] = model.shard.detach().float().numpy()
            res[f"{key}_c{c}_k{k}_grad"] = model.shard.grad.float().numpy()
            res[f"{key}_c{c}_k{k}_wgrad"] = head.weight.grad.float().numpy()
    np.savez(os.path.join(out_dir, f"r{rank}.npz"), **res)
    dist.destroy_process_group()


def _loss_with_delta(ref, output, returns, prev, resp_mask, value_clip, delta):
    """MegatronCritic's loss_func body with another huber_delta (the worker hard-codes 10000)."""
    vpreds = output[:, -L - 1:-1].contiguous().squeeze(-1)
    loss, metrics = ref.losses.compute_ppo_critic_loss(values=vpreds, returns=returns, prev_values=prev,
                                                        value_clip=value_clip, huber_delta=delta,
                                                        loss_agg_func=None, loss_mask=resp_mask[:, -L:])
    metrics["critic/final_value_loss"] = loss.detach()
    return loss, metrics


def main():
    out = {"w": value_weight().float().numpy()}
    for tp, cp, sp in GRIDS:
        with tempfile.TemporaryDirectory() as tmp:
            mp.spawn(_worker, args=(tp, cp, sp, os.path.join(tmp, "init"), tmp), nprocs=tp * cp, join=True)
            ranks = [dict(np.load(os.path.join(tmp, f"r{r}.npz"))) for r in range(tp * cp)]
        for r in ranks:
            for key, v in r.items():
                if key in out and not re.search(r"_c\d+_k\d+_", key):
                    assert np.array_equal(out[key], v, equal_nan=True), key  # the same on every rank
                out[key] = v
        for (suffix, lens), (hsuf, _) in itertools.product(BATCHES.items(), HYPER.items()):
            if hsuf and suffix:
                continue
            ids, mask, _, resp_mask, _ = batch(*lens)
            key = f"tp{tp}_cp{cp}_sp{int(sp)}{suffix}{hsuf}"
            returns, prev = targets(ids.shape[0], 31 + len(suffix) + len(hsuf))
            out[f"{key}_n"] = mask.sum(-1).numpy()
            out[f"{key}_r"] = np.array(lens[1])
            out[f"{key}_returns"] = returns.numpy()
            out[f"{key}_prev_values"] = prev.numpy()
            out[f"{key}_mask"] = resp_mask[:, -L:].numpy()
    path = os.path.join(HERE, "golden_critic.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
