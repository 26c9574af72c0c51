"""Response-rows golden fixtures: the reference's own layout code run on tiny seeded batches, on the CPU:
    python tests/golden/make_golden_response_rows.py  ->  tests/golden/golden_response_rows.npz

Three paths, each executed as the reference wrote it (functions and methods extracted from its source with `ast` and
compiled in place; nothing is copied into this repository, only numerical outputs are stored):
  - FSDP `FSDPActor.forward_batch` (rlinf/workers/actor/fsdp_actor_worker.py) and `compute_logprobs`, both branches:
    without packing (`logits[:, -L-1:-1]`), and with packing through `prepare_pack_fsdp`, `pack_fsdp_input`,
    `pack_sequences`, `unpack_fsdp_logprobs` and `unpack_sequences` (rlinf/hybrid_engines/fsdp/utils.py), for
    variable_seq_lengths (no padding) and enable_dynamic_batch_size (eos-padded to max_tokens_per_mbs);
    `compute_logprobs_from_logits` / `compute_entropy_from_logits` come from rlinf/utils/utils.py.
  - Megatron `MegatronActor.get_forward_step_func` (megatron_actor_worker.py: the label and label-mask construction and
    `logits_processor`) around `MegatronModelManager.custom_forward` with `preprocess_packed_seqs` /
    `postprocess_packed_seqs` (rlinf/hybrid_engines/megatron/utils.py), at tp 1 and 2 over gloo processes, with
    variable and fixed (`padding_seqlen`) packed lengths, both the training output (`return_loss`) and the inference
    output (`* response_mask`).  `vocab_parallel_entropy_and_log_probs` is the reference's, with the non-aliasing
    stand-ins of make_golden_vp.py; `parallel_state` is a stand-in whose tensor-parallel group is the gloo world.
The model is a stand-in: hidden = E[input_ids] + Pe[position] (fp32, H 64), logits = hidden @ W^T (V 512).  Each case
stores the hidden states the model saw (in the model's input shape), the flattened token ids, the plan's inputs and
the reference's [bsz, L] log-probs and entropies, masked columns included.
"""
from __future__ import annotations

import ast
import contextlib
import copy
import os
import sys
import tempfile
import types

import numpy as np
import torch
import torch.distributed as dist
import torch.multiprocessing as mp
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from ref_loader import REFERENCE_ROOT, load_reference  # noqa: E402

V, H, NPOS = 512, 64, 128
PAD = 3  # eos / pad token id
TEMPERATURE = 0.7
PROMPTS = [3, 6, 1, 4, 2]   # p_b <= MAX_PROMPT
RESPONSES = [5, 0, 8, 2, 7]  # r_b <= L: an empty response and a full one
MAX_PROMPT, L = 6, 8
S = MAX_PROMPT + L


class Cfg(dict):
    def __getattr__(self, k):
        try:
            return self[k]
        except KeyError as e:
            raise AttributeError(k) from e

    def get(self, k, d=None):
        return dict.get(self, k, d)


def to_cfg(d):
    return Cfg({k: to_cfg(v) if isinstance(v, dict) else v for k, v in d.items()})


def extract(path, names, globs, class_name=None):
    """Compile the named functions (methods of class_name when given) of a reference file into globs."""
    tree = ast.parse(open(path).read())
    body = tree.body
    if class_name is not None:
        body = next(n for n in tree.body if isinstance(n, ast.ClassDef) and n.name == class_name).body
    found = {}
    for node in body:
        if isinstance(node, ast.FunctionDef) and node.name in names:
            node.decorator_list = []
            mod = ast.Module(body=[node], type_ignores=[])
            ast.fix_missing_locations(mod)
            exec(compile(mod, path, "exec"), globs)
            found[node.name] = globs[node.name]
    assert set(found) == set(names), set(names) - set(found)
    return found


def batch():
    """[bsz, S]: prompts left-padded to MAX_PROMPT, responses right-padded to L (the rollout's layout)."""
    g = torch.Generator().manual_seed(7)
    bsz = len(PROMPTS)
    ids = torch.full((bsz, S), PAD, dtype=torch.int64)
    mask = torch.zeros((bsz, S), dtype=torch.bool)
    for b, (p, r) in enumerate(zip(PROMPTS, RESPONSES)):
        ids[b, MAX_PROMPT - p:MAX_PROMPT + r] = torch.randint(4, V, (p + r,), generator=g)
        mask[b, MAX_PROMPT - p:MAX_PROMPT + r] = True
    pos = (torch.cumsum(mask.long(), -1) - 1).clamp(min=0)
    resp_mask = mask.clone()
    resp_mask[:, :MAX_PROMPT] = False
    return ids, mask, pos, resp_mask


def weights():
    g = torch.Generator().manual_seed(11)
    E = torch.randn(V, H, generator=g)
    Pe = 0.5 * torch.randn(NPOS, H, generator=g)
    W = 0.4 * torch.randn(V, H, generator=g)
    return E, Pe, W


class FsdpModel:
    """logits = (E[input_ids] + Pe[position_ids]) @ W^T; keeps the hidden states it saw."""

    def __init__(self, E, Pe, W):
        self.E, self.Pe, self.W, self.hidden = E, Pe, W, None

    def __call__(self, input_ids, attention_mask, position_ids, use_cache, **kw):
        self.hidden = self.E[input_ids] + self.Pe[position_ids]
        return types.SimpleNamespace(logits=self.hidden @ self.W.T)


def fsdp_cases(ref, E, Pe, W):
    fsdp_utils = os.path.join(REFERENCE_ROOT, "rlinf/hybrid_engines/fsdp/utils.py")
    actor = os.path.join(REFERENCE_ROOT, "rlinf/workers/actor/fsdp_actor_worker.py")
    globs = {"torch": torch}
    extract(fsdp_utils, ["pack_sequences", "unpack_sequences", "prepare_pack_fsdp", "pack_fsdp_input",
                         "unpack_fsdp_logprobs"], globs)
    globs.update(compute_logprobs_from_logits=ref.utils.compute_logprobs_from_logits,
                 compute_entropy_from_logits=ref.utils.compute_entropy_from_logits, Worker=None)
    fns = extract(actor, ["forward_batch", "compute_logprobs"], globs, "FSDPActor")
    ids, mask, pos, _ = batch()
    out = {}
    for name, dyn, var in (("fsdp_padded", False, False), ("fsdp_packed_var", False, True),
                           ("fsdp_packed_fixed", True, False)):
        model = FsdpModel(E, Pe, W)
        self = types.SimpleNamespace(
            enable_dynamic_batch_size=dyn, variable_seq_lengths=var, max_tokens_per_mbs=64, response_len=L,
            tokenizer=types.SimpleNamespace(eos_token_id=PAD), amp_context=contextlib.nullcontext(), model=model,
            entropy_op_type="torch",
            cfg=to_cfg({"actor": {"model": {"encoder_seq_length": S}}, "data": {"max_prompt_length": MAX_PROMPT},
                        "algorithm": {"sampling_params": {"temperature": TEMPERATURE}}}))
        self.compute_logprobs = types.MethodType(fns["compute_logprobs"], self)
        m_batch = {"input_ids": ids, "attention_mask": mask, "position_ids": pos,
                   "prompt_lengths": torch.tensor(PROMPTS), "response_lengths": torch.tensor(RESPONSES)}
        with torch.no_grad():
            lp, ent = fns["forward_batch"](self, m_batch, calculate_entropy=True)
        h = model.hidden
        tokens = ids.reshape(-1) if not (dyn or var) else None
        if tokens is None:  # the packed stream the model saw
            starts = [MAX_PROMPT - p for p in PROMPTS]
            ends = [MAX_PROMPT + r for r in RESPONSES]
            tokens = globs["pack_sequences"](ids, starts, ends, 64, PAD, dyn)
        out[f"{name}_hidden"] = h.numpy()
        out[f"{name}_tokens"] = tokens.numpy()
        out[f"{name}_logprobs"] = lp.numpy()
        out[f"{name}_entropy"] = ent.numpy()
    return out


# ---- Megatron, over gloo ------------------------------------------------------------------------------------------
class MegatronModel:
    pre_process = post_process = True

    def __init__(self, E, Pe, W, rank, P):
        self.E, self.Pe, self.W, self.rank, self.P, self.hidden = E, Pe, W, rank, P, None

    def __call__(self, input_ids, attention_mask, position_ids, packed_seq_params, **kw):
        T = input_ids.shape[1]
        self.hidden = self.E[input_ids] + self.Pe[torch.arange(T)][None]  # [1, T, H]
        Vs = V // self.P
        return (self.hidden @ self.W.T)[..., self.rank * Vs:(self.rank + 1) * Vs].contiguous()


def _megatron_worker(rank, P, init_file, out_dir):
    dist.init_process_group("gloo", init_method=f"file://{init_file}", rank=rank, world_size=P)
    torch.set_num_threads(1)
    import make_golden_vp as VP

    ce = types.ModuleType("megatron.core.tensor_parallel.cross_entropy")
    ce.VocabParallelCrossEntropy = VP._CEUtils
    for name in ("megatron", "megatron.core", "megatron.core.tensor_parallel"):
        sys.modules.setdefault(name, types.ModuleType(name))
    sys.modules["megatron.core.tensor_parallel.cross_entropy"] = ce
    vp_cls = VP._reference_class()

    class parallel_state:  # noqa: N801 - Megatron's module name
        get_tensor_model_parallel_world_size = staticmethod(dist.get_world_size)
        get_context_parallel_world_size = staticmethod(lambda: 1)
        get_context_parallel_rank = staticmethod(lambda: 0)

    PackedSeqParams = lambda **kw: types.SimpleNamespace(**kw)  # noqa: E731
    mutils = os.path.join(REFERENCE_ROOT, "rlinf/hybrid_engines/megatron/utils.py")
    dist_py = os.path.join(REFERENCE_ROOT, "rlinf/utils/distributed.py")
    manager = os.path.join(REFERENCE_ROOT, "rlinf/hybrid_engines/megatron/megatron_model_manager.py")
    actor = os.path.join(REFERENCE_ROOT, "rlinf/workers/actor/megatron_actor_worker.py")
    globs = {"torch": torch, "copy": copy, "parallel_state": parallel_state, "PackedSeqParams": PackedSeqParams,
             "Optional": None, "_VocabParallelEntropyAndCrossEntropy": vp_cls, "unwrap_model": lambda m: m}
    extract(mutils, ["preprocess_packed_seqs", "postprocess_packed_seqs"], globs)
    extract(dist_py, ["vocab_parallel_entropy_and_log_probs"], globs)
    custom_forward = extract(manager, ["custom_forward"], globs, "MegatronModelManager")["custom_forward"]
    step = extract(actor, ["get_forward_step_func"], globs, "MegatronActor")["get_forward_step_func"]

    E, Pe, W = weights()
    ids, mask, pos, resp_mask = batch()
    res = {}
    for var in (True, False):
        for return_loss in (True, False):
            model = MegatronModel(E, Pe, W, rank, P)
            self = types.SimpleNamespace(
                variable_seq_lengths=var, enable_dynamic_batch_size=False, encoder_seq_length=S, response_len=L,
                calculate_entropy=True, calculate_entropy_loss=True, return_loss=return_loss,
                custom_forward=custom_forward, transformer_config=types.SimpleNamespace(sequence_parallel=False),
                cfg=to_cfg({"algorithm": {"sampling_params": {"temperature": TEMPERATURE}}}))
            fwd = step(self)
            b = {"input_ids": ids, "attention_mask": mask, "position_ids": pos, "response_mask": resp_mask}
            b = {k: types.SimpleNamespace(cuda=lambda v=v: v) for k, v in b.items()}  # `.cuda()` is the identity
            with torch.no_grad():
                output, _ = fwd(iter([b]), model)
            key = f"{'var' if var else 'fixed'}_{'train' if return_loss else 'infer'}"
            if return_loss:  # what loss_func reads
                res[f"{key}_logprobs"] = output["log_probs"][:, -L - 1:-1].numpy()
                res[f"{key}_entropy"] = output["entropy"][:, -L - 1:-1].numpy()
            else:
                res[f"{key}_logprobs"] = output.numpy()
            if return_loss:
                _, psp = globs["preprocess_packed_seqs"](ids, mask, padding_seqlen=None if var else S)
                res[f"{key}_cu"] = psp.cu_seqlens_q_padded.numpy()
                res[f"{key}_hidden"] = model.hidden.numpy()
                res[f"{key}_tokens"] = globs["preprocess_packed_seqs"](
                    ids, mask, padding_seqlen=None if var else S)[0].reshape(-1).numpy()
    np.savez(os.path.join(out_dir, f"r{rank}.npz"), **res)
    dist.destroy_process_group()


def megatron_cases():
    out = {}
    for P in (1, 2):
        with tempfile.TemporaryDirectory() as tmp:
            mp.spawn(_megatron_worker, args=(P, os.path.join(tmp, "init"), tmp), nprocs=P, join=True)
            ranks = [dict(np.load(os.path.join(tmp, f"r{k}.npz"))) for k in range(P)]
        for k in range(1, P):
            for key in ranks[0]:
                assert np.array_equal(ranks[k][key], ranks[0][key], equal_nan=True), key
        for key, v in ranks[0].items():
            out[f"megatron_tp{P}_{key}"] = v
    return out


def main():
    ref = load_reference()
    E, Pe, W = weights()
    out = {"W": W.numpy(), "prompt_lengths": np.array(PROMPTS), "response_lengths": np.array(RESPONSES),
           "seq_lengths": np.array(PROMPTS) + np.array(RESPONSES),
           "meta": np.array([V, H, MAX_PROMPT, L, S, PAD]), "temperature": np.array(TEMPERATURE)}
    out.update(fsdp_cases(ref, E, Pe, W))
    out.update(megatron_cases())
    path = os.path.join(HERE, "golden_response_rows.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
