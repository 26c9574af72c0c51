"""Plain OpenVLA decode fixture: the installed transformers' real `generate` with the reference's logits processor and
the reference's post-processing, on the CPU:
    python tests/golden/make_golden_openvla_decode.py  ->  tests/golden/golden_openvla_decode.npz

A tiny randomly initialised bf16 `LlamaForCausalLM` (vocab 32064, hidden 64, one layer), built from a local config
with nothing downloaded, stands in for the Prismatic backbone.  `VLALogitsProcessor` is extracted with `ast` from the
unmodified reference model file (models/embodiment/openvla/openvla_action_model.py; importing that module pulls in the
Prismatic stack) and passed as `logits_processor`, with the kwargs the rollout worker passes (huggingface_worker.py:
do_sample, temperature, top_k, top_p = 1.0, max_new_tokens = 7) plus the output flags of predict_action_batch.  The
statements of predict_action_batch after `generate` (`action_tokens = ...` through `chunk_actions = ...`) then run as
written on a stub `self` (vocab_size 32000, bin_centers, norm stats with a masked dimension, n_action_bins 256).

Cases: greedy; sampling at (T, k) in SAMPLE_CASES; and `tie`, greedy and (1.0, 50) sampling with duplicated window rows
in lm_head.weight so that the argmax and the 50th value tie.  Stored, per case: each step's last-position hidden row
`hidden` [B, 7, 64], the raw-logit and processed-score window slices `logits` / `scores` [B, 7, 256], `outside_inf`
(every processed score outside the window is -inf), `tokens` (sequences[:, -7:]), `logprob` (chunk_logprobs) and
`actions`; and the window rows of lm_head.weight (`w_window`, and `tie_w_window`)."""
from __future__ import annotations

import ast
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

V, VOCAB, NBINS, ADIM, HID = 32064, 32000, 256, 7, 64
LO, HI = VOCAB - NBINS, VOCAB
B, PROMPT = 4, 6
SAMPLE_CASES = ((1.0, 0), (1.0, 50), (0.6, 50))
MASK_OFF = 2
FILE = "rlinf/models/embodiment/openvla/openvla_action_model.py"


def case_name(do_sample, T=1.0, k=0, tie=False):
    return ("tie_" if tie else "") + (f"T{T:g}_k{k}" if do_sample else "greedy")


CASES = [case_name(False)] + [case_name(True, T, k) for T, k in SAMPLE_CASES] + [case_name(False, tie=True),
                                                                                  case_name(True, 1.0, 50, tie=True)]


def bins():
    edges = np.linspace(-1, 1, NBINS)
    centers = (edges[:-1] + edges[1:]) / 2.0
    rng = np.random.default_rng(11)
    q01 = rng.uniform(-2.0, -0.1, ADIM)
    q99 = q01 + rng.uniform(0.2, 3.0, ADIM)
    mask = np.ones(ADIM, dtype=bool)
    mask[MASK_OFF] = False
    return centers, q01, q99, mask


def extract(path):
    """(the VLALogitsProcessor class source, the statements of predict_action_batch after generate), compiled."""
    tree = ast.parse(open(path).read())
    proc = next(n for n in ast.walk(tree) if isinstance(n, ast.ClassDef) and n.name == "VLALogitsProcessor")
    cls = next(n for n in ast.walk(tree) if isinstance(n, ast.ClassDef) and n.name == "OpenVLAForRLActionPrediction")
    body = next(n for n in cls.body if isinstance(n, ast.FunctionDef) and n.name == "predict_action_batch").body
    i0 = next(i for i, s in enumerate(body) if isinstance(s, ast.Assign) and ast.unparse(s.targets[0]) == "action_tokens")
    i1 = next(i for i, s in enumerate(body) if isinstance(s, ast.Assign) and ast.unparse(s.targets[0]) == "chunk_actions")
    mods = [ast.Module(body=[proc], type_ignores=[]), ast.Module(body=body[i0:i1 + 1], type_ignores=[])]
    for m in mods:
        ast.fix_missing_locations(m)
    return compile(mods[0], path, "exec"), compile(mods[1], path, "exec")


def make_model(tie: bool):
    from transformers import LlamaConfig, LlamaForCausalLM

    cfg = LlamaConfig(vocab_size=V, hidden_size=HID, intermediate_size=128, num_hidden_layers=1, num_attention_heads=2,
                      num_key_value_heads=2, max_position_embeddings=64, pad_token_id=VOCAB, bos_token_id=1,
                      eos_token_id=2, tie_word_embeddings=False)
    torch.manual_seed(1234)
    model = LlamaForCausalLM(cfg).to(torch.bfloat16).eval()
    with torch.no_grad():
        w = model.lm_head.weight
        w.mul_(20.0)  # logits of order 1, so that T and top-k change the distribution
        if tie:
            w[LO + 40] = w[LO + 7]    # the duplicate of a lower window row: an exact tie wherever either is the argmax
            for j in range(60):       # rows 100..159 repeat 60..119 (every bf16 dot product ties pairwise)
                w[LO + 100 + j] = w[LO + 60 + j]
    return model


def run(model, proc_cls, post, utils, do_sample, T, k, seed):
    from transformers import LogitsProcessorList

    g = torch.Generator().manual_seed(77)
    input_ids = torch.randint(3, VOCAB, (B, PROMPT), generator=g)
    input_ids[:, 0] = 1
    attention_mask = torch.ones_like(input_ids, dtype=torch.bool)
    torch.manual_seed(seed)
    with torch.no_grad():
        generated_results = model.generate(
            input_ids, attention_mask=attention_mask, output_scores=True, output_logits=True, output_hidden_states=True,
            return_dict_in_generate=True, do_sample=do_sample, logits_processor=LogitsProcessorList([proc_cls(NBINS)]),
            temperature=T, top_k=k, top_p=1.0, max_new_tokens=ADIM, pad_token_id=VOCAB)
    centers, q01, q99, mask = bins()
    self_ = types.SimpleNamespace(vocab_size=VOCAB, config=types.SimpleNamespace(n_action_bins=NBINS), action_dim=ADIM,
                                  num_action_chunks=1, bin_centers=centers,
                                  _get_action_stats=lambda: {"q01": list(q01), "q99": list(q99), "mask": list(mask)})
    ns = {"self": self_, "generated_results": generated_results, "calculate_values": False, "np": np, "torch": torch,
          "compute_logprobs_from_logits": utils.compute_logprobs_from_logits, "forward_inputs": {}}
    exec(post, ns)
    raw = torch.stack(generated_results.logits, 1)          # [B, 7, V] fp32
    scores = torch.stack(generated_results.scores, 1)
    hidden = ns["last_hidden_states"]
    assert hidden.dtype == torch.bfloat16 and hidden.shape == (B, ADIM, HID)
    # the stored hidden rows are the LM head's inputs: lm_head(hidden) is the raw logits
    assert torch.equal(model.lm_head(hidden).float(), raw)
    outside = torch.cat([scores[..., :LO], scores[..., HI:]], -1)
    return {"hidden": hidden.float().numpy(), "logits": raw[..., LO:HI].numpy(), "scores": scores[..., LO:HI].numpy(),
            "outside_inf": np.array(bool(torch.isneginf(outside).all())),
            "tokens": ns["action_tokens"].numpy(), "logprob": ns["chunk_logprobs"].float().numpy(),
            "actions": np.asarray(ns["actions"], dtype=np.float64)}


def main():
    import ref_loader

    ref = ref_loader.load_reference()
    proc_code, post = extract(os.path.join(ref_loader.REFERENCE_ROOT, FILE))
    pns = {}
    exec(proc_code, {"LogitsProcessor": __import__("transformers").LogitsProcessor, "torch": torch}, pns)
    proc_cls = pns["VLALogitsProcessor"]
    centers, q01, q99, mask = bins()
    out = {"bin_centers": centers, "q01": q01, "q99": q99, "mask": mask}
    for tie in (False, True):
        model = make_model(tie)
        out[("tie_" if tie else "") + "w_window"] = model.lm_head.weight[LO:HI].detach().float().numpy()
        runs = [(False, 1.0, 0)] + ([(True, T, k) for T, k in SAMPLE_CASES] if not tie else [(True, 1.0, 50)])
        for i, (do_sample, T, k) in enumerate(runs):
            n = case_name(do_sample, T, k, tie)
            r = run(model, proc_cls, post, ref.utils, do_sample, T, k, 500 + 10 * tie + i)
            for key, val in r.items():
                out[f"{n}_{key}"] = val
            kept = np.isfinite(r["scores"]).sum(-1)
            print(n, "kept per row", kept.min(), kept.max(), "outside -inf", bool(r["outside_inf"]))
    path = os.path.join(HERE, "golden_openvla_decode.npz")
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
