"""OpenVLA-OFT rollout action-token fixture: the reference's own sampling step on the CPU:
    python tests/golden/make_golden_action_sample.py  ->  tests/golden/golden_action_sample.npz

The statements of `OpenVLAOFTForRLActionPrediction.predict_action_batch` from the action-bin window mask
(`logits_tensor[..., : self.vocab_size - ...] = -torch.inf`) through `chunk_logprobs = ...`, and the whole
`_unnormalize_actions`, are extracted with `ast` from the unmodified model file
(models/embodiment/openvla_oft/rlinf/openvla_oft_action_model.py) and executed in place with a stub `self` (vocab_size,
config.n_action_bins, action_dim, bin_centers, unnorm_key, get_action_stats), synthetic `logits_tensor` [B, 7 C, V]
fp32, the installed transformers' TopKLogitsWarper and the reference's compute_logprobs_from_logits.  Only numerical
outputs are stored.

Shape: V = 320 with vocab_size 300 and 256 bins (window [44, 300), 255 bin centres), action_dim 7, num_action_chunks 1
and 2.  Logits lie on a 1/64 grid, so dividing by T creates no new tie.  Planted rows per batch item (positions 0..6):
0 the row's maximum outside the window, 1 an exact tie at the argmax, 2..4 an exact tie at the k-th value of
k = 50, 8, 1, 5 / 6 a dominant column at the window's first / last column (the bin clip).  The q01 / q99 statistics
have mask = False at dimension 3.

Stored: per c{C}: logits [B, 7 C, V]; the bins (bin_centers, q01, q99, mask).  Greedy (c{C}_greedy_*): tokens,
log-probs, actions.  Sample mode per (T, k) (c{C}_T{T}_k{k}_*): the reference's processed_logprob_tensor over the window
[B, 7 C, 256] (`table`) and its own multinomial draws with their log-probs and actions."""
from __future__ import annotations

import ast
import os
import sys
import types

import numpy as np
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

V, VOCAB, NBINS, ADIM = 320, 300, 256, 7
LO, HI = VOCAB - NBINS, VOCAB
B = 3
CHUNKS = (1, 2)
CASES = ((1.0, 0), (1.6, 0), (1.0, 50), (0.6, 8), (1.0, 1), (1.0, 300))
TIE_KS = (50, 8, 1)
MASK_OFF = 3
FILE = "rlinf/models/embodiment/openvla_oft/rlinf/openvla_oft_action_model.py"


def case_name(C, T, k):
    return f"c{C}_T{T:g}_k{k}"


def bins():
    edges = np.linspace(-1, 1, NBINS)
    centers = (edges[:-1] + edges[1:]) / 2.0
    rng = np.random.default_rng(7)
    q01 = rng.uniform(-2.0, -0.1, ADIM)
    q99 = q01 + rng.uniform(0.2, 3.0, ADIM)
    mask = np.ones(ADIM, dtype=bool)
    mask[MASK_OFF] = False
    return centers, q01, q99, mask


def extract(path):
    """(the sampling statements of predict_action_batch, the _unnormalize_actions function), compiled."""
    src = open(path).read()
    tree = ast.parse(src)
    cls = next(n for n in ast.walk(tree) if isinstance(n, ast.ClassDef) and n.name == "OpenVLAOFTForRLActionPrediction")
    fns = {n.name: n for n in cls.body if isinstance(n, ast.FunctionDef)}
    body = fns["predict_action_batch"].body
    i0 = next(i for i, s in enumerate(body) if isinstance(s, ast.Assign) and "n_action_bins" in ast.unparse(s)
              and ast.unparse(s.targets[0]).startswith("logits_tensor["))
    i1 = next(i for i, s in enumerate(body) if isinstance(s, ast.Assign) and ast.unparse(s.targets[0]) == "chunk_logprobs")
    step = ast.Module(body=body[i0:i1 + 1], type_ignores=[])
    unnorm = fns["_unnormalize_actions"]
    unnorm.decorator_list = []
    mod_u = ast.Module(body=[unnorm], type_ignores=[])
    for m in (step, mod_u):
        ast.fix_missing_locations(m)
    return compile(step, path, "exec"), compile(mod_u, path, "exec")


def make_logits(C, seed):
    """[B, 7 C, V] on a 1/64 grid with the planted rows at positions 0..6 of each batch item."""
    g = torch.Generator().manual_seed(seed)
    R = ADIM * C
    x = torch.round(torch.randn(B, R, V, generator=g, dtype=torch.float64) * 2.0 * 64) / 64
    for b in range(B):
        x[b, 0, :LO] = 30.0 + torch.arange(LO, dtype=torch.float64) / 8   # the maximum lies outside the window
        x[b, 0, HI:] = 40.0
        cols = LO + torch.randperm(HI - LO, generator=g)[:2]
        x[b, 1, LO:HI] = torch.clamp(x[b, 1, LO:HI], max=4.0)
        x[b, 1, cols] = 6.0                                               # a tie at the argmax
        for j, k in enumerate(TIE_KS):                                    # a tie at the k-th value
            r = 2 + j
            cols = LO + torch.randperm(HI - LO, generator=g)[:k + 1]
            x[b, r, LO:HI] = torch.clamp(x[b, r, LO:HI], max=3.0)
            x[b, r, cols[:k - 1]] = 8.0 + torch.arange(k - 1, dtype=torch.float64) / 16
            x[b, r, cols[k - 1:k + 1]] = 6.0
        x[b, 5, LO] = 12.0                                                # window edges: the bin clip
        x[b, 6, HI - 1] = 12.0
    return x.to(torch.float32)


def run_reference(step, unnorm, utils, logits, C, do_sample, T, k, seed):
    from transformers.generation import TopKLogitsWarper

    centers, q01, q99, mask = bins()
    norm = types.SimpleNamespace(BOUNDS="bounds", BOUNDS_Q99="bounds_q99")
    uns = {"np": np, "NormalizationType": norm, "ACTION_PROPRIO_NORMALIZATION_TYPE": norm.BOUNDS_Q99}
    exec(unnorm, uns)
    self_ = types.SimpleNamespace(vocab_size=VOCAB, config=types.SimpleNamespace(n_action_bins=NBINS),
                                  action_dim=ADIM, num_action_chunks=C, bin_centers=centers, unnorm_key="fixture",
                                  get_action_stats=lambda key: {"q01": list(q01), "q99": list(q99), "mask": mask})
    self_._unnormalize_actions = types.MethodType(uns["_unnormalize_actions"], self_)
    ns = {"self": self_, "logits_tensor": logits.clone(), "do_sample": do_sample,
          "kwargs": {"temperature": T, "top_k": k, "top_p": 1.0}, "torch": torch, "F": F, "np": np,
          "TopKLogitsWarper": TopKLogitsWarper, "compute_logprobs_from_logits": utils.compute_logprobs_from_logits}
    torch.manual_seed(seed)
    exec(step, ns)
    out = {"tokens": ns["idxs"].numpy(), "logprob": ns["chunk_logprobs"].numpy(), "actions": ns["actions"]}
    if do_sample:
        out["table"] = ns["processed_logprob_tensor"][..., LO:HI].numpy()
    return out


def main():
    import ref_loader

    ref = ref_loader.load_reference()
    step, unnorm = extract(os.path.join(ref_loader.REFERENCE_ROOT, FILE))
    centers, q01, q99, mask = bins()
    out = {"bin_centers": centers, "q01": q01, "q99": q99, "mask": mask}
    for C in CHUNKS:
        logits = make_logits(C, 300 + C)
        out[f"c{C}_logits"] = logits.numpy()
        g = run_reference(step, unnorm, ref.utils, logits, C, False, 1.0, 0, 0)
        for key in ("tokens", "logprob", "actions"):
            out[f"c{C}_greedy_{key}"] = g[key]
        for i, (T, k) in enumerate(CASES):
            s = run_reference(step, unnorm, ref.utils, logits, C, True, T, k, 1000 * C + i)
            n = case_name(C, T, k)
            for key in ("tokens", "logprob", "actions", "table"):
                out[f"{n}_{key}"] = s[key]
            print(n, "kept per row", np.isfinite(s["table"]).sum(-1).min(), np.isfinite(s["table"]).sum(-1).max())
    path = os.path.join(HERE, "golden_action_sample.npz")
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
