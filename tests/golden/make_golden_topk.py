"""Top-k filtered action-head fixture: the reference's own training forward on the CPU:
    python tests/golden/make_golden_topk.py  ->  tests/golden/golden_topk.npz

The `if compute_logprobs:` block of `default_forward` is extracted with `ast` from both unmodified model files
(models/embodiment/openvla_oft/rlinf/openvla_oft_action_model.py and models/embodiment/openvla/openvla_action_model.py)
and executed in place with a stub `self` (action_dim, num_action_chunks, vocab_size, config.n_action_bins), synthetic
`outputs.logits` [B, S, V] fp32, the installed transformers' TopKLogitsWarper and the reference's
compute_logprobs_from_logits / compute_entropy_from_logits.  Both files must give the same bits; only numerical
outputs are stored.

Shape: V = 320 with vocab_size 300 and 256 bins (window [44, 300)), action_dim 7, num_action_chunks 1 and 2, and
(T, k) in (1.0, 50), (1.6, 8), (1.0, 1), (1.0, 1000 >= V).  Logits lie on a 1/64 grid, so every gap between two
values is far above one ulp and dividing by T creates no new tie.  Planted rows per batch item: one whose top-k set
misses the window, one whose target is filtered, one with an exact tie at the k-th value of each k, and the rest
biased toward the window.

Stored per logits set c{C}: logits [B, S, V] and target [B, 7 C]; per case c{C}_T{T}_k{k}: logprob, entropy, the
log-prob-only gradient (upstream g_lp) and the combined gradient (g_lp and g_h) over the [:, -7C-1:-1] slice.  The
reference's entropy gradient is NaN wherever a column is masked (autograd through -inf * 0), so the combined gradient
is stored as the reference gives it."""
from __future__ import annotations

import ast
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import ref_loader  # noqa: E402

V, VOCAB, BINS, ADIM = 320, 300, 256, 7
LO, HI = VOCAB - BINS, VOCAB
B = 2
CHUNKS = (1, 2)
CASES = ((1.0, 50), (1.6, 8), (1.0, 1), (1.0, 1000))
TIE_KS = (50, 8, 1)
FILES = ("rlinf/models/embodiment/openvla_oft/rlinf/openvla_oft_action_model.py",
         "rlinf/models/embodiment/openvla/openvla_action_model.py")


def case_name(C, T, k):
    return f"c{C}_T{T:g}_k{k}"


def logprob_block(path):
    """The body of `if compute_logprobs:` in default_forward, compiled."""
    tree = ast.parse(open(path).read())
    fn = next(n for n in ast.walk(tree) if isinstance(n, ast.FunctionDef) and n.name == "default_forward")
    node = next(n for n in ast.walk(fn) if isinstance(n, ast.If) and isinstance(n.test, ast.Name)
                and n.test.id == "compute_logprobs")
    mod = ast.Module(body=node.body, type_ignores=[])
    ast.fix_missing_locations(mod)
    return compile(mod, path, "exec")


def make_logits(C, seed):
    """[B, S, V] on a 1/64 grid and [B, 7 C] targets, with the planted rows in the [:, -7C-1:-1] slice."""
    g = torch.Generator().manual_seed(seed)
    S = ADIM * C + 3
    R = ADIM * C
    x = torch.round(torch.randn(B, S, V, generator=g, dtype=torch.float64) * 3.0 * 64) / 64
    x[:, :, LO:HI] += 2.0  # rows biased toward the window
    tgt = torch.randint(LO, HI, (B, R), generator=g)
    p0 = S - R - 1
    for b in range(B):
        # row 0: the top-k set misses the window (64 large columns outside it, k <= 50 of them are the top)
        r = p0
        x[b, r, :LO] = 20.0 + torch.arange(LO, dtype=torch.float64) / 8
        x[b, r, HI:] = 20.0 + torch.arange(V - HI, dtype=torch.float64) / 8
        # row 1: the target column is far below the rest (filtered for every k < V)
        x[b, p0 + 1, int(tgt[b, 1])] = -20.0
        # rows 2..4: an exact tie at the k-th value of k = 50, 8, 1 inside the window, the target on one of the ties
        for j, k in enumerate(TIE_KS):
            r = p0 + 2 + j
            cols = LO + 3 + torch.randperm(HI - LO - 3, generator=g)[:k + 1]
            x[b, r] = torch.clamp(x[b, r], max=5.0)
            x[b, r, cols[:k - 1]] = 12.0 + torch.arange(k - 1, dtype=torch.float64) / 4
            x[b, r, cols[k - 1:k + 1]] = 9.0
            tgt[b, 2 + j] = int(cols[k])
    return x.to(torch.float32), tgt


def run_reference(code, utils, logits, target, C, T, k, g_lp, g_h):
    x = logits.clone().requires_grad_(True)
    self_ = types.SimpleNamespace(action_dim=ADIM, num_action_chunks=C, vocab_size=VOCAB,
                                  config=types.SimpleNamespace(n_action_bins=BINS))
    from transformers.generation import TopKLogitsWarper

    ns = {"self": self_, "outputs": types.SimpleNamespace(logits=x), "kwargs": {"temperature": T, "top_k": k},
          "action_tokens": target, "compute_entropy": True, "torch": torch, "TopKLogitsWarper": TopKLogitsWarper,
          "compute_logprobs_from_logits": utils.compute_logprobs_from_logits,
          "compute_entropy_from_logits": utils.compute_entropy_from_logits}
    exec(code, ns)
    lp, ent = ns["logprobs"], ns["entropy"]
    (d_lp,) = torch.autograd.grad(lp, x, grad_outputs=g_lp, retain_graph=True)
    (d_all,) = torch.autograd.grad((lp, ent), x, grad_outputs=(g_lp, g_h))
    R = ADIM * C
    sl = slice(x.shape[1] - R - 1, x.shape[1] - 1)
    return lp.detach(), ent.detach(), d_lp[:, sl], d_all[:, sl]


def main():
    ref = ref_loader.load_reference()
    codes = [logprob_block(os.path.join(ref_loader.REFERENCE_ROOT, f)) for f in FILES]
    out = {}
    for C in CHUNKS:
        logits, tgt = make_logits(C, 100 + C)
        out[f"c{C}_logits"] = logits.numpy()
        out[f"c{C}_target"] = tgt.numpy()
        g = torch.Generator().manual_seed(200 + C)
        g_lp = torch.randn(tgt.shape, generator=g)
        g_h = torch.randn(tgt.shape, generator=g)
        out[f"c{C}_g_lp"] = g_lp.numpy()
        out[f"c{C}_g_h"] = g_h.numpy()
        for T, k in CASES:
            res = [run_reference(code, ref.utils, logits, tgt, C, T, k, g_lp, g_h) for code in codes]
            for a, b in zip(res[0], res[1]):
                assert torch.equal(a.nan_to_num(1e30), b.nan_to_num(1e30)), "the two model files disagree"
            lp, ent, d_lp, d_all = res[0]
            n = case_name(C, T, k)
            out[f"{n}_logprob"] = lp.numpy()
            out[f"{n}_entropy"] = ent.numpy()
            out[f"{n}_grad_lp"] = d_lp.numpy()
            out[f"{n}_grad_all"] = d_all.numpy()
            print(n, "nan rows", int(torch.isnan(lp).sum()), "-inf", int(torch.isneginf(lp).sum()))
    path = os.path.join(HERE, "golden_topk.npz")
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
