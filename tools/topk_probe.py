"""Times the top-k filtered log-prob / entropy kernels (ops.logprobs_entropy_from_logits(..., top_k=k), csrc/topk.cu)
on bf16 OpenVLA logits [8192, 32064] with the 256-bin window, against today's unfiltered full-row forward on the same
tensor and the reference's eager chain (logits / T, torch.topk threshold, masked_fill, the window writes,
cross_entropy, log_softmax entropy), forward and forward + backward; and the fused head (ops.linear_logprobs_entropy(...,
top_k=k), X [8192, 4096]) forward + backward against the materialised chain.  Prints one JSON line with the card name and power
limit read in the same run.

    python tools/topk_probe.py [--reps 5] [--iters 20]

Each time is the median over --reps of CUDA-event timings of --iters calls after warm-up; the variants alternate within
every rep.  GB/s counts one read of the logits forward, and one read plus one write of [N, V] backward."""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from rlinf_b200 import ops  # noqa: E402
from tools.lmhead_probe import card, timed  # noqa: E402

N, V, K = 8192, 32064, 50
WINDOW = (32000 - 256, 32000)


def eager_chain(x, tgt, T, k):
    """The OpenVLA heads' training forward (openvla_oft_action_model.py:537-559) in eager PyTorch."""
    z = x / T
    thr = torch.topk(z, k, dim=-1).values[..., -1, None]
    z = z.masked_fill(z < thr, -float("inf"))
    z[..., :WINDOW[0]] = -float("inf")
    z[..., WINDOW[1]:] = -float("inf")
    lp = -F.cross_entropy(z, tgt, reduction="none")
    logp = F.log_softmax(z, dim=-1)
    p = logp.exp()
    ent = -torch.where(p > 0, p * logp, 0.0).sum(-1)
    return lp, ent


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    name, plim = card()
    g = torch.Generator(device="cuda").manual_seed(0)
    x = (torch.randn(N, V, generator=g, device="cuda") * 2.5).to(torch.bfloat16)
    x[:, WINDOW[0]:WINDOW[1]] += 2.0
    tgt = torch.randint(WINDOW[0], WINDOW[1], (N,), generator=g, device="cuda")
    xg = x.clone().requires_grad_(True)
    T = 1.0

    def full_row_fwd():
        ops.logprobs_entropy_from_logits(x, tgt, T)

    def topk_fwd():
        ops.logprobs_entropy_from_logits(x, tgt, T, WINDOW, top_k=K)

    def eager_fwd():
        with torch.no_grad():
            eager_chain(x, tgt, T, K)

    def full_row_fb():
        xg.grad = None
        lp, ent = ops.logprobs_entropy_from_logits(xg, tgt, T)
        (lp.sum() + ent.sum()).backward()

    def topk_fb():
        xg.grad = None
        lp, ent = ops.logprobs_entropy_from_logits(xg, tgt, T, WINDOW, top_k=K)
        (lp.nan_to_num(0.0).sum() + ent.sum()).backward()

    def eager_fb():
        xg.grad = None
        lp, ent = eager_chain(xg, tgt, T, K)
        lp.nan_to_num(0.0).sum().backward()  # the entropy's autograd is NaN under the mask (DESIGN §2)

    fns = {"full_row_fwd": full_row_fwd, "topk_fwd": topk_fwd, "eager_fwd": eager_fwd, "full_row_fwd_bwd": full_row_fb,
           "topk_fwd_bwd": topk_fb, "eager_fwd_bwd": eager_fb}
    for f in fns.values():
        f()
        f()
    times = {k: [] for k in fns}
    for _ in range(args.reps):
        for k, f in fns.items():
            times[k].append(timed(f, args.iters))
    med = {k: statistics.median(v) for k, v in times.items()}
    spread = {k: round((max(v) - min(v)) / statistics.median(v), 3) for k, v in times.items()}
    rb = N * V * 2
    res = {"card": name, "power_limit": plim, "N": N, "V": V, "dtype": "bf16", "window": list(WINDOW), "top_k": K,
           "ms": {k: round(v, 4) for k, v in med.items()}, "rel_spread": spread,
           "topk_fwd_gbps": round(rb / med["topk_fwd"] / 1e6, 1),
           "full_row_fwd_gbps": round(rb / med["full_row_fwd"] / 1e6, 1),
           "topk_fwd_over_full_row_fwd": round(med["topk_fwd"] / med["full_row_fwd"], 3),
           "topk_fwd_over_eager_fwd": round(med["topk_fwd"] / med["eager_fwd"], 3),
           "topk_fwd_bwd_over_eager_fwd_bwd": round(med["topk_fwd_bwd"] / med["eager_fwd_bwd"], 3),
           "gate_fwd_within_2x_full_row": med["topk_fwd"] <= 2.0 * med["full_row_fwd"],
           "gate_fwd_faster_than_eager": med["topk_fwd"] < med["eager_fwd"]}
    res["fused_head"] = fused_head(args)
    print(json.dumps(res))


def fused_head(args, N=8192, H=4096):
    """ops.linear_logprobs_entropy(..., top_k=K) forward + backward against the materialised chain (bf16 X.W^T, the
    logits-level top-k op, backward through the matmul), and the forward's row-block count."""
    g = torch.Generator(device="cuda").manual_seed(1)
    x = torch.randn(N, H, generator=g, device="cuda").to(torch.bfloat16).requires_grad_(True)
    w = (torch.randn(V, H, generator=g, device="cuda") * H ** -0.5).to(torch.bfloat16).requires_grad_(True)
    tgt = torch.randint(WINDOW[0], WINDOW[1], (N,), generator=g, device="cuda")

    def fused():
        x.grad = w.grad = None
        lp, ent = ops.linear_logprobs_entropy(x, w, tgt, 1.0, WINDOW, top_k=K)
        (lp.nan_to_num(0.0, neginf=0.0).sum() + ent.sum()).backward()

    def materialised():
        x.grad = w.grad = None
        lp, ent = ops.logprobs_entropy_from_logits(x @ w.T, tgt, 1.0, WINDOW, top_k=K)
        (lp.nan_to_num(0.0, neginf=0.0).sum() + ent.sum()).backward()

    fns = {"fused_fwd_bwd": fused, "materialised_fwd_bwd": materialised}
    for f in fns.values():
        f()
        f()
    times = {k: [] for k in fns}
    for _ in range(args.reps):
        for k, f in fns.items():
            times[k].append(timed(f, max(1, args.iters // 4)))
    med = {k: statistics.median(v) for k, v in times.items()}
    tile_rows = (ops.LMHEAD_TOPK_ROW_BLOCK or (512 << 20) // (128 * (-(-V // 4) * 4) * 4) * 128)
    return {"N": N, "H": H, "V": V, "ms": {k: round(v, 3) for k, v in med.items()},
            "rel_spread": {k: round((max(v) - min(v)) / statistics.median(v), 3) for k, v in times.items()},
            "row_blocks": -(-N // min(N, tile_rows)),
            "fused_over_materialised": round(med["fused_fwd_bwd"] / med["materialised_fwd_bwd"], 3),
            "gate_fused_faster_than_materialised": med["fused_fwd_bwd"] < med["materialised_fwd_bwd"]}


if __name__ == "__main__":
    main()
