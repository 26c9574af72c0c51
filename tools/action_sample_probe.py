"""Times the OpenVLA-OFT rollout's action-token step on the device against its eager PyTorch restatement.

  - logits level: ops.sample_action_tokens (csrc/action_sample.cu) on bf16 [bsz, 56, 32064] in-place slices,
    bsz in {64, 256}, greedy and sample with top_k in {0, 50}, against predict_action_batch :350-410 in eager PyTorch
    (the window writes, / T, the top-k threshold, log_softmax, exp, multinomial or argmax, the `.cpu()` numpy
    de-tokenisation, and compute_logprobs_from_logits on the masked logits);
  - fused: ops.linear_sample_action_tokens (csrc/lmhead_sample.cu) at bsz 256, H = 4096, against the full-vocabulary
    hidden @ W.T followed by the same chain.

    python tools/action_sample_probe.py [--reps 5] [--iters 20]

Each time is the median over --reps of CUDA-event timings of --iters calls after warm-up; the variants alternate within
every rep.  Prints one JSON line with the card name and power limit read in the same run.  Needs a CUDA device."""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys

import numpy as np
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from rlinf_b200 import ops  # noqa: E402
from tools.lmhead_probe import card, timed  # noqa: E402

V, VOCAB, NBINS, ADIM, POS = 32064, 32000, 256, 7, 56
WINDOW = (VOCAB - NBINS, VOCAB)


def stats_tables():
    edges = np.linspace(-1, 1, NBINS)
    centers = (edges[:-1] + edges[1:]) / 2.0
    low, high = np.linspace(-1.0, -0.1, ADIM), np.linspace(0.2, 1.1, ADIM)
    mask = np.ones(ADIM, dtype=bool)
    mask[-1] = False
    return centers, low, high, mask


def eager_chain(logits, do_sample, T, k, tables):
    """predict_action_batch :350-410 in eager PyTorch and numpy, as the reference runs it."""
    centers, low, high, mask = tables
    logits[..., :VOCAB - NBINS] = -torch.inf
    logits[..., VOCAB:] = -torch.inf
    if do_sample:
        z = logits / T
        if k > 0:
            thr = torch.topk(z, min(k, z.size(-1)), dim=-1).values[..., -1, None]
            z = z.masked_fill(z < thr, -torch.inf)
        probs = F.log_softmax(z, dim=-1).exp()
        idx = torch.multinomial(probs.view(-1, V), num_samples=1, replacement=True).view(z.shape[:2])
    else:
        z = logits
        idx = z.argmax(dim=-1)
    tok = idx.reshape(-1, ADIM).cpu().numpy()
    d = np.clip(VOCAB - tok - 1, a_min=0, a_max=centers.shape[0] - 1)
    n = np.asarray([centers[da] for da in d]).reshape(-1, ADIM)
    actions = np.where(mask, 0.5 * (n + 1) * (high - low + 1e-8) + low, n).reshape(idx.shape)
    z[..., :VOCAB - NBINS] = -torch.inf
    z[..., VOCAB:] = -torch.inf
    lp = -F.cross_entropy(z.reshape(-1, V).float(), idx.reshape(-1), reduction="none")
    return idx, lp, actions


def logits_case(bsz, do_sample, k, bins, tables, args):
    g = torch.Generator(device="cuda").manual_seed(bsz + k)
    full = (torch.randn(bsz, POS + 2, V, generator=g, device="cuda") * 2.0).to(torch.bfloat16)
    x = full[:, 1:-1]
    step = [0]

    def device():
        step[0] += 1
        ops.sample_action_tokens(x, WINDOW, do_sample=do_sample, top_k=k, seed=0, offset=step[0], bins=bins)

    def eager():
        eager_chain(x, do_sample, 1.0, k, tables)

    return compare(device, eager, args, read=bsz * POS * NBINS * 2, written=20 * bsz * POS)


def fused_case(bsz, do_sample, k, bins, tables, args, H=4096):
    g = torch.Generator(device="cuda").manual_seed(7)
    hidden = torch.randn(bsz, POS, H, generator=g, device="cuda").to(torch.bfloat16)
    w = (torch.randn(V, H, generator=g, device="cuda") * H ** -0.5).to(torch.bfloat16)
    step = [0]

    def device():
        step[0] += 1
        ops.linear_sample_action_tokens(hidden, w, WINDOW, do_sample=do_sample, top_k=k, seed=0, offset=step[0],
                                        bins=bins)

    def eager():
        eager_chain(hidden @ w.T, do_sample, 1.0, k, tables)

    return compare(device, eager, args, read=bsz * POS * H * 2 + NBINS * H * 2, written=20 * bsz * POS)


def compare(device, eager, args, read, written):
    fns = {"device": device, "eager": eager}
    for f in fns.values():
        f()
        f()
    times = {n: [] for n in fns}
    for _ in range(args.reps):
        for n, f in fns.items():
            times[n].append(timed(f, args.iters))
    med = {n: statistics.median(v) for n, v in times.items()}
    return {"ms": {n: round(v, 4) for n, v in med.items()},
            "rel_spread": {n: round((max(v) - min(v)) / statistics.median(v), 3) for n, v in times.items()},
            "device_over_eager": round(med["device"] / med["eager"], 4),
            "device_gbps": round((read + written) / med["device"] / 1e6, 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("action_sample_probe: needs a CUDA device")
    name, plim = card()
    tables = stats_tables()
    bins = ops.ActionBins(VOCAB, *tables)
    res = {"card": name, "power_limit": plim, "V": V, "window": list(WINDOW), "positions": POS, "logits_bf16": {}}
    for bsz in (64, 256):
        for mode, do_sample, k in (("greedy", False, 0), ("sample_k0", True, 0), ("sample_k50", True, 50)):
            res["logits_bf16"][f"bsz{bsz}_{mode}"] = logits_case(bsz, do_sample, k, bins, tables, args)
    res["fused_h4096_bsz256"] = {mode: fused_case(256, do_sample, k, bins, tables, args)
                                 for mode, do_sample, k in (("greedy", False, 0), ("sample_k50", True, 50))}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
