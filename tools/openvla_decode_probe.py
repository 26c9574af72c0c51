"""Times a 7-step plain OpenVLA action decode on the device against the reference's eager generate chain.

  - ours: ops.linear_sample_action_tokens per step (csrc/lmhead_sample.cu over the 256 window rows, the sampler, the
    counter advance) writing column j of [B, 7] buffers, eager and captured in one CUDA graph;
  - reference: per step the full hidden @ W.T [B, 32064], VLALogitsProcessor (clone, -inf outside [31744, 32000)),
    / T, TopKLogitsWarper(50), softmax and multinomial, every step's scores kept; at the end stack, the window fill,
    log_softmax, gather and the `.cpu()` numpy de-tokenisation (openvla_action_model.py:453-471,610-756).
The backbone is excluded on both sides: every step's hidden rows are made beforehand.

    python tools/openvla_decode_probe.py [--reps 5] [--iters 20]

Times are medians over --reps of CUDA-event timings of --iters decodes after warm-up, the variants alternating within
every rep.  Device time and launch count come from one separate torch.profiler pass per variant, host syncs from
torch.cuda.set_sync_debug_mode("warn").  Prints one JSON line with the card name and power limit read in the same run.
Needs a CUDA device."""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import warnings

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from rlinf_b200 import ops  # noqa: E402
from tools.lmhead_probe import card, timed  # noqa: E402

V, VOCAB, NBINS, A, H, K, T = 32064, 32000, 256, 7, 4096, 50, 1.0
WINDOW = (VOCAB - NBINS, VOCAB)


def tables():
    edges = np.linspace(-1, 1, NBINS)
    mask = np.ones(A, dtype=bool)
    mask[-1] = False
    return (edges[:-1] + edges[1:]) / 2.0, np.linspace(-1.0, -0.1, A), np.linspace(0.2, 1.1, A), mask


def reference(hs, w, tab):
    centers, low, high, mask = tab
    scores = []
    toks = []
    for j in range(A):
        logits = (hs[j] @ w.T).float()
        s = logits.clone()                                   # VLALogitsProcessor
        s[:, :VOCAB - NBINS] = -torch.inf
        s[:, VOCAB:] = -torch.inf
        s = s / T                                            # TemperatureLogitsWarper
        thr = torch.topk(s, K)[0][..., -1, None]             # TopKLogitsWarper
        s = s.masked_fill(s < thr, -torch.inf)
        tok = torch.multinomial(torch.softmax(s, -1), num_samples=1)[:, 0]
        scores.append(s)
        toks.append(tok)
    tokens = torch.stack(toks, 1)
    z = torch.stack(scores, 1)
    z[..., :VOCAB - NBINS] = -torch.inf
    z[..., VOCAB:] = -torch.inf
    lp = torch.log_softmax(z, -1).gather(-1, tokens[..., None])[..., 0]
    t = tokens.cpu().numpy()
    d = np.clip(VOCAB - t - 1, a_min=0, a_max=centers.shape[0] - 1)
    n = np.asarray([centers[da] for da in d])
    actions = np.where(mask, 0.5 * (n + 1) * (high - low + 1e-8) + low, n)
    return tokens, lp, actions


def profile(fn):
    """(device microseconds, device ops) of one call, from torch.profiler."""
    from torch.profiler import ProfilerActivity, profile as prof

    torch.cuda.synchronize()
    with prof(activities=[ProfilerActivity.CUDA]) as p:
        fn()
        torch.cuda.synchronize()
    ev = [e for e in p.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    return round(sum(e.device_time_total for e in ev), 1), len(ev)


def host_syncs(fn):
    torch.cuda.synchronize()
    with warnings.catch_warnings(record=True) as rec:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            fn()
        finally:
            torch.cuda.set_sync_debug_mode("default")
    # torch warns once per process that the mode is a prototype; that warning is not a sync
    return sum("synchroniz" in str(r.message) and "prototype" not in str(r.message) for r in rec)


def case(B, bins, tab, args):
    g = torch.Generator(device="cuda").manual_seed(B)
    hs = torch.randn(A, B, H, generator=g, device="cuda").to(torch.bfloat16)
    w = (torch.randn(V, H, generator=g, device="cuda") * H ** -0.5).to(torch.bfloat16)
    ctr = torch.zeros(1, dtype=torch.int64, device="cuda")
    out = (torch.empty(B, A, dtype=torch.int64, device="cuda"), torch.empty(B, A, device="cuda"),
           torch.empty(B, A, dtype=torch.float64, device="cuda"))

    def ours():
        for j in range(A):
            ops.linear_sample_action_tokens(hs[j], w, WINDOW, do_sample=True, temperature=T, top_k=K, seed=0,
                                            counter=ctr, bins=bins, out=out, column=j)

    ours()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        ours()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        ours()
    fns = {"ours_eager": ours, "ours_graph": graph.replay, "reference": lambda: reference(hs, w, tab)}
    for f in fns.values():
        f()
        f()
    times = {n: [] for n in fns}
    for _ in range(args.reps):
        for n, f in fns.items():
            times[n].append(timed(f, args.iters))
    med = {n: statistics.median(v) for n, v in times.items()}
    res = {"ms": {n: round(v, 4) for n, v in med.items()},
           "rel_spread": {n: round((max(v) - min(v)) / statistics.median(v), 3) for n, v in times.items()},
           "eager_over_reference": round(med["ours_eager"] / med["reference"], 4),
           "graph_over_reference": round(med["ours_graph"] / med["reference"], 4)}
    res["host_syncs"] = {n: host_syncs(f) for n, f in fns.items()}  # before any profiler pass
    for n in ("ours_eager", "reference"):
        us, nops = profile(fns[n])
        res.setdefault("device_us", {})[n] = us
        res.setdefault("device_ops", {})[n] = nops
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("openvla_decode_probe: needs a CUDA device")
    name, plim = card()
    tab = tables()
    bins = ops.ActionBins(VOCAB, *tab)
    res = {"card": name, "power_limit": plim, "V": V, "H": H, "window": list(WINDOW), "steps": A, "top_k": K,
           "head_rows_fraction": round(NBINS / V, 5)}
    for B in (32, 128, 256):
        res[f"B{B}"] = case(B, bins, tab, args)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
