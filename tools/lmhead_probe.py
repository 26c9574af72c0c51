"""Times the fused LM-head log-prob / entropy kernels (ops.linear_logprobs_entropy) against the GEMM alone and the
materialised path (X @ W.T, then ops.logprobs_entropy_from_logits), forward and forward + backward, and their peak
memory.  Prints one JSON line with the card name and power limit read in the same run.

    python tools/lmhead_probe.py [--reps 5] [--iters 20]

Each time is the median over --reps of CUDA-event timings of --iters launches after warm-up; the variants alternate
within every rep.  TFLOP/s use 2 N V H (forward) and 6 N V H (forward + backward) over the window's columns and are
compared with the data-sheet 989 TFLOP/s dense bf16 of the H100 SXM."""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from rlinf_b200 import ops  # noqa: E402

DATASHEET_BF16_TFLOPS = 989.0
SHAPES = [  # (name, N, H, V, window)
    ("qwen2.5-1.5b", 16384, 1536, 151936, None),
    ("qwen2.5-7b", 16384, 3584, 152064, None),
    ("openvla-256bins", 8192, 4096, 32064, (32000 - 256, 32000)),
]


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i",
                              str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout
        name, plim = (s.strip() for s in out.strip().split(","))
        return name, plim
    except Exception:  # noqa: BLE001
        return torch.cuda.get_device_name(), "unknown"


def timed(fn, iters):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / iters


def peak_of(fn):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    fn()
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() - base


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    name, plim = card()
    res = {"card": name, "power_limit": plim, "datasheet_bf16_tflops": DATASHEET_BF16_TFLOPS, "shapes": {}}
    for tag, N, H, V, window in SHAPES:
        g = torch.Generator(device="cuda").manual_seed(0)
        x = torch.randn(N, H, generator=g, device="cuda").to(torch.bfloat16)
        w = (torch.randn(V, H, generator=g, device="cuda") * H ** -0.5).to(torch.bfloat16)
        lo, hi = window or (0, V)
        tgt = torch.randint(lo, hi, (N,), generator=g, device="cuda")
        xg, wg = x.clone().requires_grad_(True), w.clone().requires_grad_(True)

        def gemm():
            torch.matmul(x, w.T)

        def fused_fwd():
            ops.linear_logprobs_entropy(x, w, tgt, window=window)

        def mat_fwd():
            ops.logprobs_entropy_from_logits(torch.matmul(x, w.T), tgt, window=window)

        def fused_fb():
            xg.grad = wg.grad = None
            lp, ent = ops.linear_logprobs_entropy(xg, wg, tgt, window=window)
            (lp.sum() + ent.sum()).backward()

        def mat_fb():
            xg.grad = wg.grad = None
            lp, ent = ops.logprobs_entropy_from_logits(torch.matmul(xg, wg.T), tgt, window=window)
            (lp.sum() + ent.sum()).backward()

        fns = {"gemm_only_fwd": gemm, "fused_fwd": fused_fwd, "materialised_fwd": mat_fwd, "fused_fwd_bwd": fused_fb,
               "materialised_fwd_bwd": mat_fb}
        for f in fns.values():  # warm-up
            f()
            f()
        times = {k: [] for k in fns}
        for _ in range(args.reps):
            for k, f in fns.items():
                times[k].append(timed(f, args.iters))
        med = {k: statistics.median(v) for k, v in times.items()}
        W = hi - lo
        fl = 2.0 * N * W * H
        r = {"N": N, "H": H, "V": V, "window": [lo, hi], "ms": {k: round(v, 4) for k, v in med.items()},
             "fused_fwd_tflops": round(fl / med["fused_fwd"] / 1e9, 1),
             "fused_fwd_bwd_tflops": round(3 * fl / med["fused_fwd_bwd"] / 1e9, 1),
             "gemm_only_tflops": round(2.0 * N * V * H / med["gemm_only_fwd"] / 1e9, 1),
             "fused_fwd_over_gemm": round(med["fused_fwd"] / med["gemm_only_fwd"], 3),
             "fused_fwd_over_materialised_fwd": round(med["fused_fwd"] / med["materialised_fwd"], 3),
             "fused_fwd_bwd_over_materialised": round(med["fused_fwd_bwd"] / med["materialised_fwd_bwd"], 3),
             "peak_bytes": {"fused_fwd_bwd": peak_of(fused_fb), "materialised_fwd_bwd": peak_of(mat_fb)}}
        res["shapes"][tag] = r
        del x, w, xg, wg
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
