"""Times the OpenVLA value head (ops.vla_value_head, csrc/vla_value_head.cu) against the eager bf16 chain.

    python tools/vla_value_head_probe.py [--reps 5] [--iters 50] [--out FILE]

Shapes: H = 4096, O in {1, 8, 25} (chunk_level, and action_level at C = 8 and 25), N in {40, 128, 1024, 4096}.  The
eager chain is an nn.Sequential of the same layers in bf16 (Linear, GELU, Linear, GELU, Linear without bias) with the
same parameters and inputs.  For each shape and each of forward (under no_grad) and forward + backward:
  - call time: the median over --reps of CUDA-event timings of --iters back-to-back calls after warm-up, the new op
    and the eager chain alternating within every rep (host launch cost included: it is what a caller waits for);
  - kernel time and launch count: the sum of the kernels' durations and their number in one torch.profiler pass;
  - bytes and FLOPs from the shapes (below), and the share of the larger of the HBM bound (3.35 TB/s) and the dense
    bf16 tensor-core bound (989 TFLOP/s) of the H100 SXM data sheet, over the kernel time.
Prints one JSON line with the card name and power limit read in the same run.  Needs a CUDA device."""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from rlinf_b200 import ops  # noqa: E402
from tools.lmhead_probe import card, timed  # noqa: E402

H = 4096
OS = (1, 8, 25)
NS = (40, 128, 1024, 4096)
HBM, TC = 3.35e12, 989e12


def model(N, O):
    """(bytes, flops) of forward and of forward + backward: every weight and row read once per pass, every output and
    gradient written once; the saved pre-activations (1280 B a row) written by the forward and read by the backward."""
    w = 2 * (512 * H + 512 + 128 * 512 + 128 + O * 128)
    rows = 2 * N * H
    f_flops = 2 * N * (512 * H + 128 * 512 + O * 128)
    f_bytes = w + rows + 2 * N * O
    fb_bytes = f_bytes + 1280 * N * 2 + w + rows + 2 * N * O + rows + w  # + backward: weights, rows, gv, dX, grads
    return (f_bytes, f_flops), (fb_bytes, 3 * f_flops)


def make(N, O):
    g = torch.Generator().manual_seed(N * 100 + O)

    def r(*shape, std=1.0):
        return (torch.randn(*shape, generator=g) * std).to(torch.bfloat16).cuda()

    params = [r(512, H, std=(2 / 512) ** 0.5), r(512, std=0.1), r(128, 512, std=(2 / 128) ** 0.5), r(128, std=0.1),
              r(O, 128, std=0.02)]
    return r(N, H), params, r(N, O)


def kernel_time(fn):
    from torch.profiler import ProfilerActivity, profile

    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    ev = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    return sum(e.device_time for e in ev) / 1e3, len(ev)  # ms, launches


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("vla_value_head_probe needs a CUDA device")
    name, plim = card()
    rows = []
    for O in OS:
        for N in NS:
            x, params, gv = make(N, O)
            xs = x.clone().requires_grad_(True)
            ps = [p.clone().requires_grad_(True) for p in params]
            seq = torch.nn.Sequential(torch.nn.Linear(H, 512), torch.nn.GELU(), torch.nn.Linear(512, 128),
                                      torch.nn.GELU(), torch.nn.Linear(128, O, bias=False)).cuda().to(torch.bfloat16)
            with torch.no_grad():
                for p, q in zip(seq.parameters(), params):
                    p.copy_(q)
            xe = x.clone().requires_grad_(True)

            def op_f():
                with torch.no_grad():
                    ops.vla_value_head(x, *params)

            def op_fb():
                v = ops.vla_value_head(xs, *ps)
                torch.autograd.grad(v, [xs] + ps, gv)

            def eg_f():
                with torch.no_grad():
                    seq(x)

            def eg_fb():
                v = seq(xe)
                torch.autograd.grad(v, [xe] + list(seq.parameters()), gv)

            fns = {"op_fwd": op_f, "eager_fwd": eg_f, "op_fwd_bwd": op_fb, "eager_fwd_bwd": eg_fb}
            for fn in fns.values():
                for _ in range(3):
                    fn()
            torch.cuda.synchronize()
            times = {k: [] for k in fns}
            for _ in range(a.reps):
                for k, fn in fns.items():
                    times[k].append(timed(fn, a.iters))
            (fb_, ff_), (bb_, bf_) = model(N, O)
            row = {"O": O, "N": N}
            for k, fn in fns.items():
                kt, nl = kernel_time(fn)
                by, fl = (fb_, ff_) if k.endswith("_fwd") else (bb_, bf_)
                bound = max(by / HBM, fl / TC)
                row[k] = {"call_us": round(statistics.median(times[k]) * 1e3, 2), "kernel_us": round(kt * 1e3, 2),
                          "launches": nl, "bytes": by, "flops": fl,
                          "bound": "hbm" if by / HBM >= fl / TC else "tensor",
                          "share_of_bound": round(bound / (kt * 1e-3), 4) if kt > 0 else None}
            row["fwd_call_ratio"] = round(row["op_fwd"]["call_us"] / row["eager_fwd"]["call_us"], 3)
            row["fwd_bwd_call_ratio"] = round(row["op_fwd_bwd"]["call_us"] / row["eager_fwd_bwd"]["call_us"], 3)
            rows.append(row)
            print(f"O={O:2d} N={N:5d}  fwd {row['op_fwd']['call_us']:8.1f} us ({row['op_fwd']['kernel_us']:7.1f} kernel,"
                  f" {row['op_fwd']['launches']} launches) vs eager {row['eager_fwd']['call_us']:8.1f} "
                  f"({row['eager_fwd']['kernel_us']:7.1f}, {row['eager_fwd']['launches']})   fwd+bwd "
                  f"{row['op_fwd_bwd']['call_us']:8.1f} ({row['op_fwd_bwd']['kernel_us']:7.1f}, "
                  f"{row['op_fwd_bwd']['launches']}) vs eager {row['eager_fwd_bwd']['call_us']:8.1f} "
                  f"({row['eager_fwd_bwd']['kernel_us']:7.1f}, {row['eager_fwd_bwd']['launches']})", flush=True)
    res = {"probe": "vla_value_head", "card": name, "power_limit": plim, "H": H, "reps": a.reps, "iters": a.iters,
           "rows": rows}
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
