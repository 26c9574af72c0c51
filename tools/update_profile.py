"""Where the update phase spends its device time, per kernel.

    python tools/update_profile.py TRACE_DIR [--B 4096 --T 512 --obs 128 --act 8 --update-epoch 8 --minibatches 8]

Builds the bench.py workload (default: its config), runs warm-up iterations, then profiles ONE `update_phase()`
under torch.profiler (CUDA activities).  Prints one row per kernel (total ms, calls, share of the phase) and a JSON
line with the same table; the Chrome trace goes to TRACE_DIR/update_phase.pt.trace.json.  The phase time is taken
with CUDA events around the profiled phase, so it includes launch gaps and the profiler's own overhead; kernel
times come from the CUPTI activity records.  Needs a GPU.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
from collections import defaultdict

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("trace_dir")
    ap.add_argument("--B", type=int, default=4096)
    ap.add_argument("--T", type=int, default=512)
    ap.add_argument("--obs", type=int, default=128)
    ap.add_argument("--act", type=int, default=8)
    ap.add_argument("--update-epoch", type=int, default=8)
    ap.add_argument("--minibatches", type=int, default=8)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile

    from rlinf_b200.config import synthetic_ppo_config
    from rlinf_b200.runner import EmbodiedRunner

    assert torch.cuda.is_available(), "update_profile.py needs a GPU"
    torch.cuda.set_device(0)
    cfg = synthetic_ppo_config(B=a.B, T=a.T, obs_dim=a.obs, action_dim=a.act, update_epoch=a.update_epoch,
                               num_minibatches=a.minibatches)
    run = EmbodiedRunner(cfg)
    for _ in range(max(a.warmup, 3)):  # the rollout graph is captured on the 2nd iteration
        run.run_iteration()
    run.update_rollout_weights()
    run.rollout_phase()
    torch.cuda.synchronize()

    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        e0.record()
        run.update_phase()
        e1.record()
        torch.cuda.synchronize()
    phase_ms = e0.elapsed_time(e1)

    tot, cnt = defaultdict(float), defaultdict(int)
    for ev in prof.events():
        if ev.device_type == torch.autograd.DeviceType.CUDA:
            tot[ev.name] += ev.device_time_total / 1e3
            cnt[ev.name] += 1
    rows = sorted(tot, key=lambda k: -tot[k])
    kern_ms = sum(tot.values())
    os.makedirs(a.trace_dir, exist_ok=True)
    trace = os.path.join(a.trace_dir, "update_phase.pt.trace.json")
    prof.export_chrome_trace(trace)

    gpu = torch.cuda.get_device_name(0)
    print(f"{gpu}; update phase {phase_ms:.2f} ms (CUDA events, profiler on), kernels {kern_ms:.2f} ms")
    print(f"{'total ms':>10} {'calls':>6} {'share':>7}  kernel")
    for k in rows:
        print(f"{tot[k]:10.3f} {cnt[k]:6d} {100 * tot[k] / phase_ms:6.1f}%  {k[:150]}")
    print(json.dumps({"gpu": gpu, "phase_ms": phase_ms, "kernel_ms": kern_ms, "trace": trace,
                      "kernels": [{"name": k, "ms": tot[k], "calls": cnt[k], "share": tot[k] / phase_ms}
                                  for k in rows]}))


if __name__ == "__main__":
    main()
