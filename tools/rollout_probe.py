"""ms per T-step rollout for the three implementations (tc = persistent wgmma kernel, fused = fp32 SIMT persistent
kernel, graph = per-kernel CUDA graph), CUDA events, device Philox.
usage: python tools/rollout_probe.py [--chunks C] [--action-dim A] [--episode-stats] [B ...]
With --chunks C > 1 (num_action_chunks; T stays 512 env steps = 512 / C chunk steps) only tc and graph run.
--episode-stats: A/B of the training episode statistics (env/* metrics) per implementation - two runners, rollouts
with statistics off and on alternated in one process, median ms of each and the relative difference."""
import statistics
import argparse
import os
import subprocess
import sys

import torch
sys.path.insert(0, '.')
from rlinf_b200.config import synthetic_ppo_config
from rlinf_b200.runner import EmbodiedRunner

ap = argparse.ArgumentParser()
ap.add_argument("--chunks", type=int, default=1)
ap.add_argument("--action-dim", type=int, default=None, help="A per sub-step (default 8, or 32 // C when chunked)")
ap.add_argument("--episode-stats", action="store_true")
ap.add_argument("B", type=int, nargs="*")
args = ap.parse_args()
Cn = args.chunks
A = args.action_dim or (8 if Cn == 1 else min(8, 32 // Cn))
Bs = args.B or [512, 1024, 2048, 4096]
T = 512
try:
    power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True).stdout.strip()
except OSError:
    power = "unknown"
print(f"{torch.cuda.get_device_name()} power limit {power}; obs 128, A {A}, C {Cn}, T {T} env steps", flush=True)
for B in Bs:
    row = {}
    modes = (("tc", "tc"), ("fused", True), ("graph", False)) if Cn == 1 else (("tc", "tc"), ("graph", False))
    if os.environ.get("RB200_PROBE_MODES"):
        modes = tuple(m for m in modes if m[0] in os.environ["RB200_PROBE_MODES"].split(","))
    if args.episode_stats:
        for name, mode in modes:
            cfg = synthetic_ppo_config(B=B, T=T, obs_dim=128, action_dim=A, **{"rollout.fused_kernel": mode,
                                                                                "actor.model.num_action_chunks": Cn})
            runs = {}
            for stats in (False, True):
                runs[stats] = EmbodiedRunner(cfg)
                runs[stats].rollout.episode_stats = stats
                for _ in range(3):
                    runs[stats].rollout_phase()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            ts = {False: [], True: []}
            for i in range(12):
                for stats in ((False, True) if i % 2 == 0 else (True, False)):
                    e0.record(); runs[stats].rollout_phase(); e1.record(); torch.cuda.synchronize()
                    ts[stats].append(e0.elapsed_time(e1))
            off, on = statistics.median(ts[False]), statistics.median(ts[True])
            print(f"B={B} T={T} C={Cn} A={A} {name}: stats off {off:.3f} ms, on {on:.3f} ms, "
                  f"{100.0 * (on - off) / off:+.2f} % (min {min(ts[False]):.3f} / {min(ts[True]):.3f}); "
                  f"episodes {int(runs[True].rollout.episode_sums[0].item())}", flush=True)
            del runs
            torch.cuda.empty_cache()
        continue
    for name, mode in modes:
        cfg = synthetic_ppo_config(B=B, T=T, obs_dim=128, action_dim=A, **{"rollout.fused_kernel": mode,
                                                                            "actor.model.num_action_chunks": Cn})
        run = EmbodiedRunner(cfg)
        for _ in range(3):
            run.rollout_phase()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ts = []
        for _ in range(4):
            e0.record(); run.rollout_phase(); e1.record(); torch.cuda.synchronize()
            ts.append(e0.elapsed_time(e1))
        row[name] = min(ts)
        b = run.buffer
        row[name + "_chk"] = (float(b.rewards.mean()), float(b.prev_values.mean()), int(b.dones.sum()))
        del run
        torch.cuda.empty_cache()
    print(f"B={B} T={T} C={Cn} ms/rollout: " + " ".join(f"{k}={v:.2f}" if isinstance(v, float) else f"{k}={v}" for k, v in row.items()), flush=True)
