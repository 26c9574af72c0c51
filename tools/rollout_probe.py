"""ms per T-step rollout for the three implementations (tc = persistent wgmma kernel, fused = fp32 SIMT persistent
kernel, graph = per-kernel CUDA graph), CUDA events, device Philox.  usage: python tools/rollout_probe.py [B ...]"""
import sys
import torch
sys.path.insert(0, '.')
from rlinf_b200.config import synthetic_ppo_config
from rlinf_b200.runner import EmbodiedRunner

Bs = [int(x) for x in sys.argv[1:]] or [512, 1024, 2048, 4096]
T = 512
for B in Bs:
    row = {}
    import os
    modes = (("tc", "tc"), ("fused", True), ("graph", False))
    if os.environ.get("RB200_PROBE_MODES"):
        modes = tuple(m for m in modes if m[0] in os.environ["RB200_PROBE_MODES"].split(","))
    for name, mode in modes:
        cfg = synthetic_ppo_config(B=B, T=T, obs_dim=128, action_dim=8, **{"rollout.fused_kernel": mode})
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
    print(f"B={B} T={T} ms/rollout: " + " ".join(f"{k}={v:.2f}" if isinstance(v, float) else f"{k}={v}" for k, v in row.items()), flush=True)
