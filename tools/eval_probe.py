"""ms per EmbodiedRunner.evaluate() (policy mean + synthetic env + episode statistics, CUDA-graph replay, one device-to-
host copy of 4 doubles) at B eval envs and 512 env steps, obs 128, CUDA events after warm-up.
usage: python tools/eval_probe.py [B ...]        (default 4096; rows for C = 1 and C = 4, A = 8)"""
import subprocess
import sys

import torch
sys.path.insert(0, '.')
from rlinf_b200.config import Cfg, synthetic_ppo_config
from rlinf_b200.runner import EmbodiedRunner

Bs = [int(x) for x in sys.argv[1:]] or [4096]
T, obs, A = 512, 128, 8
try:
    power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True).stdout.strip()
except OSError:
    power = "unknown"
print(f"{torch.cuda.get_device_name()} power limit {power}; obs {obs}, A {A}, {T} env steps per evaluate()", flush=True)
for B in Bs:
    for Cn in (1, 4):
        cfg = synthetic_ppo_config(B=256, T=8 * Cn, obs_dim=obs, action_dim=A, **{"actor.model.num_action_chunks": Cn})
        cfg.env["eval"] = Cfg({"total_num_envs": B, "max_episode_steps": 128, "max_steps_per_rollout_epoch": T,
                               "rollout_epoch": 1, "auto_reset": True, "ignore_terminations": False})
        run = EmbodiedRunner(cfg)
        for _ in range(3):
            m = run.evaluate()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ts = []
        for _ in range(5):
            e0.record()
            m = run.evaluate()
            e1.record()
            torch.cuda.synchronize()
            ts.append(e0.elapsed_time(e1))
        print(f"B={B} C={Cn} ms/evaluate: min {min(ts):.2f} median {sorted(ts)[2]:.2f} "
              f"kernels/epoch {run.evaluator.graph_kernel_count} episodes {m['eval/num_trajectories']} "
              f"return {m.get('eval/return', float('nan')):.4f}", flush=True)
        del run
        torch.cuda.empty_cache()
