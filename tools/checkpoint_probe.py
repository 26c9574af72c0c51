"""ms per EmbodiedRunner.save_checkpoint() and load_checkpoint() at config 2 (B 4096, T 512, obs 128, A 8; optimiser
state of one iteration), host clock from the call to a device synchronise after it, median of several calls.  The
checkpoint directory is a temporary directory (local disk), removed at the end.
usage: python tools/checkpoint_probe.py [calls]        (default 7)"""
import os
import subprocess
import sys
import tempfile
import time

import torch
sys.path.insert(0, '.')
from rlinf_b200.config import Cfg, synthetic_ppo_config
from rlinf_b200.runner import EmbodiedRunner

n = int(sys.argv[1]) if len(sys.argv) > 1 else 7
B, T, obs, A = 4096, 512, 128, 8
try:
    power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i",
                            str(torch.cuda.current_device())], capture_output=True, text=True).stdout.strip()
except OSError:
    power = "unknown"
print(f"{torch.cuda.get_device_name()} power limit {power}; B {B}, T {T}, obs {obs}, A {A}", flush=True)
with tempfile.TemporaryDirectory() as tmp:
    cfg = synthetic_ppo_config(B=B, T=T, obs_dim=obs, action_dim=A)
    cfg.runner.logger = Cfg({"log_path": tmp, "experiment_name": "probe"})
    run = EmbodiedRunner(cfg)
    run.run_iteration()
    torch.cuda.synchronize()

    def timed(fn):
        ts = []
        for _ in range(n + 1):  # the first call is warm-up (pinned-memory allocation, file creation)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            ts.append(1e3 * (time.perf_counter() - t0))
        ts = sorted(ts[1:])
        return ts[len(ts) // 2], ts[0], ts[-1]

    path = run.save_checkpoint()
    size = sum(os.path.getsize(os.path.join(d, f)) for d, _, fs in os.walk(path) for f in fs)
    for what, fn in (("save_checkpoint", run.save_checkpoint), ("load_checkpoint", lambda: run.load_checkpoint(path))):
        med, lo, hi = timed(fn)
        print(f"{what}: median {med:.2f} ms (min {lo:.2f}, max {hi:.2f}) over {n} calls; {size / 2**20:.2f} MiB on disk",
              flush=True)
