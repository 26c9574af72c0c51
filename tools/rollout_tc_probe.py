"""Where a step of the persistent tensor-core rollout (csrc/rollout_tc.cu) spends its cycles.

usage: python tools/rollout_tc_probe.py [--chunks C] [--rollouts N] [B]

Compiles rollout_tc.cu with -DRB200_ROLLOUT_TC_PROBE into a temporary directory, links it with the other objects of
the in-tree build (`python -m rlinf_b200.build` first), loads that library instead of the in-tree one and times
rollouts of T = 512 env steps at B (default 4096), obs 128, with training episode statistics.  Prints the per-role
clock64() table of the last rollout: per step (chunk step when C > 1), mean over CTAs and the slowest CTA, in SM
cycles and in µs at the clock the kernel ran at (chain cycles of CTA 0 over the CUDA-event time of the launch).
The default build has no probe code."""
import argparse
import glob
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from rlinf_b200 import build as B  # noqa: E402

ROWS = [  # slot, name, kind: "wait" = summed wait cycles, "t" = summed (stamp - obs-ready stamp), "n" = count
    (0, "producer: waits on empty (unsuccessful)", "wait"),
    (1, "producer: unsuccessful empty waits (count)", "n"),
    (2, "producer: stages issued (count)", "n"),
    (3, "env warpgroup: waits on full", "wait"),
    (4, "actor warpgroup: waits on full", "wait"),
    (5, "value warpgroup: waits on full", "wait"),
    (6, "obs-ready -> actor tower done", "t"),
    (7, "obs-ready -> actions sampled", "t"),
    (8, "obs-ready -> env product (x.W_s) done", "t"),
    (9, "obs-ready -> value head seen by the env warps", "t"),
    (11, "obs-ready -> value tower done", "t"),
    (12, "obs-ready -> value head done", "t"),
    (10, "obs-ready -> next obs-ready (the step)", "t"),
]


def build_probe_lib(out_dir: str) -> str:
    objdir = os.path.join(B.PKG_DIR, "build")
    if not B.is_fresh():
        raise SystemExit("run `python -m rlinf_b200.build` first: the probe library links the in-tree objects")
    src = os.path.join(B.CSRC, "rollout_tc.cu")
    obj = os.path.join(out_dir, "rollout_tc_probe.o")
    subprocess.run([B._nvcc(), *B.NVCC_FLAGS, "-DRB200_ROLLOUT_TC_PROBE", "-c", src, "-o", obj], check=True)
    objs = [o for o in sorted(glob.glob(os.path.join(objdir, "*.o"))) if os.path.basename(o) != "rollout_tc.o"]
    lib = os.path.join(out_dir, "librlinf_b200_probe.so")
    subprocess.run([B._nvcc(), "-shared", "-gencode", "arch=compute_90a,code=sm_90a", "-Xcompiler", "-fPIC", "-o", lib,
                    obj, *objs, "-lcudart"], check=True)
    return lib


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--chunks", type=int, default=1)
    ap.add_argument("--rollouts", type=int, default=3, help="timed rollouts (after 2 warm-up ones)")
    ap.add_argument("B", type=int, nargs="?", default=4096)
    args = ap.parse_args()
    Cn, T, A = args.chunks, 512, (8 if args.chunks == 1 else min(8, 32 // args.chunks))

    import ctypes as C

    import torch
    from rlinf_b200 import _lib as L
    from rlinf_b200.config import synthetic_ppo_config
    from rlinf_b200.runner import EmbodiedRunner

    with tempfile.TemporaryDirectory() as tmp:
        L.LIB_PATH = build_probe_lib(tmp)
        lib = L.load()
        lib.rb200_rollout_tc_probe_buffer.argtypes = [C.c_void_p]
        nslots = lib.rb200_rollout_tc_probe_slots()
        cfg = synthetic_ppo_config(B=args.B, T=T, obs_dim=128, action_dim=A,
                                   **{"rollout.fused_kernel": "tc", "actor.model.num_action_chunks": Cn})
        run = EmbodiedRunner(cfg)
        assert run.rollout.impl == "tc"
        grid = (args.B + 31) // 32
        buf = torch.zeros(grid, nslots, dtype=torch.int64, device="cuda")
        L.check(lib.rb200_rollout_tc_probe_buffer(buf.data_ptr()), "rollout_tc_probe_buffer")
        for _ in range(2):
            run.rollout_phase()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ms = []
        for _ in range(args.rollouts):
            e0.record(); run.rollout_phase(); e1.record(); torch.cuda.synchronize()
            ms.append(e0.elapsed_time(e1))
        v = buf.cpu().double()

    steps = T // Cn
    assert int(v[0, 13]) == steps, f"probe counted {int(v[0, 13])} steps, expected {steps}"
    per_step = v / steps
    mhz = v[0, 10].item() / (min(ms) * 1e3)  # chain cycles of CTA 0 over the rollout phase's time: a lower bound
    print(f"{torch.cuda.get_device_name()}; B {args.B}, C {Cn}, T {T} env steps, {grid} CTAs; rollout phase "
          f"{' / '.join(f'{x:.2f}' for x in ms)} ms; clock from the probe >= {mhz:.0f} MHz")
    print(f"{'per step (chunk step)':52s} {'mean cycles':>12s} {'max CTA':>10s} {'mean µs':>9s}")
    for slot, name, kind in ROWS:
        col = per_step[:, slot]
        us = f"{col.mean().item() / mhz:9.2f}" if kind != "n" else " " * 9
        print(f"{name:52s} {col.mean().item():12.1f} {col.max().item():10.1f} {us}")


if __name__ == "__main__":
    main()
