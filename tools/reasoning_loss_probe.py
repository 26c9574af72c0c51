"""Times the reasoning actor's fused loss (algorithms.reasoning_actor_loss, csrc/token_loss.cu), forward + backward,
against the reference's eager chain run on the same GPU (tests/reasoning_loss_oracle.py: the worker's loss block in
the reference's op order, with its two host syncs per call), and reports kernels per call (torch.profiler; those
the library launched counted apart) and host syncs (torch.cuda.set_sync_debug_mode).  The whole-head case -
ops.linear_logprobs_entropy at N 16,384, H 1536, V 151,936, then the loss - shows the loss's share of the head.
Prints one JSON line with the card name and power limit read in the same run, and also writes it to --out if given.

    python tools/reasoning_loss_probe.py [--reps 5] [--iters 50] [--out result.json]

Each time is the median over --reps of CUDA-event timings of --iters calls after warm-up; fused and eager alternate
within every rep."""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import warnings

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from rlinf_b200 import _lib, ops  # noqa: E402
from rlinf_b200.algorithms import reasoning_actor_loss  # noqa: E402
from reasoning_loss_oracle import reasoning_actor_loss as eager_chain  # noqa: E402

SHAPES = [(1, 28672), (8, 1024), (64, 4096)]
FULL = dict(kl_penalty_type="k3", kl_beta=0.05, entropy_bonus=0.01, importance_sampling_fix=True,
            importance_sampling_clip=2.0)


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


def inputs(bsz, L, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    lp = -torch.rand(bsz, L, generator=g, device="cuda") * 3.0
    old = lp + torch.randn(bsz, L, generator=g, device="cuda") * 0.3
    roll = old + torch.randn(bsz, L, generator=g, device="cuda") * 0.2
    return dict(logprobs=lp, old_logprobs=old, rollout_logprobs=roll,
                advantages=torch.randn(bsz, L, generator=g, device="cuda"),
                entropy=torch.rand(bsz, L, generator=g, device="cuda") * 2.0,
                ref_logprobs=lp + torch.randn(bsz, L, generator=g, device="cuda") * 0.5,
                loss_mask=torch.rand(bsz, L, generator=g, device="cuda") < 0.7)


def fused_step(c, full, lp, ent):
    lp.grad = None
    ent.grad = None
    loss, _ = reasoning_actor_loss(lp, c["advantages"], c["loss_mask"], recomputed_logprobs=c["old_logprobs"],
                                   rollout_logprobs=c["rollout_logprobs"] if full else None,
                                   ref_logprobs=c["ref_logprobs"] if full else None, entropy=ent if full else None,
                                   loss_agg_func="token-mean", **(FULL if full else {}))
    loss.backward()


def eager_step(c, full):
    eager_chain(c["logprobs"], c["advantages"], c["loss_mask"], c["old_logprobs"],
                entropy=c["entropy"] if full else None, ref_logprobs=c["ref_logprobs"] if full else None,
                rollout_logprobs=c["rollout_logprobs"] if full else None,
                recomputed_logprobs=c["old_logprobs"] if full else None, loss_agg="token-mean",
                kl_penalty_type=FULL["kl_penalty_type"], kl_beta=FULL["kl_beta"] if full else 0.0,
                entropy_bonus=FULL["entropy_bonus"] if full else 0.0, importance_sampling_fix=full,
                importance_sampling_clip=2.0)


def launches(fn):
    """(CUDA kernels in a torch.profiler trace of one call, of which launched by librlinf_b200)."""
    lib = _lib.load()
    torch.cuda.synchronize()
    n0 = lib.rb200_launch_count()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    ours = lib.rb200_launch_count() - n0
    return sum(1 for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA
               and "memcpy" not in e.name.lower() and "memset" not in e.name.lower()), ours


def host_syncs(fn):
    """Synchronising calls torch.cuda.set_sync_debug_mode reports for one call."""
    torch.cuda.synchronize()
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            fn()
        finally:
            torch.cuda.set_sync_debug_mode("default")
    return [str(x.message)[:120] for x in w if "synchroniz" in str(x.message).lower()
            and "prototype" not in str(x.message).lower()]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    args = ap.parse_args()
    name, plim = card()
    res = {"card": name, "power_limit": plim, "cases": []}
    for bsz, L in SHAPES:
        c = inputs(bsz, L)
        for full in (False, True):
            lp = c["logprobs"].clone().requires_grad_(True)
            ent = c["entropy"].clone().requires_grad_(True)
            f = lambda: fused_step(c, full, lp, ent)  # noqa: E731
            e = lambda: eager_step(c, full)  # noqa: E731
            for _ in range(5):
                f()
                e()
            tf, te = [], []
            for _ in range(args.reps):
                tf.append(timed(f, args.iters))
                te.append(timed(e, args.iters))
            fs, es = host_syncs(f), host_syncs(e)
            (fk, fl), (ek, _) = launches(f), launches(e)
            row = {"bsz": bsz, "L": L, "kl_k3_entropy_is_fix": full, "fused_ms": statistics.median(tf),
                   "eager_ms": statistics.median(te), "fused_kernels": fk, "fused_library_launches": fl,
                   "eager_kernels": ek, "fused_host_syncs": len(fs), "eager_host_syncs": len(es),
                   "fused_sync_messages": fs}
            row["speedup"] = row["eager_ms"] / row["fused_ms"]
            res["cases"].append(row)
            print(json.dumps(row), flush=True)

    # whole head: fused LM head forward + backward, without and with the loss
    N, H, V = 16384, 1536, 151936
    g = torch.Generator(device="cuda").manual_seed(1)
    x = torch.randn(1, N, H, generator=g, device="cuda").to(torch.bfloat16).requires_grad_(True)
    w = (torch.randn(V, H, generator=g, device="cuda") * (2.0 / H ** 0.5)).to(torch.bfloat16).requires_grad_(True)
    tgt = torch.randint(0, V, (1, N), generator=g, device="cuda")
    c = inputs(1, N, seed=2)
    glp, gh = torch.randn(1, N, device="cuda") * 1e-4, torch.randn(1, N, device="cuda") * 1e-4

    def head_only():
        lp, ent = ops.linear_logprobs_entropy(x, w, tgt)
        torch.autograd.backward((lp, ent), (glp, gh))

    def head_and_loss():
        lp, ent = ops.linear_logprobs_entropy(x, w, tgt)
        fused_step(dict(c, logprobs=lp), True, lp, ent)

    for _ in range(3):
        head_only()
        head_and_loss()
    th, tl = [], []
    for _ in range(args.reps):
        th.append(timed(head_only, 5))
        tl.append(timed(head_and_loss, 5))
    head = {"N": N, "H": H, "V": V, "head_fwd_bwd_ms": statistics.median(th),
            "head_plus_loss_fwd_bwd_ms": statistics.median(tl)}
    total = head["head_plus_loss_fwd_bwd_ms"]
    head["loss_share"] = (total - head["head_fwd_bwd_ms"]) / total
    res["whole_head"] = head
    print(json.dumps(head), flush=True)
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
