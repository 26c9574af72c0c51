"""Times one rank's share of the vocabulary-parallel LM-head log-prob / entropy ops on one GPU, for P ranks of the
qwen2.5-7b vocabulary (N 16,384, H 3584, V 152,064), and their peak memory:
  fused          ops.lmhead_vp_partials + ops.vp_combine (+ ops.lmhead_vp_backward): no logits tensor
  materialised   X @ W_k^T, then the logits-level shard ops (ops.logits_vp_partials / logits_vp_backward) and the two
                 gradient GEMMs
  reference      an eager restatement of the reference's per-rank arithmetic (_VocabParallelEntropyAndCrossEntropy on
                 fp32 logits of X @ W_k^T, its four all-reduces left out), forward and its backward
The collectives are not timed there: the records of the other ranks are this rank's repeated (the combine's work
does not depend on their values).  With two or more GPUs it also times the fused op over 2 ranks on NCCL
(`nccl_two_rank`: host wall time per call, forward and forward + backward, all-gather and fp32 all-reduce included),
run as a child `torch.distributed.run` of this script.  Prints one JSON line with the card name and power limit read
in the same run.

    python tools/lmhead_vp_probe.py [--reps 5] [--iters 10] [--ranks 2 4 8]

Each time is the median over --reps of CUDA-event timings of --iters calls after warm-up; the variants alternate
within every rep."""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from rlinf_b200 import ops  # noqa: E402
from tools.lmhead_probe import card, peak_of, timed  # noqa: E402

N, H, V = 16384, 3584, 152064


def reference_rank(logits, tgt, vocab_start, g_h, g_ce):
    """The reference's per-rank forward and backward arithmetic with world size 1 collectives, eager fp32."""
    z = logits.float()
    m = z.max(dim=-1, keepdim=True).values
    norm = z - m
    e = norm.exp()
    s = e.sum(dim=-1, keepdim=True)
    softmax = e.div_(s)
    sp = (softmax * z).sum(dim=-1, keepdim=True)
    entropy = m.squeeze(-1) + s.log().squeeze(-1) - sp.squeeze(-1)
    Vs = z.shape[-1]
    mask = (tgt < vocab_start) | (tgt >= vocab_start + Vs)
    mt = (tgt - vocab_start).masked_fill(mask, 0)
    pred = norm.gather(1, mt[:, None])[:, 0].masked_fill(mask, 0.0)
    logp = pred - s.log().squeeze(-1)
    # backward (softmax and norm_logits are what the reference saves)
    grad = softmax * (-g_ce[:, None])
    rows = torch.nonzero(~mask)[:, 0]
    grad[rows, mt[rows]] += g_ce[rows]
    grad += g_h[:, None] * softmax * (sp - norm)
    return logp, entropy, grad


def nccl_worker(args):
    """One of 2 NCCL ranks: the fused op over the world group, host wall time per call after a barrier."""
    import time

    import torch.distributed as dist

    local = int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    rank, P = dist.get_rank(), dist.get_world_size()
    g = torch.Generator(device="cuda").manual_seed(0)  # the same hidden states and targets on both ranks
    x = torch.randn(N, H, generator=g, device="cuda").to(torch.bfloat16).requires_grad_(True)
    tgt = torch.randint(0, V, (N,), generator=g, device="cuda")
    Vs = V // P
    w = (torch.randn(Vs, H, device="cuda") * H ** -0.5).to(torch.bfloat16).requires_grad_(True)

    def fwd():
        with torch.no_grad():
            ops.vocab_parallel_linear_logprobs_entropy(x, w, tgt, group=dist.group.WORLD)

    def fwd_bwd():
        x.grad = w.grad = None
        lp, ent = ops.vocab_parallel_linear_logprobs_entropy(x, w, tgt, group=dist.group.WORLD)
        (lp.sum() + ent.sum()).backward()

    out = {}
    for tag, fn in (("fused_fwd", fwd), ("fused_fwd_bwd", fwd_bwd)):
        fn()
        fn()
        times = []
        for _ in range(args.reps):
            torch.cuda.synchronize()
            dist.barrier()
            t0 = time.perf_counter()
            for _ in range(args.iters):
                fn()
            torch.cuda.synchronize()
            times.append((time.perf_counter() - t0) * 1e3 / args.iters)
        out[tag] = round(statistics.median(times), 4)
    if rank == 0:
        print(json.dumps({"P": P, "Vs": Vs, "ms": out}), flush=True)
    dist.destroy_process_group()


def nccl_two_rank(args):
    """Runs nccl_worker on 2 GPUs; its JSON, or why there is none."""
    import socket
    import subprocess

    if torch.cuda.device_count() < 2:
        return "not measured: fewer than 2 GPUs"
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2",
                        "--master-addr", "127.0.0.1", "--master-port", str(port), os.path.abspath(__file__),
                        "--nccl-worker", "--reps", str(args.reps), "--iters", str(args.iters)],
                       capture_output=True, text=True, timeout=1200)
    lines = [ln for ln in r.stdout.splitlines() if ln.startswith("{")]
    if r.returncode != 0 or not lines:
        return f"failed (exit {r.returncode}): {r.stderr[-500:]}"
    return json.loads(lines[-1])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--ranks", type=int, nargs="+", default=[2, 4, 8])
    ap.add_argument("--nccl-worker", action="store_true", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.nccl_worker:
        return nccl_worker(args)
    name, plim = card()
    res = {"card": name, "power_limit": plim, "N": N, "H": H, "V": V, "ranks": {}}
    g = torch.Generator(device="cuda").manual_seed(0)
    x = torch.randn(N, H, generator=g, device="cuda").to(torch.bfloat16)
    tgt = torch.randint(0, V, (N,), generator=g, device="cuda")
    glp = torch.randn(N, generator=g, device="cuda")
    gh = torch.randn(N, generator=g, device="cuda")
    for P in args.ranks:
        Vs = V // P
        k = P - 1  # the last rank: its shard holds 1/P of the targets
        w = (torch.randn(Vs, H, generator=g, device="cuda") * H ** -0.5).to(torch.bfloat16)

        def fused_fwd():
            rec = ops.lmhead_vp_partials(x, w, tgt, k, P)
            return ops.vp_combine(rec[None].expand(P, N, 4), tgt, Vs)

        def fused_fb():
            lp, ent, lse = fused_fwd()
            return ops.lmhead_vp_backward(x, w, tgt, k, P, lse, ent, glp, gh)

        def mat_fwd():
            logits = torch.matmul(x, w.T)
            rec = ops.logits_vp_partials(logits, tgt, k, P)
            return logits, ops.vp_combine(rec[None].expand(P, N, 4), tgt, Vs)

        def mat_fb():
            logits, (lp, ent, lse) = mat_fwd()
            dl = ops.logits_vp_backward(logits, tgt, k, lse, ent, glp, gh)
            return torch.matmul(dl, w), torch.matmul(dl.T, x)

        def ref_fwd():
            return reference_rank(torch.matmul(x, w.T), tgt, k * Vs, gh, glp)

        def ref_fb():
            logp, ent, grad = ref_fwd()
            gb = grad.to(torch.bfloat16)
            return torch.matmul(gb, w), torch.matmul(gb.T, x)

        fns = {"fused_fwd": fused_fwd, "fused_fwd_bwd": fused_fb, "materialised_fwd": mat_fwd,
               "materialised_fwd_bwd": mat_fb, "reference_fwd": ref_fwd, "reference_fwd_bwd": ref_fb}
        for f in fns.values():  # warm-up
            f()
            f()
        times = {kk: [] for kk in fns}
        for _ in range(args.reps):
            for kk, f in fns.items():
                times[kk].append(timed(f, args.iters))
        med = {kk: statistics.median(v) for kk, v in times.items()}
        res["ranks"][P] = {
            "Vs": Vs, "ms": {kk: round(v, 4) for kk, v in med.items()},
            "fused_fwd_over_materialised": round(med["fused_fwd"] / med["materialised_fwd"], 3),
            "fused_fwd_bwd_over_materialised": round(med["fused_fwd_bwd"] / med["materialised_fwd_bwd"], 3),
            "fused_fwd_bwd_over_reference": round(med["fused_fwd_bwd"] / med["reference_fwd_bwd"], 3),
            "peak_bytes": {kk: peak_of(f) for kk, f in fns.items()}}
        del w
        torch.cuda.empty_cache()
    res["nccl_two_rank"] = nccl_two_rank(args)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
