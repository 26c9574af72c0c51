"""Time ops.response_logprobs_entropy (the LM head on the response rows only) against today's route - the fused op
over every row the reference computes, plus the reference's unpack into [bsz, L] - and against the fused op alone on a
contiguous [R, H] tensor of the same rows, for the three batch layouts of the reasoning workers:

    padded        [8, 8192] with L 7168           H 1536, V 151,936   (today: bsz * L rows, logits[:, -L-1:-1])
    fsdp_packed   16,384 packed tokens            H 1536, V 151,936   (today: every packed row, then a per-sequence
                                                                       unpack loop)
    megatron_thd  one rank's shard at TP 2        H 3584, V 152,064   (today: every packed row, then a per-sequence
                                                                       unpack with one .item() each)

Response lengths are seeded and well below L on average; they are printed.  The Megatron case times one rank's share
(the vocabulary shard of 76,032 columns) without the all-gather of records, which needs a second GPU.
Forward and forward + backward times are CUDA-event medians; peak memory is torch's allocator peak per call.
Prints one JSON line with the card name and power limit read in the same run.
    python tools/response_rows_probe.py [--iters 10] [--out OUT.json]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from rlinf_b200 import ops  # noqa: E402
from rlinf_b200 import response_rows as RR  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i",
                              str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout
        name, plim = (s.strip() for s in out.strip().split(","))
        return name, plim
    except Exception:  # noqa: BLE001
        return torch.cuda.get_device_name(), "unknown"


def timed(fn, iters):
    """(median ms, peak bytes above the starting allocation) of fn()."""
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    fn()
    torch.cuda.synchronize()
    return sorted(ts)[len(ts) // 2], torch.cuda.max_memory_allocated() - base


def unpack_loop(values, starts, lengths, bsz, L):
    """The reference's unpack: one slice per sequence, with its length read on the host, stacked into [bsz, L]."""
    rows = []
    for b in range(bsz):
        s, n = int(starts[b].item()), int(lengths[b].item())
        rows.append(torch.cat([values[s:s + n], values.new_zeros(L - n)]))
    return torch.stack(rows)


def case(name, H, V, bsz, L, r, x, tok, plan, full_rows, full_targets, starts, iters):
    w = (torch.randn(V, H, device="cuda") * (2.0 / H ** 0.5)).to(torch.bfloat16)
    glp = torch.randn(bsz, L, device="cuda")
    gh = torch.randn(bsz, L, device="cuda")
    T = tok.numel()
    idx = plan.index(tok.reshape(-1), T)
    R = idx.R
    hc = x.reshape(T, H)[idx.rows].contiguous()
    tg = idx.targets.clone()
    rl = r.cuda()

    def new(bwd):
        def f():
            xx, ww = x.detach().requires_grad_(bwd), w.detach().requires_grad_(bwd)
            lp, ent = ops.response_logprobs_entropy(xx, ww, tok, plan)
            if bwd:
                ((lp * glp).sum() + (ent * gh).sum()).backward()
        return f

    def contiguous(bwd):
        def f():
            hh, ww = hc.detach().requires_grad_(bwd), w.detach().requires_grad_(bwd)
            lp, ent = ops.linear_logprobs_entropy(hh, ww, tg)
            if bwd:
                (lp.sum() + ent.sum()).backward()
        return f

    def today(bwd):
        def f():
            xx, ww = x.detach().requires_grad_(bwd), w.detach().requires_grad_(bwd)
            h = full_rows(xx)
            lp, ent = ops.linear_logprobs_entropy(h, ww, full_targets)
            lp, ent = lp.reshape(-1), ent.reshape(-1)
            if starts is None:  # padded: already [bsz, L]
                lpc, entc = lp.view(bsz, L), ent.view(bsz, L)
            else:
                lpc, entc = unpack_loop(lp, starts, rl, bsz, L), unpack_loop(ent, starts, rl, bsz, L)
            if bwd:
                ((lpc * glp).sum() + (entc * gh).sum()).backward()
        return f

    res = {"layout": name, "H": H, "V": V, "bsz": bsz, "response_len": L, "T": T,
           "response_lengths": r.tolist(), "rows_today": int(full_targets.numel()), "rows_new": R}
    for key, mk in (("new", new), ("contiguous_R", contiguous), ("today", today)):
        res[f"{key}_fwd_ms"], res[f"{key}_fwd_peak_bytes"] = timed(mk(False), iters)
        res[f"{key}_fwd_bwd_ms"], res[f"{key}_fwd_bwd_peak_bytes"] = timed(mk(True), iters)
    for k in ("fwd", "fwd_bwd"):
        res[f"{k}_new_over_contiguous"] = res[f"new_{k}_ms"] / res[f"contiguous_R_{k}_ms"]
        res[f"{k}_speedup_over_today"] = res[f"today_{k}_ms"] / res[f"new_{k}_ms"]
    del w
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("response_rows_probe needs a CUDA device")
    torch.manual_seed(0)
    g = torch.Generator().manual_seed(0)
    results = []

    # padded: [8, 8192], L 7168
    bsz, S, L, H, V = 8, 8192, 7168, 1536, 151936
    r = torch.randint(256, 3072, (bsz,), generator=g)
    x = (torch.randn(bsz, S, H, device="cuda")).to(torch.bfloat16)
    tok = torch.randint(0, V, (bsz, S), device="cuda")
    plan = RR.padded(bsz, S, L, r)
    results.append(case("padded", H, V, bsz, L, r, x, tok, plan, lambda xx: xx[:, -L - 1:-1], tok[:, -L:], None,
                        args.iters))
    del x, tok

    # FSDP packed: 16,384 tokens
    bsz, L, H, V, T = 16, 4096, 1536, 151936, 16384
    p = torch.randint(128, 512, (bsz,), generator=g)
    r = torch.randint(64, 1024, (bsz,), generator=g)
    assert int((p + r).sum()) <= T
    plan = RR.fsdp_packed(p, r, 1024, response_len=L)
    x = torch.randn(1, T, H, device="cuda").to(torch.bfloat16)
    tok = torch.randint(0, V, (1, T), device="cuda")
    tflat = tok.reshape(-1)
    nxt = torch.cat([tflat[1:], tflat[:1]])
    a = (torch.cumsum(p + r, 0) - r).cuda()
    results.append(case("fsdp_packed", H, V, bsz, L, r, x, tok, plan, lambda xx: xx.reshape(T, H), nxt, a - 1,
                        args.iters))
    del x, tok

    # Megatron THD, one rank's vocabulary shard at TP 2
    bsz, L, H, Vfull = 16, 4096, 3584, 152064
    p = torch.randint(128, 512, (bsz,), generator=g)
    r = torch.randint(64, 1024, (bsz,), generator=g)
    n = p + r
    cu = torch.zeros(bsz + 1, dtype=torch.int64)
    cu[1:] = torch.cumsum(n + n % 2, 0)
    T = int(cu[-1])
    plan = RR.megatron_thd(cu, n, r, response_len=L)
    x = torch.randn(T, 1, H, device="cuda").to(torch.bfloat16)
    tok = torch.randint(0, Vfull // 2, (T, 1), device="cuda")
    tflat = tok.reshape(-1)
    nxt = torch.cat([tflat[1:], tflat[:1]])
    a = (cu[:-1] + n - r).cuda()
    results.append(case("megatron_thd_tp2_shard", H, Vfull // 2, bsz, L, r, x, tok, plan, lambda xx: xx.reshape(T, H),
                        nxt, a - 1, args.iters))

    name, plim = card()
    line = json.dumps({"probe": "response_rows", "gpu": name, "power_limit": plim, "results": results})
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
