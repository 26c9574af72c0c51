"""Times the reasoning critic on one GPU: the value-head kernels alone (csrc/value_head.cu), and
ops.megatron_response_values + algorithms.reasoning_critic_loss forward and backward against the reference's eager
chain restated in plain torch (a bf16 Linear on every packed row, .float(), postprocess_packed_seqs' per-sequence
unpack loop with its .item() calls, the [:, -L-1:-1] slice, compute_ppo_critic_loss's ops with the explained-variance
sums, and autograd).  The batch is one packed micro-batch of T = 12,288 rows (the config's max_tokens_per_mbs) with
R / T = 0.70, at tp = cp = 1 and, for the value-head stages, TP rank 0 of an emulated tp 2 sequence-parallel grid.
Reports times, each kernel's bytes over its time as a fraction of 3.35 TB/s (kernels timed as --iters calls captured
in one CUDA graph, so the host's launch overhead is not counted), launches and host syncs per call, and the card name
and power limit read in the same run; prints one JSON line, also written to --out if given.

    python tools/critic_probe.py [--reps 5] [--iters 50] [--out result.json]

Each time is the median over --reps of CUDA-event timings of --iters calls after warm-up; fused and eager alternate
within every rep."""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from rlinf_b200 import ops  # noqa: E402
from rlinf_b200 import response_rows as RR  # noqa: E402
from rlinf_b200.algorithms import reasoning_critic_loss  # noqa: E402
from reasoning_loss_probe import card, host_syncs, launches, timed  # noqa: E402

HBM = 3.35e12  # bytes/s, H100 SXM data sheet
SHAPES = [1536, 3584]
VALUE_CLIP = 0.5


def batch(H, seed=0):
    """8 sequences of 1,536 packed rows (prompts 460 / 536, responses 1,076 / 1,000): T 12,288, R 8,532."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    p = torch.full((8,), 460)
    r = torch.full((8,), 1076)
    p[3], r[3] = 536, 1000
    n = p + r
    cu = torch.cat([torch.zeros(1, dtype=torch.int64), torch.cumsum(n, 0)])
    T, L, P = int(cu[-1]), int(r.max()), int(p.max())
    x = torch.randn(T, 1, H, generator=g, device="cuda").to(torch.bfloat16)
    w = (torch.randn(1, H, generator=g, device="cuda") * (2.0 / H ** 0.5)).to(torch.bfloat16)
    # the padded [bsz, S] layout postprocess_packed_seqs unpacks into: prompts right-aligned at P, responses after
    S = P + L
    attn = torch.zeros(8, S, dtype=torch.bool)
    for b in range(8):
        attn[b, P - int(p[b]):P + int(r[b])] = True
    mask = (torch.arange(L)[None] < r[:, None]).cuda()
    ret = torch.randn(8, L, generator=g, device="cuda")
    prev = torch.randn(8, L, generator=g, device="cuda") * 0.1
    return dict(x=x, w=w, cu=cu, n=n, r=r, T=T, L=L, R=int(r.sum()), attn=attn.cuda(), cu_dev=cu.cuda(), mask=mask,
                ret=ret, prev=prev)


def eager_step(c, x, lin):
    """The reference's chain, restated: MegatronCritic forward step + postprocess_packed_seqs + loss_func."""
    out = lin(x).float()  # [T, 1, 1]: LinearForLastLayer
    out = out.transpose(0, 1)  # [1, T, 1]
    bsz, S = c["attn"].shape
    full = torch.zeros(bsz, S, 1, device=out.device, dtype=out.dtype)
    for i in range(bsz):
        s = c["attn"][i].sum().item()
        start = c["cu_dev"][i].item()
        full[i, c["attn"][i]] = out[0, start:start + s]
    L = c["L"]
    v = full[:, -L - 1:-1].contiguous().squeeze(-1)
    ret, prev, m = c["ret"], c["prev"], c["mask"]
    vpc = prev + (v - prev).clamp(-VALUE_CLIP, VALUE_CLIP)
    e1, e2 = ret - v, ret - vpc

    def huber(e):
        return torch.where(e.abs() < 1e4, 0.5 * e * e, 1e4 * (e.abs() - 0.5e4))

    vl = torch.max(huber(e1), huber(e2))
    loss = (vl * m).sum() / m.sum() if not (~m).all() else (vl * m).sum()
    clip = ((vpc - prev).abs() > VALUE_CLIP).float().mean()
    rr, ee = ret[m], (ret - v.detach())[m]
    stats = torch.stack([torch.tensor(float(rr.numel()), device=rr.device), rr.sum(), (rr * rr).sum(), ee.sum(),
                         (ee * ee).sum(), clip, loss.detach()])
    loss.backward()
    return stats


def fused_step(c, x, w, plan):
    v = ops.megatron_response_values(x, w, plan)
    loss, _ = reasoning_critic_loss(v, c["ret"], c["prev"], c["mask"], value_clip=VALUE_CLIP)
    loss.backward()


def graph_time(fn, iters):
    """ms per call of `iters` calls captured in one CUDA graph: kernel time without the host's launch overhead."""
    st = torch.cuda.Stream()
    st.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(st):
        for _ in range(3):
            fn()
    torch.cuda.current_stream().wait_stream(st)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        for _ in range(iters):
            fn()
    graph.replay()
    t = timed(graph.replay, 3) / iters
    del graph
    return t


def kernel_times(c, iters, reps):
    """Value-head kernels alone at TP rank 0 of tp 1 (all rows) and of an emulated tp 2 SP grid (its shard)."""
    out = {}
    H = c["w"].shape[1]
    for tp in (1, 2):
        plan = RR.megatron_parallel(c["cu"], c["n"], c["r"], response_len=c["L"], tp_size=tp,
                                    sequence_parallel=tp > 1)
        Ts = c["T"] // tp
        xs = c["x"][:Ts, 0]
        idx = plan.index(torch.zeros(8, c["L"], dtype=torch.int64, device="cuda"), Ts, 0, 0)
        rows = idx.send if idx.sp else idx.rows
        n = rows.numel()
        g = torch.randn(n, device="cuda")
        fwd = lambda: ops.value_head_rows(xs, rows, c["w"])  # noqa: E731
        dx = lambda: ops.value_head_backward(xs, rows, g, c["w"], idx.hidden_map, True, False)  # noqa: E731
        dw = lambda: ops.value_head_backward(xs, rows, g, c["w"], idx.hidden_map, False, True)  # noqa: E731
        row = {"tp": tp, "rows": n, "shard_rows": Ts}
        for name, fn, nbytes in (("fwd", fwd, n * H * 2), ("bwd_dx", dx, Ts * H * 2), ("bwd_dw", dw, n * H * 2)):
            t = statistics.median(graph_time(fn, iters) for _ in range(reps))
            row[f"{name}_us"] = t * 1e3
            row[f"{name}_hbm_fraction"] = nbytes / (t * 1e-3) / HBM
        out[f"tp{tp}"] = row
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    args = ap.parse_args()
    name, plim = card()
    res = {"card": name, "power_limit": plim, "hbm_bytes_per_s": HBM, "cases": []}
    for H in SHAPES:
        c = batch(H)
        plan = RR.megatron_parallel(c["cu"], c["n"], c["r"], response_len=c["L"])
        xf = c["x"].clone().requires_grad_(True)
        wf = c["w"].clone().requires_grad_(True)
        xe = c["x"].clone().requires_grad_(True)
        lin = torch.nn.Linear(H, 1, bias=False, device="cuda", dtype=torch.bfloat16)
        with torch.no_grad():
            lin.weight.copy_(c["w"])

        def f():
            xf.grad = wf.grad = None
            fused_step(c, xf, wf, plan)

        def e():
            xe.grad = lin.weight.grad = None
            eager_step(c, xe, lin)

        for _ in range(5):
            f()
            e()
        tf, te = [], []
        for _ in range(args.reps):
            tf.append(timed(f, args.iters))
            te.append(timed(e, args.iters))
        fs, es = host_syncs(f), host_syncs(e)
        (fk, fl), (ek, _) = launches(f), launches(e)
        row = {"H": H, "T": c["T"], "R": c["R"], "R_over_T": c["R"] / c["T"], "bsz": 8, "L": c["L"],
               "fused_ms": statistics.median(tf), "eager_ms": statistics.median(te), "fused_kernels": fk,
               "fused_library_launches": fl, "eager_kernels": ek, "fused_host_syncs": len(fs),
               "eager_host_syncs": len(es), "kernels": kernel_times(c, args.iters, args.reps)}
        row["speedup"] = row["eager_ms"] / row["fused_ms"]
        res["cases"].append(row)
        print(json.dumps(row), flush=True)
    big = next(r for r in res["cases"] if r["H"] == 3584)["kernels"]["tp1"]
    res["goals"] = {
        "value_head_kernels_60pct_hbm_at_H3584": all(big[f"{k}_hbm_fraction"] >= 0.6 for k in ("fwd", "bwd_dx",
                                                                                                 "bwd_dw")),
        "fused_no_slower_than_eager": all(r["fused_ms"] <= r["eager_ms"] for r in res["cases"]),
    }
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
