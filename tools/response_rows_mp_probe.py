"""Time one rank's share of ops.megatron_response_logprobs_entropy (the LM head on the response rows of a Megatron
rank's hidden shard) on one GPU, and count both routes' collective bytes from the shapes:

    qwen2.5-7b   TP 4, SP on, CP 1   H 3584, V 152,064 (Megatron's padded vocabulary; shard 38,016)
    qwen2.5-1.5b TP 2, SP on, CP 2   H 1536, V 152,064 (151,936 padded to a multiple of 128 * tp; shard 76,032)

Each is a packed micro-batch of about 32k tokens with seeded prompt and response lengths (printed).  Timed on rank
(tp 0, cp 0), forward + backward, the three routes alternated in each of --rounds rounds (--iters calls per route per
round, CUDA events around each route's calls): the median and the range over the rounds of each time, and of the
per-round ratios stages / contiguous and megatron / stages, so a clock or ordering drift shows as spread:
    stages      the op's local work: plan kernel, pack, unpad of the TP-gathered rows (all TP ranks' sends emulated on
                this device), head partials and combine on R_c rows, values to cells; backward cell gradients, head
                backward, the bf16 send layout and the unpack of the received rows
    contiguous  the head alone (partials + combine, backward) on a contiguous [R_c, H] tensor of the same rows
    megatron    today's SP route: the same head on all T_c rows (the all-gathered stream), dX left as the rank's share
                (vocab_parallel_linear_logprobs_entropy's reduce_hidden_grad=False), before any unpacking
Collective bytes per micro-batch and rank, forward and backward, of both routes; the bf16 reduce-scatter of R_c rows
against an fp32 one.  NCCL times of the two routes need tp * cp GPUs and are reported as not measured.
Prints one JSON line with the card name and power limit read in the same run.
    python tools/response_rows_mp_probe.py [--rounds 9] [--iters 5] [--out OUT.json]
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from rlinf_b200 import ops  # noqa: E402
from rlinf_b200 import response_rows as RR  # noqa: E402
from tools.response_rows_probe import card  # noqa: E402

SHAPES = {"qwen2.5-7b": dict(H=3584, V=152064, tp=4, cp=1), "qwen2.5-1.5b": dict(H=1536, V=152064, tp=2, cp=2)}
TOKENS, L = 32768, 4096


def lengths(tp, cp, seed):
    """Prompts U[128, 1024), responses U[64, L]: sequences until ~32k tokens, padded as preprocess_packed_seqs pads."""
    g = torch.Generator().manual_seed(seed)
    align = 2 * cp * tp if cp > 1 else tp
    p, r, N = [], [], []
    while sum(N) < TOKENS:
        p.append(int(torch.randint(128, 1024, (1,), generator=g)))
        r.append(int(torch.randint(64, L + 1, (1,), generator=g)))
        n = p[-1] + r[-1]
        N.append(n + (align - n % align) % align)
    cu = torch.cat([torch.zeros(1, dtype=torch.int64), torch.cumsum(torch.tensor(N), 0)])
    return torch.tensor(p), torch.tensor(r), cu


def alternated(fns, rounds, iters):
    """{name: [ms per call in each round]}: every round times each fn for `iters` calls, one after another."""
    for fn in fns.values():  # warm-up
        fn()
    torch.cuda.synchronize()
    out = {k: [] for k in fns}
    for _ in range(rounds):
        for k, fn in fns.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(iters):
                fn()
            b.record()
            torch.cuda.synchronize()
            out[k].append(a.elapsed_time(b) / iters)
    return out


def spread(xs):
    xs = sorted(xs)
    return {"median": round(xs[len(xs) // 2], 3), "min": round(xs[0], 3), "max": round(xs[-1], 3)}


def peak_mib(fn):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    fn()
    torch.cuda.synchronize()
    return round((torch.cuda.max_memory_allocated() - base) / 2 ** 20, 1)


def case(name, H, V, tp, cp, rounds, iters):
    p, r, cu = lengths(tp, cp, seed=1)
    n = p + r
    bsz = len(p)
    plan = RR.megatron_parallel(cu, n, r, response_len=L, tp_size=tp, cp_size=cp, sequence_parallel=True)
    T_c = int(cu[-1]) // cp
    Ts = T_c // tp
    Vs = V // tp
    g = torch.Generator(device="cuda").manual_seed(2)
    stream = torch.randn(T_c, H, generator=g, device="cuda").to(torch.bfloat16)
    w = (torch.randn(Vs, H, generator=g, device="cuda") * (2.0 / H ** 0.5)).to(torch.bfloat16)
    responses = torch.randint(0, V, (bsz, L), generator=g, device="cuda")
    glp = torch.randn(bsz, L, generator=g, device="cuda")
    gh = torch.randn(bsz, L, generator=g, device="cuda")
    counts = plan.counts(T_c)
    idx = [plan.index(responses, Ts, k, 0) for k in range(tp)]
    ix = idx[0]
    R = ix.R
    shape = (bsz, L)

    def stages():
        i0 = plan.index(responses, Ts, 0, 0)
        sends = torch.stack([ops.mp_pack(stream[k * Ts:(k + 1) * Ts], idx[k]) for k in range(tp)])
        hc = ops.mp_unpad(sends, i0)
        rec = ops.lmhead_vp_partials(hc, w, i0.targets, 0, tp)
        lp, ent, lse = ops.vp_combine(rec.expand(tp, -1, -1), i0.targets, Vs)
        vals = ops.mp_values(lp, ent, i0)
        ops.mp_to_cells(vals.expand(cp, -1, -1), i0, shape)
        a, b = ops.mp_cell_grads(glp, gh, i0)
        dx32, _ = ops.lmhead_vp_backward(hc, w, i0.targets, 0, tp, lse, ent, a, b)
        send = ops.mp_pack_grad(dx32, i0)
        buf = ops.mp_grad_buffer(i0, H)
        buf[:-1] = send[0]
        ops.mp_unpack_grad(buf, i0)

    hc0 = stream[ix.rows].contiguous()
    a0, b0 = ops.mp_cell_grads(glp, gh, ix)

    def contiguous():
        rec = ops.lmhead_vp_partials(hc0, w, ix.targets, 0, tp)
        lp, ent, lse = ops.vp_combine(rec.expand(tp, -1, -1), ix.targets, Vs)
        ops.lmhead_vp_backward(hc0, w, ix.targets, 0, tp, lse, ent, a0, b0)

    tg_all = torch.randint(0, V, (T_c,), generator=g, device="cuda")
    g_all = torch.randn(T_c, generator=g, device="cuda")

    def megatron():
        rec = ops.lmhead_vp_partials(stream, w, tg_all, 0, tp)
        lp, ent, lse = ops.vp_combine(rec.expand(tp, -1, -1), tg_all, Vs)
        ops.lmhead_vp_backward(stream, w, tg_all, 0, tp, lse, ent, g_all, g_all)

    t = alternated({"stages": stages, "contiguous": contiguous, "megatron": megatron}, rounds, iters)
    ratio = [a / b for a, b in zip(t["stages"], t["contiguous"])]
    speedup = [a / b for a, b in zip(t["megatron"], t["stages"])]
    Rmax_c = max(1, max(sum(x) for x in counts))
    ours_fwd = (tp * ix.Rmax_k * H * 2 if tp > 1 else 0) + (tp * R * 16 if tp > 1 else 0) + (
        cp * Rmax_c * 8 if cp > 1 else 0)
    ours_bwd = tp * ix.Rmax_k * H * 2 if tp > 1 else 0
    meg_fwd = (T_c * H * 2 if tp > 1 else 0) + (tp * T_c * 16 if tp > 1 else 0) + (cp * T_c * 8 if cp > 1 else 0)
    meg_bwd = T_c * H * 2 if tp > 1 else 0
    return {
        "shape": name, "H": H, "V": V, "tp": tp, "cp": cp, "sp": True, "bsz": bsz, "prompt_lengths": p.tolist(),
        "response_lengths": r.tolist(), "T_c": T_c, "R_c": R, "Rmax_k": ix.Rmax_k, "R_c_over_T_c": round(R / T_c, 4),
        "counts": counts,
        "rounds": rounds, "iters_per_round": iters,
        "ms_stages_fwd_bwd": spread(t["stages"]), "ms_contiguous_fwd_bwd": spread(t["contiguous"]),
        "ms_megatron_all_rows_fwd_bwd": spread(t["megatron"]),
        "stages_over_contiguous": spread(ratio), "speedup_vs_megatron_route": spread(speedup),
        "peak_mib_stages": peak_mib(stages), "peak_mib_megatron": peak_mib(megatron),
        "bytes_fwd": {"ours": ours_fwd, "megatron": meg_fwd},
        "bytes_bwd": {"ours_bf16_reduce_scatter": ours_bwd, "fp32_reduce_scatter_of_R_c_rows": 2 * ours_bwd,
                      "megatron_bf16_reduce_scatter": meg_bwd},
        "nccl_fwd_bwd": "not measured: this probe times one rank on one GPU",
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=9)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--out")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("response_rows_mp_probe needs a CUDA device")
    name, plim = card()
    res = {"gpu": name, "power_limit": plim, "cases": [case(k, rounds=a.rounds, iters=a.iters, **v) for k, v in SHAPES.items()]}
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
