"""2-rank NCCL worker of the vocabulary-parallel log-prob ops (launched by
tests/test_gpu_lmhead_vp.py::test_vp_two_rank_nccl_matches_emulation with torchrun).

Each rank holds one half of lm_head.weight (and of the logits).  The fused op and the logits drop-ins run over the real
process group; each rank then emulates both ranks on its own device and checks that the distributed results are
bit-identical to the emulation: with two ranks the fp32 all-reduce of dX is a single addition."""
import json
import os
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    from rlinf_b200 import ops

    N, H, V, temp = 300, 512, 32064, 0.7
    g = torch.Generator(device="cuda").manual_seed(0)  # same inputs on both ranks
    x = torch.randn(N, H, generator=g, device="cuda").to(torch.bfloat16)
    w = (torch.randn(V, H, generator=g, device="cuda") * (2.0 / H ** 0.5)).to(torch.bfloat16)
    tgt = torch.randint(0, V, (N,), generator=g, device="cuda")
    glp = torch.randn(N, generator=g, device="cuda")
    gh = torch.randn(N, generator=g, device="cuda")
    Vs = V // world
    checks = {}

    # fused op over the group
    xx = x.clone().requires_grad_(True)
    ws = w[rank * Vs:(rank + 1) * Vs].clone().requires_grad_(True)
    lp, ent = ops.vocab_parallel_linear_logprobs_entropy(xx, ws, tgt, temperature=temp)
    (lp * glp + ent * gh).sum().backward()
    both = [torch.empty_like(lp) for _ in range(world)]
    dist.all_gather(both, lp)
    checks["ranks_identical_logprob"] = all(torch.equal(b, both[0]) for b in both)
    dist.all_gather(both, ent)
    checks["ranks_identical_entropy"] = all(torch.equal(b, both[0]) for b in both)

    # the same two ranks emulated on this device
    shards = [w[k * Vs:(k + 1) * Vs] for k in range(world)]
    rec = torch.stack([ops.lmhead_vp_partials(x, shards[k], tgt, k, world, temp) for k in range(world)])
    elp, eent, lse_e = ops.vp_combine(rec, tgt, Vs)
    parts = [ops.lmhead_vp_backward(x, shards[k], tgt, k, world, lse_e, eent, glp, gh, temp) for k in range(world)]
    edx = parts[0][0]
    for k in range(1, world):
        edx = edx + parts[k][0]
    checks["fused_logprob"] = torch.equal(lp, elp)
    checks["fused_entropy"] = torch.equal(ent, eent)
    checks["fused_dX"] = torch.equal(xx.grad, edx.to(torch.bfloat16))
    checks["fused_dW_shard"] = torch.equal(ws.grad, parts[rank][1])

    # the weight shard frozen, and dX left un-summed for a caller that reduces it itself
    xx = x.clone().requires_grad_(True)
    lp, ent = ops.vocab_parallel_linear_logprobs_entropy(xx, w[rank * Vs:(rank + 1) * Vs], tgt, temperature=temp,
                                                         reduce_hidden_grad=False)
    (lp * glp + ent * gh).sum().backward()
    checks["fused_dX_share_unreduced"] = torch.equal(xx.grad, parts[rank][0].to(torch.bfloat16))

    # logits drop-ins on the rank's [bsz, L, Vs] shard of the logits
    logits = (x.float() @ w.float().T).view(3, N // 3, V)
    t3 = tgt.view(3, N // 3)
    shard = logits[..., rank * Vs:(rank + 1) * Vs].contiguous().requires_grad_(True)
    dent, dlp = ops.vocab_parallel_entropy_and_log_probs(shard, t3)
    (dlp.reshape(-1) * glp + dent.reshape(-1) * gh).sum().backward()
    rec = torch.stack([ops.logits_vp_partials(logits[..., k * Vs:(k + 1) * Vs], t3, k, world) for k in range(world)])
    llp, lent, llse = ops.vp_combine(rec, t3, Vs)
    checks["dropin_logprob"] = torch.equal(dlp.reshape(-1), llp)
    checks["dropin_entropy"] = torch.equal(dent.reshape(-1), lent)
    want = ops.logits_vp_backward(logits[..., rank * Vs:(rank + 1) * Vs], t3, rank, llse, lent, glp, gh)
    checks["dropin_dlogits"] = torch.equal(shard.grad.reshape(N, Vs), want)
    lp2 = ops.vocab_parallel_log_probs_from_logits(shard.detach(), t3)
    checks["log_probs_from_logits"] = torch.equal(lp2.reshape(-1), llp)

    out = {"rank": rank, "checks": checks, "ok": all(checks.values())}
    res = [None] * world
    dist.all_gather_object(res, out)
    if rank == 0:
        with open(os.environ["RB200_DIST_OUT"], "w") as fh:
            json.dump({"ok": all(r["ok"] for r in res), "ranks": res}, fh)
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
