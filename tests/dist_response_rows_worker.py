"""2-rank NCCL worker of ops.response_logprobs_entropy (launched by
tests/test_gpu_response_rows.py::test_two_rank_nccl_matches_emulation with torchrun).

Each rank holds one half of lm_head.weight; the op runs over the real process group on a packed batch, and each rank
checks its results against both ranks emulated on its own device over the plan's rows gathered by torch indexing: log-probs,
entropies and its weight shard's gradient bit-identical, and dX zero outside the responses."""
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
    from rlinf_b200 import response_rows as RR

    H, V, temp = 512, 32064, 0.7
    p, r = [5, 9, 3, 7], [40, 0, 64, 17]
    plan = RR.fsdp_packed(p, r, 16, response_len=64)
    T = sum(p) + sum(r)
    g = torch.Generator(device="cuda").manual_seed(0)  # same inputs on both ranks
    x = torch.randn(1, T, H, generator=g, device="cuda").to(torch.bfloat16)
    w = (torch.randn(V, H, generator=g, device="cuda") * (2.0 / H ** 0.5)).to(torch.bfloat16)
    tok = torch.randint(0, V, (1, T), generator=g, device="cuda")
    glp = torch.randn(len(p), 64, generator=g, device="cuda")
    gh = torch.randn(len(p), 64, generator=g, device="cuda")
    Vs = V // world
    ws = w[rank * Vs:(rank + 1) * Vs].clone().requires_grad_(True)
    xx = x.clone().requires_grad_(True)
    lp, ent = ops.response_logprobs_entropy(xx, ws, tok, plan, temperature=temp, group=dist.group.WORLD)
    (lp * glp + ent * gh).sum().backward()
    # both ranks emulated on this device, on the plan's rows gathered by torch indexing
    idx = plan.index(tok.reshape(-1), T)
    hc = x.reshape(T, H)[idx.rows]
    shards = [w[k * Vs:(k + 1) * Vs] for k in range(world)]
    rec = torch.stack([ops.lmhead_vp_partials(hc, shards[k], idx.targets, k, world, temp) for k in range(world)])
    elp, eent, lse = ops.vp_combine(rec, idx.targets, Vs)
    z = torch.zeros(1, device="cuda")
    cells = lambda v, s: torch.cat([v, z])[s:][idx.cell_map].view(lp.shape)  # noqa: E731
    glp_c = torch.cat([glp.reshape(-1), z])[idx.cells[1:]]
    gh_c = torch.cat([gh.reshape(-1), z])[idx.cells[:-1]]
    dx_k, dw_k = ops.lmhead_vp_backward(hc, shards[rank], idx.targets, rank, world, lse, eent, glp_c, gh_c, temp)
    checks = {
        "logprob": torch.equal(lp, cells(elp, 0)),
        "entropy": torch.equal(ent, cells(eent, 1)),
        "dW_shard": torch.equal(ws.grad, dw_k),
        "dX_outside_zero": not xx.grad.reshape(T, H)[idx.hidden_map < 0].any(),
    }
    if rank == 0:
        with open(os.environ["RB200_DIST_OUT"], "w") as fh:
            json.dump({"ok": all(checks.values()), **checks}, fh)
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
