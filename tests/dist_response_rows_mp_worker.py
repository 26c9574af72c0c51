"""tp x cp NCCL worker of ops.megatron_response_logprobs_entropy (launched by
tests/test_gpu_response_rows_mp.py::test_nccl_matches_emulation with torch.distributed.run,
RB200_GRID = "tp,cp,sp,sparse"; sparse lengths leave every CP rank but the first without a prediction row).

Ranks are laid out as Megatron's, TP fastest: rank = c * tp + k.  Every rank builds the same batch, runs the op on its
own hidden shard and vocabulary shard over real TP and CP groups, and checks itself against the whole grid emulated
on its own device through the op's stages: log-probs and entropies bit-identical, d_weight_shard bit-identical, dX
equal within bf16 rounding of the reduction order and zero exactly where the emulation's is."""
import json
import os
import sys

import torch
import torch.distributed as dist

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    grid = [int(x) for x in os.environ["RB200_GRID"].split(",")]
    tp, cp, sp, sparse = grid[0], grid[1], bool(grid[2]), bool(grid[3])
    assert world == tp * cp
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    import test_gpu_response_rows_mp as T
    from rlinf_b200 import ops

    tp_groups = [dist.new_group([c * tp + k for k in range(tp)]) for c in range(cp)]
    cp_groups = [dist.new_group([c * tp + k for c in range(cp)]) for k in range(tp)]
    c, k = rank // tp, rank % tp
    H, V = 512, 32768
    s = T._setup(tp, cp, sp, H, V, sparse=sparse)
    w = T._weights(H, V)
    L = s["responses"].shape[1]
    g = torch.Generator(device="cuda").manual_seed(9)
    g_lp = torch.randn(len(s["n"]), L, generator=g, device="cuda")
    g_ent = torch.randn(len(s["n"]), L, generator=g, device="cuda")
    Vs = V // tp
    Ts = s["T_c"] // tp if sp else s["T_c"]
    x = (s["streams"][c][k * Ts:(k + 1) * Ts] if sp else s["streams"][c])[:, None].clone().requires_grad_(True)
    ws = w[k * Vs:(k + 1) * Vs].clone().requires_grad_(True)
    lp, ent = ops.megatron_response_logprobs_entropy(x, ws, s["responses"], s["plan"], temperature=T.TEMP,
                                                     tp_group=tp_groups[c], cp_group=cp_groups[k])
    (lp * g_lp + ent * g_ent).sum().backward()
    e = T._emulate(s["plan"], s["streams"], w, s["responses"], tp, cp, sp, g_lp, g_ent)
    elp, eent = e["out"][c][k]
    edx = e["dx"][c][k]
    got = x.grad[:, 0].float()
    checks = {
        "logprob": torch.equal(lp, elp),
        "entropy": torch.equal(ent, eent),
        "dW_shard": torch.equal(ws.grad, e["dw"][c][k]),
        "dX_zero_pattern": torch.equal(got.ne(0).any(-1), edx.ne(0).any(-1)),
        "dX_close": torch.allclose(got, edx.float(), rtol=0.02, atol=0.02 * float(edx.float().abs().max()) + 1e-6),
    }
    ok = torch.tensor([int(all(checks.values()))], device="cuda")
    dist.all_reduce(ok, op=dist.ReduceOp.MIN)
    if rank == 0:
        with open(os.environ["RB200_DIST_OUT"], "w") as fh:
            json.dump({"ok": bool(ok.item()), **checks}, fh)
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
