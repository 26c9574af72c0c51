"""tp x cp NCCL worker of ops.megatron_response_values (launched by tests/test_gpu_critic.py::test_nccl_matches_emulation
with torch.distributed.run, RB200_GRID = "tp,cp,sp").

Ranks are laid out as Megatron's, TP fastest: rank = c * tp + k.  Every rank builds the same batch, runs the op on its
own hidden shard over real TP and CP groups, drives it with reasoning_critic_loss, and checks itself against the whole
grid emulated on its own device through the op's stages: values, dX and d value_weight bit-identical."""
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
    tp, cp, sp = (int(x) for x in os.environ["RB200_GRID"].split(","))
    sp = bool(sp)
    assert world == tp * cp
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    import test_gpu_critic as T
    from rlinf_b200 import ops
    from rlinf_b200.algorithms import reasoning_critic_loss

    tp_groups = [dist.new_group([c * tp + k for k in range(tp)]) for c in range(cp)]
    cp_groups = [dist.new_group([c * tp + k for c in range(cp)]) for k in range(tp)]
    c, k = rank // tp, rank % tp
    s = T._setup(tp, cp, sp, 512)
    _, hid = T._shards(s)
    x = hid[c][k][:, None].clone().requires_grad_(True)
    w = s["w"].clone().requires_grad_(True)
    v = ops.megatron_response_values(x, w, s["plan"], tp_group=tp_groups[c], cp_group=cp_groups[k])
    mask = (torch.arange(s["L"])[None] < s["r"][:, None]).cuda()
    ret = v.detach() + 0.3
    prev = v.detach() - 0.2
    loss, _ = reasoning_critic_loss(v, ret, prev, mask, value_clip=0.5)
    loss.backward()
    e0 = T._emulate(s)
    vv = e0["out"][0][0].clone().requires_grad_(True)
    reasoning_critic_loss(vv, ret, prev, mask, value_clip=0.5)[0].backward()
    e = T._emulate(s, vv.grad)
    checks = {
        "values": torch.equal(v, e["out"][c][k]),
        "dX": torch.equal(x.grad[:, 0], e["dx"][c][k]),
        "dW": torch.equal(w.grad, e["dw"][c][k]),
    }
    ok = torch.tensor([int(all(checks.values()))], device="cuda")
    dist.all_reduce(ok, op=dist.ReduceOp.MIN)
    if rank == 0:
        with open(os.environ["RB200_DIST_OUT"], "w") as fh:
            json.dump({"ok": bool(ok.item()), **checks}, fh)
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
