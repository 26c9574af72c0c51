"""2-rank NCCL worker of the reasoning step bookkeeping (launched by
tests/test_gpu_reasoning_step.py::test_nccl_two_ranks_match_emulation with torch.distributed.run).

Each rank runs compute_rollout_metrics(_dynamic) on its fixture batch and the actor's loss_func epilogue over the
fixture's micro-batches with real NCCL collectives, and checks itself against the torch oracle: at two ranks an fp32
sum has one result, so the match is bit for bit."""
import json
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(HERE, "golden"))


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist.init_process_group("nccl", device_id=dev)
    import make_golden_reasoning_step as G
    import reasoning_step_oracle as O
    from rlinf_b200.algorithms import MegatronLossEpilogue, step_metrics
    from rlinf_b200.utils import distributed as RD

    ok = True
    for case in ("values", "dynamic"):
        host = [G.rollout_batch(case, r) for r in range(world)]
        b = {k: (v.to(dev) if isinstance(v, torch.Tensor) else v) for k, v in host[rank].items()}
        fn = RD.compute_rollout_metrics_dynamic if case == "dynamic" else RD.compute_rollout_metrics
        m, pl, dl = fn(b, 12, G.L)
        want = O.rollout_metrics(host, G.L, dynamic=case == "dynamic")
        ok &= list(m) == list(want) and all(m[k] == want[k] for k in m)
        ok &= np.array_equal(dl.cpu().numpy(), np.concatenate([h["response_lengths"].numpy() for h in host]))
    ep = MegatronLossEpilogue("actor", num_microbatches=G.N_MB, early_stop_imp_ratio=G.EARLY_STOP)
    final = G.ACTOR_KEYS.index("actor/final_loss")
    rows = []
    for mb in range(G.N_MB):
        vals, loss, mask = G.actor_inputs(rank, mb, world)
        scaled, md = ep(loss.to(dev), {k: vals[i].to(dev) for i, k in enumerate(G.ACTOR_KEYS)}, mask.to(dev), mb)
        per = [(G.actor_inputs(q, mb, world)[0].numpy(), np.float32(G.actor_inputs(q, mb, world)[1]), None)
               for q in range(world)]
        want = O.epilogue(per, final, G.ACTOR_KEYS.index("actor/ratio"), 0, G.EARLY_STOP)[rank]
        ok &= float(scaled) == float(want[1]) and [float(md[k]) for k in G.ACTOR_KEYS] == [float(x) for x in want[2]]
        rows.append(want[2])
    step = step_metrics(ep)
    ok &= list(step.values()) == [float(x) for x in O.step_finish(rows)]
    flags = torch.tensor([int(ok)], device=dev)
    dist.all_reduce(flags, op=dist.ReduceOp.MIN)
    if rank == 0:
        with open(os.environ["RB200_DIST_OUT"], "w") as fh:
            json.dump({"ok": bool(flags.item())}, fh)
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
