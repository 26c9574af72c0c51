"""2-rank NCCL worker for checkpoint save and resume (launched by
tests/test_gpu_checkpoint.py::test_two_rank_nccl_resume with torchrun).

Each rank runs 4 iterations straight, then 2 iterations that save checkpoints/global_step_2 (each rank its own
rank_{r}/ state, rank 0 the actor's files), then a new runner resumed from that directory runs the remaining 2.  Every
rank checks that the resumed parameters, optimiser state, last rollout and non-rollout/* metrics equal the straight
run's; rank 0 writes the verdict to $RB200_DIST_OUT/result.npz."""
import gc
import math
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    from rlinf_b200.config import Cfg, synthetic_ppo_config
    from rlinf_b200.runner import EmbodiedRunner

    out = os.environ["RB200_DIST_OUT"]

    def cfg(name, resume=None):
        c = synthetic_ppo_config(B=256, T=16, obs_dim=32, action_dim=2, update_epoch=1, num_minibatches=2,
                                 world_size=world, **{"env.train.max_episode_steps": 6, "env.train.p_term": 0.05})
        c.runner.max_epochs, c.runner.save_interval = 4, 2
        c.runner.logger = Cfg({"log_path": os.path.join(out, name), "experiment_name": "exp"})
        if resume:
            c.runner.resume_dir = resume
        return c

    def state(run):
        torch.cuda.synchronize()
        opt, buf = run.actor.optimizer, run.buffer
        # optimiser state: the step count and skip flag (the norm and clip coefficient come from fp64 atomics)
        return [t.cpu().clone() for t in (run.actor.model.flat_params, opt.exp_avg, opt.exp_avg_sq, opt.state[[0, 3]],
                                          buf.states, buf.actions, buf.prev_logprobs, buf.rewards, buf.dones)]

    run = EmbodiedRunner(cfg("straight"))
    straight = run.run()
    want = state(run)
    del run
    EmbodiedRunner(cfg("split")).run(2)
    gc.collect()  # the dropped runners' graphs must not be destroyed while the resumed runner captures its own
    ckdir = os.path.join(out, "split", "exp", "checkpoints", "global_step_2")
    resumed = EmbodiedRunner(cfg("split", resume=ckdir))
    rest = resumed.run()
    got = state(resumed)
    ok = resumed.global_step == 4 and len(rest) == 2 and all(torch.equal(a, b) for a, b in zip(want, got))
    bad = [k for a, b in zip(straight[2:], rest) for k in a
           if not k.startswith("rollout/") and not (a[k] == b[k] or (math.isnan(a[k]) and math.isnan(b[k])))]
    ok = ok and not bad and sorted(os.listdir(ckdir)) == ["actor", "rank_0", "rank_1"]
    flags = torch.tensor([int(ok)], device="cuda")
    dist.all_reduce(flags, op=dist.ReduceOp.MIN)
    if rank == 0:
        np.savez(os.path.join(out, "result.npz"), ok=np.asarray(bool(flags.item())), report=np.array(bad or ["-"]))
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
