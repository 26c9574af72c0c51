"""2-rank NCCL worker for the training rollouts' env/* metrics (launched by
tests/test_gpu_train_env_metrics.py::test_two_rank_nccl_env_metrics with torchrun).

Each rank owns half of the training environments.  After every run_iteration() rank 0 checks that both ranks report the
same env/* metrics and that they are the metrics of the sum of the ranks' own episode statistics."""
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
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    from rlinf_b200.config import synthetic_ppo_config
    from rlinf_b200.runner import EmbodiedRunner, eval_metrics_from_sums

    cfg = synthetic_ppo_config(B=256, T=16, obs_dim=32, action_dim=2,
                               **{"env.train.max_episode_steps": 6, "env.train.p_term": 0.05})
    run = EmbodiedRunner(cfg)
    ok, report = True, []
    for _ in range(2):
        got = {k: v for k, v in run.run_iteration().items() if k.startswith("env/")}
        local_sums = run.rollout.episode_sums.cpu().tolist()
        all_got, all_sums = [None] * world, [None] * world
        dist.all_gather_object(all_got, got)
        dist.all_gather_object(all_sums, local_sums)
        want = eval_metrics_from_sums([sum(s[i] for s in all_sums) for i in range(4)], "env")
        ok = ok and all(g == all_got[0] for g in all_got) and want["env/num_trajectories"] > 0
        ok = ok and all(abs(got[k] - want[k]) <= 1e-12 * max(1.0, abs(want[k])) for k in want)
        report.append({"got": all_got, "want": want})
    if rank == 0:
        with open(os.environ["RB200_DIST_OUT"], "w") as fh:
            json.dump({"ok": bool(ok), "iterations": report}, fh)
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
