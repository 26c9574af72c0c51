"""2-rank NCCL evaluation worker (launched by tests/test_gpu_eval.py::test_two_rank_nccl_evaluate with torchrun).

Each rank owns half of the eval environments and evaluates them with injected noise; EmbodiedRunner.evaluate sums the
four episode statistics over the ranks with one all-reduce.  Every rank also runs the CPU evaluation oracle on its own
half; rank 0 gathers the per-rank oracle records and checks that both ranks report the same metrics and that they are
the oracle's over the union of the ranks' episodes."""
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
    from eval_oracle import EvalOracle, draw_eval_noise, metrics_from_records
    from rlinf_b200.config import Cfg, synthetic_ppo_config
    from rlinf_b200.runner import EmbodiedRunner

    cfg = synthetic_ppo_config(B=64, T=8, obs_dim=32, action_dim=2)
    cfg.env["eval"] = Cfg({"total_num_envs": 96, "max_episode_steps": 6, "max_steps_per_rollout_epoch": 20,
                           "rollout_epoch": 1, "auto_reset": True, "ignore_terminations": False, "p_term": 0.05})
    run = EmbodiedRunner(cfg)
    assert run.eval_env.num_envs == 96 // world
    params = {k: p.detach().cpu().clone() for k, p in run.actor.model.named_parameters()}
    orc = EvalOracle(cfg, params, B=96 // world)
    noise, init = draw_eval_noise(cfg, orc.B, torch.Generator().manual_seed(100 + rank))
    _, rec = orc.evaluate(noise, init)
    got = run.evaluate(env_noise=noise.cuda(), initial_states=init.cuda())
    all_got = [None] * world
    all_rec = [None] * world
    dist.all_gather_object(all_got, got)
    dist.all_gather_object(all_rec, {k: v.tolist() for k, v in rec.items()})
    if rank == 0:
        want = metrics_from_records([{k: torch.tensor(v) for k, v in r.items()} for r in all_rec])
        counts = [len(r["return"]) for r in all_rec]
        ok = all(g == all_got[0] for g in all_got) and got["eval/num_trajectories"] == sum(counts)
        ok = ok and all(abs(got[k] - want[k]) <= 1e-4 * max(1.0, abs(want[k])) for k in want)
        with open(os.environ["RB200_DIST_OUT"], "w") as fh:
            json.dump({"ok": bool(ok), "got": all_got, "want": want, "counts": counts}, fh)
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
