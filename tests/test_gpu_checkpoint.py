"""Checkpoint save and exact resume of EmbodiedRunner.

The main test runs N = 4 iterations straight and compares them with 2 iterations, a save, a NEW runner resumed from
that directory (runner.resume_dir) and the 2 remaining iterations: parameters, both Adam moments, the optimiser's
device state, every tensor of the last rollout and every metric must be equal.  The one exception is the rollout/*
metrics, which rb200_masked_stats sums with fp64 atomics (they differ at the last bits between two runs of the same
code); they are compared at 1e-6 relative.  Likewise the gradient norm and clip coefficient in the optimiser's device
state: rb200_grad_sqnorm sums the squares with fp64 atomics, so they are compared at 1e-12 relative (the step count
and the skip flag exactly; the parameters, which read the coefficient rounded to fp32, exactly)."""
import gc
import math
import os
import socket
import subprocess
import sys

import numpy as np
import pytest
import torch

@pytest.fixture(autouse=True)
def _collect_dropped_runners():
    """Runners dropped earlier may sit in reference cycles: collect them now, so that their CUDA graphs are not
    destroyed by an automatic collection while this test captures a graph (which invalidates the capture)."""
    gc.collect()


ROLLOUT_KEYS = ("states", "actions", "prev_logprobs", "prev_values", "rewards", "dones", "terminations", "truncations")


def _cfg(tmp, mode, C=1, B=64, obs=32, A=4, auto_reset=True, evaluate=False, save_interval=2, **over):
    from rlinf_b200.config import Cfg, synthetic_ppo_config

    cfg = synthetic_ppo_config(B=B, T=8 * C, obs_dim=obs, action_dim=A, update_epoch=1, num_minibatches=2,
                               **{"actor.model.num_action_chunks": C, "rollout.fused_kernel": mode,
                                  # 8 chunk steps x B envs in 2 mini-batches, whatever C is
                                  "actor.global_batch_size": 4 * B, "actor.micro_batch_size": 4 * B,
                                  "env.train.auto_reset": auto_reset, "env.train.max_episode_steps": 3 * C + 2,
                                  "env.train.p_term": 0.05, **over})
    cfg.runner.max_epochs = 4
    cfg.runner.save_interval = save_interval
    cfg.runner.logger = Cfg({"log_path": str(tmp), "experiment_name": "exp"})
    if evaluate:
        cfg.runner.val_check_interval = 2
        cfg.env["eval"] = Cfg({"total_num_envs": 48, "max_episode_steps": 5, "max_steps_per_rollout_epoch": 4 * C,
                               "rollout_epoch": 2, "auto_reset": True, "ignore_terminations": False, "p_term": 0.05})
    return cfg


def _state(run):
    torch.cuda.synchronize()
    opt = run.actor.optimizer
    out = {"flat_params": run.actor.model.flat_params, "exp_avg": opt.exp_avg, "exp_avg_sq": opt.exp_avg_sq,
           "optimizer.state": opt.state}
    out.update({f"buffer.{k}": getattr(run.buffer, k) for k in ROLLOUT_KEYS})
    return {k: v.detach().cpu().clone() for k, v in out.items()}


def _assert_same(a, b):
    for k in a:
        if k == "optimizer.state":  # step, last norm, last coef, skipped
            assert torch.equal(a[k][[0, 3]], b[k][[0, 3]]), k
            torch.testing.assert_close(a[k][1:3], b[k][1:3], rtol=1e-12, atol=0, msg=k)
        else:
            assert torch.equal(a[k], b[k]), k


def _assert_same_metrics(ms_a, ms_b):
    assert len(ms_a) == len(ms_b)
    for a, b in zip(ms_a, ms_b):
        assert sorted(a) == sorted(b)
        for k, v in a.items():
            w = b[k]
            if k.startswith("rollout/"):  # rb200_masked_stats: fp64 atomics
                assert abs(v - w) <= 1e-6 * abs(v) or (math.isnan(v) and math.isnan(w)), (k, v, w)
            else:
                assert v == w or (math.isnan(v) and math.isnan(w)), (k, v, w)


CASES = {
    # name: (rollout.fused_kernel, num_action_chunks, extra config)
    "tc": ("tc", 1, {}),
    "simt": (True, 1, {}),
    "graph": (False, 1, {}),
    "tc_c4": ("tc", 4, {}),
    "graph_c4": (False, 4, {}),
    "tc_noreset": ("tc", 1, {"auto_reset": False}),
    "graph_c4_noreset": (False, 4, {"auto_reset": False}),
    "simt_eval": (True, 1, {"evaluate": True}),
    "graph_c4_eval": (False, 4, {"evaluate": True}),
    # 2 optimiser steps per iteration: warm-up ends in iteration 3, after the resume
    "tc_critic_warmup": ("tc", 1, {"actor.optim.critic_warmup_steps": 5}),
    "graph_cosine_lr": (False, 1, {"actor.optim.lr_scheduler": "cosine", "actor.optim.total_training_steps": 4,
                                   "actor.optim.lr_warmup_steps": 1, "actor.optim.min_lr_rate": 0.1}),
    "tc_graph_update": ("tc", 1, {"actor.cuda_graph_update": True}),
    "simt_graph_update_warmup": (True, 1, {"actor.cuda_graph_update": True, "actor.optim.critic_warmup_steps": 5}),
}


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(CASES))
def test_resume_is_exact(tmp_path, case):
    from rlinf_b200.runner import EmbodiedRunner

    mode, C, extra = CASES[case]
    kw = {k: extra[k] for k in ("auto_reset", "evaluate") if k in extra}
    over = {k: v for k, v in extra.items() if k not in kw}
    straight_dir, split_dir = tmp_path / "straight", tmp_path / "split"
    run = EmbodiedRunner(_cfg(straight_dir, mode, C, **kw, **over))
    straight = run.run()
    want = _state(run)
    assert run.global_step == 4 and len(straight) == 4
    if kw.get("evaluate"):
        assert "eval/num_trajectories" in straight[1] and "eval/num_trajectories" in straight[3]
    assert "env/num_trajectories" in straight[3]

    first = EmbodiedRunner(_cfg(split_dir, mode, C, **kw, **over))
    first.run(2)  # saves checkpoints/global_step_2 (save_interval 2)
    ckdir = split_dir / "exp" / "checkpoints" / "global_step_2"
    assert sorted(os.listdir(ckdir)) == ["actor", "rank_0"]
    del first
    gc.collect()  # before the resumed runner captures graphs
    cfg = _cfg(split_dir, mode, C, **kw, **over)
    cfg.runner.resume_dir = str(ckdir)
    resumed = EmbodiedRunner(cfg)
    assert resumed.global_step == 2
    rest = resumed.run()  # max_epochs - global_step = 2 iterations
    assert resumed.global_step == 4 and len(rest) == 2
    _assert_same(want, _state(resumed))
    _assert_same_metrics(straight[2:], rest)
    # the last step saved too (check_progress: step == max_steps)
    assert os.path.isdir(split_dir / "exp" / "checkpoints" / "global_step_4")


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["tc", False])
def test_load_into_live_runner_with_captured_graphs(tmp_path, mode):
    """load_checkpoint() into a runner that has captured its rollout, evaluation and optimiser-step graphs: restored in
    place, the graphs replay the resumed run exactly."""
    from rlinf_b200.runner import EmbodiedRunner

    over = {"actor.cuda_graph_update": True, "evaluate": True}
    ref = EmbodiedRunner(_cfg(tmp_path / "ref", mode, **over))
    straight = ref.run()
    want = _state(ref)

    run = EmbodiedRunner(_cfg(tmp_path / "live", mode, **over))
    run.run(3)  # saves global_step_2; graphs captured and replayed
    run.evaluate()  # the second evaluation captures the eval graph (and moves the eval env on)
    assert run.actor._step_graphs and run.evaluator._graph is not None
    if mode is False:
        assert run.rollout._graph is not None
    run.load_checkpoint(tmp_path / "live" / "exp" / "checkpoints" / "global_step_2")
    assert run.global_step == 2
    rest = run.run()
    _assert_same(want, _state(run))
    _assert_same_metrics(straight[2:], rest)


def _fixture_state_dict(golden, name="c1"):
    """A state dict in the reference's names, order, shapes and dtypes: the reference's seeded values where the fixture
    stores them (every tensor but the hidden-layer matrices), a seeded draw with the recorded RMS for the matrices."""
    z = golden("ckpt")
    g = torch.Generator().manual_seed(5)
    sd = {}
    for i, (n, shape) in enumerate(zip(z[f"{name}_names"].tolist(), z[f"{name}_shapes"].tolist())):
        if f"{name}_value_{i}" in z:
            sd[n] = torch.from_numpy(z[f"{name}_value_{i}"].copy())
        else:
            dims = tuple(int(d) for d in shape.split(","))
            rms = math.sqrt(float(z[f"{name}_sumsq"][i]) / math.prod(dims))
            sd[n] = torch.randn(dims, generator=g) * rms
    return sd


def _check_against_fixture(sd, z, name):
    assert list(sd) == z[f"{name}_names"].tolist()
    assert [",".join(str(d) for d in v.shape) for v in sd.values()] == z[f"{name}_shapes"].tolist()
    assert [str(v.dtype) for v in sd.values()] == z[f"{name}_dtypes"].tolist()
    assert all(v.device.type == "cpu" for v in sd.values())


@pytest.mark.gpu
@pytest.mark.parametrize("name,C,mode", [("c1", 1, "tc"), ("c4", 4, False)])
def test_full_weights_match_reference_state_dict(tmp_path, golden, name, C, mode):
    from rlinf_b200.runner import EmbodiedRunner

    run = EmbodiedRunner(_cfg(tmp_path, mode, C, obs=128, A=8))
    path = run.save_checkpoint()
    assert path.endswith(os.path.join("exp", "checkpoints", "global_step_0"))
    sd = torch.load(os.path.join(path, "actor", "model_state_dict", "full_weights.pt"), weights_only=True)
    _check_against_fixture(sd, golden("ckpt"), name)
    for n, p in run.actor.model.named_parameters():
        assert torch.equal(sd[n], p.cpu()), n
    for f in ("actor/trainer_state.pt", "rank_0/runner_state.pt"):
        torch.load(os.path.join(path, f), weights_only=True)


@pytest.mark.gpu
@pytest.mark.parametrize("name,C,value,gran", [("novalue", 1, False, "action_level"), ("chunkvalue", 4, True, "chunk_level")])
def test_policy_state_dict_layout_matches_reference(golden, name, C, value, gran):
    """The layouts the runner does not build (no value head, one value per chunk): the policy's state_dict, which is
    what full_weights.pt holds."""
    from rlinf_b200.policy import MLPPolicy

    pol = MLPPolicy(128, 8, C, add_value_head=value, value_granularity=gran)
    sd = {k: v.cpu() for k, v in pol.state_dict().items()}
    _check_against_fixture(sd, golden("ckpt"), name)


@pytest.mark.gpu
def test_ckpt_path_loads_reference_weights(tmp_path, golden):
    from rlinf_b200.runner import EmbodiedRunner

    sd = _fixture_state_dict(golden)
    pt = tmp_path / "full_weights.pt"
    torch.save(sd, pt)
    cfg = _cfg(tmp_path, "tc", obs=128, A=8, evaluate=True)
    cfg.runner.ckpt_path = str(pt)
    a = EmbodiedRunner(cfg)
    for n, p in a.actor.model.named_parameters():
        assert torch.equal(p.cpu(), sd[n]), n
    b = EmbodiedRunner(_cfg(tmp_path, "tc", obs=128, A=8, evaluate=True))
    b.actor.model.load_state_dict(sd)
    assert torch.equal(a.actor.model.flat_params, b.actor.model.flat_params)
    ma, mb = a.evaluate(), b.evaluate()
    assert ma == mb and ma["eval/num_trajectories"] > 0

    bad = dict(sd, extra=torch.zeros(1))
    torch.save(bad, pt)
    with pytest.raises(ValueError, match="unexpected keys"):
        EmbodiedRunner(cfg)
    bad = dict(sd, **{"actor_mean.bias": torch.zeros(4)})
    torch.save(bad, pt)
    with pytest.raises(ValueError, match="actor_mean.bias"):
        EmbodiedRunner(cfg)


@pytest.mark.gpu
def test_resume_errors(tmp_path):
    from rlinf_b200.runner import EmbodiedRunner

    run = EmbodiedRunner(_cfg(tmp_path, False))
    run.run(1)
    path = run.save_checkpoint()
    for over, field in (({"B": 32}, "total_num_envs"), ({"obs": 64}, "obs_dim"), ({"A": 2}, "action_dim")):
        cfg = _cfg(tmp_path, False, **over)
        cfg.runner.resume_dir = path
        with pytest.raises(ValueError, match=field):
            EmbodiedRunner(cfg)
    with pytest.raises(ValueError, match="eval_total_num_envs"):  # saved without evaluation, resumed with it
        EmbodiedRunner(_cfg(tmp_path, False, evaluate=True)).load_checkpoint(path)
    # the name and the content disagree
    moved = str(tmp_path / "exp" / "checkpoints" / "global_step_7")
    os.rename(path, moved)
    with pytest.raises(ValueError, match="step 7"):
        run.load_checkpoint(moved)
    # a directory with only the actor's files (as the reference writes it): weights only, through ckpt_path
    ref_dir = tmp_path / "ref" / "global_step_3"
    os.makedirs(ref_dir / "actor" / "model_state_dict")
    torch.save(run.actor.model.state_dict(), ref_dir / "actor" / "model_state_dict" / "full_weights.pt")
    with pytest.raises(ValueError, match="ckpt_path"):
        run.load_checkpoint(ref_dir)
    with pytest.raises(ValueError, match="divisible"):
        EmbodiedRunner(_cfg(tmp_path, False, evaluate=True, save_interval=3))
    cfg = _cfg(tmp_path, False)
    del cfg.runner["logger"]
    with pytest.raises(ValueError, match="log_path"):
        EmbodiedRunner(cfg)


@pytest.mark.gpu
def test_two_rank_nccl_resume(tmp_path):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    worker = os.path.join(os.path.dirname(os.path.abspath(__file__)), "dist_checkpoint_worker.py")
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2",
                        "--master-addr", "127.0.0.1", "--master-port", str(port), worker],
                       env=dict(os.environ, RB200_DIST_OUT=str(tmp_path)), capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    res = np.load(tmp_path / "result.npz")
    assert bool(res["ok"]), res["report"]
