"""CPU checks of policy evaluation: the evaluation oracle (tests/eval_oracle.py) against goldens produced by the
reference's own EnvWorker / MultiStepRolloutWorker / ManiskillEnv / compute_evaluate_metrics code
(tests/golden/make_golden_r7.py), the product's progress rule against the reference check_progress, and config
validation."""
import numpy as np
import pytest
import torch

from eval_oracle import EvalOracle

CASES = ("c1_auto", "c1_noreset_2ep", "c2_term", "ignore_term", "c1_auto_2ep", "none")


def _fixture_params(seed, obs_dim, act_dim, chunks):
    """make_golden_r5.fixture_params: the oracle's seeded init with non-trivial biases."""
    from oracle import rl_oracle as O

    p = O.mlp_init(obs_dim, act_dim, chunks, seed=seed)
    g = torch.Generator().manual_seed(seed + 1)
    for n in p:
        if p[n].dim() == 1 or n == "actor_logstd":
            p[n] = p[n] + 0.05 * torch.randn(p[n].shape, generator=g)
    return p


def _case(z, name):
    B, T, C, obs, A, auto_reset, epochs, ignore, mes = (int(x) for x in z[name + "_meta"])
    cfg = {"env": {"train": {"seed": int(z[name + "_env_seed"])},
                   "eval": {"total_num_envs": B, "max_steps_per_rollout_epoch": T, "auto_reset": bool(auto_reset),
                            "rollout_epoch": epochs, "ignore_terminations": bool(ignore), "max_episode_steps": mes,
                            "p_term": float(z[name + "_p_term"])}},
           "actor": {"model": {"obs_dim": obs, "action_dim": A, "num_action_chunks": C}}}
    params = _fixture_params(int(z[name + "_param_seed"]), obs, A, C)
    noise = torch.from_numpy(z[name + "_env_noise"]).reshape(epochs, T // C, B, -1)
    return cfg, params, noise, torch.from_numpy(z[name + "_initial_states"])


@pytest.mark.parametrize("name", CASES)
def test_eval_oracle_matches_reference(golden, name):
    z = golden("r7")
    cfg, params, noise, init = _case(z, name)
    metrics, rec = EvalOracle(cfg, params).evaluate(noise, init)
    n = int(z[name + "_num_trajectories"])
    assert metrics["eval/num_trajectories"] == n
    assert rec["return"].numel() == n
    if n == 0:
        assert metrics == {"eval/num_trajectories": 0}
        return
    for key in ("return", "episode_len", "reward"):
        want = torch.from_numpy(z[name + "_ep_" + key])
        torch.testing.assert_close(rec[key].float(), want, rtol=1e-5, atol=1e-6, msg=key)  # record order
        assert metrics["eval/" + key] == pytest.approx(float(z[name + "_agg_" + key]), rel=1e-5, abs=1e-7), key


def test_golden_cases_cover_the_eval_semantics(golden):
    z = golden("r7")
    meta = {n: z[n + "_meta"] for n in CASES}
    assert any(m[2] > 1 for m in meta.values())                      # chunked
    assert any(m[5] == 0 and m[6] == 2 for m in meta.values())      # no auto-reset, two epochs
    assert any(m[5] == 1 and m[6] == 2 for m in meta.values())      # auto-reset state carried over epochs
    assert any(m[7] == 1 for m in meta.values())                    # ignore_terminations
    assert int(z["none_num_trajectories"]) == 0
    # without auto-reset only the first done of each env and epoch counts
    B, _, _, _, _, _, epochs, _, _ = meta["c1_noreset_2ep"]
    assert int(z["c1_noreset_2ep_num_trajectories"]) <= B * epochs


def test_progress_rule_matches_reference_check_progress(golden):
    from rlinf_b200.runner import should_evaluate

    table = golden("r7")["check_progress"]
    assert len(table) > 100 and table[:, 3].any() and not table[:, 3].all()
    for step, max_steps, interval, run_val in table:
        assert should_evaluate(int(step), int(max_steps), int(interval)) == bool(run_val), (step, max_steps, interval)


def test_max_steps_rule():
    from rlinf_b200.config import Cfg
    from rlinf_b200.runner import max_steps

    assert max_steps(Cfg({"max_epochs": 10})) == 10
    assert max_steps(Cfg({"max_epochs": 10, "max_steps": -1})) == 10
    assert max_steps(Cfg({"max_epochs": 10, "max_steps": 4})) == 4
    assert max_steps(Cfg({"max_epochs": 3, "max_steps": 40})) == 3


def test_config_validation():
    from rlinf_b200.config import Cfg, synthetic_ppo_config
    from rlinf_b200.runner import check_eval_config

    cfg = synthetic_ppo_config(B=64, T=8)
    assert check_eval_config(cfg) == 0  # evaluation stays off by default
    cfg.runner.val_check_interval = 5
    with pytest.raises(ValueError, match="env.eval"):
        check_eval_config(cfg)
    cfg.env["eval"] = Cfg({"total_num_envs": 64, "max_episode_steps": 16, "auto_reset": True})
    with pytest.raises(ValueError, match="max_steps_per_rollout_epoch"):
        check_eval_config(cfg)
    cfg.env.eval.max_steps_per_rollout_epoch = 32
    assert check_eval_config(cfg) == 5
    cfg.runner.val_check_interval = -1
    assert check_eval_config(cfg) == -1


def test_metrics_from_sums():
    from rlinf_b200.runner import eval_metrics_from_sums

    assert eval_metrics_from_sums([0.0, 0.0, 0.0, 0.0]) == {"eval/num_trajectories": 0}
    m = eval_metrics_from_sums([4.0, -2.0, 40.0, -0.2])
    assert m == {"eval/return": -0.5, "eval/episode_len": 10.0, "eval/reward": -0.05, "eval/num_trajectories": 4}
    assert isinstance(m["eval/num_trajectories"], int)
    assert np.isfinite(list(m.values())).all()
