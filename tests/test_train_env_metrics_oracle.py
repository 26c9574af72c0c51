"""CPU checks of the training rollouts' episode statistics (env/* metrics): the oracle (tests/train_env_metrics_oracle.py)
against goldens produced by the reference's own EnvWorker._run_interact_once / env_interact_step, ManiskillEnv and
compute_evaluate_metrics code (tests/golden/make_golden_r8.py), two consecutive rollouts per case."""
import pytest
import torch

from train_env_metrics_oracle import KEYS, TrainEnvMetricsOracle, env_metrics, oracle_cfg

CASES = ("c1_std", "c1_always", "noreset", "c2_term", "none", "two_ranks")


def fixture_params(seed, obs_dim, act_dim, chunks):
    """make_golden_r5.fixture_params: the oracle's seeded init with non-trivial biases."""
    from oracle import rl_oracle as O

    p = O.mlp_init(obs_dim, act_dim, chunks, seed=seed)
    g = torch.Generator().manual_seed(seed + 1)
    for n in p:
        if p[n].dim() == 1 or n == "actor_logstd":
            p[n] = p[n] + 0.05 * torch.randn(p[n].shape, generator=g)
    return {n: v.detach().clone() for n, v in p.items()}


def case_inputs(z, name):
    """(meta dict, params, per rank: (initial_states, [(policy_noise, env_noise) per rollout]))."""
    B, T, C, obs, A, auto_reset, always, mes, ranks = (int(x) for x in z[name + "_meta"])
    meta = dict(B=B, T=T, C=C, obs=obs, A=A, auto_reset=bool(auto_reset), always=bool(always), mes=mes, ranks=ranks,
                p_term=float(z[name + "_p_term"]), env_seed=int(z[name + "_env_seed"]))
    params = fixture_params(int(z[name + "_param_seed"]), obs, A, C)
    nc = T // C
    per_rank = []
    for rank in range(ranks):
        k = f"{name}_rank{rank}_"
        en = torch.from_numpy(z[k + "env_noise"])
        rollouts = [(torch.from_numpy(z[k + f"r{r}_policy_noise"]), en[r * nc:(r + 1) * nc]) for r in range(2)]
        per_rank.append((torch.from_numpy(z[k + "initial_states"]), rollouts))
    return meta, params, per_rank


@pytest.mark.parametrize("name", CASES)
def test_train_env_metrics_oracle_matches_reference(golden, name):
    z = golden("r8")
    m, params, per_rank = case_inputs(z, name)
    cfg = oracle_cfg(m["B"], m["T"], m["C"], m["obs"], m["A"], m["auto_reset"], m["always"], m["mes"], m["p_term"],
                     m["env_seed"])
    oracles = [TrainEnvMetricsOracle(cfg, params, init) for init, _ in per_rank]
    for r in range(2):
        recs = []
        for rank, (orc, (_, rollouts)) in enumerate(zip(oracles, per_rank)):
            pn, en = rollouts[r]
            rec, batch = orc.rollout(pn, en)
            k = f"{name}_rank{rank}_r{r}_"
            # same trajectory as the reference (rewards carry the bootstrap, the statistics do not)
            torch.testing.assert_close(batch["rewards"], torch.from_numpy(z[k + "rewards"]), rtol=1e-5, atol=1e-6)
            for key in KEYS:
                want = torch.from_numpy(z[k + "ep_" + key])
                got = rec[key].float()
                assert got.shape == want.shape, (key, got.shape, want.shape)
                if key == "episode_len":  # the flags are bit-exact, so are the lengths
                    assert torch.equal(got, want)
                else:  # the oracle's MLP rounds differently from the reference's in the last bit
                    torch.testing.assert_close(got, want, rtol=1e-5, atol=1e-6, msg=key)
            recs.append(rec)
        metrics = env_metrics(recs)
        n = int(z[f"{name}_r{r}_num_trajectories"])
        assert metrics["env/num_trajectories"] == n
        if n == 0:
            assert metrics == {"env/num_trajectories": 0}
            continue
        for key in KEYS:
            assert metrics["env/" + key] == pytest.approx(float(z[f"{name}_r{r}_agg_" + key]), rel=1e-6), key


def test_golden_cases_cover_the_record_rules(golden):
    z = golden("r8")
    meta = {n: z[n + "_meta"] for n in CASES}
    assert any(m[2] > 1 and m[7] % m[2] != 0 for m in meta.values())  # chunked, max_episode_steps not a multiple of C
    assert any(m[5] == 0 for m in meta.values())                      # no auto-reset
    assert any(m[6] == 1 for m in meta.values())                      # "always" bootstrap
    assert any(m[8] == 2 for m in meta.values())                      # two ranks
    assert int(z["none_r0_num_trajectories"]) == 0 and int(z["none_r1_num_trajectories"]) == 0
    # without auto-reset every env records once per rollout, at its last chunk step
    assert int(z["noreset_r0_num_trajectories"]) == int(meta["noreset"][0])


def test_env_metrics_from_sums():
    from rlinf_b200.runner import eval_metrics_from_sums

    assert eval_metrics_from_sums([0.0, 0.0, 0.0, 0.0], "env") == {"env/num_trajectories": 0}
    m = eval_metrics_from_sums([4.0, -2.0, 40.0, -0.2], "env")
    assert m == {"env/return": -0.5, "env/episode_len": 10.0, "env/reward": -0.05, "env/num_trajectories": 4}
    # the default prefix stays eval/
    assert eval_metrics_from_sums([1.0, -1.0, 2.0, -0.5]) == {"eval/return": -1.0, "eval/episode_len": 2.0,
                                                             "eval/reward": -0.5, "eval/num_trajectories": 1}


def test_records_train_episodes_rule():
    from rlinf_b200.config import Cfg
    from rlinf_b200.runner import records_train_episodes

    assert records_train_episodes(Cfg({"auto_reset": True}))
    assert records_train_episodes(Cfg({"auto_reset": False}))
    assert records_train_episodes(Cfg({"auto_reset": True, "ignore_terminations": True}))
    assert not records_train_episodes(Cfg({"auto_reset": False, "ignore_terminations": True}))
