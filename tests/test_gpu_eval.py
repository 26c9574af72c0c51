"""Policy evaluation on the device: eval-mode inference (rb200_mlp_mean), the episode statistics kernels and the whole
EmbodiedRunner.evaluate loop against the CPU restatement in tests/eval_oracle.py."""
import math

import numpy as np
import pytest
import torch

from eval_oracle import EvalOracle, draw_eval_noise
from oracle import rl_oracle as O

pytestmark = pytest.mark.gpu


def _eval_cfg(B=64, obs=32, A=2, C=1, eval_B=48, eval_T=24, max_ep=6, auto_reset=True, epochs=1, ignore=False,
              p_term=0.05, graph=True, interval=0, **over):
    from rlinf_b200.config import Cfg, synthetic_ppo_config

    cfg = synthetic_ppo_config(B=B, T=8 * C, obs_dim=obs, action_dim=A, **{"rollout.enable_cuda_graph": graph}, **over)
    cfg.actor.model.num_action_chunks = C
    cfg.runner.val_check_interval = interval
    cfg.env["eval"] = Cfg({"total_num_envs": eval_B, "max_episode_steps": max_ep, "max_steps_per_rollout_epoch": eval_T,
                           "rollout_epoch": epochs, "auto_reset": auto_reset, "ignore_terminations": ignore,
                           "p_term": p_term})
    return cfg


def _params(run):
    return {n: p.detach().cpu().clone() for n, p in run.actor.model.named_parameters()}


@pytest.mark.parametrize("obs,A,C,B", [(128, 8, 1, 4096), (42, 8, 1, 40), (32, 2, 4, 256)])
def test_mlp_mean_matches_oracle(obs, A, C, B):
    from rlinf_b200.policy import MLPPolicy

    pol = MLPPolicy(obs, A, num_action_chunks=C, seed=3)
    params = {n: p.detach().cpu().clone() for n, p in pol.named_parameters()}
    g = torch.Generator().manual_seed(1)
    states = torch.randn(B, obs, generator=g)
    chunk_actions, res = pol.predict_action_batch({"states": states.cuda()}, mode="eval")
    out = O.mlp_forward(params, states, None, want_entropy=False, want_values=True)
    mean = out["mean"]
    torch.testing.assert_close(chunk_actions.reshape(B, -1).cpu(), mean, rtol=1e-4, atol=1e-4)
    assert chunk_actions.shape == (B, C, A)
    # log_prob of the mean under Normal(mean, std) (mlp_policy.py:275) and the value head
    want_lp = (-out["logstd"] - 0.5 * math.log(2 * math.pi)).expand(B, -1)
    torch.testing.assert_close(res["prev_logprobs"].cpu(), want_lp, rtol=1e-5, atol=1e-5)
    torch.testing.assert_close(res["prev_values"].cpu(), out["values"], rtol=1e-4, atol=1e-4)
    # without log-probs / values the action is the same
    a2, lp2, v2 = pol.mean(states.cuda(), calculate_logprobs=False, calculate_values=False)
    assert lp2 is None and v2 is None
    assert torch.equal(a2, chunk_actions.reshape(B, -1))


def _host_stats(rewards, dones, auto_reset):
    """Host restatement of rb200_episode_stats_step over S steps: rewards [S,B,C] fp32, dones [S,B] bool."""
    S, B, C = rewards.shape
    ret = np.zeros(B, np.float32)
    ln = np.zeros(B, np.int64)
    prev = np.zeros(B, bool)
    acc = np.zeros((B, 4), np.float64)
    episodes = np.full((S, B, 3), np.nan, np.float32)
    for s in range(S):
        for c in range(C):
            ret = (ret + rewards[s, :, c]).astype(np.float32)
        ln = ln + C
        d = dones[s]
        newly = d if auto_reset else d & ~prev
        prev = prev | d
        rew = (ret / ln.astype(np.float32)).astype(np.float32)
        for b in np.nonzero(newly)[0]:
            acc[b] += (1.0, float(ret[b]), float(ln[b]), float(rew[b]))
            episodes[s, b] = (ret[b], ln[b], rew[b])
        if auto_reset:
            ret = np.where(d, np.float32(0), ret).astype(np.float32)
            ln = np.where(d, 0, ln)
    return acc, episodes


@pytest.mark.parametrize("auto_reset", [True, False])
@pytest.mark.parametrize("C", [1, 3])
def test_episode_stats_kernels_vs_host(auto_reset, C):
    from rlinf_b200 import _lib as L

    lib = L.load()
    S, B = 40, 1000
    rng = np.random.default_rng(C + 2 * auto_reset)
    rewards = rng.standard_normal((S, B, C)).astype(np.float32)
    dones = rng.random((S, B)) < 0.1
    want_acc, want_ep = _host_stats(rewards, dones, auto_reset)

    def run():
        ret = torch.zeros(B, device="cuda")
        ln = torch.zeros(B, dtype=torch.int32, device="cuda")
        prev = torch.zeros(B, dtype=torch.uint8, device="cuda")
        acc = torch.zeros(B, 4, dtype=torch.float64, device="cuda")
        out = torch.zeros(4, dtype=torch.float64, device="cuda")
        ep = torch.zeros(S, B, 3, device="cuda")
        r_dev = torch.from_numpy(rewards).cuda()
        d_dev = torch.zeros(S, B, C, dtype=torch.uint8)
        d_dev[:, :, C - 1] = torch.from_numpy(dones)
        d_dev = d_dev.cuda()
        for s in range(S):
            L.check(lib.rb200_episode_stats_step(L.ptr(r_dev[s]), L.ptr(d_dev[s]), B, C, int(auto_reset), L.ptr(ret),
                                                 L.ptr(ln), L.ptr(prev), L.ptr(acc), L.ptr(ep[s]), L.stream_ptr()))
        L.check(lib.rb200_episode_stats_reduce(L.ptr(acc), B, L.ptr(out), L.stream_ptr()))
        return acc.cpu().numpy(), ep.cpu().numpy(), out.cpu().numpy()

    acc, ep, out = run()
    np.testing.assert_array_equal(acc[:, 0], want_acc[:, 0])             # counts exact
    np.testing.assert_array_equal(ep, want_ep)                           # per-episode fp32 values bit-exact (NaN = none)
    np.testing.assert_allclose(acc, want_acc, rtol=1e-12, atol=0)
    np.testing.assert_allclose(out, want_acc.sum(0), rtol=1e-12, atol=0)
    assert out[0] == want_acc[:, 0].sum()
    acc2, ep2, out2 = run()
    assert acc2.tobytes() == acc.tobytes() and out2.tobytes() == out.tobytes()


EVAL_CASES = {
    "c1_auto": dict(C=1),
    "c1_noreset_2ep": dict(C=1, auto_reset=False, epochs=2, max_ep=10),
    "c2_auto": dict(C=2, p_term=0.1),
    "c4_auto": dict(C=4, eval_T=32),
    "c2_noreset": dict(C=2, auto_reset=False, max_ep=8),
    "ignore_term": dict(C=1, ignore=True, max_ep=5),
    "c1_auto_2ep": dict(C=1, epochs=2, max_ep=7),
    "none_finished": dict(C=1, p_term=0.0, max_ep=100),
}


@pytest.mark.parametrize("case", sorted(EVAL_CASES))
def test_evaluate_matches_oracle(case):
    from rlinf_b200.runner import EmbodiedRunner

    cfg = _eval_cfg(**EVAL_CASES[case])
    run = EmbodiedRunner(cfg)
    orc = EvalOracle(cfg, _params(run))
    noise, init = draw_eval_noise(cfg, orc.B, torch.Generator().manual_seed(11))
    want, _ = orc.evaluate(noise, init)
    got = run.evaluate(env_noise=noise.cuda(), initial_states=init.cuda())
    assert set(got) == set(want)
    assert got["eval/num_trajectories"] == want["eval/num_trajectories"]
    if case == "none_finished":
        assert got == {"eval/num_trajectories": 0}
    else:
        assert want["eval/num_trajectories"] > 0
    for k in got:
        assert got[k] == pytest.approx(want[k], rel=1e-4, abs=1e-6), k


def test_episode_records_match_oracle_order():
    """The per-step episode records of the device loop, in env_evaluate_step's order, against the oracle's."""
    from rlinf_b200.runner import EmbodiedRunner

    cfg = _eval_cfg(C=2, epochs=2, auto_reset=False, max_ep=6)
    run = EmbodiedRunner(cfg)
    orc = EvalOracle(cfg, _params(run))
    noise, init = draw_eval_noise(cfg, orc.B, torch.Generator().manual_seed(5))
    _, rec = orc.evaluate(noise, init)
    ev = run.evaluator
    eps = torch.zeros(ev.rollout_epoch, ev.n_chunk_steps, ev.B, 3, device="cuda")
    ev.run(env_noise=noise.cuda(), initial_states=init.cuda(), episodes=eps)
    eps = eps.cpu().reshape(-1, 3)
    eps = eps[~torch.isnan(eps[:, 0])]
    assert eps.shape[0] == rec["return"].numel()
    assert torch.equal(eps[:, 1], rec["episode_len"].float())
    torch.testing.assert_close(eps[:, 0], rec["return"], rtol=1e-4, atol=1e-5)
    torch.testing.assert_close(eps[:, 2], rec["reward"], rtol=1e-4, atol=1e-5)


def test_graph_replay_and_fresh_runners_bit_identical():
    from rlinf_b200.runner import EmbodiedRunner

    def metrics(graph, calls=3):
        run = EmbodiedRunner(_eval_cfg(C=2, epochs=2, graph=graph, eval_B=256, eval_T=64, max_ep=12))
        return [run.evaluate() for _ in range(calls)], run

    with_graph, run = metrics(True)
    assert run.evaluator._graph is not None and run.evaluator.graph_kernel_count > 0
    without_graph, run2 = metrics(False)
    assert run2.evaluator._graph is None
    assert with_graph == without_graph  # python floats: bit-identical
    again, _ = metrics(True)
    assert again == with_graph
    assert with_graph[0] != with_graph[1]  # fresh noise (device counter) on every evaluation


def test_training_untouched_by_evaluation():
    from rlinf_b200.runner import EmbodiedRunner, should_evaluate

    def train(interval):
        cfg = _eval_cfg(B=64, obs=32, A=2, interval=interval, **{"runner.max_epochs": 3})
        run = EmbodiedRunner(cfg)
        ms = [run.run_iteration() for _ in range(3)]
        return run, ms

    r0, m0 = train(0)
    r1, m1 = train(1)
    assert torch.equal(r0.actor.model.flat_params, r1.actor.model.flat_params)
    b0, b1 = r0.buffer.as_batch(), r1.buffer.as_batch()
    for k in ("rewards", "dones", "prev_values", "prev_logprobs"):
        assert torch.equal(b0[k], b1[k]), k
    assert torch.equal(b0["forward_inputs"]["states"], b1["forward_inputs"]["states"])
    for step, (a, b) in enumerate(zip(m0, m1), start=1):
        assert not any(k.startswith("eval/") for k in a)
        assert any(k.startswith("eval/") for k in b) == should_evaluate(step, 3, 1)
        assert {k: v for k, v in b.items() if not k.startswith("eval/")}.keys() == a.keys()
    # interval 2 of 3 steps: step 2 (multiple) and step 3 (last)
    r2, m2 = train(2)
    assert ["eval/num_trajectories" in m for m in m2] == [False, True, True]


def test_evaluate_at_scale():
    from rlinf_b200.runner import EmbodiedRunner

    B = 4096
    cfg = _eval_cfg(B=256, obs=128, A=8, eval_B=B, eval_T=512, max_ep=128, ignore=True)
    run = EmbodiedRunner(cfg)
    m = run.evaluate()
    assert m["eval/num_trajectories"] == 4 * B
    assert m["eval/episode_len"] == 128.0
    assert all(math.isfinite(v) for v in m.values())
    m2 = run.evaluate()  # graph replay
    assert m2["eval/num_trajectories"] == 4 * B and m2["eval/episode_len"] == 128.0


def test_two_rank_nccl_evaluate(tmp_path):
    import json
    import os
    import socket
    import subprocess
    import sys

    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    outp = tmp_path / "dist_eval.json"
    worker = os.path.join(os.path.dirname(os.path.abspath(__file__)), "dist_eval_worker.py")
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2",
                        "--master-addr", "127.0.0.1", "--master-port", str(port), worker],
                       env=dict(os.environ, RB200_DIST_OUT=str(outp)), capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    res = json.loads(outp.read_text())
    assert res["ok"], res


def test_config_without_eval_section_and_default_off():
    from rlinf_b200.config import synthetic_ppo_config
    from rlinf_b200.runner import EmbodiedRunner

    cfg = synthetic_ppo_config(B=64, T=8, obs_dim=32, action_dim=2)
    run = EmbodiedRunner(cfg)
    assert run.evaluator is None and run.val_check_interval == 0
    with pytest.raises(ValueError, match="env.eval"):
        run.evaluate()
