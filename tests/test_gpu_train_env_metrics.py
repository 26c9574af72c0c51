"""Episode statistics of the training rollouts (env/* metrics) on the five rollout paths: the persistent tensor-core
kernel (C = 1 and chunked), the persistent SIMT kernel and the per-kernel CUDA-graph loop (C = 1 and chunked).
Against the CPU oracle (tests/train_env_metrics_oracle.py) with injected noise over two consecutive rollouts; the
rollout buffers bit-identical with and without statistics; the tensor-core kernel against the per-kernel loop on the
device random streams; the runner's env/* metrics; two ranks over NCCL."""
import json
import os
import socket
import subprocess
import sys

import pytest
import torch

from train_env_metrics_oracle import TrainEnvMetricsOracle

# (rollout.fused_kernel, num_action_chunks)
PATHS = {"tc": ("tc", 1), "tc_chunked": ("tc", 2), "simt": (True, 1), "graph": (False, 1), "graph_chunked": (False, 2)}


def _runner(mode, B, nc, obs, A, Cn, **over):
    from rlinf_b200.config import synthetic_ppo_config
    from rlinf_b200.runner import EmbodiedRunner

    cfg = synthetic_ppo_config(B=B, T=nc * Cn, obs_dim=obs, action_dim=A,
                               **{"actor.model.num_action_chunks": Cn, "rollout.fused_kernel": mode, **over})
    run = EmbodiedRunner(cfg)
    ro = run.rollout
    assert ro._tc == (mode == "tc") and ro._fused == (mode is True)
    return cfg, run


def _device_rollout(run, s0, pn, en):
    """RolloutWorker.generate with injected draws: s0 = the observations of a fresh env reset (None: the episodes carry
    over from the previous rollout).  Returns the reduced [count, sum return, sum length, sum reward]."""
    ro, buf = run.rollout, run.buffer
    if s0 is not None:
        buf.states[0].copy_(s0)
        run.env.elapsed.zero_()
        ro.ep_ret.zero_()
        ro.ep_len.zero_()
    else:
        buf.states[0].copy_(buf.states[buf.T])
    ro.started = True
    ro.ep_acc.zero_()
    ro._one_rollout(policy_noise=pn[: buf.T].cuda(), env_noise=en.cuda())
    return ro.ep_acc.sum(0).cpu()


def _draws(g, B, nc, obs, A, Cn):
    pn = torch.randn(nc + 1, B, Cn * A, generator=g)
    parts = []
    for _ in range(Cn):
        parts += [torch.randn(nc, B, obs + 1, generator=g), torch.rand(nc, B, 1, generator=g)]
    parts.append(torch.randn(nc, B, obs, generator=g))
    return pn, torch.cat(parts, -1)


def _check_sums(got, rec):
    n = rec["return"].numel()
    assert int(got[0]) == n
    assert float(got[2]) == float(rec["episode_len"].double().sum())  # flags bit-exact -> lengths exact
    for i, k in ((1, "return"), (3, "reward")):
        want = float(rec[k].double().sum())
        assert abs(float(got[i]) - want) <= 1e-4 * max(1.0, abs(want)), (k, float(got[i]), want)


@pytest.mark.gpu
@pytest.mark.parametrize("path,Cn,auto_reset", [
    ("tc", 1, True), ("tc", 1, False), ("tc_chunked", 2, True), ("tc_chunked", 4, False), ("tc_chunked", 4, True),
    ("simt", 1, True), ("simt", 1, False),
    ("graph", 1, True), ("graph", 1, False), ("graph_chunked", 2, True), ("graph_chunked", 4, False),
])
def test_train_env_metrics_vs_oracle(path, Cn, auto_reset):
    mode = PATHS[path][0]
    B, nc, obs, A = 80, 8, 32, 3
    # max_episode_steps not a multiple of C: truncations on inner sub-steps; episodes span the two rollouts
    cfg, run = _runner(mode, B, nc, obs, A, Cn, **{"env.train.p_term": 0.05, "env.train.max_episode_steps": 2 * Cn + 3,
                                                   "env.train.auto_reset": auto_reset})
    g = torch.Generator().manual_seed(17 * Cn + B + int(auto_reset))
    params = {n: p.detach().cpu().clone() for n, p in run.actor.model.named_parameters()}
    draws = [_draws(g, B, nc, obs, A, Cn) for _ in range(2)]
    inits = [torch.randn(B, obs, generator=g) for _ in range(1 if auto_reset else 2)]
    orc = TrainEnvMetricsOracle(cfg, params, inits)
    total = 0
    for r in range(2):
        rec, _ = orc.rollout(*draws[r])
        s0 = inits[r] if (r == 0 or not auto_reset) else None
        got = _device_rollout(run, None if s0 is None else s0.cuda(), *draws[r])
        _check_sums(got, rec)
        torch.testing.assert_close(run.rollout.ep_ret.cpu(), orc.returns, rtol=1e-4, atol=1e-4)
        total += rec["return"].numel()
    assert total > 0


def _stats_off_buffers(mode, Cn, stats):
    _, run = _runner(mode, 96, 8, 32, 3, Cn, **{"env.train.p_term": 0.05, "env.train.max_episode_steps": 7})
    run.rollout.episode_stats = stats
    out = []
    for _ in range(3):  # graph paths: eager, capture + replay, replay
        run.rollout_phase()
        torch.cuda.synchronize()
        b = run.buffer
        out.append({n: getattr(b, n).cpu().clone() for n in (
            "states", "actions", "prev_logprobs", "prev_values", "rewards", "dones", "terminations", "truncations",
            "final_obs", "final_values")})
        out[-1]["elapsed"] = run.env.elapsed.cpu().clone()
    return out, run


@pytest.mark.gpu
@pytest.mark.parametrize("path", list(PATHS))
def test_statistics_leave_the_buffers_untouched(path):
    mode, Cn = PATHS[path]
    off, _ = _stats_off_buffers(mode, Cn, False)
    on, run = _stats_off_buffers(mode, Cn, True)
    for r in range(3):
        for k in off[r]:
            assert torch.equal(off[r][k], on[r][k]), (r, k)
    assert int(run.rollout.episode_sums[0].item()) > 0


def _device_rng_sums(mode, Cn, B=4096, T=512, obs=128, A=8):
    _, run = _runner(mode, B, T // Cn, obs, A, Cn, **{"env.train.p_term": 0.01, "env.train.max_episode_steps": 50})
    sums = []
    for _ in range(3):
        run.rollout_phase()
        sums.append(run.rollout.episode_sums.cpu().clone())
    return sums


@pytest.mark.gpu
@pytest.mark.parametrize("Cn", [1, 4])
def test_tc_kernel_matches_graph_loop_on_device_rng(Cn):
    """Terminations and truncations depend only on the draws and the elapsed counts, so counts and lengths agree
    exactly between the implementations; returns up to the fp32 rounding of the two GEMM paths."""
    a, b = _device_rng_sums("tc", Cn), _device_rng_sums(False, Cn)
    for r in range(3):
        assert a[r][0] == b[r][0] and a[r][2] == b[r][2], (r, a[r], b[r])
        for i in (1, 3):
            assert abs(float(a[r][i] - b[r][i])) <= 1e-4 * abs(float(b[r][i])), (r, i, a[r], b[r])
    assert float(a[2][0]) > 0


@pytest.mark.gpu
def test_runner_reports_env_metrics_deterministically():
    def run_once():
        _, run = _runner(False, 128, 16, 32, 2, 1, **{"env.train.p_term": 0.05, "env.train.max_episode_steps": 9})
        return [{k: v for k, v in run.run_iteration().items() if k.startswith("env/")} for _ in range(3)]

    a, b = run_once(), run_once()  # iterations 2 and 3 replay the captured graph
    for m in a:
        assert set(m) == {"env/return", "env/episode_len", "env/reward", "env/num_trajectories"}
        assert isinstance(m["env/num_trajectories"], int) and m["env/num_trajectories"] > 0
    assert a == b


@pytest.mark.gpu
@pytest.mark.parametrize("path", ["tc", "graph"])
def test_runner_without_finished_episodes(path):
    _, run = _runner(PATHS[path][0], 64, 8, 32, 2, 1, **{"env.train.p_term": 0.0, "env.train.max_episode_steps": 1000})
    for _ in range(2):
        m = run.run_iteration()
        assert {k: v for k, v in m.items() if k.startswith("env/")} == {"env/num_trajectories": 0}


@pytest.mark.gpu
def test_eval_metrics_unchanged_by_training_statistics():
    from rlinf_b200.config import Cfg, synthetic_ppo_config
    from rlinf_b200.runner import EmbodiedRunner

    def run_once(stats):
        cfg = synthetic_ppo_config(B=64, T=8, obs_dim=32, action_dim=2,
                                   **{"env.train.p_term": 0.05, "env.train.max_episode_steps": 9})
        cfg.runner.val_check_interval = 1
        cfg.env["eval"] = Cfg({"total_num_envs": 64, "max_episode_steps": 6, "max_steps_per_rollout_epoch": 12,
                               "auto_reset": True, "p_term": 0.05})
        run = EmbodiedRunner(cfg)
        run.rollout.episode_stats = stats
        out = []
        for _ in range(2):
            m = run.run_iteration()
            assert ("env/num_trajectories" in m) == stats
            out.append({k: v for k, v in m.items() if k.startswith("eval/")})
        return out

    a, b = run_once(True), run_once(False)
    assert a == b and a[0]["eval/num_trajectories"] > 0


@pytest.mark.gpu
def test_two_rank_nccl_env_metrics(tmp_path):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    outp = tmp_path / "dist_env_metrics.json"
    worker = os.path.join(os.path.dirname(os.path.abspath(__file__)), "dist_train_env_metrics_worker.py")
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2",
                        "--master-addr", "127.0.0.1", "--master-port", str(port), worker],
                       env=dict(os.environ, RB200_DIST_OUT=str(outp)), capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    res = json.loads(outp.read_text())
    assert res["ok"], res
