"""The persistent tensor-core rollout (csrc/rollout_tc.cu) at the benchmark's network shapes: its buffers equal the
per-kernel loop's over two consecutive rollouts on the device Philox streams, with full and partial last CTAs and the
truncation bootstrap (N = 64 value passes) on every done."""
import pytest
import torch

from test_gpu_rollout_tc import _compare, _cpu_batch

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("B,obs", [
    (40, 128),    # second CTA owns 8 of its 32 environment slots
    (4096, 128),  # the benchmark's B: 128 full CTAs
    (4097, 128),  # one environment in the last CTA
    (40, 96),     # three W_s stages per step
])
def test_rollout_tc_matches_per_kernel_path_at_bench_shapes(B, obs):
    from rlinf_b200.config import synthetic_ppo_config
    from rlinf_b200.runner import EmbodiedRunner

    T, act = 12, 8
    bufs = []
    for mode in ("tc", False):
        cfg = synthetic_ppo_config(B=B, T=T, obs_dim=obs, action_dim=act, **{"rollout.fused_kernel": mode,
                                                                              "env.train.p_term": 0.03,
                                                                              "env.train.max_episode_steps": 5,
                                                                              "algorithm.bootstrap_type": "always"})
        run = EmbodiedRunner(cfg)
        assert run.rollout._tc == (mode == "tc")
        out = []
        for _ in range(2):
            run.rollout_phase()
            torch.cuda.synchronize()
            out.append(_cpu_batch(run.buffer.as_batch()))
            out[-1]["elapsed"] = run.env.elapsed.cpu().clone()
        bufs.append(out)
        del run
    for r in range(2):
        a, b = bufs[0][r], bufs[1][r]
        assert torch.equal(a["elapsed"], b["elapsed"]), r
        _compare(a, b, rtol=2e-3, atol=2e-4)
    assert bool(bufs[0][1]["dones"].any()) and bool(bufs[0][1]["truncations"].any())
