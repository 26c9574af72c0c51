"""The persistent tensor-core rollout kernel with num_action_chunks = C > 1 (rb200_rollout_tc, C > 1): env.chunk_step
semantics (maniskill_env.py:327-375 - C sub-steps without reset, flags OR-ed over the chunk on its last column, one
auto-reset per chunk) and the bootstrap on the chunk's last sub-step (env_worker.py:719-758), against the oracle with
injected noise, against the per-kernel chunked loop on the device Philox streams, the `auto` selection, and a full
T = 512 iteration.  The envelope check at the end runs without a GPU."""
import ctypes as C

import pytest
import torch

from oracle.runner_oracle import RunnerOracle


def _cpu_batch(b):
    return {k: (_cpu_batch(v) if isinstance(v, dict) else v.detach().cpu().clone()) for k, v in b.items()}


def _compare(b, ob, rtol=1e-4, atol=2e-5):
    for k in ("dones", "terminations", "truncations"):
        assert torch.equal(b[k], ob[k]), k
    for k in ("rewards", "prev_values", "prev_logprobs"):
        torch.testing.assert_close(b[k], ob[k], rtol=rtol, atol=atol, msg=k)
    torch.testing.assert_close(b["forward_inputs"]["states"], ob["forward_inputs"]["states"], rtol=rtol, atol=atol)
    torch.testing.assert_close(b["forward_inputs"]["action"], ob["forward_inputs"]["action"], rtol=rtol, atol=atol)


def _chunked_cfg(B, nc, obs, A, Cn, **over):
    from rlinf_b200.config import synthetic_ppo_config

    return synthetic_ppo_config(B=B, T=nc * Cn, obs_dim=obs, action_dim=A, **{"actor.model.num_action_chunks": Cn,
                                                                             **over})


@pytest.mark.gpu
@pytest.mark.parametrize("B,obs,A,Cn,bootstrap_type,auto_reset", [
    (40, 32, 3, 2, "standard", True),     # second CTA owns 8 of its 32 environment slots
    (96, 128, 8, 4, "always", True),      # config-2 network shapes, bootstrap on every done
    (1000, 128, 4, 8, "standard", True),  # 32 CTAs, last one partial
    (64, 32, 4, 8, "standard", True),     # C = 8, C*A = 32
    (64, 64, 2, 3, "standard", False),    # no auto-reset: no bootstrap, elapsed keeps counting
])
def test_rollout_tc_chunked_vs_oracle(B, obs, A, Cn, bootstrap_type, auto_reset):
    from rlinf_b200.runner import EmbodiedRunner

    nc = 10
    # max_episode_steps is not a multiple of C: truncations land on inner sub-steps and are OR-ed into the last column
    cfg = _chunked_cfg(B, nc, obs, A, Cn, **{"rollout.fused_kernel": "tc", "env.train.p_term": 0.03,
                                             "env.train.max_episode_steps": 2 * Cn + 1,
                                             "env.train.auto_reset": auto_reset,
                                             "algorithm.bootstrap_type": bootstrap_type})
    run = EmbodiedRunner(cfg)
    assert run.rollout._tc and run.buffer.rewards.shape == (nc, B, Cn)
    orc = RunnerOracle(cfg, params={n: p.detach().cpu().clone() for n, p in run.actor.model.named_parameters()})
    g = torch.Generator().manual_seed(B + obs + Cn)
    pn = torch.randn(nc + 1, B, Cn * A, generator=g)
    parts = []
    for _ in range(Cn):
        parts += [torch.randn(nc, B, obs + 1, generator=g), torch.rand(nc, B, 1, generator=g)]
    parts.append(torch.randn(nc, B, obs, generator=g))
    en = torch.cat(parts, -1)
    if auto_reset:
        s0 = torch.randn(B, obs, generator=g)
        orc.env.state = s0.clone()
        orc.obs = {"states": orc.env.state}
    ob = orc.rollout(policy_noise=pn, env_noise=en)
    if not auto_reset:  # the oracle resets the envs at the start of the rollout
        s0 = ob["forward_inputs"]["states"][0]
        run.env.elapsed.zero_()
    run.rollout.started = True
    run.buffer.states[0].copy_(s0)
    run.rollout._one_rollout(policy_noise=pn[:nc].cuda(), env_noise=en.cuda())
    torch.cuda.synchronize()
    b = _cpu_batch(run.buffer.as_batch())
    assert bool(ob["truncations"].any()) and bool(ob["terminations"].any())
    for k in ("dones", "terminations", "truncations"):
        assert not bool(b[k][:, :, :-1].any()), k  # flags only on the last sub-step of a chunk
    _compare(b, ob)
    assert (run.env.elapsed.cpu() == orc.env.elapsed).all()


@pytest.mark.gpu
def test_rollout_tc_chunked_matches_per_kernel_path_on_device_rng():
    """Same Philox streams and draw order as the per-kernel chunked loop: flags and elapsed counters agree exactly over
    three consecutive rollouts (auto-reset draws included), floats up to the fp32 summation order of the GEMM paths."""
    from rlinf_b200.runner import EmbodiedRunner

    B, nc, obs, A, Cn = 300, 8, 32, 3, 4
    bufs = []
    for mode in ("tc", False):
        cfg = _chunked_cfg(B, nc, obs, A, Cn, **{"rollout.fused_kernel": mode, "env.train.p_term": 0.03,
                                                 "env.train.max_episode_steps": 5,
                                                 "algorithm.bootstrap_type": "always"})
        run = EmbodiedRunner(cfg)
        assert run.rollout._tc == (mode == "tc")
        out = []
        for _ in range(3):
            run.rollout_phase()
            torch.cuda.synchronize()
            out.append(_cpu_batch(run.buffer.as_batch()))
            out[-1]["elapsed"] = run.env.elapsed.cpu().clone()
        bufs.append(out)
    for r in range(3):
        a, b = bufs[0][r], bufs[1][r]
        assert torch.equal(a["elapsed"], b["elapsed"]), r
        _compare(a, b, rtol=2e-3, atol=2e-4)
    assert bool(bufs[0][2]["dones"].any())


@pytest.mark.gpu
def test_rollout_tc_chunked_selection():
    from rlinf_b200.runner import EmbodiedRunner

    def worker(B, obs, A, Cn, mode="auto"):
        return EmbodiedRunner(_chunked_cfg(B, 4, obs, A, Cn, **{"rollout.fused_kernel": mode})).rollout

    # `auto` keeps the per-kernel loop for chunked policies at every size (faster on the H100, DESIGN.md §6)
    for B, obs, A in ((4096, 128, 4), (640, 128, 4), (320, 128, 4), (1024, 8, 2)):
        w = worker(B, obs, A, 4)
        assert not w._tc and not w._fused, (B, obs, A)
    assert worker(640, 128, 4, 4, "tc")._tc
    with pytest.raises(ValueError, match="num_action_chunks"):
        worker(1024, 40, 4, 4, "tc")
    for mode in ("simt", True):
        with pytest.raises(ValueError, match="num_action_chunks"):
            worker(1024, 128, 4, 4, mode)


@pytest.mark.gpu
def test_rollout_tc_chunked_full_iteration():
    """One full iteration (T = 512 env steps, C = 4, A = 8, B = 1024) on the kernel and the device RNG.  Without state
    and reward noise every reward is recomputable from the buffer: each chunk is replayed on the host from states[n]
    and actions[n], and every flagged chunk must carry gamma * V(final_obs) on its last column."""
    from oracle import rl_oracle as O
    from rlinf_b200.runner import EmbodiedRunner

    B, T, obs, A, Cn = 1024, 512, 128, 8, 4
    nc = T // Cn
    cfg = _chunked_cfg(B, nc, obs, A, Cn, **{"rollout.fused_kernel": "tc", "env.train.noise_std": 0.0,
                                             "env.train.reward_noise_std": 0.0})
    run = EmbodiedRunner(cfg)
    assert run.rollout._tc
    params = {n: p.detach().cpu().clone() for n, p in run.actor.model.named_parameters()}
    run.update_rollout_weights()  # run_iteration, with the rollout buffer read before the update consumes it
    run.rollout_phase()
    torch.cuda.synchronize()
    b = _cpu_batch(run.buffer.as_batch())
    assert run.update_phase()
    for k in ("rewards", "prev_values", "prev_logprobs"):
        assert torch.isfinite(b[k]).all(), k
    states, actions = b["forward_inputs"]["states"], b["forward_inputs"]["action"]
    assert torch.isfinite(states).all() and float(states.abs().max()) < 8.0
    for k in ("dones", "terminations", "truncations"):
        assert not bool(b[k][:, :, :-1].any()), k
    # the first truncation closes env step max_episode_steps, i.e. chunk row max_episode_steps / C
    first = int(cfg.env.train.max_episode_steps) // Cn
    tr = b["truncations"][:, :, -1]
    assert bool(tr[first].any()) and not bool(tr[1:first].any())
    w_s, w_a = run.env.w_s.cpu(), run.env.w_a.cpu()
    s = states.reshape(nc * B, obs)
    raw = []
    for c in range(Cn):
        s = torch.tanh(s @ w_s + actions.reshape(nc * B, Cn * A)[:, c * A:(c + 1) * A] @ w_a)
        raw.append(-(s * s).sum(-1) / obs)
    raw = torch.stack(raw, -1).reshape(nc, B, Cn)
    v_final = O.mlp_forward(params, s, None, want_entropy=False)["values"][:, 0].detach().reshape(nc, B)
    flag = b["dones"][1:, :, -1]  # bootstrap_type "always"
    assert bool(flag.any())
    expect = raw.clone()
    expect[..., -1] += torch.where(flag, float(cfg.algorithm.gamma) * v_final, torch.zeros_like(v_final))
    torch.testing.assert_close(b["rewards"], expect, rtol=1e-4, atol=2e-5)


def test_rollout_tc_supported_envelope():
    from rlinf_b200 import _lib as L

    lib = L.load()

    def ok(obs, A, Cn, value_dim=None):
        lay = L.MlpLayout()
        L.check(lib.rb200_mlp_layout_init(C.byref(lay), obs, A * Cn, Cn if value_dim is None else value_dim, 256),
                "mlp_layout_init")
        return lib.rb200_rollout_tc_supported(C.byref(lay), Cn, 1024) == 0

    assert ok(128, 8, 4) and ok(32, 4, 8)
    assert not ok(40, 4, 2) and not ok(160, 4, 2) and not ok(128, 9, 2)
    assert not ok(128, 4, 4, value_dim=1) and not ok(32, 2, 9, value_dim=8)
    # C = 1: the unchunked kernel's envelope
    assert ok(128, 4, 1) and not ok(128, 9, 1) and not ok(128, 4, 1, value_dim=0)
