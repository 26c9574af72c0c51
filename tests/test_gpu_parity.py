"""GPU parity: CUDA path (through the C ABI) vs the CPU oracle and the reference-generated goldens.

Bar: bit-exact for masks, indices and the un-normalised GAE / GRPO-score recurrences;
<= 1e-4 relative (stated per test) for normalised advantages, losses, metrics, gradients, policy
outputs and optimiser results.
"""
import numpy as np
import pytest
import torch

from oracle import rl_oracle as O

pytestmark = pytest.mark.gpu

RTOL = 1e-4


def _t(a):
    a = np.asarray(a)
    return torch.from_numpy(np.ascontiguousarray(a)).reshape(a.shape)


def _cuda(t):
    return None if t is None else t.cuda()


def _synth(seed, nc, B, C, p_done=0.05):
    g = torch.Generator().manual_seed(seed)
    r = torch.randn(nc, B, C, generator=g)
    v = torch.randn(nc + 1, B, C, generator=g)
    d = torch.rand(nc + 1, B, C, generator=g) < p_done
    d[0] = False
    return r, v, d


def rank_consistent(ours: torch.Tensor, ref: torch.Tensor):
    """Ranks agree up to ties: ours_i < ours_j implies ref_i <= ref_j, and vice versa. (Both are monotone maps
    of the same bit-exact raw advantages; a 1-ulp difference in mean/std may merge or split ties but never swaps.)"""
    o, r = ours.flatten().cpu().double().numpy(), ref.flatten().cpu().double().numpy()
    order = np.lexsort((r, o))  # primary key o, ties ordered by r
    assert (np.diff(r[order]) >= 0).all()
    order = np.lexsort((o, r))
    assert (np.diff(o[order]) >= 0).all()


# ---------------------------------------------------------------------------------------------
def test_loss_mask_golden_and_random(golden):
    from rlinf_b200 import ops

    g = golden("adv")
    for name in g["adv_cases"]:
        mask, msum = ops.loss_mask(_t(g[f"adv_{name}_dones"]))
        assert torch.equal(mask.cpu(), _t(g[f"adv_{name}_mask"])), name
        assert torch.equal(msum.contiguous().cpu(), _t(g[f"adv_{name}_mask_sum"])), name
    for seed, (nc, B, C, pd) in enumerate([(64, 200, 1, 0.01), (31, 77, 3, 0.05), (5, 1, 2, 0.5), (512, 4096, 1, 0.005)]):
        _, _, d = _synth(seed, nc, B, C, pd)
        mask, msum = ops.loss_mask(d)
        om, os_ = O.loss_mask_from_dones(d)
        assert torch.equal(mask.cpu(), om) and torch.equal(msum.cpu(), os_)
        assert msum.dtype == torch.int64 and mask.dtype == torch.bool


@pytest.mark.parametrize("B", [160, 33, 4096])
@pytest.mark.parametrize("use_mask", [False, True])
def test_gae_raw_bit_exact_vs_oracle(B, use_mask):
    from rlinf_b200 import ops

    T = 512 if B == 4096 else 77
    r, v, d = _synth(B, T, B, 1, 0.01)
    r, v, d = r[..., 0], v[..., 0], d[..., 0]
    m = (torch.rand(T, B) < 0.8) if use_mask else None
    adv, ret, stats = ops.gae(r, v, d, 0.99, 0.95, m, want_stats=True)
    oa, orr = O.gae(r, v, d, 0.99, 0.95, normalize_advantages=False)
    assert torch.equal(ret.cpu(), orr)
    assert torch.equal(adv.cpu(), oa)
    sel = oa[m] if m is not None else oa.flatten()
    st = stats.cpu()
    assert st[0].item() == sel.numel()
    # per-tile fp32 partial sums folded into fp64 totals: ~1e-7 relative on the second moment
    np.testing.assert_allclose(st[1].item(), sel.double().sum().item(), rtol=1e-6, atol=1e-2)
    np.testing.assert_allclose(st[2].item(), (sel.double() ** 2).sum().item(), rtol=1e-6)


def test_gae_golden_raw_and_critic_free(golden):
    from rlinf_b200 import ops

    g = golden("adv")
    for name in g["adv_cases"]:
        gamma, lam = g[f"adv_{name}_hp"]
        p = O.chunks_to_steps(_t(g[f"adv_{name}_rewards"]), _t(g[f"adv_{name}_dones"]), _t(g[f"adv_{name}_values"]))
        adv, ret, _ = ops.gae(p["rewards"].contiguous(), p["values"].contiguous(), p["dones"].contiguous(),
                              float(gamma), float(lam))
        assert torch.equal(adv.cpu(), _t(g[f"adv_{name}_gae_raw_adv"])), name
        assert torch.equal(ret.cpu(), _t(g[f"adv_{name}_gae_raw_ret"])), name
    adv, ret, _ = ops.gae(_t(g["adv_critic_free_rewards"]), None, _t(g["adv_critic_free_dones"]), 0.9, 0.8)
    assert torch.equal(adv.cpu(), _t(g["adv_critic_free_adv"])) and torch.equal(ret.cpu(), _t(g["adv_critic_free_ret"]))


@pytest.mark.parametrize("mk", ["nomask", "mask"])
def test_calculate_adv_and_returns_gae_golden(golden, mk):
    """Through the plugin entry point, normalised (tolerance 1e-4 rel + 1e-6 abs; ranks consistent)."""
    import rlinf_b200.algorithms as A

    g = golden("adv")
    for name in g["adv_cases"]:
        gamma, lam = g[f"adv_{name}_hp"]
        lm = _t(g[f"adv_{name}_mask"]) if mk == "mask" else None
        lms = _t(g[f"adv_{name}_mask_sum"]) if mk == "mask" else None
        C = g[f"adv_{name}_rewards"].shape[-1]
        res = A.calculate_adv_and_returns(
            task_type="embodied", adv_type="gae", rewards=_t(g[f"adv_{name}_rewards"]),
            dones=_t(g[f"adv_{name}_dones"]), values=_t(g[f"adv_{name}_values"]), gamma=float(gamma),
            gae_lambda=float(lam), group_size=8, reward_type="action_level", num_action_chunks=C,
            loss_mask=lm, loss_mask_sum=lms, prev_logprobs=None, teacher_logprobs=None, advantage_mode=None)
        assert set(res) == {"advantages", "returns"}
        ref_a, ref_r = _t(g[f"adv_{name}_gae_{mk}_adv"]), _t(g[f"adv_{name}_gae_{mk}_ret"])
        assert res["advantages"].shape == ref_a.shape
        assert torch.equal(res["returns"].cpu(), ref_r), name  # returns are not normalised: bit-exact
        torch.testing.assert_close(res["advantages"].cpu(), ref_a, rtol=RTOL, atol=1e-6)
        rank_consistent(res["advantages"], ref_a)


def test_grpo_golden(golden):
    import rlinf_b200.algorithms as A
    from rlinf_b200 import ops

    g = golden("adv")
    n = 0
    for name in g["adv_cases"]:
        if f"adv_{name}_grpo_adv" not in g:
            continue
        n += 1
        C = g[f"adv_{name}_rewards"].shape[-1]
        res = A.calculate_adv_and_returns(
            task_type="embodied", adv_type="grpo", rewards=_t(g[f"adv_{name}_rewards"]),
            dones=_t(g[f"adv_{name}_dones"]), values=_t(g[f"adv_{name}_values"]), gamma=1.0, gae_lambda=1.0,
            group_size=8, reward_type="action_level", num_action_chunks=C, loss_mask=_t(g[f"adv_{name}_mask"]),
            loss_mask_sum=_t(g[f"adv_{name}_mask_sum"]))
        assert set(res) == {"advantages"}
        torch.testing.assert_close(res["advantages"].cpu(), _t(g[f"adv_{name}_grpo_adv"]), rtol=RTOL, atol=1e-6)
        p = O.chunks_to_steps(_t(g[f"adv_{name}_rewards"]), _t(g[f"adv_{name}_dones"]))
        sc = ops.grpo_scores(p["rewards"].contiguous(), p["dones"].contiguous())
        assert torch.equal(sc.cpu().reshape(-1, 8), _t(g[f"adv_{name}_grpo_scores"])), name  # bit-exact
    assert n >= 2


def test_reasoning_branch_golden(golden):
    import rlinf_b200.algorithms as A

    g = golden("adv")
    adv, ret = A.calculate_adv_and_returns(task_type="reasoning", adv_type="gae", rewards=_t(g["reason_rewards"]),
                                           loss_mask=_t(g["reason_mask"]), values=_t(g["reason_values"]), gamma=1.0,
                                           gae_lambda=0.95, normalize_advantages=False)
    assert torch.equal(adv.cpu(), _t(g["reason_gae_adv"])) and torch.equal(ret.cpu(), _t(g["reason_gae_ret"]))
    adv, ret = A.calculate_adv_and_returns(task_type="reasoning", adv_type="grpo", rewards=_t(g["reason_rewards"]),
                                           loss_mask=_t(g["reason_mask"]), group_size=4)
    assert ret is None
    torch.testing.assert_close(adv.cpu(), _t(g["reason_grpo_adv"]), rtol=RTOL, atol=1e-6)


def test_gather_rows_bit_exact(golden):
    from rlinf_b200 import ops

    g = golden("indexing")
    perm = _t(g["idx_perm"])
    for k, drop in (("rewards", False), ("dones", True), ("prev_values", True), ("prev_logprobs", False), ("states", False)):
        src = _t(g["idx_in_" + k])
        if drop:
            src = src[:-1]
        flat = src.reshape(-1, *src.shape[2:]).contiguous()
        out = ops.gather_rows(flat.view(torch.uint8) if flat.dtype == torch.bool else flat, perm)
        ref = _t(g["idx_out_" + k])
        assert torch.equal(out.cpu().view(ref.dtype) if ref.dtype == torch.bool else out.cpu(), ref), k
    # big: N = 4096*512 rows of 128 floats would be 1 GB; use 2^18 rows x 128 floats and a seeded permutation
    n = 1 << 18
    src = torch.randn(n, 128)
    perm = O.shuffle_indices(n, 1234)
    out = ops.gather_rows(src, perm)
    assert torch.equal(out.cpu(), src[perm])


def _loss_case(g, name):
    pre = f"loss_{name}_"
    bsz, C, A, use_ratio, dual, clamp = [int(x) for x in g[pre + "cfg"]]
    lpt, lt, rt = [str(x) for x in g[pre + "types"]]
    hp = dict(clip_ratio_high=0.28, clip_ratio_low=0.2, value_clip=0.2, huber_delta=1.5,
              max_episode_steps=50 if use_ratio else None, critic_warmup=False)
    if dual:
        hp["clip_ratio_c"] = 3.0
    if clamp:
        hp["clip_log_ratio_min"], hp["clip_log_ratio_max"] = -0.2, 0.25
    return pre, A, lpt, lt, rt, hp


# critic/value_clip_ratio is pure rounding noise in the reference (SURVEY.md A9): compared loosely.
LOOSE = {"critic/value_clip_ratio": 0.05}


def test_policy_loss_golden_all_cases(golden):
    import rlinf_b200.algorithms as A

    g = golden("loss")
    for name in g["loss_cases"]:
        pre, Adim, lpt, lt, rt, hp = _loss_case(g, name)
        has_mask = (pre + "mask") in g
        ac = lt == "actor_critic"
        new = _t(g[pre + "new"]).cuda().requires_grad_(True)
        val = _t(g[pre + "val"]).cuda().requires_grad_(True)
        kw = dict(task_type="embodied", loss_type=lt, logprob_type=lpt, reward_type=rt, single_action_dim=Adim,
                  logprobs=new, old_logprobs=_t(g[pre + "old"]), advantages=_t(g[pre + "adv"]),
                  returns=_t(g[pre + "ret"]) if ac else None, values=val if ac else None,
                  prev_values=_t(g[pre + "prev_v"]) if ac else None,
                  loss_mask=_t(g[pre + "mask"]) if has_mask else None,
                  loss_mask_sum=_t(g[pre + "mask_sum"]) if has_mask else None, **hp)
        loss, metrics = A.policy_loss(**kw)
        loss.backward()
        torch.testing.assert_close(loss.detach().cpu(), _t(g[pre + "loss"]), rtol=RTOL, atol=1e-7, msg=name)
        dnew = new.grad if new.grad is not None else torch.zeros_like(new)
        torch.testing.assert_close(dnew.cpu(), _t(g[pre + "dnew"]), rtol=RTOL, atol=1e-8, msg=name)
        if ac:
            dval = val.grad if val.grad is not None else torch.zeros_like(val)
            torch.testing.assert_close(dval.cpu(), _t(g[pre + "dval"]), rtol=RTOL, atol=1e-8, msg=name)
        keys = [str(k) for k in g[pre + "metric_keys"]]
        assert sorted(metrics) == keys, (name, sorted(metrics), keys)
        assert all(isinstance(v, float) for v in metrics.values())  # embodied: Python floats (SURVEY A10)
        for k, ref in zip(keys, g[pre + "metric_vals"]):
            tol = LOOSE.get(k, RTOL)
            np.testing.assert_allclose(metrics[k], ref, rtol=tol, atol=max(tol * 1e-2, 1e-7), err_msg=f"{name}:{k}")


def test_registered_loss_takes_preprocessed_kwargs(golden):
    """The registry-level callables accept the output of preprocess_loss_inputs (drop-in into the
    reference's LOSS_REGISTRY): compare against the oracle on reduced inputs."""
    import rlinf_b200.algorithms as A

    g = golden("loss")
    for name in ("ac_action_mask", "actor_token"):
        pre, Adim, lpt, lt, rt, hp = _loss_case(g, name)
        ac = lt == "actor_critic"
        p = O.reduce_loss_inputs(_t(g[pre + "new"]), _t(g[pre + "old"]), _t(g[pre + "adv"]), lpt, Adim,
                                 _t(g[pre + "mask"]), _t(g[pre + "mask_sum"]),
                                 _t(g[pre + "val"]) if ac else None, _t(g[pre + "prev_v"]) if ac else None,
                                 _t(g[pre + "ret"]) if ac else None, rt)
        kw = {k: (_cuda(v) if isinstance(v, torch.Tensor) else v) for k, v in p.items()}
        kw["logprobs"] = kw["logprobs"].requires_grad_(True)
        loss, metrics = A.LOSS_REGISTRY[lt](**kw, **hp)
        torch.testing.assert_close(loss.detach().cpu(), _t(g[pre + "loss"]), rtol=RTOL, atol=1e-7)
        assert all(isinstance(v, torch.Tensor) for v in metrics.values())


def test_policy_loss_large_matches_oracle():
    """N = 2^18 samples, A = 8, action_level actor_critic with mask + fused gather (idx)."""
    from rlinf_b200 import ops

    n, A = 1 << 18, 8
    g = torch.Generator().manual_seed(0)
    old = -1 + 0.3 * torch.randn(n, A, generator=g)
    new = old + 0.05 * torch.randn(n, A, generator=g)
    adv, ret, pv = torch.randn(n, 1, generator=g), torch.randn(n, 1, generator=g), torch.randn(n, 1, generator=g)
    val = pv + 0.1 * torch.randn(n, 1, generator=g)
    mask = torch.rand(n, 1, generator=g) < 0.9
    perm = O.shuffle_indices(n, 1234)
    hp = dict(clip_ratio_low=0.2, clip_ratio_high=0.2, value_clip=0.2, huber_delta=10.0)
    # our kernel gathers rollout rows through idx; the current-policy outputs are in micro-batch order
    loss, metrics, d_lp, d_v, _ = ops.ppo_loss(logprobs=new[perm].cuda(), values=val[perm].cuda(), old_logprobs=old.cuda(),
                                               advantages=adv.cuda(), returns=ret.cuda(), prev_values=pv.cuda(),
                                               loss_mask=mask.cuda(), idx=perm.cuda(), C_chunks=1, A_dim=A,
                                               logprob_type="action_level", **hp)
    newp = new[perm].clone().requires_grad_(True)
    valp = val[perm].clone().requires_grad_(True)
    oloss, ometrics = O.policy_loss_embodied("actor_critic", newp, old[perm], adv[perm], "action_level", A,
                                             loss_mask=mask[perm], values=valp, prev_values=pv[perm],
                                             returns=ret[perm], **hp)
    oloss.backward()
    torch.testing.assert_close(loss.cpu().reshape(()), oloss.detach(), rtol=RTOL, atol=1e-7)
    torch.testing.assert_close(d_lp.cpu(), newp.grad, rtol=RTOL, atol=1e-10)
    torch.testing.assert_close(d_v.cpu(), valp.grad, rtol=RTOL, atol=1e-10)
    m = metrics.cpu()
    from rlinf_b200 import _lib as L
    for slot, key in L.M_KEYS.items():
        if key in ometrics and key not in LOOSE:
            np.testing.assert_allclose(m[slot].item(), ometrics[key], rtol=RTOL, atol=1e-7, err_msg=key)


def test_deferred_normalisation_equals_materialised():
    from rlinf_b200 import ops

    T, B, A = 64, 256, 8
    r, v, d = _synth(3, T, B, 1, 0.02)
    adv, ret, stats = ops.gae(r[..., 0], v[..., 0], d[..., 0], 0.99, 0.95, None, want_stats=True)
    n = T * B
    g = torch.Generator().manual_seed(1)
    old = (-1 + 0.3 * torch.randn(n, A, generator=g)).cuda()
    new = old + 0.05 * torch.randn(n, A, generator=g).cuda()
    common = dict(logprobs=new, old_logprobs=old, C_chunks=1, A_dim=A, logprob_type="action_level")
    l1, m1, g1, _, _ = ops.ppo_loss(advantages=adv.reshape(n, 1), adv_stats=stats[:3].contiguous(), **common)
    advn = ops.normalize_(adv.clone(), stats[:3].contiguous())
    l2, m2, g2, _, _ = ops.ppo_loss(advantages=advn.reshape(n, 1), **common)
    assert torch.equal(l1, l2) and torch.equal(g1, g2)


def test_mlp_forward_backward_adamw_golden(golden):
    from rlinf_b200.policy import FlatAdamW, MLPPolicy

    g = golden("policy")
    names = [str(n) for n in g["pol_names"]]
    pol = MLPPolicy(obs_dim=12, action_dim=3, num_action_chunks=1)
    assert [n for n, _ in pol.named_parameters()] == names
    from test_oracle_golden import _golden_view, _policy_grads, _policy_init

    p0 = _policy_init(golden, names)
    pol.load_state_dict(p0)
    states, action = _t(g["pol_states"]).cuda(), _t(g["pol_action"]).cuda()
    out = pol.forward_train(states, action)
    torch.testing.assert_close(out["logprobs"].cpu(), _t(g["pol_logprobs"]), rtol=RTOL, atol=1e-5)
    torch.testing.assert_close(out["entropy"].cpu(), _t(g["pol_entropy"]), rtol=RTOL, atol=1e-6)
    torch.testing.assert_close(out["values"].cpu(), _t(g["pol_values"]), rtol=RTOL, atol=1e-5)
    pol.flat_grads.zero_()
    pol.backward(_t(g["pol_wl"]).cuda(), _t(g["pol_wv"]).cuda(), _t(g["pol_we"]).cuda())
    worst = 0.0
    for n, gr in pol.named_grads():
        got, ref = _golden_view(g, "pol_g_" + n, gr.cpu())
        # parameter gradients are sums over samples with cancellation: the bar is 1e-4 relative per element plus 1e-5 of
        # the tensor's own scale (round 1 used rtol 1e-3; measured max |diff| / max |ref| is printed)
        torch.testing.assert_close(got, ref, rtol=RTOL, atol=1e-5 * max(1.0, ref.abs().max().item()), msg=n)
        worst = max(worst, ((got - ref).abs().max() / ref.abs().max().clamp_min(1e-30)).item())
    print(f"max |dW - ref| / max |ref| over parameter tensors: {worst:.2e}")
    # optimiser: 3 steps with the fixture's seeded gradients
    for n, gr in pol.named_grads():
        gr.copy_(_policy_grads(p0)[n])
    opt = FlatAdamW(pol, lr=3e-4, value_lr=1e-3, clip_grad=0.5)
    norms = []
    for _ in range(3):
        opt.step()
        norms.append(opt.last_grad_norm().item())
        # the golden run clips IN PLACE (torch clip_grad_norm_) and keeps the clipped grads for the next
        # step; the kernel applies the coefficient on the fly, so replay the in-place scaling here
        pol.flat_grads.mul_(opt.state[2].float())
    np.testing.assert_allclose(norms, g["pol_gradnorms"], rtol=1e-5)
    for n, p in pol.named_parameters():
        torch.testing.assert_close(*_golden_view(g, "pol_p3_" + n, p.cpu()), rtol=1e-5, atol=1e-7, msg=n)
    assert opt.state[0].item() == 3


def test_mlp_config2_shapes_vs_oracle():
    """obs=128, act=8, n=5000 rows (not a tile multiple), gathered by idx; fwd + bwd vs the oracle."""
    from rlinf_b200.policy import MLPPolicy

    pol = MLPPolicy(obs_dim=128, action_dim=8, seed=7)
    params = {n: p.detach().cpu().clone().requires_grad_(True) for n, p in pol.named_parameters()}
    g = torch.Generator().manual_seed(5)
    N, n = 8192, 5000
    states, action = torch.randn(N, 128, generator=g), torch.randn(N, 8, generator=g)
    idx = torch.randperm(N, generator=g)[:n]
    out = pol.forward_train(states.cuda(), action.cuda(), idx=idx.cuda())
    o = O.mlp_forward(params, states[idx], action[idx])
    torch.testing.assert_close(out["logprobs"].cpu(), o["logprobs"], rtol=RTOL, atol=1e-5)
    torch.testing.assert_close(out["values"].cpu(), o["values"], rtol=RTOL, atol=1e-5)
    wl, wv = torch.randn(n, 8, generator=g) / n, torch.randn(n, 1, generator=g) / n
    ((o["logprobs"] * wl).sum() + (o["values"] * wv).sum()).backward()
    pol.flat_grads.zero_()
    pol.backward(wl.cuda(), wv.cuda(), None)
    worst = 0.0
    for name, gr in pol.named_grads():
        ref = params[name].grad
        torch.testing.assert_close(gr.cpu(), ref, rtol=RTOL, atol=2e-5 * max(ref.abs().max().item(), 1e-6), msg=name)
        worst = max(worst, ((gr.cpu() - ref).abs().max() / ref.abs().max().clamp_min(1e-30)).item())
    print(f"config-2 shapes: max |dW - ref| / max |ref| over parameter tensors: {worst:.2e}")


def test_mlp_sample_given_noise_vs_oracle():
    from rlinf_b200.policy import MLPPolicy

    pol = MLPPolicy(obs_dim=16, action_dim=4, seed=3)
    params = {n: p.detach().cpu() for n, p in pol.named_parameters()}
    g = torch.Generator().manual_seed(2)
    states, noise = torch.randn(300, 16, generator=g), torch.randn(300, 4, generator=g)
    a, lp, v = pol.sample(states.cuda(), noise=noise.cuda())
    oa, olp, ov = O.mlp_sample(params, states, noise)
    torch.testing.assert_close(a.cpu(), oa, rtol=RTOL, atol=1e-5)
    torch.testing.assert_close(lp.cpu(), olp, rtol=RTOL, atol=1e-5)
    torch.testing.assert_close(v.cpu(), ov, rtol=RTOL, atol=1e-5)
    # Philox path: statistics only (parity is on GIVEN noise, not on the RNG stream)
    a2, lp2, _ = pol.sample(states.cuda().repeat(40, 1), seed=11, offset=0)
    z = (a2 - a2.mean(0)) / a2.std(0)
    assert abs(z.mean().item()) < 0.05 and abs(z.std().item() - 1) < 0.05
    a3, _, _ = pol.sample(states.cuda().repeat(40, 1), seed=11, offset=0)
    assert torch.equal(a2, a3)
    # consecutive env steps (device counter t, t+1) must draw independent noise: the Philox offset advances by 4 words per
    # step, curand_normal consumes 2 (a stride of 1 made the angle word of step t the radius word of step t+1,
    # correlation of z_t^2 and z_{t+1}^2 about -0.06)
    big = torch.zeros(20000, 16, device="cuda")
    ctr = torch.zeros(1, dtype=torch.int64, device="cuda")
    zs = []
    for t in range(2):
        ctr.fill_(t)
        at, _, _ = pol.sample(big, seed=5, offset=0, counter=ctr)
        zs.append((at - at.mean(0)) / at.std(0))
    c = torch.corrcoef(torch.stack([(zs[0] ** 2).flatten(), (zs[1] ** 2).flatten()]))[0, 1].item()
    assert abs(c) < 0.015, c
    assert not torch.equal(zs[0], zs[1])


def test_reward_filter_golden(golden):
    from rlinf_b200 import ops

    g = golden("filter")
    for name in g["filt_cases"]:
        G, lo, hi, with_mask = g[f"filt_{name}_cfg"]
        r, d = _t(g[f"filt_{name}_rewards"]), _t(g[f"filt_{name}_dones"])
        mask = ops.loss_mask(d)[0] if with_mask else None
        out = ops.reward_filter(r, mask, int(G), float(lo), float(hi))
        ref = _t(g[f"filt_{name}_mask"])
        assert out.shape == ref.shape and torch.equal(out.cpu(), ref), name


def test_rollout_metrics_golden(golden):
    from rlinf_b200.metric_utils import compute_rollout_metrics

    g = golden("filter")
    buf = {k: _t(g["rm_" + k]).cuda() for k in ("rewards", "advantages", "returns", "loss_mask")}
    m = compute_rollout_metrics(buf)
    keys = [str(k) for k in g["rm_keys"]]
    assert sorted(m) == keys
    np.testing.assert_allclose([m[k] for k in keys], g["rm_vals"], rtol=1e-5, atol=1e-7)
    m2 = compute_rollout_metrics({"rewards": buf["rewards"], "advantages": buf["advantages"]})
    np.testing.assert_allclose(m2["advantages_max"], buf["advantages"].max().item())


@pytest.mark.parametrize("kind", ["k1", "abs", "k2", "k3"])
def test_kl_penalty_golden_and_grad(golden, kind):
    import rlinf_b200.algorithms.utils as U

    g = golden("loss")
    a, b = _t(g["kl_a"]), _t(g["kl_b"])
    ac = a.cuda().requires_grad_(True)
    out = U.kl_penalty(ac, b.cuda(), kind)
    torch.testing.assert_close(out.detach().cpu(), _t(g[f"kl_{kind}"]), rtol=1e-5, atol=1e-6)
    w = torch.linspace(-1, 1, a.numel())
    (out * w.cuda()).sum().backward()
    ar = a.clone().requires_grad_(True)
    (O.kl_penalty(ar, b, kind) * w).sum().backward()
    torch.testing.assert_close(ac.grad.cpu(), ar.grad, rtol=1e-5, atol=1e-6)
