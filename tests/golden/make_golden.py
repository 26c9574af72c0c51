"""Generate golden input/output vectors by EXECUTING the unmodified reference.

Run here (build container) only:  python tests/golden/make_golden.py
Writes tests/golden/*.npz (small, committed).  The reference's own tests hold no
golden vector for this path (SURVEY.md §4), so these fixtures - outputs of the
reference itself on seeded inputs - are what pins the oracle and the CUDA path.
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from ref_loader import load_reference  # noqa: E402


def _np(x):
    if isinstance(x, torch.Tensor):
        return x.detach().cpu().numpy().copy()
    return np.asarray(x)


def synth_rollout(seed, nc, B, C, p_done=0.05):
    g = torch.Generator().manual_seed(seed)
    rewards = torch.randn(nc, B, C, generator=g)
    values = torch.randn(nc + 1, B, C, generator=g)
    dones = torch.rand(nc + 1, B, C, generator=g) < p_done
    dones[0] = False
    return rewards, values, dones


def gen_adv(ref, out):
    cases = []
    #      name        seed nc  B  C  gamma lam  p_done
    specs = [("c1", 0, 32, 64, 1, 0.99, 0.95, 0.05),
             ("yaml", 1, 50, 96, 1, 0.8, 0.9, 0.02),
             ("chunk4", 2, 12, 40, 4, 0.99, 0.95, 0.05),
             ("nodone", 3, 40, 33, 1, 0.99, 0.95, 0.0),
             ("ragged", 4, 17, 21, 1, 0.97, 0.9, 0.2)]
    for name, seed, nc, B, C, gamma, lam, pd in specs:
        r, v, d = synth_rollout(seed, nc, B, C, pd)
        mask, mask_sum = ref.metric_utils.compute_loss_mask(d)
        out[f"adv_{name}_rewards"], out[f"adv_{name}_values"], out[f"adv_{name}_dones"] = _np(r), _np(v), _np(d)
        out[f"adv_{name}_hp"] = np.array([gamma, lam], dtype=np.float64)
        out[f"adv_{name}_mask"], out[f"adv_{name}_mask_sum"] = _np(mask), _np(mask_sum.contiguous())
        common = dict(task_type="embodied", rewards=r, dones=d, values=v, gamma=gamma,
                      gae_lambda=lam, group_size=8, reward_type="action_level",
                      num_action_chunks=C, prev_logprobs=None, teacher_logprobs=None,
                      advantage_mode=None)
        for mk, (lm, lms) in {"nomask": (None, None), "mask": (mask, mask_sum)}.items():
            res = ref.registry.calculate_adv_and_returns(adv_type="gae", loss_mask=lm, loss_mask_sum=lms, **common)
            out[f"adv_{name}_gae_{mk}_adv"], out[f"adv_{name}_gae_{mk}_ret"] = _np(res["advantages"].contiguous()), _np(res["returns"].contiguous())
        # un-normalised GAE (direct registry fn call on step-major tensors) for the bit-exact check
        p = ref.alg_utils.preprocess_embodied_advantages_inputs(adv_type="gae", loss_mask=None, loss_mask_sum=None, **{k: common[k] for k in ("rewards", "dones", "values", "reward_type")})
        a, rt = ref.advantages.compute_gae_advantages_and_returns(rewards=p["rewards"], values=p["values"], dones=p["dones"], gamma=gamma, gae_lambda=lam, normalize_advantages=False)
        out[f"adv_{name}_gae_raw_adv"], out[f"adv_{name}_gae_raw_ret"] = _np(a.contiguous()), _np(rt.contiguous())
        if B % 8 == 0:
            res = ref.registry.calculate_adv_and_returns(adv_type="grpo", loss_mask=mask, loss_mask_sum=mask_sum, **common)
            out[f"adv_{name}_grpo_adv"] = _np(res["advantages"].contiguous())
            assert "returns" not in res
            sc = ref.alg_utils.calculate_scores(rewards=p["rewards"], dones=p["dones"], batch_size=B, n_steps=nc * C, group_size=8)["rewards"]
            out[f"adv_{name}_grpo_scores"] = _np(sc.contiguous())
        cases.append(name)
    # critic-free GAE (values None) on step-major input
    r, v, d = synth_rollout(7, 20, 16, 1, 0.1)
    a, rt = ref.advantages.compute_gae_advantages_and_returns(rewards=r[..., 0], values=None, dones=d[..., 0], gamma=0.9, gae_lambda=0.8, normalize_advantages=False)
    out["adv_critic_free_rewards"], out["adv_critic_free_dones"] = _np(r[..., 0]), _np(d[..., 0])
    out["adv_critic_free_adv"], out["adv_critic_free_ret"] = _np(a), _np(rt)
    # reasoning branch
    g = torch.Generator().manual_seed(11)
    bsz, L = 16, 24
    rew = torch.randn(bsz, generator=g)
    vals = torch.randn(bsz, L, generator=g)
    lens = torch.randint(4, L + 1, (bsz,), generator=g)
    lm = torch.arange(L).unsqueeze(0) < lens.unsqueeze(1)
    adv, ret = ref.registry.calculate_adv_and_returns(task_type="reasoning", adv_type="gae", rewards=rew, loss_mask=lm, values=vals, gamma=1.0, gae_lambda=0.95, normalize_advantages=False)
    out["reason_rewards"], out["reason_values"], out["reason_mask"] = _np(rew), _np(vals), _np(lm)
    out["reason_gae_adv"], out["reason_gae_ret"] = _np(adv), _np(ret)
    adv, ret = ref.registry.calculate_adv_and_returns(task_type="reasoning", adv_type="grpo", rewards=rew, loss_mask=lm, group_size=4)
    assert ret is None
    out["reason_grpo_adv"] = _np(adv)
    out["adv_cases"] = np.array(cases)


def gen_loss(ref, out):
    cases = []
    specs = [
        # name, seed, bsz, C, A, logprob_type, loss_type, mask?, ratio-agg?, dual-clip?, clamp?
        ("ac_action", 0, 96, 1, 8, "action_level", "actor_critic", False, False, False, False),
        ("ac_action_mask", 1, 80, 1, 8, "action_level", "actor_critic", True, False, False, False),
        ("ac_action_ratio", 2, 64, 1, 8, "action_level", "actor_critic", True, True, False, False),
        ("ac_chunk3", 3, 48, 3, 7, "action_level", "actor_critic", True, False, True, True),
        ("actor_token", 4, 40, 2, 7, "token_level", "actor", True, False, False, False),
        ("actor_chunklvl", 5, 56, 4, 7, "chunk_level", "actor", False, False, True, False),
        ("ac_allmasked", 6, 32, 1, 8, "action_level", "actor_critic", "zero", False, False, False),
    ]
    for name, seed, bsz, C, A, lpt, lt, use_mask, use_ratio, dual, clamp in specs:
        g = torch.Generator().manual_seed(100 + seed)
        old = -1.0 + 0.3 * torch.randn(bsz, C * A, generator=g)
        new = (old + 0.15 * torch.randn(bsz, C * A, generator=g)).requires_grad_(True)
        reward_type = "chunk_level" if lpt == "chunk_level" else "action_level"
        per = 1 if reward_type == "chunk_level" else C
        adv = torch.randn(bsz, per, generator=g)
        ret = torch.randn(bsz, per, generator=g)
        prev_v = torch.randn(bsz, per, generator=g)
        val = (prev_v + 0.3 * torch.randn(bsz, per, generator=g)).requires_grad_(True)
        if use_mask == "zero":
            mask = torch.zeros(bsz, per, dtype=torch.bool)
        elif use_mask:
            mask = torch.rand(bsz, per, generator=g) < 0.7
        else:
            mask = None
        mask_sum = torch.randint(1, 50, (bsz, 1), generator=g).expand(bsz, per).contiguous() if mask is not None else None
        kw = dict(task_type="embodied", loss_type=lt, logprob_type=lpt, reward_type=reward_type,
                  single_action_dim=A, logprobs=new, old_logprobs=old, advantages=adv,
                  returns=ret if lt == "actor_critic" else None,
                  values=val if lt == "actor_critic" else None,
                  prev_values=prev_v if lt == "actor_critic" else None,
                  clip_ratio_high=0.28, clip_ratio_low=0.2, value_clip=0.2, huber_delta=1.5,
                  loss_mask=mask, loss_mask_sum=mask_sum,
                  max_episode_steps=50 if use_ratio else None, critic_warmup=False)
        if dual:
            kw["clip_ratio_c"] = 3.0
        if clamp:
            kw["clip_log_ratio_min"], kw["clip_log_ratio_max"] = -0.2, 0.25
        loss, metrics = ref.registry.policy_loss(**kw)
        loss.backward()
        pre = f"loss_{name}_"
        out[pre + "old"], out[pre + "new"], out[pre + "adv"] = _np(old), _np(new), _np(adv)
        out[pre + "ret"], out[pre + "prev_v"], out[pre + "val"] = _np(ret), _np(prev_v), _np(val)
        if mask is not None:
            out[pre + "mask"], out[pre + "mask_sum"] = _np(mask), _np(mask_sum)
        out[pre + "cfg"] = np.array([bsz, C, A, int(use_ratio), int(dual), int(clamp)], dtype=np.int64)
        out[pre + "types"] = np.array([lpt, lt, reward_type])
        out[pre + "loss"] = _np(loss)
        out[pre + "dnew"] = _np(new.grad if new.grad is not None else torch.zeros_like(new))
        if lt == "actor_critic":
            out[pre + "dval"] = _np(val.grad if val.grad is not None else torch.zeros_like(val))
        keys = sorted(metrics)
        out[pre + "metric_keys"] = np.array(keys)
        out[pre + "metric_vals"] = np.array([float(metrics[k]) for k in keys], dtype=np.float64)
        cases.append(name)
    out["loss_cases"] = np.array(cases)
    # kl_penalty
    g = torch.Generator().manual_seed(5)
    a, b = torch.randn(257, generator=g), torch.randn(257, generator=g)
    out["kl_a"], out["kl_b"] = _np(a), _np(b)
    for kind in ("k1", "abs", "k2", "k3"):
        out[f"kl_{kind}"] = _np(ref.alg_utils.kl_penalty(a, b, kind))


def gen_filter_and_metrics(ref, out):
    import torch.distributed as dist
    cases = []
    for name, seed, nc, B, C, G, lo, hi, with_mask in [("f1", 0, 12, 32, 1, 8, -1.0, 1.0, True),
                                                         ("f2", 1, 9, 24, 2, 4, -0.5, 2.0, False),
                                                         ("f3", 2, 20, 64, 1, 8, 0.0, 100.0, True)]:
        r, v, d = synth_rollout(seed, nc, B, C, 0.1)
        batch = {"rewards": r, "dones": d}
        res = ref.utils.preprocess_embodied_batch(batch, rollout_epoch=1, auto_reset=not with_mask,
                                                  ignore_terminations=False, reward_type="action_level",
                                                  filter_rewards=True, group_size=G, rewards_lower_bound=lo,
                                                  rewards_upper_bound=hi)
        out[f"filt_{name}_rewards"], out[f"filt_{name}_dones"] = _np(r), _np(d)
        out[f"filt_{name}_cfg"] = np.array([G, lo, hi, int(with_mask)], dtype=np.float64)
        out[f"filt_{name}_mask"] = _np(res["loss_mask"].contiguous())
        cases.append(name)
    out["filt_cases"] = np.array(cases)
    # compute_rollout_metrics needs a process group: 1-rank gloo
    if not dist.is_initialized():
        import os
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        os.environ.setdefault("MASTER_PORT", "29533")
        dist.init_process_group("gloo", rank=0, world_size=1)
    g = torch.Generator().manual_seed(21)
    buf = {"rewards": torch.randn(16, 24, 1, generator=g), "advantages": torch.randn(16, 24, 1, generator=g),
           "returns": torch.randn(16, 24, 1, generator=g), "loss_mask": torch.rand(16, 24, 1, generator=g) < 0.7}
    m = ref.metric_utils.compute_rollout_metrics(buf)
    for k, v in buf.items():
        out["rm_" + k] = _np(v)
    keys = sorted(m)
    out["rm_keys"] = np.array(keys)
    out["rm_vals"] = np.array([float(m[k]) for k in keys])


def gen_indexing(ref, out):
    g = torch.Generator().manual_seed(9)
    T, B = 6, 10
    batch = {
        "rewards": torch.randn(T, B, 1, generator=g),
        "dones": torch.rand(T + 1, B, 1, generator=g) < 0.2,
        "prev_values": torch.randn(T + 1, B, 1, generator=g),
        "prev_logprobs": torch.randn(T, B, 3, generator=g),
        "forward_inputs": {"states": torch.randn(T, B, 5, generator=g), "action": torch.randn(T, B, 3, generator=g)},
    }
    gen = torch.Generator()
    gen.manual_seed(1234 + 3)
    perm = torch.randperm(T * B, generator=gen)
    res = ref.nested.process_nested_dict_for_train(batch, perm)
    out["idx_perm"] = _np(perm)
    for k in ("rewards", "dones", "prev_values", "prev_logprobs"):
        out["idx_in_" + k], out["idx_out_" + k] = _np(batch[k]), _np(res[k])
    out["idx_in_states"], out["idx_out_states"] = _np(batch["forward_inputs"]["states"]), _np(res["forward_inputs"]["states"])
    # epoch merge
    E = 2
    x = torch.arange(E * 3 * 4 * 2, dtype=torch.float32).reshape(E * 3, 4, 2)
    out["merge_in"], out["merge_out"] = _np(x), _np(ref.nested.process_nested_dict_for_adv({"x": x}, E)["x"].contiguous())
    # a large-N permutation checksum (bit-exact RNG stream): N = 4096*512
    gen.manual_seed(1234)
    big = torch.randperm(4096 * 512, generator=gen)
    out["idx_big_head"] = _np(big[:64])
    out["idx_big_checksum"] = np.array([int((big * torch.arange(big.numel())).sum() % (2**61 - 1))], dtype=np.int64)


def policy_grads(params):
    """Seeded gradients the fixture's three optimiser steps consume (the tests regenerate them)."""
    g = torch.Generator().manual_seed(4)
    return {n: 1e-2 * torch.randn(p.shape, generator=g) for n, p in params.items()}


def gen_policy(ref, out):
    from make_golden_r5 import snapshot

    torch.manual_seed(42)
    pol = ref.mlp_policy.MLPPolicy(obs_dim=12, action_dim=3, num_action_chunks=1, add_value_head=True, add_q_head=False)
    with torch.no_grad():  # make biases / logstd non-trivial
        for p in pol.parameters():
            if p.dim() == 1:
                p.add_(0.05 * torch.randn_like(p))
        pol.actor_logstd.add_(0.1 * torch.randn_like(pol.actor_logstd))
    names = [n for n, _ in pol.named_parameters()]
    out["pol_names"] = np.array(names)
    p0 = {n: p.detach().clone() for n, p in pol.named_parameters()}
    for n, p in p0.items():  # initial parameters: value head / policy halves in two files (each < 1 MB)
        out[("pinit_v:" if n.startswith("value_head") else "pinit:") + "pol_p_" + n] = _np(p)
    g = torch.Generator().manual_seed(3)
    states = torch.randn(37, 12, generator=g)
    action = torch.randn(37, 3, generator=g)
    o = pol.default_forward({"states": states, "action": action})
    out["pol_states"], out["pol_action"] = _np(states), _np(action)
    out["pol_logprobs"], out["pol_entropy"], out["pol_values"] = _np(o["logprobs"]), _np(o["entropy"]), _np(o["values"])
    # gradient of a scalar functional, for the backward kernel
    wl = torch.randn(37, 3, generator=g)
    wv = torch.randn(37, 1, generator=g)
    we = torch.randn(37, 3, generator=g)
    s = (o["logprobs"] * wl).sum() + (o["values"] * wv).sum() + (o["entropy"] * we).sum()
    s.backward()
    out["pol_wl"], out["pol_wv"], out["pol_we"] = _np(wl), _np(wv), _np(we)
    for n, p in pol.named_parameters():
        out.update({"pol_g_" + n + k: v for k, v in snapshot(p.grad).items()})
        p.grad = policy_grads(p0)[n]
    # 3 AdamW steps with the reference's grouping / clipping semantics (no_shard path)
    actor = [p for n, p in pol.named_parameters() if "value_head" not in n]
    critic = [p for n, p in pol.named_parameters() if "value_head" in n]
    opt = torch.optim.AdamW([{"params": actor, "lr": 3e-4, "betas": (0.9, 0.999)},
                             {"params": critic, "lr": 1e-3, "betas": (0.9, 0.999)}], eps=1e-8, weight_decay=1e-2)
    norms = []
    for step in range(3):
        gn = torch.nn.utils.clip_grad_norm_(pol.parameters(), 0.5)
        norms.append(float(gn))
        opt.step()
        # keep the same grads (deterministic known-answer)
    out["pol_gradnorms"] = np.array(norms)
    for n, p in pol.named_parameters():
        out.update({"pol_p3_" + n + k: v for k, v in snapshot(p).items()})


def gen_next(ref, out):
    """SURVEY §8(f) rank 4: registry entries next in line (decoupled PPO loss, raw / reinforce++ advantages)."""
    # ---- reasoning advantages: raw, reinpp ----
    g = torch.Generator().manual_seed(11)
    bsz, L, G = 24, 13, 4
    rewards = torch.randn(bsz, generator=g)
    lens = torch.randint(2, L + 1, (bsz,), generator=g)
    mask = torch.arange(L)[None, :] < lens[:, None]
    lp = -1 + 0.3 * torch.randn(bsz, L, generator=g)
    rlp = lp + 0.1 * torch.randn(bsz, L, generator=g)
    out["next_rewards"], out["next_mask"], out["next_lp"], out["next_rlp"] = _np(rewards), _np(mask), _np(lp), _np(rlp)
    out["next_group_size"] = np.array([G], dtype=np.int64)
    for name, kw in (("raw", dict(adv_type="raw", normalize_advantages=False)),
                     ("raw_norm", dict(adv_type="raw", normalize_advantages=True)),
                     ("reinpp", dict(adv_type="reinpp")),
                     ("reinpp_kl", dict(adv_type="reinpp", kl_beta=0.05, logprob=lp, ref_logprob=rlp,
                                        kl_penalty_type="k3"))):
        a, r = ref.registry.calculate_adv_and_returns(task_type="reasoning", rewards=rewards.clone(), loss_mask=mask,
                                                      group_size=G, **kw)
        assert r is None
        out["next_adv_" + name] = _np(a)
    try:
        ref.registry.calculate_adv_and_returns(task_type="reasoning", adv_type="reinpp", rewards=rewards.clone(),
                                               loss_mask=mask, group_size=G, use_reinpp_baseline=True)
        out["next_reinpp_baseline_raises"] = np.array([0])
    except IndexError:
        out["next_reinpp_baseline_raises"] = np.array([1])

    # ---- decoupled PPO actor-critic loss ----
    cases = []
    specs = [
        # name, seed, bsz, C, A, logprob_type, mask?, ratio-agg?, dual?, proximal (given/versions/none), threshold
        ("dec_none", 0, 64, 1, 8, "action_level", False, False, False, "none", None),
        ("dec_given_mask", 1, 72, 1, 8, "action_level", True, False, True, "given", 1.15),
        ("dec_versions", 2, 48, 2, 7, "action_level", True, True, False, "versions", None),
        ("dec_versions_chunk", 3, 40, 3, 7, "chunk_level", False, False, True, "versions", 1.05),
    ]
    for name, seed, bsz, C, A, lpt, use_mask, use_ratio, dual, prox, thr in specs:
        g = torch.Generator().manual_seed(300 + seed)
        old = -1.0 + 0.3 * torch.randn(bsz, C * A, generator=g)
        new = (old + 0.15 * torch.randn(bsz, C * A, generator=g)).requires_grad_(True)
        reward_type = "chunk_level" if lpt == "chunk_level" else "action_level"
        per = 1 if reward_type == "chunk_level" else C
        adv = torch.randn(bsz, per, generator=g)
        ret = torch.randn(bsz, per, generator=g)
        prev_v = torch.randn(bsz, per, generator=g)
        val = (prev_v + 0.3 * torch.randn(bsz, per, generator=g)).requires_grad_(True)
        mask = (torch.rand(bsz, per, generator=g) < 0.7) if use_mask else None
        mask_sum = torch.randint(1, 50, (bsz, 1), generator=g).expand(bsz, per).contiguous() if use_mask else None
        proximal = (old + 0.05 * torch.randn(bsz, C * A, generator=g)) if prox == "given" else None
        versions = torch.randint(-1, 6, (bsz, 1), generator=g).expand(bsz, C * A).contiguous().float() \
            if prox == "versions" else None
        kw = dict(task_type="embodied", loss_type="decoupled_actor_critic", logprob_type=lpt, reward_type=reward_type,
                  single_action_dim=A, logprobs=new, old_logprobs=old, advantages=adv, returns=ret, values=val,
                  prev_values=prev_v, clip_ratio_high=0.28, clip_ratio_low=0.2, value_clip=0.2, huber_delta=1.5,
                  loss_mask=mask, loss_mask_sum=mask_sum, max_episode_steps=50 if use_ratio else None,
                  critic_warmup=False, proximal_logprobs=proximal, versions=versions,
                  current_version=5.0 if prox == "versions" else None, behave_weight_threshold=thr)
        if dual:
            kw["clip_ratio_c"] = 3.0
        loss, metrics = ref.registry.policy_loss(**kw)
        loss.backward()
        pre = f"dec_{name}_"
        out[pre + "old"], out[pre + "new"], out[pre + "adv"] = _np(old), _np(new), _np(adv)
        out[pre + "ret"], out[pre + "prev_v"], out[pre + "val"] = _np(ret), _np(prev_v), _np(val)
        if mask is not None:
            out[pre + "mask"], out[pre + "mask_sum"] = _np(mask), _np(mask_sum)
        if proximal is not None:
            out[pre + "proximal"] = _np(proximal)
        if versions is not None:
            out[pre + "versions"] = _np(versions)
        out[pre + "cfg"] = np.array([bsz, C, A, int(use_ratio), int(dual), -1 if thr is None else 1], dtype=np.int64)
        out[pre + "thr"] = np.array([0.0 if thr is None else thr], dtype=np.float64)
        out[pre + "types"] = np.array([lpt, reward_type, prox])
        out[pre + "loss"] = _np(loss)
        out[pre + "dnew"] = _np(new.grad if new.grad is not None else torch.zeros_like(new))
        out[pre + "dval"] = _np(val.grad if val.grad is not None else torch.zeros_like(val))
        keys = sorted(metrics)
        out[pre + "metric_keys"] = np.array(keys)
        out[pre + "metric_vals"] = np.array([float(metrics[k]) for k in keys], dtype=np.float64)
        cases.append(name)
    out["dec_cases"] = np.array(cases)

    # ---- grpo_video advantages (step-level video rewards) ----
    g = torch.Generator().manual_seed(21)
    steps, B, G = 7, 24, 4
    vr = torch.randn(steps, B, generator=g)
    vm = (torch.rand(steps, B, generator=g) < 0.8).float()
    out["vid_rewards"], out["vid_mask"] = _np(vr), _np(vm)
    for mode in ("frame", "video"):
        a, r = ref.advantages.compute_grpo_video_advantages(rewards=vr.clone(), loss_mask=vm, group_size=G,
                                                            advantage_mode=mode)
        assert r is None
        out["vid_adv_" + mode] = _np(a)

    # ---- OPD (on-policy distillation): advantages + actor loss ----
    g = torch.Generator().manual_seed(22)
    Tn, B, C, tok = 6, 10, 2, 7
    student = -1.0 + 0.3 * torch.randn(Tn + 1, B, C * tok, generator=g)
    teacher = student + 0.2 * torch.randn(Tn + 1, B, C * tok, generator=g)
    lmask = torch.rand(Tn, B, C, generator=g) < 0.8
    a, r = ref.advantages.compute_opd_advantages(prev_logprobs=student, teacher_logprobs=teacher, loss_mask=lmask,
                                                 normalize_advantages=False, num_action_chunks=C)
    assert r is None
    out["opd_student"], out["opd_teacher"], out["opd_mask"], out["opd_adv"] = _np(student), _np(teacher), _np(lmask), _np(a)
    n = Tn * B
    lp = (student[:Tn].reshape(n, C, tok) + 0.05 * torch.randn(n, C, tok, generator=g)).requires_grad_(True)
    adv = a.reshape(n, C, tok).contiguous()
    m2 = lmask.reshape(n, C)
    msum = torch.randint(1, 40, (n, 1), generator=g).expand(n, C).contiguous()
    for name, mes in (("mean", None), ("ratio", 50)):
        if lp.grad is not None:
            lp.grad = None
        loss, metrics = ref.losses.compute_opd_actor_loss(logprobs=lp, advantages=adv, loss_mask=m2, loss_mask_sum=msum,
                                                          max_episode_steps=mes)
        loss.backward()
        out[f"opd_{name}_loss"], out[f"opd_{name}_dlp"] = _np(loss), _np(lp.grad)
        keys = sorted(metrics)
        out[f"opd_{name}_metric_keys"] = np.array(keys)
        out[f"opd_{name}_metric_vals"] = np.array([float(metrics[k]) for k in keys], dtype=np.float64)
    out["opd_lp"], out["opd_msum"] = _np(lp), _np(msum)


def main():
    ref = load_reference()
    torch.set_num_threads(1)
    for fn, name in ((gen_adv, "adv"), (gen_loss, "loss"), (gen_indexing, "indexing"), (gen_policy, "policy"),
                     (gen_filter_and_metrics, "filter"), (gen_next, "next")):
        out = {}
        fn(ref, out)
        for part in ("pinit_v", "pinit", ""):  # "<file suffix>:" key prefixes route arrays to golden_<name>_<suffix>.npz
            sel = {k.split(":", 1)[-1]: out.pop(k) for k in list(out) if not part or k.startswith(part + ":")}
            if sel:
                path = os.path.join(HERE, f"golden_{name}{'_' + part if part else ''}.npz")
                np.savez_compressed(path, **sel)
                print(name, part, len(sel), "arrays ->", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
