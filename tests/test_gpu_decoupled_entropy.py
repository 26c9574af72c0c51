"""GPU checks of the decoupled actor-critic loss with the entropy bonus and one weight version per batch, against
reference-generated goldens (tests/golden/golden_async.npz), and of the fixed-order rb200_masked_moments."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _t(a):
    return torch.from_numpy(np.ascontiguousarray(np.asarray(a)))


def _case(g, name):
    pre = f"dec_{name}_"
    bsz, Cc, A, use_ratio, has_thr, k, accum = (int(x) for x in g[pre + "cfg"])
    thr, ent_bonus = (float(x) for x in g[pre + "hp"])
    lpt, rt = (str(x) for x in g[pre + "types"])
    has_mask = (pre + "mask") in g.files
    return dict(pre=pre, bsz=bsz, C=Cc, A=A, U=1 if rt == "chunk_level" else Cc, ratio=bool(use_ratio),
                thr=thr if has_thr > 0 else None, bonus=ent_bonus, k=k, accum=accum, lpt=lpt, rt=rt, has_mask=has_mask)


def _kernel_call(g, c, decoupled):
    from rlinf_b200 import ops

    pre, bsz, U = c["pre"], c["bsz"], c["U"]
    dev = torch.device("cuda")

    def unit(key):
        return _t(g[pre + key]).to(dev).reshape(bsz, U) if (pre + key) in g.files else None

    return ops.ppo_loss(
        logprobs=_t(g[pre + "new"]).to(dev), old_logprobs=_t(g[pre + "old"]).to(dev), advantages=unit("adv"),
        values=unit("val"), returns=unit("ret"), prev_values=unit("prev_v"), loss_mask=unit("mask"),
        loss_mask_sum=unit("mask_sum"), entropy=_t(g[pre + "ent"]).to(dev), C_chunks=c["C"], A_dim=c["A"],
        logprob_type=c["lpt"], clip_ratio_low=0.2, clip_ratio_high=0.28, clip_ratio_c=3.0, value_clip=0.2,
        huber_delta=1.5, max_episode_steps=50 if c["ratio"] else None, entropy_bonus=c["bonus"],
        loss_scale=1.0 / c["accum"], _decoupled=decoupled)


def _check_metrics(g, c, metrics, tag):
    pre = c["pre"]
    keys = [str(k) for k in g[pre + "metric_keys"]]
    assert sorted(metrics) == keys, (tag, sorted(metrics), keys)
    for k, want in zip(keys, g[pre + "metric_vals"]):
        if k == "critic/value_clip_ratio":  # rounding-noise metric (SURVEY A9)
            continue
        np.testing.assert_allclose(float(metrics[k]), want, rtol=1e-4, atol=2e-7, err_msg=f"{tag} {k}")


def test_scalar_version_entry_with_entropy_matches_reference(golden):
    from rlinf_b200 import _lib as L
    from rlinf_b200.algorithms.losses import _decoupled_metrics_dict

    g = golden("async")
    for name in (str(x) for x in g["dec_cases"]):
        c = _case(g, name)
        pre = c["pre"]
        loss, raw, d_lp, d_v, d_e = _kernel_call(
            g, c, dict(version=c["k"] - 1, current_version=c["k"] + 1, behave_weight_threshold=c["thr"]))
        torch.testing.assert_close(loss.cpu().reshape(()), _t(g[pre + "loss"]).reshape(()), rtol=1e-5, atol=1e-7)
        torch.testing.assert_close(d_lp.cpu(), _t(g[pre + "dnew"]), rtol=1e-4, atol=1e-9)
        torch.testing.assert_close(d_v.cpu(), _t(g[pre + "dval"]), rtol=1e-4, atol=1e-9)
        torch.testing.assert_close(d_e.cpu(), _t(g[pre + "dent"]), rtol=1e-4, atol=1e-9)
        metrics = _decoupled_metrics_dict(raw, as_float=True)
        host = raw.tolist()
        metrics["actor/entropy_loss"] = host[L.DM_ENTROPY]
        metrics["actor/total_loss"] = host[16]
        _check_metrics(g, c, metrics, f"{name}/scalar")


def test_scalar_version_is_bit_identical_to_per_token_versions(golden):
    g = golden("async")
    for name in (str(x) for x in g["dec_cases"]):
        c = _case(g, name)
        scalar = _kernel_call(g, c, dict(version=c["k"] - 1, current_version=c["k"] + 1,
                                         behave_weight_threshold=c["thr"]))
        versions = torch.full((c["bsz"], c["C"] * c["A"]), float(c["k"] - 1), device="cuda")
        per_token = _kernel_call(g, c, dict(versions=versions, current_version=c["k"] + 1,
                                            behave_weight_threshold=c["thr"]))
        for a, b in zip(scalar, per_token):
            assert torch.equal(a, b), name


def test_registry_decoupled_loss_with_entropy_matches_reference(golden):
    """The registry's fused route (policy_loss, task_type embodied) now takes the entropy term of the decoupled loss."""
    import rlinf_b200.algorithms as A

    g = golden("async")
    for name in (str(x) for x in g["dec_cases"]):
        c = _case(g, name)
        pre = c["pre"]
        new = _t(g[pre + "new"]).cuda().requires_grad_(True)
        val = _t(g[pre + "val"]).cuda().requires_grad_(True)
        ent = _t(g[pre + "ent"]).cuda().requires_grad_(True)
        kw = dict(task_type="embodied", loss_type="decoupled_actor_critic", logprob_type=c["lpt"], reward_type=c["rt"],
                  single_action_dim=c["A"], logprobs=new, old_logprobs=_t(g[pre + "old"]), advantages=_t(g[pre + "adv"]),
                  returns=_t(g[pre + "ret"]), values=val, prev_values=_t(g[pre + "prev_v"]), clip_ratio_high=0.28,
                  clip_ratio_low=0.2, clip_ratio_c=3.0, value_clip=0.2, huber_delta=1.5,
                  loss_mask=_t(g[pre + "mask"]) if c["has_mask"] else None,
                  loss_mask_sum=_t(g[pre + "mask_sum"]) if c["has_mask"] else None,
                  max_episode_steps=50 if c["ratio"] else None, critic_warmup=False,
                  versions=torch.full((c["bsz"], c["C"] * c["A"]), float(c["k"] - 1)),
                  current_version=c["k"] + 1, behave_weight_threshold=c["thr"], entropy=ent,
                  entropy_type=c["rt"], entropy_bonus=c["bonus"], loss_scale=1.0 / c["accum"])
        loss, metrics = A.policy_loss(**kw)
        loss.backward()
        torch.testing.assert_close(loss.detach().cpu(), _t(g[pre + "loss"]).reshape(()), rtol=1e-5, atol=1e-7)
        torch.testing.assert_close(new.grad.cpu(), _t(g[pre + "dnew"]), rtol=1e-4, atol=1e-9)
        torch.testing.assert_close(val.grad.cpu(), _t(g[pre + "dval"]), rtol=1e-4, atol=1e-9)
        torch.testing.assert_close(ent.grad.cpu(), _t(g[pre + "dent"]), rtol=1e-4, atol=1e-9)
        _check_metrics(g, c, metrics, f"{name}/registry")


def test_masked_moments_repeat_bit_for_bit():
    """Config-2 size (T 512 x B 4096): every call gives the same bits, within fp64 rounding of an fp64 sum."""
    from rlinf_b200 import ops

    gen = torch.Generator(device="cuda").manual_seed(5)
    x = torch.randn(512 * 4096, device="cuda", generator=gen) * 1.7 + 0.3
    m = torch.rand(512 * 4096, device="cuda", generator=gen) < 0.8
    first = ops.masked_moments(x, m)
    for _ in range(8):
        assert torch.equal(ops.masked_moments(x, m), first)
    xd = x.double()[m]
    want = torch.stack([torch.tensor(float(xd.numel()), dtype=torch.float64, device="cuda"), xd.sum(),
                        (xd * xd).sum()])
    torch.testing.assert_close(first, want, rtol=1e-12, atol=0)
    nomask = ops.masked_moments(x)
    assert torch.equal(ops.masked_moments(x), nomask) and float(nomask[0]) == x.numel()


def test_masked_normalization_of_flat_advantages_matches_reference(golden):
    from rlinf_b200.utils import masked_normalization

    g = golden("async")
    adv, mask = _t(g["mn_adv"]).cuda(), _t(g["mn_mask"]).cuda()
    torch.testing.assert_close(masked_normalization(adv, mask).cpu(), _t(g["mn_out_masked"]), rtol=1e-6, atol=1e-6)
    torch.testing.assert_close(masked_normalization(adv).cpu(), _t(g["mn_out_plain"]), rtol=1e-6, atol=1e-6)
