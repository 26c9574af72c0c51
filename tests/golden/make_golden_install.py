"""golden_install.npz for tests/test_install_reference.py, recorded from the UNMODIFIED reference executed in place
(tests/golden/ref_loader.py; run by hand where the reference tree exists): registry entry names, the parameter lists of
the registered callables and the logits helpers, and the kwargs the reference's dispatchers (registry.py:77-124) hand
the registered callable for the kwargs its workers build, captured by recording stand-ins.

    python tests/golden/make_golden_install.py
"""
from __future__ import annotations

import inspect
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import ref_loader  # noqa: E402


def worker_kwargs():
    T, B, A = 6, 8, 3
    g = torch.Generator().manual_seed(0)
    rewards, values = torch.randn(T, B, 1, generator=g), torch.randn(T + 1, B, 1, generator=g)
    dones = torch.zeros(T + 1, B, 1, dtype=torch.bool)
    adv_kw = dict(task_type="embodied", rewards=rewards, dones=dones, values=values, prev_logprobs=None,
                  teacher_logprobs=None, num_action_chunks=1, gamma=0.99, gae_lambda=0.95, group_size=4,
                  reward_type="action_level", loss_mask=None, loss_mask_sum=None, advantage_mode=None)
    adv = {}
    for adv_type in ("gae", "grpo", "raw", "reinpp"):
        kw = dict(adv_kw, adv_type=adv_type)
        if adv_type != "gae":
            lm = torch.ones(T, B, 1, dtype=torch.bool)
            kw.update(loss_mask=lm, loss_mask_sum=lm.sum(0, keepdim=True).expand_as(lm))
        adv[adv_type] = kw
    n = T * B
    loss_kw = dict(loss_type="actor_critic", logprob_type="action_level", reward_type="action_level", single_action_dim=A,
                   logprobs=torch.randn(n, A, generator=g), values=torch.randn(n, 1, generator=g),
                   old_logprobs=torch.randn(n, A, generator=g), advantages=torch.randn(n, 1, generator=g),
                   returns=torch.randn(n, 1, generator=g), prev_values=torch.randn(n, 1, generator=g), clip_ratio_high=0.2,
                   clip_ratio_low=0.2, value_clip=0.2, huber_delta=10.0, loss_mask=None, loss_mask_sum=None,
                   max_episode_steps=80, task_type="embodied", critic_warmup=False)
    loss = {t: dict(loss_kw, loss_type=t) for t in ("actor_critic", "actor", "decoupled_actor_critic")}
    return adv, loss


class _Recorded(Exception):
    pass


def _put_value(out, key, v):  # n: None, t: tensor, s: python scalar / string
    if v is None:
        out[f"n:{key}"] = np.zeros(0)
    elif isinstance(v, torch.Tensor):
        out[f"t:{key}"] = v.detach().contiguous().numpy()
    else:
        assert isinstance(v, (bool, int, float, str)), (key, type(v))
        out[f"s:{key}"] = np.asarray(v)


def main():
    ref = ref_loader.load_reference()
    import importlib

    importlib.import_module("rlinf.algorithms.loss_scales")
    reg = ref.registry
    out = {}
    for tag, r in (("adv", reg.ADV_REGISTRY), ("loss", reg.LOSS_REGISTRY), ("loss_scale", reg.LOSS_SCALE_REGISTRY)):
        out[f"reg:{tag}"] = np.asarray(sorted(r))
        if tag == "loss_scale":
            continue
        for name, fn in r.items():
            rows = []
            for pname, p in inspect.signature(inspect.unwrap(fn)).parameters.items():
                has = p.default is not inspect.Parameter.empty
                rows.append("|".join((pname, p.kind.name, "1" if has else "0", repr(p.default) if has else "")))
            out[f"sig:{tag}:{name}"] = np.asarray(rows)
    for name in ("compute_logprobs_from_logits", "compute_entropy_from_logits"):
        out[f"util:{name}"] = np.asarray(list(inspect.signature(getattr(ref.utils, name)).parameters))

    adv, loss = worker_kwargs()
    for tag, registry, dispatch, cases in (("adv", reg.ADV_REGISTRY, reg.calculate_adv_and_returns, adv),
                                           ("loss", reg.LOSS_REGISTRY, reg.policy_loss, loss)):
        saved = dict(registry)
        try:
            for case, kw in cases.items():
                seen = {}

                def make(name):
                    def rec(**kwargs):
                        seen["name"], seen["kwargs"] = name, kwargs
                        raise _Recorded()
                    return rec

                for name in saved:
                    registry[name] = make(name)
                try:
                    dispatch(**kw)
                except _Recorded:
                    pass
                out[f"target:{tag}:{case}"] = np.asarray(seen["name"])
                for k, v in seen["kwargs"].items():
                    if k == "loss_agg_func":  # a callable default of the reference; selected inside the fused kernel here
                        continue
                    _put_value(out, f"call:{tag}:{case}:{k}", v)
        finally:
            registry.clear()
            registry.update(saved)
    path = os.path.join(HERE, "golden_install.npz")
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), "bytes,", len(out), "arrays")


if __name__ == "__main__":
    main()
