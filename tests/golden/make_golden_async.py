"""Generate tests/golden/golden_async.npz from the UNMODIFIED reference (RLinf v0.4.0), for the async PPO pieces.

    python tests/golden/make_golden_async.py

Runs, on seeded inputs, through the stub import of ref_loader.py (SURVEY.md §8c); only outputs are stored:
  dec_*  registry.policy_loss(loss_type="decoupled_actor_critic") followed by the async worker's entropy term and
         gradient-accumulation division (async_ppo_fsdp_worker.py:441-463: reshape_entropy + masked_mean), with
         versions = k - 1 for every token and current_version = k + 1; loss, metrics and the gradients of the
         log-probs, values and entropy.  Token, action and chunk log-prob levels, with and without a behaviour-weight
         threshold, a loss mask and masked_mean_ratio (max_episode_steps).
  mn_*   masked_normalization (rlinf/utils/distributed.py) of flattened advantages with a loss mask, as the worker
         applies it after the shuffle (async_ppo_fsdp_worker.py:293-297).
"""
from __future__ import annotations

import importlib
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from ref_loader import load_reference  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden_async.npz")


def _np(t):
    return t.detach().cpu().numpy() if isinstance(t, torch.Tensor) else np.asarray(t)


# name, seed, bsz, C, A, logprob_type, mask?, ratio-agg?, threshold, entropy_bonus, k (learner version), grad_accum
SPECS = [
    ("token_plain", 0, 40, 2, 7, "token_level", False, False, None, 0.01, 3, 1),
    ("token_mask_thr", 1, 48, 2, 7, "token_level", True, False, 1.2, 0.05, 1, 2),
    ("action_mask_ratio", 2, 56, 3, 6, "action_level", True, True, None, 0.02, 4, 1),
    ("action_thr_ratio", 3, 64, 2, 8, "action_level", True, True, 1.1, 0.03, 2, 4),
    ("chunk_plain_thr", 4, 36, 1, 8, "chunk_level", False, False, 1.3, 0.01, 5, 1),
    ("chunk_mask_ratio", 5, 44, 1, 5, "chunk_level", True, True, None, 0.04, 1, 2),
]


def gen_loss(ref, out):
    utils = ref.utils
    cases = []
    for name, seed, bsz, C, A, lpt, use_mask, use_ratio, thr, ent_bonus, k, accum in SPECS:
        g = torch.Generator().manual_seed(700 + seed)
        old = -1.0 + 0.3 * torch.randn(bsz, C * A, generator=g)
        new = (old + 0.15 * torch.randn(bsz, C * A, generator=g)).requires_grad_(True)
        reward_type = "chunk_level" if lpt == "chunk_level" else "action_level"
        per = 1 if reward_type == "chunk_level" else C
        adv = torch.randn(bsz, per, generator=g)
        ret = torch.randn(bsz, per, generator=g)
        prev_v = torch.randn(bsz, per, generator=g)
        val = (prev_v + 0.3 * torch.randn(bsz, per, generator=g)).requires_grad_(True)
        ent = (0.5 + 0.2 * torch.rand(bsz, C * A, generator=g)).requires_grad_(True)
        mask = (torch.rand(bsz, per, generator=g) < 0.7) if use_mask else None
        mask_sum = torch.randint(1, 50, (bsz, 1), generator=g).expand(bsz, per).contiguous() if use_mask else None
        versions = torch.full((bsz, C * A), float(k - 1))
        kw = dict(task_type="embodied", loss_type="decoupled_actor_critic", logprob_type=lpt, reward_type=reward_type,
                  single_action_dim=A, logprobs=new, old_logprobs=old, advantages=adv, returns=ret, values=val,
                  prev_values=prev_v, clip_ratio_high=0.28, clip_ratio_low=0.2, clip_ratio_c=3.0, value_clip=0.2,
                  huber_delta=1.5, loss_mask=mask, loss_mask_sum=mask_sum,
                  max_episode_steps=50 if use_ratio else None, critic_warmup=False, proximal_logprobs=None,
                  versions=versions, current_version=k + 1, behave_weight_threshold=thr)
        loss, metrics = ref.registry.policy_loss(**kw)
        entropy = utils.reshape_entropy(ent, entropy_type=reward_type, action_dim=A, batch_size=bsz)
        entropy_loss = utils.masked_mean(entropy, mask=mask)
        loss = loss - ent_bonus * entropy_loss
        loss = loss / accum
        loss.backward()
        metrics = dict(metrics)
        metrics["actor/entropy_loss"] = float(entropy_loss.detach().item())
        metrics["actor/total_loss"] = float(loss.detach().item())
        pre = f"dec_{name}_"
        out[pre + "old"], out[pre + "new"], out[pre + "adv"] = _np(old), _np(new), _np(adv)
        out[pre + "ret"], out[pre + "prev_v"], out[pre + "val"], out[pre + "ent"] = _np(ret), _np(prev_v), _np(val), _np(ent)
        if mask is not None:
            out[pre + "mask"], out[pre + "mask_sum"] = _np(mask), _np(mask_sum)
        out[pre + "cfg"] = np.array([bsz, C, A, int(use_ratio), -1 if thr is None else 1, k, accum], dtype=np.int64)
        out[pre + "hp"] = np.array([0.0 if thr is None else thr, ent_bonus], dtype=np.float64)
        out[pre + "types"] = np.array([lpt, reward_type])
        out[pre + "loss"] = _np(loss)
        out[pre + "dnew"] = _np(new.grad if new.grad is not None else torch.zeros_like(new))
        out[pre + "dval"] = _np(val.grad if val.grad is not None else torch.zeros_like(val))
        out[pre + "dent"] = _np(ent.grad if ent.grad is not None else torch.zeros_like(ent))
        keys = sorted(metrics)
        out[pre + "metric_keys"] = np.array(keys)
        out[pre + "metric_vals"] = np.array([float(metrics[k_]) for k_ in keys], dtype=np.float64)
        cases.append(name)
    out["dec_cases"] = np.array(cases)


def gen_masked_norm(ref, out):
    sys.modules["rlinf.scheduler"].Tracer = object
    dist = importlib.import_module("rlinf.utils.distributed")
    g = torch.Generator().manual_seed(801)
    adv = 0.4 + 1.7 * torch.randn(64 * 3, 1, generator=g)  # [T*B, C] after the flatten
    mask = torch.rand(64 * 3, 1, generator=g) < 0.8
    out["mn_adv"], out["mn_mask"] = _np(adv), _np(mask)
    real_cuda = torch.Tensor.cuda
    torch.Tensor.cuda = lambda self, *a, **k: self  # no GPU here: the reference moves the statistics with .cuda()
    try:
        out["mn_out_masked"] = _np(dist.masked_normalization(adv.clone(), mask))
        out["mn_out_plain"] = _np(dist.masked_normalization(adv.clone(), None))
    finally:
        torch.Tensor.cuda = real_cuda


def main():
    ref = load_reference()
    out: dict = {}
    gen_loss(ref, out)
    gen_masked_norm(ref, out)
    np.savez_compressed(OUT, **out)
    print(f"wrote {OUT} ({os.path.getsize(OUT)} bytes, {len(out)} arrays)")


if __name__ == "__main__":
    main()
