"""The reasoning-loss oracle (tests/reasoning_loss_oracle.py) against the unmodified reference's worker loss blocks
(tests/golden/golden_reasoning_loss.npz, tests/golden/make_golden_reasoning_loss.py): bit for bit in fp32, loss,
metrics and both gradients, for every case.  Also pins the one deviation of the fused op as a fact: the reference's
fast path (an empty first row) returns a different metrics key set, the fused op the normal one.  CPU only."""
import json
import os

import numpy as np
import pytest
import torch

from reasoning_loss_oracle import reasoning_actor_loss

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "golden_reasoning_loss.npz")
NORMAL_KEYS = {"actor/policy_loss", "actor/policy_loss_abs", "actor/ratio", "actor/ratio_abs", "actor/clipped_ratio",
               "actor/dual_cliped_ratio", "actor/approx_kl", "actor/clip_fraction", "actor/final_loss",
               "actor/entropy_loss", "actor/kl_loss", "actor/rollout_train_kl"}


def _golden():
    return np.load(GOLDEN)


def _cases():
    return sorted({k.split("__")[0] for k in _golden().files})


def run_case(g, case, dtype=torch.float32):
    """The oracle on the fixture's inputs of `case` (cast to dtype) -> (cfg, loss, metrics, d_lp, d_ent)."""
    cfg = json.loads(str(g[f"{case}__cfg"]))
    t = {k: torch.from_numpy(g[f"{case}__in_{k}"]) for k in ("logprobs", "old_logprobs", "rollout_logprobs",
                                                              "advantages", "entropy", "ref_logprobs", "loss_mask")}
    t = {k: v if v.dtype == torch.bool else v.to(dtype) for k, v in t.items()}
    out = reasoning_actor_loss(
        t["logprobs"], t["advantages"], t["loss_mask"], t["old_logprobs"],
        entropy=t["entropy"] if cfg["with_entropy"] else None, ref_logprobs=t["ref_logprobs"],
        rollout_logprobs=t["rollout_logprobs"], recomputed_logprobs=t["old_logprobs"], loss_agg=cfg["loss_agg"],
        clip_ratio_low=cfg["clip_ratio_low"], clip_ratio_high=cfg["clip_ratio_high"], clip_ratio_c=cfg["clip_ratio_c"],
        clip_log_ratio_min=cfg.get("clip_log_ratio_min"), clip_log_ratio_max=cfg.get("clip_log_ratio_max"),
        entropy_bonus=cfg["entropy_bonus"], kl_beta=cfg["kl_beta"], kl_penalty_type=cfg["kl_penalty"],
        kl_order=cfg["worker"], importance_sampling_fix=cfg["importance_sampling_fix"],
        importance_sampling_clip=cfg["importance_sampling_clip"])
    return (cfg, t) + out


def _same(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return a.shape == b.shape and np.array_equal(a.view(np.uint32) if a.dtype == np.float32 else a,
                                                 b.view(np.uint32) if b.dtype == np.float32 else b)


@pytest.mark.parametrize("case", _cases())
def test_oracle_reproduces_reference_bit_for_bit(case):
    g = _golden()
    cfg, _, loss, metrics, d_lp, d_ent = run_case(g, case)
    assert _same(loss.numpy(), g[f"{case}__loss"])
    ref_keys = {k.split("__m_", 1)[1] for k in g.files if k.startswith(f"{case}__m_")}
    assert set(metrics) == NORMAL_KEYS
    for k in ref_keys & set(metrics):
        assert _same(metrics[k].numpy().reshape(g[f"{case}__m_{k}"].shape), g[f"{case}__m_{k}"]), k
    assert _same(d_lp.numpy(), g[f"{case}__d_logprobs"])
    if cfg["with_entropy"]:
        assert _same(d_ent.numpy(), g[f"{case}__d_entropy"])


def test_fixture_covers_the_issue_cases():
    g = _golden()
    cfgs = {c: json.loads(str(g[f"{c}__cfg"])) for c in _cases()}
    assert {c["loss_agg"] for c in cfgs.values()} == {"token-mean", "seq-mean-token-sum", "seq-mean-token-mean"}
    assert {(c["kl_penalty"], c["worker"]) for c in cfgs.values() if c["kl_beta"] > 0} >= {
        (k, w) for k in ("k1", "abs", "k2", "k3") for w in ("fsdp", "megatron")}
    assert any(c["importance_sampling_fix"] for c in cfgs.values())
    assert any(c["with_entropy"] and c["entropy_bonus"] > 0 for c in cfgs.values())
    assert any(not c["with_entropy"] for c in cfgs.values())
    assert np.isnan(g["empty_row_seq_token_mean_nan__loss"])  # the reference's 0/0 for an empty row


def test_fast_path_key_set_deviation():
    """The reference's fast path (losses.py:204-217) returns actor/token_num and actor/policy_loss_mbs_mean and no
    actor/ratio_abs; choosing keys on the device's mask would take a host sync, so the fused op keeps the normal set.
    Every key both sets share holds the same value, and the reference's extra keys are 0."""
    g = _golden()
    for case in ("fast_path_first_row_empty", "fast_path_seq_mean"):
        ref_keys = {k.split("__m_", 1)[1] for k in g.files if k.startswith(f"{case}__m_")}
        assert ref_keys ^ NORMAL_KEYS == {"actor/token_num", "actor/policy_loss_mbs_mean", "actor/ratio_abs"}
        for k in ("actor/token_num", "actor/policy_loss_mbs_mean", "actor/policy_loss", "actor/ratio"):
            assert float(g[f"{case}__m_{k}"]) == 0.0
        _, _, _, metrics, _, _ = run_case(g, case)
        assert float(metrics["actor/ratio_abs"]) == 0.0
