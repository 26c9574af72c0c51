"""Argument checks of ops.token_policy_loss / algorithms.reasoning_actor_loss / policy_loss's loss_agg_func route,
all raised before anything touches a device, and the ctypes mirror of rb200_token_loss_args against the C compiler's
layout.  CPU only."""
import ctypes
import os
import shutil
import subprocess

import pytest
import torch

from rlinf_b200 import _lib, ops
from rlinf_b200.algorithms import policy_loss, reasoning_actor_loss

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _args(bsz=2, L=5, **over):
    lp = -torch.rand(bsz, L)
    kw = dict(logprobs=lp, old_logprobs=lp.clone(), advantages=torch.randn(bsz, L),
              loss_mask=torch.ones(bsz, L, dtype=torch.bool))
    kw.update(over)
    return kw


def _call(**over):
    kw = _args(**over)
    extra = {k: kw.pop(k) for k in list(kw) if k not in ("logprobs", "old_logprobs", "advantages", "loss_mask")}
    return ops.token_policy_loss(kw["logprobs"], kw["old_logprobs"], kw["advantages"], kw["loss_mask"], **extra)


@pytest.mark.parametrize("name", ["logprobs", "old_logprobs", "advantages"])
def test_non_fp32_log_probs_assert_with_the_reference_message(name):
    with pytest.raises(AssertionError, match=f"{name} must be float32 to keep numerical stability"):
        _call(**{name: torch.zeros(2, 5, dtype=torch.float64)})


def test_hyper_parameter_errors():
    with pytest.raises(AssertionError, match="clip_ratio_c must be greater than 1.0"):
        _call(clip_ratio_c=1.0)
    with pytest.raises(ValueError, match="unknown kl_penalty"):
        _call(kl_penalty="k4", kl_beta=0.1)
    with pytest.raises(NotImplementedError):
        _call(kl_penalty="full", kl_beta=0.1)
    with pytest.raises(ValueError, match="kl_order"):
        _call(kl_order="deepspeed")
    with pytest.raises(ValueError, match="Unsupported loss aggregation method"):
        _call(loss_agg="seq-sum")
    with pytest.raises(ValueError, match="requires both rollout_logprobs and recomputed_logprobs"):
        _call(importance_sampling_fix=True, importance_sampling_clip=2.0)


def test_shape_and_dtype_errors():
    with pytest.raises(ValueError, match="advantages has shape"):
        _call(advantages=torch.zeros(2, 4))
    with pytest.raises(ValueError, match="loss_mask has shape"):
        _call(loss_mask=torch.ones(2, 6, dtype=torch.bool))
    with pytest.raises(ValueError, match="loss_mask must be bool or uint8"):
        _call(loss_mask=torch.ones(2, 5))
    with pytest.raises(ValueError, match="entropy has shape"):
        _call(entropy=torch.zeros(5, 2))
    with pytest.raises(ValueError, match=r"must be \[bsz, L\]"):
        _call(logprobs=torch.zeros(10), old_logprobs=torch.zeros(10), advantages=torch.zeros(10))
    with pytest.raises(ValueError, match="ref_logprobs must be torch.float32"):
        _call(ref_logprobs=torch.zeros(2, 5, dtype=torch.bfloat16), kl_beta=0.1)


def test_reasoning_actor_loss_errors():
    kw = _args()
    with pytest.raises(ValueError, match="needs old_logprobs"):
        reasoning_actor_loss(kw["logprobs"], kw["advantages"], kw["loss_mask"])
    with pytest.raises(ValueError, match="seq_mean_token_mean"):
        reasoning_actor_loss(kw["logprobs"], kw["advantages"], kw["loss_mask"], old_logprobs=kw["old_logprobs"],
                             loss_agg_func=lambda v, m: v.mean())


def test_policy_loss_rejects_what_it_cannot_aggregate():
    def seq_mean_token_sum(values, mask, dim=-1):
        raise AssertionError("never called")

    kw = dict(_args(), task_type="reasoning", clip_ratio_low=0.2, clip_ratio_high=0.2)
    with pytest.raises(ValueError, match="masked_mean, seq_mean_token_sum or seq_mean_token_mean"):
        policy_loss(loss_type="actor", loss_agg_func=lambda v, m: v.mean(), **kw)
    with pytest.raises(ValueError, match="loss_type='actor' only"):
        policy_loss(loss_type="actor_critic", loss_agg_func=seq_mean_token_sum, **kw)


def test_token_loss_args_layout_matches_the_c_compiler(tmp_path):
    cls = _lib.TokenLossArgs
    lines = [f'  printf("sizeof %zu\\n", sizeof(rb200_token_loss_args));']
    for f in cls._fields_:
        lines.append(f'  printf("{f[0]} %zu %zu\\n", offsetof(rb200_token_loss_args, {f[0]}), '
                     f'sizeof(((rb200_token_loss_args*)0)->{f[0]}));')
    src = tmp_path / "layout.c"
    src.write_text("#include <stddef.h>\n#include <stdio.h>\n#include \"rlinf_b200.h\"\nint main(void) {\n" +
                   "\n".join(lines) + "\n  return 0;\n}\n")
    cc = os.environ.get("CC") or shutil.which("gcc") or shutil.which("cc")
    assert cc, "no host C compiler (gcc) found"
    exe = tmp_path / "layout"
    subprocess.run([cc, "-std=c99", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    out = subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split("\n")
    got = {line.split()[0]: tuple(int(v) for v in line.split()[1:]) for line in out if line}
    assert got.pop("sizeof") == (ctypes.sizeof(cls),)
    for name, _ in cls._fields_:
        field = getattr(cls, name)
        assert got[name] == (field.offset, field.size), name
