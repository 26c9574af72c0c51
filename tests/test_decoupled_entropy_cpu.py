"""CPU checks of the decoupled actor-critic loss with the worker's entropy term and one weight version per batch
(tests/golden/golden_async.npz, generated from the reference by make_golden_async.py): the oracle restatement against
the reference's outputs, and the ctypes mirror of rb200_dppo_scalar_version_args against the C compiler."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import torch

from oracle import rl_oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _t(a):
    a = np.asarray(a)
    return torch.from_numpy(np.ascontiguousarray(a)).reshape(a.shape)


def oracle_decoupled_with_entropy(g, name, new, val, ent):
    """registry.policy_loss (decoupled_actor_critic) - entropy_bonus * masked_mean(entropy, loss_mask), / grad_accum
    (async_ppo_fsdp_worker.py:441-463), with the batch's single version k - 1 and current_version k + 1."""
    pre = f"dec_{name}_"
    bsz, Cc, A, use_ratio, has_thr, k, accum = (int(x) for x in g[pre + "cfg"])
    thr, ent_bonus = (float(x) for x in g[pre + "hp"])
    lpt, rt = (str(x) for x in g[pre + "types"])
    mask = _t(g[pre + "mask"]) if (pre + "mask") in g.files else None
    loss, metrics = O.policy_loss_embodied(
        "decoupled_actor_critic", new, _t(g[pre + "old"]), _t(g[pre + "adv"]), lpt, A, loss_mask=mask,
        loss_mask_sum=_t(g[pre + "mask_sum"]) if mask is not None else None, values=val,
        prev_values=_t(g[pre + "prev_v"]), returns=_t(g[pre + "ret"]), reward_type=rt,
        versions=torch.full((bsz, Cc * A), float(k - 1)), clip_ratio_high=0.28, clip_ratio_low=0.2, clip_ratio_c=3.0,
        value_clip=0.2, huber_delta=1.5, max_episode_steps=50 if use_ratio else None, critic_warmup=False,
        current_version=k + 1, behave_weight_threshold=thr if has_thr > 0 else None)
    entropy_loss = O.entropy_term(ent, rt, A, bsz, mask)
    loss = (loss - ent_bonus * entropy_loss) / accum
    metrics["actor/entropy_loss"] = float(entropy_loss.detach())
    metrics["actor/total_loss"] = float(loss.detach())
    return loss, metrics


def test_oracle_decoupled_loss_with_entropy_matches_reference(golden):
    g = golden("async")
    assert len(g["dec_cases"]) == 6
    for name in (str(c) for c in g["dec_cases"]):
        pre = f"dec_{name}_"
        new = _t(g[pre + "new"]).requires_grad_(True)
        val = _t(g[pre + "val"]).requires_grad_(True)
        ent = _t(g[pre + "ent"]).requires_grad_(True)
        loss, metrics = oracle_decoupled_with_entropy(g, name, new, val, ent)
        loss.backward()
        torch.testing.assert_close(loss.detach(), _t(g[pre + "loss"]), rtol=1e-6, atol=1e-7, msg=name)
        torch.testing.assert_close(new.grad, _t(g[pre + "dnew"]), rtol=1e-6, atol=1e-9, msg=name)
        torch.testing.assert_close(val.grad, _t(g[pre + "dval"]), rtol=1e-6, atol=1e-9, msg=name)
        torch.testing.assert_close(ent.grad, _t(g[pre + "dent"]), rtol=1e-6, atol=1e-9, msg=name)
        keys = [str(k) for k in g[pre + "metric_keys"]]
        assert sorted(metrics) == keys, (name, sorted(metrics), keys)
        np.testing.assert_allclose([float(metrics[k]) for k in keys], g[pre + "metric_vals"], rtol=1e-6, atol=1e-7,
                                   err_msg=name)


def test_oracle_masked_normalization_of_flat_advantages(golden):
    g = golden("async")
    adv, mask = _t(g["mn_adv"]), _t(g["mn_mask"])
    torch.testing.assert_close(O.masked_normalization(adv, mask), _t(g["mn_out_masked"]), rtol=1e-6, atol=1e-7)
    torch.testing.assert_close(O.masked_normalization(adv), _t(g["mn_out_plain"]), rtol=1e-6, atol=1e-7)


def test_scalar_version_struct_layout_matches_ctypes(tmp_path):
    from rlinf_b200 import _lib

    cname, cls = "rb200_dppo_scalar_version_args", _lib.DppoScalarVersionArgs
    lines = [f'  printf("sizeof %zu\\n", sizeof({cname}));']
    for f in cls._fields_:
        lines.append(f'  printf("{f[0]} %zu %zu\\n", offsetof({cname}, {f[0]}), sizeof((({cname}*)0)->{f[0]}));')
    src = tmp_path / "layout.c"
    src.write_text("#include <stddef.h>\n#include <stdio.h>\n#include \"rlinf_b200.h\"\nint main(void) {\n" +
                   "\n".join(lines) + "\n  return 0;\n}\n")
    cc = os.environ.get("CC") or shutil.which("gcc") or shutil.which("cc")
    assert cc, "no host C compiler (gcc) found"
    exe = tmp_path / "layout"
    subprocess.run([cc, "-std=c99", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    out = subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split("\n")
    got = {line.split()[0]: tuple(int(v) for v in line.split()[1:]) for line in out if line}
    assert got["sizeof"] == (C.sizeof(cls),)
    for f in cls._fields_:
        d = getattr(cls, f[0])
        assert got[f[0]] == (d.offset, d.size), f[0]
    assert _lib.SIGNATURES["rb200_decoupled_ppo_loss_scalar_version"][1][0] == C.POINTER(cls)
