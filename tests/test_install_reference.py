"""INTEGRATION.md's install() against the reference's registries as recorded in tests/golden/golden_install.npz: every
entry gets replaced, the kwargs the reference's dispatchers (registry.py:77-124) hand the registered callable reach the
replacement, and without a GPU the replacement refuses to compute on the host (Rb200Error) instead of falling back."""
import inspect

import numpy as np
import pytest
import torch


@pytest.fixture()
def installed(golden):
    g = golden("install")
    saved = tuple({n: (lambda **kw: None) for n in g[f"reg:{t}"]} for t in ("adv", "loss", "loss_scale"))
    import rlinf_b200.plugin as plugin

    regs = tuple(dict(r) for r in saved)  # stand-ins for the reference's ADV_REGISTRY / LOSS_REGISTRY / LOSS_SCALE_REGISTRY
    done = plugin.install(*regs)
    yield g, regs, saved, done


def test_install_replaces_every_reference_entry(installed):
    g, regs, saved, done = installed
    import rlinf_b200.algorithms as A

    assert sorted(done["adv"]) == sorted(saved[0]) == sorted(A.ADV_REGISTRY)
    assert sorted(done["loss"]) == sorted(saved[1]) == sorted(A.LOSS_REGISTRY)
    assert sorted(done["loss_scale"]) == sorted(saved[2]) == sorted(A.LOSS_SCALE_REGISTRY)
    for name, fn in regs[0].items():
        assert fn is A.ADV_REGISTRY[name]
    # signature compatibility: every parameter the reference callable names is accepted by the replacement
    for tag, old_reg, new_reg in (("adv", saved[0], A.ADV_REGISTRY), ("loss", saved[1], A.LOSS_REGISTRY)):
        for name in old_reg:
            new_sig = inspect.signature(new_reg[name])
            new_kw = any(p.kind is inspect.Parameter.VAR_KEYWORD for p in new_sig.parameters.values())
            for row in g[f"sig:{tag}:{name}"]:
                pname, kind, has_default, default = str(row).split("|", 3)
                if kind in ("VAR_KEYWORD", "VAR_POSITIONAL"):
                    continue
                assert pname in new_sig.parameters or new_kw, (name, pname)
                if pname == "loss_agg_func":
                    continue  # a callable default (masked_mean): the aggregation is selected inside the fused kernel
                if pname in new_sig.parameters and has_default == "1":
                    assert repr(new_sig.parameters[pname].default) == default, (name, pname)  # same defaults (e.g. A1)


def _dispatched(g, tag, case):
    """(registered name, kwargs) the reference's dispatcher handed the registered callable."""
    prefix, kw = f"call:{tag}:{case}:", {}
    for key in g.files:
        kind, _, rest = key.partition(":")
        if rest.startswith(prefix):
            v = g[key]
            kw[rest[len(prefix):]] = None if kind == "n" else (torch.from_numpy(np.array(v)) if kind == "t" else v.item())
    return str(g[f"target:{tag}:{case}"]), kw


def test_reference_dispatchers_reach_the_cuda_callables(installed):
    g, _, _, _ = installed
    import rlinf_b200.algorithms as A
    from rlinf_b200._lib import Rb200Error

    if torch.cuda.is_available():
        pytest.skip("build-container check (no GPU): on a GPU box the call would simply succeed")
    for adv_type in ("gae", "grpo", "raw", "reinpp"):
        name, kw = _dispatched(g, "adv", adv_type)
        with pytest.raises(Rb200Error):
            A.ADV_REGISTRY[name](**kw)
    for loss_type in ("actor_critic", "actor", "decoupled_actor_critic"):
        name, kw = _dispatched(g, "loss", loss_type)
        with pytest.raises(Rb200Error):
            A.LOSS_REGISTRY[name](**kw)


def test_logits_wrappers_are_signature_compatible_with_the_reference(golden):
    """SURVEY 8(f)3 drop-ins: rlinf_b200.ops.compute_logprobs_from_logits / compute_entropy_from_logits take the reference's
    positional and keyword arguments (rlinf/utils/utils.py:454-512) and, without a GPU, refuse to compute on the host."""
    g = golden("install")
    from rlinf_b200 import ops
    from rlinf_b200._lib import Rb200Error

    for name in ("compute_logprobs_from_logits", "compute_entropy_from_logits"):
        want = [str(x) for x in g[f"util:{name}"]]
        got = list(inspect.signature(getattr(ops, name)).parameters)
        assert got == want, (name, got, want)
    if not torch.cuda.is_available():
        logits, target = torch.randn(2, 3, 11), torch.randint(0, 11, (2, 3))
        with pytest.raises((Rb200Error, RuntimeError, AssertionError, OSError)):
            ops.compute_logprobs_from_logits(logits, target, op_type="torch")
