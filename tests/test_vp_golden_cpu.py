"""The vocabulary-parallel forward restated per rank (records {m, s, t, z_t}, merged in rank order) against the
reference's `_VocabParallelEntropyAndCrossEntropy` run over P = 1, 2 and 4 gloo processes (tests/golden/golden_vp.npz,
tests/golden/make_golden_vp.py), and the reference's entropy-gradient deviation pinned as a fact: its backward is the
gradient of its forward plus g_H * p * m, m the row's global max logit.  CPU only."""
import os

import numpy as np
import pytest
import torch

from oracle import rl_oracle as O

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "golden_vp.npz")


def vp_forward(logits, target, P, temperature=1.0, window=None):
    """fp64 restatement of the sharded forward: each rank's record of its [..., Vs] shard, then the rank-order merge and
    the row finish (log-probs, entropies)."""
    V = logits.shape[-1]
    Vs = V // P
    lo, hi = window or (0, V)
    z = logits.double().reshape(-1, V) / temperature
    t = target.reshape(-1)
    recs = []
    for k in range(P):
        zk = z[:, k * Vs:(k + 1) * Vs].clone()
        zk[:, :max(lo - k * Vs, 0)] = -float("inf")
        zk[:, max(min(hi - k * Vs, Vs), 0):] = -float("inf")
        m = zk.max(-1).values
        finite = torch.isfinite(m)
        d = zk - torch.where(finite, m, torch.zeros_like(m))[:, None]
        e = torch.exp(d)
        s = e.sum(-1)
        tt = torch.where(e > 0, e * d, torch.zeros_like(e)).sum(-1)
        own = (t >= max(lo, k * Vs)) & (t < min(hi, (k + 1) * Vs))
        zt = torch.where(own, zk.gather(1, (t - k * Vs).clamp(0, Vs - 1)[:, None])[:, 0], torch.zeros_like(m))
        recs.append((m, s, tt, zt))
    M = torch.stack([r[0] for r in recs]).max(0).values
    S = sum(torch.where(torch.isfinite(r[0]), torch.exp(r[0] - M) * r[1], torch.zeros_like(M)) for r in recs)
    T = sum(torch.where(torch.isfinite(r[0]), torch.exp(r[0] - M) * (r[2] + r[1] * (r[0] - M)), torch.zeros_like(M))
            for r in recs)
    lse = M + torch.log(S)
    ent = torch.log(S) - T / S
    t_in = (t >= lo) & (t < hi)
    zt = torch.stack([r[3] for r in recs]).gather(0, (t // Vs).clamp(0, P - 1)[None])[0]
    lp = torch.where(t_in, zt - lse, torch.full_like(lse, -float("inf")))
    shape = logits.shape[:-1]
    return lp.reshape(shape), ent.reshape(shape), lse.reshape(shape)


@pytest.fixture(scope="module")
def golden():
    return np.load(GOLDEN, allow_pickle=False)


@pytest.mark.parametrize("P", [1, 2, 4])
def test_vp_oracle_forward_reproduces_reference(golden, P):
    k = lambda n: torch.from_numpy(golden[f"vp{P}_{n}"])  # noqa: E731
    logits, target = k("logits"), k("target")
    lp, ent, _ = vp_forward(logits, target, P)
    torch.testing.assert_close(lp, k("logprobs").double(), rtol=1e-5, atol=1e-5)
    torch.testing.assert_close(ent, k("entropy").double(), rtol=1e-5, atol=1e-5)
    # the unsharded oracle agrees
    lp1, ent1 = O.logprobs_entropy_from_logits(logits.double(), target)[:2]
    torch.testing.assert_close(lp, lp1.double(), rtol=1e-5, atol=1e-5)
    torch.testing.assert_close(ent, ent1.double(), rtol=1e-5, atol=1e-5)


@pytest.mark.parametrize("P", [1, 2, 4])
def test_vp_reference_gradient_deviates_by_the_max_logit_term(golden, P):
    """reference gradient - autograd gradient = g_H * p * m: the entropy term mixes raw and max-shifted logits."""
    k = lambda n: torch.from_numpy(golden[f"vp{P}_{n}"])  # noqa: E731
    logits = k("logits").double().requires_grad_(True)
    target, g_h, g_ce = k("target"), k("g_h").double(), k("g_ce").double()
    logp = torch.log_softmax(logits, -1)
    ent = -(logp.exp() * logp).sum(-1)
    ce = -logp.gather(-1, target[..., None])[..., 0]
    (ent * g_h + ce * g_ce).sum().backward()
    p = logp.detach().exp()
    m = logits.detach().max(-1, keepdim=True).values
    assert (m.abs() > 1).all(), "fixture rows need a visible max logit"
    deviation = g_h[..., None] * p * m
    assert deviation.abs().max() > 1e-2
    torch.testing.assert_close(k("grad").double() - logits.grad, deviation, rtol=0, atol=1e-5)
