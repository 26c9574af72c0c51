"""ops.token_policy_loss / algorithms.reasoning_actor_loss / rb200_token_ppo_loss (csrc/token_loss.cu) on the GPU:
against the fp64 oracle (tests/reasoning_loss_oracle.py) over shapes, masks and every option, against the reference's
golden fixture, bit-identical repeats, CUDA-graph replay, no host sync, the launch count, composition with the fused
LM head (single GPU and vocabulary-parallel emulated at P = 2), and the policy_loss registry route."""
import itertools
import json
import os

import numpy as np
import pytest
import torch

from reasoning_loss_oracle import reasoning_actor_loss as oracle

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "golden_reasoning_loss.npz")
# Bars.  Loss and metrics: 1e-5 relative to the fp64 oracle, plus an absolute floor of 2^-24 * 32: every summed term
# is an fp32 value of magnitude <= 32 here (|advantage| * ratio under the dual clip 3|adv|, k3 <= 10, entropies <= 2),
# rounded once (2^-24 relative), and the sums are fp64, so a mean of such terms is off by at most 2^-24 * 32.
# Gradients: 1e-6 of the largest gradient magnitude - each gradient is one fp32 product chain of a few roundings.
METRIC_RTOL, METRIC_ATOL = 1e-5, 2.0 ** -24 * 32
GRAD_REL = 1e-6


def _inputs(bsz, L, seed, empty_rows=(), with_rr=True):
    g = torch.Generator().manual_seed(seed)
    lp = -torch.rand(bsz, L, generator=g) * 3.0
    old = lp + torch.randn(bsz, L, generator=g) * 0.3
    rollout = old + torch.randn(bsz, L, generator=g) * 0.2
    adv = torch.randn(bsz, L, generator=g)
    ent = torch.rand(bsz, L, generator=g) * 2.0
    ref = lp + torch.randn(bsz, L, generator=g) * 0.5
    mask = torch.rand(bsz, L, generator=g) < 0.7
    for r in empty_rows:
        if r < bsz:
            mask[r] = False
    return dict(logprobs=lp, old_logprobs=old, rollout_logprobs=rollout if with_rr else None, advantages=adv,
                entropy=ent, ref_logprobs=ref, loss_mask=mask)


def _close(got, want, rtol, atol, what):
    got, want = torch.as_tensor(got).double().cpu(), torch.as_tensor(want).double().cpu()
    nan = torch.isnan(want)
    assert torch.equal(torch.isnan(got), nan), f"{what}: NaN pattern differs"
    err = (got - want).abs()[~nan]
    bound = (atol + rtol * want.abs())[~nan]
    assert bool((err <= bound).all()), f"{what}: max excess {(err - bound).max().item():.3e}"


def _grad_close(got, want, what):
    got, want = got.double().cpu(), want.double().cpu()
    nan = torch.isnan(want)
    assert torch.equal(torch.isnan(got), nan), f"{what}: NaN pattern differs"
    if bool((~nan).any()):
        scale = want[~nan].abs().max().item()
        err = (got - want).abs()[~nan].max().item()
        assert err <= GRAD_REL * scale + 1e-30, f"{what}: max error {err:.3e} vs max |grad| {scale:.3e}"


def _run_gpu(ins, cfg, dev="cuda"):
    """reasoning_actor_loss on the device with autograd -> (loss, metrics, d_lp, d_ent)."""
    from rlinf_b200.algorithms import reasoning_actor_loss

    lp = ins["logprobs"].to(dev).requires_grad_(True)
    ent = ins["entropy"].to(dev).requires_grad_(True) if cfg.get("with_entropy", True) else None
    d = {k: (v.to(dev) if v is not None else None) for k, v in ins.items()}
    loss, metrics = reasoning_actor_loss(
        lp, d["advantages"], d["loss_mask"], recomputed_logprobs=d["old_logprobs"],
        rollout_logprobs=d["rollout_logprobs"], ref_logprobs=d["ref_logprobs"], entropy=ent,
        loss_agg_func=cfg["loss_agg"], clip_ratio_low=0.2, clip_ratio_high=0.28, clip_ratio_c=3.0,
        clip_log_ratio_min=cfg.get("lr_min"), clip_log_ratio_max=cfg.get("lr_max"),
        entropy_bonus=cfg.get("entropy_bonus", 0.0), kl_beta=cfg.get("kl_beta", 0.0),
        kl_penalty_type=cfg.get("kl", "kl"), kl_order=cfg.get("order", "fsdp"),
        importance_sampling_fix=cfg.get("is_fix", False), importance_sampling_clip=2.0)
    loss.backward()
    d_lp = lp.grad
    d_ent = None if ent is None else (ent.grad if ent.grad is not None else torch.zeros_like(ent))
    return loss, metrics, d_lp, d_ent


def _run_oracle(ins, cfg):
    d = {k: (v.double() if v is not None and v.dtype != torch.bool else v) for k, v in ins.items()}
    return oracle(d["logprobs"], d["advantages"], d["loss_mask"], d["old_logprobs"],
                  entropy=d["entropy"] if cfg.get("with_entropy", True) else None, ref_logprobs=d["ref_logprobs"],
                  rollout_logprobs=d["rollout_logprobs"],
                  recomputed_logprobs=d["old_logprobs"] if d["rollout_logprobs"] is not None else None,
                  loss_agg=cfg["loss_agg"], clip_ratio_low=0.2, clip_ratio_high=0.28, clip_ratio_c=3.0,
                  clip_log_ratio_min=cfg.get("lr_min"), clip_log_ratio_max=cfg.get("lr_max"),
                  entropy_bonus=cfg.get("entropy_bonus", 0.0), kl_beta=cfg.get("kl_beta", 0.0),
                  kl_penalty_type=cfg.get("kl", "kl"), kl_order=cfg.get("order", "fsdp"),
                  importance_sampling_fix=cfg.get("is_fix", False), importance_sampling_clip=2.0)


def _compare(ins, cfg, what):
    loss, metrics, d_lp, d_ent = _run_gpu(ins, cfg)
    rloss, rmetrics, rd_lp, rd_ent = _run_oracle(ins, cfg)
    _close(loss.detach(), rloss, METRIC_RTOL, METRIC_ATOL, f"{what} loss")
    assert set(metrics) == set(rmetrics), (what, set(metrics) ^ set(rmetrics))
    for k in rmetrics:
        _close(metrics[k], rmetrics[k], METRIC_RTOL, METRIC_ATOL, f"{what} {k}")
    _grad_close(d_lp, rd_lp, f"{what} d_logprobs")
    if d_ent is not None:
        _grad_close(d_ent, rd_ent, f"{what} d_entropy")


FULL = dict(kl="k3", kl_beta=0.05, entropy_bonus=0.01, is_fix=True)
SHAPES = [(1, 1), (1, 33), (7, 33), (7, 1024), (64, 1024), (1, 28672), (64, 28672)]


@pytest.mark.parametrize("bsz,L", SHAPES)
@pytest.mark.parametrize("agg", ["token-mean", "seq-mean-token-sum", "seq-mean-token-mean"])
@pytest.mark.parametrize("full", [False, True])
def test_vs_fp64_oracle_shapes(bsz, L, agg, full):
    cfg = dict(loss_agg=agg, **(FULL if full else {}))
    empty = (0,) if (full and bsz > 1) else ((bsz - 1,) if bsz > 2 else ())
    _compare(_inputs(bsz, L, seed=bsz * 7 + L, empty_rows=empty, with_rr=full), cfg, f"{bsz}x{L} {agg} full={full}")


@pytest.mark.parametrize("kl,order", list(itertools.product(["k1", "abs", "k2", "k3"], ["fsdp", "megatron"])))
@pytest.mark.parametrize("agg", ["token-mean", "seq-mean-token-mean"])
def test_vs_fp64_oracle_kl_kinds_and_orders(kl, order, agg):
    ins = _inputs(7, 1033, seed=11, empty_rows=(3,))
    ins["ref_logprobs"][0, :4] = ins["logprobs"][0, :4] + torch.tensor([25.0, -25.0, 12.0, -0.0])
    _compare(ins, dict(loss_agg=agg, kl=kl, order=order, kl_beta=0.1), f"{kl}/{order}/{agg}")


@pytest.mark.parametrize("opts", [dict(is_fix=True), dict(with_entropy=False), dict(entropy_bonus=0.0),
                                  dict(entropy_bonus=0.02), dict(lr_min=-0.2, lr_max=0.15)])
def test_vs_fp64_oracle_options(opts):
    _compare(_inputs(7, 1033, seed=5, empty_rows=(0, 4)), dict(loss_agg="seq-mean-token-sum", **opts), str(opts))


def test_strided_slices_read_in_place():
    """Megatron's log_probs[:, -L-1:-1] and response_mask[:, -L:] of wider tensors, read without copies."""
    from rlinf_b200 import ops

    bsz, L, S = 7, 1033, 1100
    ins = _inputs(bsz, L, seed=3, empty_rows=(2,))
    wide = {k: torch.zeros(bsz, S, dtype=v.dtype) for k, v in ins.items()}
    for k, v in ins.items():
        wide[k][:, S - L - 1:S - 1] = v
    sl = {k: v.cuda()[:, S - L - 1:S - 1] for k, v in wide.items()}
    assert sl["logprobs"].stride(0) == S and not sl["logprobs"].is_contiguous()
    cfg = dict(loss_agg="seq-mean-token-mean", **FULL)
    a = ops.token_policy_loss(sl["logprobs"], sl["old_logprobs"], sl["advantages"], sl["loss_mask"],
                              entropy=sl["entropy"], ref_logprobs=sl["ref_logprobs"],
                              rollout_logprobs=sl["rollout_logprobs"], recomputed_logprobs=sl["old_logprobs"],
                              loss_agg=cfg["loss_agg"], clip_ratio_c=3.0, entropy_bonus=0.01, kl_beta=0.05,
                              kl_penalty="k3", importance_sampling_fix=True, importance_sampling_clip=2.0)
    c = {k: v.cuda() for k, v in ins.items()}
    b = ops.token_policy_loss(c["logprobs"], c["old_logprobs"], c["advantages"], c["loss_mask"],
                              entropy=c["entropy"], ref_logprobs=c["ref_logprobs"],
                              rollout_logprobs=c["rollout_logprobs"], recomputed_logprobs=c["old_logprobs"],
                              loss_agg=cfg["loss_agg"], clip_ratio_c=3.0, entropy_bonus=0.01, kl_beta=0.05,
                              kl_penalty="k3", importance_sampling_fix=True, importance_sampling_clip=2.0)
    assert torch.equal(a[0], b[0]) or (torch.isnan(a[0]) and torch.isnan(b[0]))
    for k in a[1]:
        assert torch.equal(a[1][k].nan_to_num(), b[1][k].nan_to_num()), k


@pytest.mark.parametrize("case", sorted({k.split("__")[0] for k in np.load(GOLDEN).files}))
def test_matches_reference_fixture(case):
    g = np.load(GOLDEN)
    c = json.loads(str(g[f"{case}__cfg"]))
    ins = {k: torch.from_numpy(g[f"{case}__in_{k}"]) for k in ("logprobs", "old_logprobs", "rollout_logprobs",
                                                                "advantages", "entropy", "ref_logprobs", "loss_mask")}
    cfg = dict(loss_agg=c["loss_agg"], kl=c["kl_penalty"], order=c["worker"], kl_beta=c["kl_beta"],
               entropy_bonus=c["entropy_bonus"], is_fix=c["importance_sampling_fix"], with_entropy=c["with_entropy"],
               lr_min=c.get("clip_log_ratio_min"), lr_max=c.get("clip_log_ratio_max"))
    loss, metrics, d_lp, d_ent = _run_gpu(ins, cfg)
    _close(loss.detach(), torch.from_numpy(g[f"{case}__loss"]), METRIC_RTOL, METRIC_ATOL, f"{case} loss")
    for k in metrics:
        key = f"{case}__m_{k}"
        if key in g.files:
            _close(metrics[k], torch.from_numpy(g[key]).reshape(()), METRIC_RTOL, METRIC_ATOL, f"{case} {k}")
    _grad_close(d_lp, torch.from_numpy(g[f"{case}__d_logprobs"]), f"{case} d_logprobs")
    if c["with_entropy"]:
        _grad_close(d_ent, torch.from_numpy(g[f"{case}__d_entropy"]), f"{case} d_entropy")


def _fwd_bwd(c, lp, ent):
    from rlinf_b200.algorithms import reasoning_actor_loss

    loss, metrics = reasoning_actor_loss(lp, c["advantages"], c["loss_mask"], recomputed_logprobs=c["old_logprobs"],
                                         rollout_logprobs=c["rollout_logprobs"], ref_logprobs=c["ref_logprobs"],
                                         entropy=ent, loss_agg_func="seq-mean-token-mean", clip_ratio_high=0.28,
                                         entropy_bonus=0.01,
                                         kl_beta=0.05, kl_penalty_type="k3", importance_sampling_fix=True,
                                         importance_sampling_clip=2.0)
    (loss / 4).backward()
    return loss, metrics


def test_deterministic_graph_replay_no_sync_and_launch_count():
    from rlinf_b200 import _lib

    c = {k: v.cuda() for k, v in _inputs(64, 4096, seed=9, empty_rows=(5,)).items()}
    lp = c["logprobs"].clone().requires_grad_(True)
    ent = c["entropy"].clone().requires_grad_(True)

    def step():
        lp.grad = None
        ent.grad = None
        loss, metrics = _fwd_bwd(c, lp, ent)
        return loss.detach().clone(), torch.stack(list(metrics.values())).clone(), lp.grad.clone(), ent.grad.clone()

    runs = [step() for _ in range(2)]
    for a, b in zip(*runs):
        assert torch.equal(a.nan_to_num(7.0), b.nan_to_num(7.0)) and torch.equal(a.isnan(), b.isnan())

    torch.cuda.synchronize()
    n0 = _lib.load().rb200_launch_count()
    torch.cuda.set_sync_debug_mode("error")
    try:
        step()
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert _lib.load().rb200_launch_count() - n0 <= 9  # 4 forward kernels + 2 gradient scalings

    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    lp.grad = None
    ent.grad = None
    with torch.cuda.graph(graph):
        loss, metrics = _fwd_bwd(c, lp, ent)
        out = (loss.detach(), torch.stack(list(metrics.values())), lp.grad, ent.grad)
    graph.replay()
    torch.cuda.synchronize()
    for a, b in zip(runs[0], out):
        assert torch.equal(a.nan_to_num(7.0), b.nan_to_num(7.0)) and torch.equal(a.isnan(), b.isnan())


def _lmhead_case(seed=0, N_rows=(3, 200), H=1536, V=32064):
    g = torch.Generator(device="cuda").manual_seed(seed)
    bsz, L = N_rows
    x = torch.randn(bsz, L, H, generator=g, device="cuda").to(torch.bfloat16)
    w = (torch.randn(V, H, generator=g, device="cuda") * (2.0 / H ** 0.5)).to(torch.bfloat16)
    tgt = torch.randint(0, V, (bsz, L), generator=g, device="cuda")
    return x, w, tgt


def _fp64_head_and_loss(x, w, tgt, c, lp_dev, ent_dev):
    """fp64 torch on the materialised logits: the oracle loss's gradients and (dX, dW) with the magnitudes of their
    summed terms, as tests/test_gpu_lmhead.py bounds them.  The loss sees the device's log-probs and entropies
    (lp_dev, ent_dev): the bf16 head moves them by ~1e-3, enough to flip a token across a clip bound, and a flip
    changes that token's whole gradient - a property of the inputs, not of the composition under test."""
    H = w.shape[1]
    X, W = x.reshape(-1, H).double(), w.double()
    logp = torch.log_softmax(X @ W.T, -1)
    p = logp.exp()
    ent = -(p * logp).sum(-1)
    shape = tgt.shape
    cpu = {k: v.cpu() for k, v in c.items()}
    _, _, glp, gh = _run_oracle(dict(cpu, logprobs=lp_dev.detach().reshape(shape).cpu(),
                                     entropy=ent_dev.detach().reshape(shape).cpu()),
                                dict(loss_agg="seq-mean-token-mean", kl="k3", kl_beta=0.05, entropy_bonus=0.01,
                                     is_fix=True))
    glp, gh = glp.reshape(-1).cuda() / 4, gh.reshape(-1).cuda() / 4
    dz = -glp[:, None] * p - gh[:, None] * p * (logp + ent[:, None])
    dz[torch.arange(dz.shape[0], device=dz.device), tgt.reshape(-1)] += glp
    return (dz @ W, dz.abs() @ W.abs()), (dz.T @ X, dz.abs().T @ X.abs())


def _bf16_close(got, ref, what):
    want, mag = ref
    err = (got.double() - want).abs()
    bound = 2.0 ** -8 * (want.abs() + mag) + 1e-3 * want.abs().max()
    assert (err - bound).max().item() <= 0, what


def _loss_inputs(lp0):
    """The loss's other inputs around the head's own log-probs lp0, so ratios and KL terms are of the usual size."""
    g = torch.Generator().manual_seed(21)
    lp0 = lp0.detach().float().cpu()
    old = lp0 + torch.randn(lp0.shape, generator=g) * 0.3
    ins = dict(old_logprobs=old, rollout_logprobs=old + torch.randn(lp0.shape, generator=g) * 0.2,
               advantages=torch.randn(lp0.shape, generator=g), ref_logprobs=lp0 + torch.randn(lp0.shape, generator=g),
               loss_mask=torch.rand(lp0.shape, generator=g) < 0.7)
    return {k: v.cuda() for k, v in ins.items()}


def test_composition_with_fused_lm_head():
    from rlinf_b200 import ops

    x, w, tgt = _lmhead_case()
    xx, ww = x.clone().requires_grad_(True), w.clone().requires_grad_(True)
    lp, ent = ops.linear_logprobs_entropy(xx, ww, tgt)
    c = _loss_inputs(lp)
    _fwd_bwd(c, lp, ent)
    rdx, rdw = _fp64_head_and_loss(x, w, tgt, c, lp, ent)
    _bf16_close(xx.grad.reshape(-1, w.shape[1]), rdx, "dX")
    _bf16_close(ww.grad, rdw, "dW")


def test_composition_with_vocab_parallel_lm_head_emulated_p2():
    from rlinf_b200 import ops

    x, w, tgt = _lmhead_case(seed=1)
    P, Vs = 2, w.shape[0] // 2
    shards = [w[k * Vs:(k + 1) * Vs] for k in range(P)]
    rec = torch.stack([ops.lmhead_vp_partials(x, shards[k], tgt, k, P) for k in range(P)])
    lp, ent, lse = ops.vp_combine(rec, tgt, Vs)
    c = _loss_inputs(lp.reshape(tgt.shape))
    lp_leaf = lp.reshape(tgt.shape).detach().requires_grad_(True)
    ent_leaf = ent.reshape(tgt.shape).detach().requires_grad_(True)
    _fwd_bwd(c, lp_leaf, ent_leaf)
    glp, gh = lp_leaf.grad.reshape(-1), ent_leaf.grad.reshape(-1)
    parts = [ops.lmhead_vp_backward(x, shards[k], tgt, k, P, lse, ent, glp, gh) for k in range(P)]
    dx = (parts[0][0] + parts[1][0]).to(torch.bfloat16)
    dw = torch.cat([p[1] for p in parts])
    rdx, rdw = _fp64_head_and_loss(x, w, tgt, c, lp, ent)
    _bf16_close(dx.reshape(-1, w.shape[1]), rdx, "dX (P = 2)")
    _bf16_close(dw, rdw, "dW (P = 2)")


def test_registry_routes_seq_mean_and_keeps_token_mean():
    """policy_loss(task_type="reasoning") with the reference's seq_mean_token_mean (matched by name) equals the
    fixture's policy loss; token-mean calls still take the embodied-path kernel and give its bits."""
    from rlinf_b200.algorithms import losses, policy_loss

    def seq_mean_token_mean(values, mask, dim=-1):  # the reference's function, by name
        raise AssertionError("never called: the aggregation runs in the kernel")

    def masked_mean(values, mask, axis=None):
        raise AssertionError("never called")

    g = np.load(GOLDEN)
    case = "agg_seq_token_mean"
    t = {k: torch.from_numpy(g[f"{case}__in_{k}"]).cuda() for k in ("logprobs", "old_logprobs", "advantages",
                                                                     "loss_mask")}
    kw = dict(task_type="reasoning", loss_type="actor", logprobs=t["logprobs"], old_logprobs=t["old_logprobs"],
              advantages=t["advantages"], loss_mask=t["loss_mask"], clip_ratio_c=3.0, clip_ratio_low=0.2,
              clip_ratio_high=0.28, fast_path_zero_loss_mask=True)
    _, metrics = policy_loss(loss_agg_func=seq_mean_token_mean, **kw)
    ref = float(g[f"{case}__m_actor/policy_loss"])
    assert abs(float(metrics["actor/policy_loss"]) - ref) <= METRIC_RTOL * abs(ref) + METRIC_ATOL
    loss_tm, m_tm = policy_loss(loss_agg_func=masked_mean, **kw)
    loss_old, m_old = losses.compute_grpo_actor_loss_fn(**kw)
    assert torch.equal(loss_tm, loss_old)
    assert all(torch.equal(m_tm[k], m_old[k]) for k in m_old)
    with pytest.raises(ValueError, match="seq_mean_token_mean"):
        policy_loss(loss_agg_func=lambda v, m: v.mean(), **kw)
