"""Tensor-level wrappers over the C ABI (one function per entry point).

All compute happens in librlinf_b200.so on the current CUDA stream; these wrappers only allocate
outputs (torch.empty) and translate pointers.  Inputs on the host are copied to the device first.
"""
from __future__ import annotations

import ctypes as C
from typing import Optional

import torch

from . import _lib as L


def loss_mask(dones: torch.Tensor):
    """compute_loss_mask (rlinf/utils/metric_utils.py:516-537). dones bool [nc+1,B,C] ->
    (mask bool [nc,B,C], mask_sum int64 [nc,B,C] expanded view of the per-env count)."""
    lib = L.load()
    if dones.dim() != 3:
        raise ValueError(f"dones must be [n_chunk_steps+1, bsz, num_action_chunks], got {tuple(dones.shape)}")
    d = L.as_u8(L.to_device(dones))
    ncp1, B, Cc = d.shape
    mask = torch.empty((ncp1 - 1, B, Cc), dtype=torch.uint8, device=d.device)
    msum = torch.empty((B,), dtype=torch.int64, device=d.device)
    L.check(lib.rb200_loss_mask(L.ptr(d), L.ptr(mask), L.ptr(msum), ncp1 - 1, B, Cc, L.stream_ptr()), "loss_mask")
    return mask.view(torch.bool), msum.view(1, B, 1).expand(ncp1 - 1, B, Cc)


def gae(rewards, values, dones, gamma, gae_lambda, loss_mask=None, want_stats=False):
    """Un-normalised GAE on step-major [T,B] tensors -> (adv, ret, stats|None)."""
    lib = L.load()
    r = L.to_device(rewards, dtype=torch.float32)
    dev = r.device
    v = L.to_device(values, dev, torch.float32)
    d = L.as_u8(L.to_device(dones, dev))
    m = L.as_u8(L.to_device(loss_mask, dev))
    T, B = r.shape
    if d.shape != (T + 1, B):
        raise ValueError(f"dones must be [T+1,B]=({T + 1},{B}), got {tuple(d.shape)}")
    if v is not None and v.shape != (T + 1, B):
        raise ValueError(f"values must be [T+1,B]=({T + 1},{B}), got {tuple(v.shape)}")
    if m is not None and m.shape != (T, B):
        raise ValueError(f"loss_mask must be [T,B]=({T},{B}), got {tuple(m.shape)}")
    adv = torch.empty_like(r)
    ret = torch.empty_like(r)
    stats = torch.empty(6, dtype=torch.float64, device=dev) if want_stats else None
    L.check(lib.rb200_gae(L.ptr(r), L.ptr(v), L.ptr(d), L.ptr(m), L.ptr(adv), L.ptr(ret), L.ptr(stats), T, B,
                          float(gamma), float(gae_lambda), L.stream_ptr()), "gae")
    return adv, ret, stats


def normalize_(x: torch.Tensor, stats: torch.Tensor, eps: float = 1e-5) -> torch.Tensor:
    """In-place (x-mean)/(std+eps) from {n,sum,sumsq} (safe_normalize's apply half)."""
    lib = L.load()
    L.check(lib.rb200_normalize(L.ptr(x), L.ptr(stats), x.numel(), float(eps), L.stream_ptr()), "normalize")
    return x


def grpo_scores(rewards, dones) -> torch.Tensor:
    lib = L.load()
    r = L.to_device(rewards, dtype=torch.float32)
    d = L.as_u8(L.to_device(dones, r.device))
    T, B = r.shape
    s = torch.empty((B,), dtype=torch.float32, device=r.device)
    L.check(lib.rb200_grpo_scores(L.ptr(r), L.ptr(d), L.ptr(s), T, B, L.stream_ptr()), "grpo_scores")
    return s


def grpo_advantages(scores, loss_mask, T, group_size, eps=1e-6) -> torch.Tensor:
    lib = L.load()
    s = L.to_device(scores, dtype=torch.float32).reshape(-1)
    m = L.as_u8(L.to_device(loss_mask, s.device))
    B = s.numel()
    adv = torch.empty((T, B), dtype=torch.float32, device=s.device)
    L.check(lib.rb200_grpo_advantages(L.ptr(s), L.ptr(m), L.ptr(adv), T, B, int(group_size), float(eps),
                                      L.stream_ptr()), "grpo_advantages")
    return adv


def absmax(x: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Maxima of |x| for x [rows, cols] (contiguous fp32, 16-byte aligned, cols % 4 == 0) as an fp32 device tensor:
    [0] max|x| and, for cols <= 256, [4 + c] max|x[:, c]| (4 + cols floats, else 1) - MLPPolicy.forward_train's
    `states_amax`."""
    lib = L.load()
    rows, cols = x.shape[0], x[0].numel()
    out = out if out is not None else torch.empty(4 + cols if cols <= 256 else 1, dtype=torch.float32, device=x.device)
    L.check(lib.rb200_absmax(L.ptr(x), rows, cols, L.ptr(out), L.stream_ptr()), "absmax")
    return out


def gather_rows(src: torch.Tensor, idx: torch.Tensor) -> torch.Tensor:
    """dst = src.reshape(N, -1)[idx] with the trailing shape kept (bit-exact row gather)."""
    lib = L.load()
    s = L.to_device(src)
    i = L.to_device(idx, s.device, torch.int64)
    n_src = s.shape[0]
    row_bytes = s[0].numel() * s.element_size() if n_src > 0 else 0
    out = torch.empty((i.numel(), *s.shape[1:]), dtype=s.dtype, device=s.device)
    if i.numel() == 0 or row_bytes == 0:
        return out
    L.check(lib.rb200_gather_rows(L.ptr(s), L.ptr(i), L.ptr(out), i.numel(), n_src, row_bytes, L.stream_ptr()),
            "gather_rows")
    return out


def ppo_loss(*, logprobs, old_logprobs, advantages, C_chunks, A_dim, logprob_type, values=None, returns=None,
             prev_values=None, loss_mask=None, loss_mask_sum=None, mask_sum_row_mod=0, idx=None, entropy=None,
             adv_stats=None, adv_norm_eps=1e-5, clip_ratio_low=0.2, clip_ratio_high=0.2, clip_ratio_c=None,
             clip_log_ratio_min=None, clip_log_ratio_max=None, value_clip=0.0, huber_delta=0.0,
             max_episode_steps=None, critic_warmup=False, entropy_bonus=0.0, loss_scale=1.0, want_grads=True,
             _decoupled=None):
    """One fused launch group. Returns (loss[1], metrics[24], d_logprobs|None, d_values|None, d_entropy|None).
    `_decoupled` (internal): dict(proximal_logprobs, versions, current_version, behave_weight_threshold) selects
    rb200_decoupled_ppo_loss (metrics in the RB200_DM_* layout); with a `version` number instead of the `versions`
    tensor (one weight version for the whole batch), rb200_decoupled_ppo_loss_scalar_version."""
    lib = L.load()
    dev = logprobs.device
    bsz = logprobs.shape[0]
    with_critic = values is not None
    lp = logprobs.contiguous()
    a = L.PpoArgs()
    a.bsz, a.C, a.A = bsz, int(C_chunks), int(A_dim)
    a.logprob_type = L.LOGPROB_TYPES[logprob_type] if isinstance(logprob_type, str) else int(logprob_type)
    a.with_critic = 1 if with_critic else 0
    keep = [lp]

    def P(t, dtype=None):
        if t is None:
            return None
        t = L.to_device(t, dev, dtype)
        keep.append(t)
        return L.ptr(t)

    a.logprobs = L.ptr(lp)
    a.values = P(values, torch.float32)
    a.entropy = P(entropy, torch.float32)
    a.idx = P(idx, torch.int64)
    a.old_logprobs = P(old_logprobs, torch.float32)
    a.advantages = P(advantages, torch.float32)
    a.returns = P(returns, torch.float32)
    a.prev_values = P(prev_values, torch.float32)
    a.loss_mask = P(L.as_u8(loss_mask) if loss_mask is not None else None)
    a.loss_mask_sum = P(loss_mask_sum, torch.int64)
    a.mask_sum_row_mod = int(mask_sum_row_mod)
    a.adv_stats = P(adv_stats, torch.float64)
    a.adv_norm_eps = float(adv_norm_eps)
    a.clip_ratio_low, a.clip_ratio_high = float(clip_ratio_low), float(clip_ratio_high)
    a.clip_ratio_c = float(clip_ratio_c) if clip_ratio_c is not None else 0.0
    if clip_ratio_c is not None and not clip_ratio_c > 1.0:
        raise AssertionError("clip_ratio_c must be greater than 1.0")  # losses.py:260
    a.has_clip_log_ratio_min = int(clip_log_ratio_min is not None)
    a.has_clip_log_ratio_max = int(clip_log_ratio_max is not None)
    a.clip_log_ratio_min = float(clip_log_ratio_min or 0.0)
    a.clip_log_ratio_max = float(clip_log_ratio_max or 0.0)
    a.value_clip = float(value_clip or 0.0)
    a.huber_delta = float(huber_delta or 0.0)
    a.max_episode_steps = int(max_episode_steps) if max_episode_steps else 0
    a.critic_warmup = int(bool(critic_warmup))
    a.entropy_bonus = float(entropy_bonus)
    a.loss_scale = float(loss_scale)
    ws = _loss_workspace(dev)
    loss = torch.empty(1, dtype=torch.float32, device=dev)
    metrics = torch.empty(L.NUM_METRICS, dtype=torch.float32, device=dev)
    d_lp = torch.empty_like(lp) if want_grads else None
    d_v = torch.empty((values.numel(),), dtype=torch.float32, device=dev).view(values.shape) if (want_grads and with_critic) else None
    d_e = torch.empty_like(keep[0]) if (want_grads and entropy is not None) else None
    a.workspace, a.loss, a.metrics = L.ptr(ws), L.ptr(loss), L.ptr(metrics)
    a.d_logprobs, a.d_values, a.d_entropy = L.ptr(d_lp), L.ptr(d_v), L.ptr(d_e)
    if _decoupled is not None and _decoupled.get("version") is not None:
        if _decoupled.get("versions") is not None or _decoupled.get("current_version") is None:
            raise ValueError("a scalar `version` needs `current_version` and excludes the `versions` tensor")
        d = L.DppoScalarVersionArgs()
        d.base = a
        d.proximal_logprobs = P(_decoupled.get("proximal_logprobs"), torch.float32)
        d.version, d.current_version = float(_decoupled["version"]), float(_decoupled["current_version"])
        thr = _decoupled.get("behave_weight_threshold")
        d.has_behave_weight_threshold, d.behave_weight_threshold = int(thr is not None), float(thr or 0.0)
        L.check(lib.rb200_decoupled_ppo_loss_scalar_version(C.byref(d), L.stream_ptr()), "decoupled_ppo_loss")
        return loss, metrics, d_lp, d_v, d_e
    if _decoupled is not None:
        d = L.DppoArgs()
        d.base = a
        d.proximal_logprobs = P(_decoupled.get("proximal_logprobs"), torch.float32)
        d.versions = P(_decoupled.get("versions"), torch.float32)
        cv, thr = _decoupled.get("current_version"), _decoupled.get("behave_weight_threshold")
        d.has_current_version, d.current_version = int(cv is not None), float(cv or 0.0)
        d.has_behave_weight_threshold, d.behave_weight_threshold = int(thr is not None), float(thr or 0.0)
        L.check(lib.rb200_decoupled_ppo_loss(C.byref(d), L.stream_ptr()), "decoupled_ppo_loss")
        return loss, metrics, d_lp, d_v, d_e
    L.check(lib.rb200_ppo_loss(C.byref(a), L.stream_ptr()), "ppo_loss")
    return loss, metrics, d_lp, d_v, d_e


def opd_loss(*, logprobs, advantages, loss_mask, loss_mask_sum, max_episode_steps=None, loss_scale=1.0, want_grads=True):
    """compute_opd_actor_loss (losses.py:427-505). logprobs/advantages [n_units, tokens]; mask/mask_sum [n_units]."""
    lib = L.load()
    lp = logprobs.contiguous()
    dev = lp.device
    n_units, g = lp.shape
    adv = L.to_device(advantages, dev, torch.float32).reshape(n_units, g)
    m = L.as_u8(L.to_device(loss_mask, dev)).reshape(n_units).contiguous()
    ms = L.to_device(loss_mask_sum, dev, torch.int64).reshape(n_units).contiguous()
    loss = torch.empty(1, dtype=torch.float32, device=dev)
    metrics = torch.empty(L.NUM_METRICS, dtype=torch.float32, device=dev)
    d_lp = torch.empty_like(lp) if want_grads else None
    L.check(lib.rb200_opd_loss(L.ptr(lp), L.ptr(adv), L.ptr(m), L.ptr(ms), n_units, g, int(max_episode_steps or 0),
                               float(loss_scale), L.ptr(_loss_workspace(dev)), L.ptr(loss), L.ptr(metrics), L.ptr(d_lp),
                               L.stream_ptr()), "opd_loss")
    return loss, metrics, d_lp


_WS: dict = {}


def _loss_workspace(dev) -> torch.Tensor:
    """Zero-initialised, self-cleaning reduction workspace of the loss kernels, one per device: the loss kernels of
    one process are stream-ordered (training loop / one CUDA graph), which is what sharing it requires."""
    key = dev.index
    ws = _WS.get(key)
    if ws is None:
        ws = torch.zeros(32, dtype=torch.float64, device=dev)
        _WS[key] = ws
    return ws


def scale_(x: torch.Tensor, s: float) -> torch.Tensor:
    lib = L.load()
    L.check(lib.rb200_scale(L.ptr(x), x.numel(), float(s), L.stream_ptr()), "scale")
    return x


def scale_by_(x: torch.Tensor, s_dev: torch.Tensor) -> torch.Tensor:
    """x *= s_dev[0] with the scalar read on the device (no host sync)."""
    lib = L.load()
    s = s_dev.reshape(1).to(torch.float32)
    L.check(lib.rb200_scale_by(L.ptr(x), x.numel(), L.ptr(s), L.stream_ptr()), "scale_by")
    return x


def reward_filter(rewards, loss_mask, group_size, lower, upper):
    """filter_rewards (embodied_fsdp_actor_worker.py:236-282): returns the new loss_mask (bool) -
    [nc,B,C] = keep & loss_mask, or [nc,B,1] when there was no loss_mask."""
    lib = L.load()
    r = L.to_device(rewards, dtype=torch.float32)
    m = L.as_u8(L.to_device(loss_mask, r.device))
    nc, B, Cc = r.shape
    if B % group_size != 0:
        raise AssertionError(f"batch {B} not divisible by group_size {group_size}")
    out = torch.empty((nc, B, Cc if m is not None else 1), dtype=torch.uint8, device=r.device)
    keep = torch.empty((B,), dtype=torch.uint8, device=r.device)
    L.check(lib.rb200_reward_filter(L.ptr(r), L.ptr(m), L.ptr(out), L.ptr(keep), nc, B, Cc, int(group_size),
                                    float(lower), float(upper), L.stream_ptr()), "reward_filter")
    return out.view(torch.bool)


_KL_MODES = {"kl": 0, "k1": 0, "abs": 1, "mse": 2, "k2": 2, "low_var_kl": 3, "k3": 3}


def kl_penalty_raw(logprob, ref_logprob, kind, want_grad=False):
    lib = L.load()
    if kind not in _KL_MODES:
        raise NotImplementedError(kind)
    a = L.to_device(logprob, dtype=torch.float32)
    b = L.to_device(ref_logprob, a.device, torch.float32)
    out = torch.empty_like(a)
    g = torch.empty_like(a) if want_grad else None
    L.check(lib.rb200_kl_penalty(L.ptr(a), L.ptr(b), L.ptr(out), L.ptr(g), a.numel(), _KL_MODES[kind],
                                 L.stream_ptr()), "kl_penalty")
    return out, g


# ---------------------------------------------------------------------------------------------------------------
# Token-level PPO-clip actor loss of the reasoning workers (csrc/token_loss.cu)
_KL_ORDERS = {"megatron": 0, "fsdp": 1}


def _rows(t, name, shape, dev, dtype=torch.float32):
    """A [bsz, L] input as (tensor, row stride): read in place when its tokens are contiguous."""
    if t is None:
        return None, 0
    if tuple(t.shape) != shape:
        raise ValueError(f"token_policy_loss: {name} has shape {tuple(t.shape)}, expected {shape} (that of logprobs)")
    if t.dtype != dtype:
        raise ValueError(f"token_policy_loss: {name} must be {dtype}, got {t.dtype}")
    if t.device != dev:
        raise ValueError(f"token_policy_loss: {name} is on {t.device}, logprobs on {dev}")
    if t.stride(1) != 1 or t.stride(0) < shape[1]:
        t = t.contiguous()
    return t, t.stride(0)


def _token_loss_cfg(logprobs, old_logprobs, advantages, loss_mask, entropy, ref_logprobs, rollout_logprobs,
                    recomputed_logprobs, loss_agg, clip_ratio_low, clip_ratio_high, clip_ratio_c, clip_log_ratio_min,
                    clip_log_ratio_max, entropy_bonus, kl_beta, kl_penalty, kl_order, importance_sampling_fix,
                    importance_sampling_clip, fast_path_zero_loss_mask):
    """Validate the arguments of token_policy_loss (before anything touches the device) -> the ABI struct's fields."""
    for name, t in (("logprobs", logprobs), ("old_logprobs", old_logprobs), ("advantages", advantages)):
        assert t.dtype == torch.float32, f"{name} must be float32 to keep numerical stability"  # losses.py:232-240
    if logprobs.dim() != 2:
        raise ValueError(f"token_policy_loss: logprobs must be [bsz, L], got {tuple(logprobs.shape)}")
    if loss_agg not in L.AGG_MODES:
        raise ValueError(f"Unsupported loss aggregation method: {loss_agg}; supported: {sorted(L.AGG_MODES)}")
    if clip_ratio_c is not None:
        assert clip_ratio_c > 1.0, "clip_ratio_c must be greater than 1.0"  # losses.py:260
    if kl_penalty == "full":
        raise NotImplementedError("kl_penalty 'full' needs the whole vocabulary's log-probs (utils.py:60-62)")
    if kl_penalty not in _KL_MODES:
        raise ValueError(f"unknown kl_penalty {kl_penalty!r}; supported: {sorted(_KL_MODES)}")
    if kl_order not in _KL_ORDERS:
        raise ValueError(f"kl_order must be one of {sorted(_KL_ORDERS)}, got {kl_order!r}")
    if importance_sampling_fix:
        if rollout_logprobs is None or recomputed_logprobs is None:
            raise ValueError("importance_sampling_fix requires both rollout_logprobs and recomputed_logprobs")
        if importance_sampling_clip is None:
            raise ValueError("importance_sampling_fix requires importance_sampling_clip")
    shape, dev = tuple(logprobs.shape), logprobs.device
    if loss_mask is None or tuple(loss_mask.shape) != shape:
        raise ValueError(f"token_policy_loss: loss_mask has shape {None if loss_mask is None else tuple(loss_mask.shape)}"
                         f", expected {shape} (that of logprobs)")
    if loss_mask.dtype not in (torch.bool, torch.uint8):
        raise ValueError(f"token_policy_loss: loss_mask must be bool or uint8, got {loss_mask.dtype}")
    if 0 in shape:
        raise ValueError(f"token_policy_loss: empty logprobs {shape}")
    named = dict(logprobs=logprobs, old_logprobs=old_logprobs, advantages=advantages,
                 loss_mask=loss_mask.view(torch.uint8) if loss_mask.dtype == torch.bool else loss_mask,
                 entropy=entropy, ref_logprobs=ref_logprobs, rollout_logprobs=rollout_logprobs,
                 recomputed_logprobs=recomputed_logprobs)
    ins = {k: _rows(t, k, shape, dev, torch.uint8 if k == "loss_mask" else torch.float32) for k, t in named.items()}
    hp = dict(clip_ratio_low=float(clip_ratio_low), clip_ratio_high=float(clip_ratio_high),
              clip_ratio_c=float(clip_ratio_c) if clip_ratio_c is not None else 0.0,
              has_clip_log_ratio_min=int(clip_log_ratio_min is not None),
              has_clip_log_ratio_max=int(clip_log_ratio_max is not None),
              clip_log_ratio_min=float(clip_log_ratio_min or 0.0), clip_log_ratio_max=float(clip_log_ratio_max or 0.0),
              entropy_bonus=float(entropy_bonus or 0.0), kl_beta=float(kl_beta or 0.0),
              importance_sampling_clip=float(importance_sampling_clip or 0.0), agg=L.AGG_MODES[loss_agg],
              kl_mode=_KL_MODES[kl_penalty], kl_order=_KL_ORDERS[kl_order],
              importance_sampling_fix=int(bool(importance_sampling_fix)),
              fast_path_zero_loss_mask=int(bool(fast_path_zero_loss_mask)))
    return ins, hp


def _token_loss_launch(lp, ent, ins, hp, want_d_lp, want_d_ent):
    if not lp.is_cuda:
        raise L.Rb200Error("token_policy_loss takes CUDA tensors; there is no CPU path")
    lib = L.load()
    dev = lp.device
    bsz, Ln = lp.shape
    a = L.TokenLossArgs()
    a.bsz, a.L = bsz, Ln
    keep = []
    for name, (t, stride) in ins.items():
        if name == "logprobs":
            t, stride = lp, lp.stride(0)
        elif name == "entropy":
            t, stride = ent, (ent.stride(0) if ent is not None else 0)
        keep.append(t)
        setattr(a, name, None if t is None else C.c_void_p(t.data_ptr()))
        setattr(a, name + "_stride", stride)
    for k, v in hp.items():
        setattr(a, k, v)
    wsb = L.load().rb200_token_loss_workspace_bytes(bsz, Ln)
    if wsb < 0:
        raise ValueError(f"token_policy_loss: unsupported shape bsz={bsz} L={Ln} (bsz <= 65535)")
    ws = torch.empty(wsb, dtype=torch.uint8, device=dev)
    loss = torch.empty(1, dtype=torch.float32, device=dev)
    metrics = torch.empty(L.TM_NUM, dtype=torch.float32, device=dev)
    d_lp = torch.empty((bsz, Ln), dtype=torch.float32, device=dev) if want_d_lp else None
    d_ent = torch.empty((bsz, Ln), dtype=torch.float32, device=dev) if want_d_ent else None
    a.workspace, a.workspace_bytes = L.ptr(ws), wsb
    a.loss, a.metrics, a.d_logprobs, a.d_entropy = L.ptr(loss), L.ptr(metrics), L.ptr(d_lp), L.ptr(d_ent)
    L.check(lib.rb200_token_ppo_loss(C.byref(a), L.stream_ptr(dev)), "token_ppo_loss")
    return loss.reshape(()), metrics, d_lp, d_ent


class _TokenPolicyLoss(torch.autograd.Function):
    """forward: one launch group writes the loss, the metrics and the gradients that are needed; backward: those
    gradients times the upstream scalar, read on the device."""

    @staticmethod
    def forward(ctx, logprobs, entropy, ins, hp):
        want_d_ent = entropy is not None and ctx.needs_input_grad[1] and hp["entropy_bonus"] > 0.0
        loss, metrics, d_lp, d_ent = _token_loss_launch(logprobs.detach(), None if entropy is None else entropy.detach(),
                                                        ins, hp, ctx.needs_input_grad[0], want_d_ent)
        ctx.grads = (d_lp, d_ent)
        ctx.mark_non_differentiable(metrics)
        return loss, metrics

    @staticmethod
    def backward(ctx, g_loss, _g_metrics):
        d_lp, d_ent = ctx.grads
        ctx.grads = None
        if d_lp is not None:
            scale_by_(d_lp, g_loss)
        if d_ent is not None:
            scale_by_(d_ent, g_loss)
        return d_lp, d_ent, None, None


def token_policy_loss(logprobs, old_logprobs, advantages, loss_mask, *, entropy=None, ref_logprobs=None,
                      rollout_logprobs=None, recomputed_logprobs=None, loss_agg: str = "token-mean",
                      clip_ratio_low: float = 0.2, clip_ratio_high: float = 0.2, clip_ratio_c: Optional[float] = None,
                      clip_log_ratio_min: Optional[float] = None, clip_log_ratio_max: Optional[float] = None,
                      entropy_bonus: float = 0.0, kl_beta: float = 0.0, kl_penalty: str = "kl", kl_order: str = "fsdp",
                      importance_sampling_fix: bool = False, importance_sampling_clip: Optional[float] = None,
                      fast_path_zero_loss_mask: bool = False):
    """Token-level PPO-clip actor loss of the reasoning workers, with its entropy and KL terms, in one device pass.

    logprobs, old_logprobs, advantages, loss_mask (bool / uint8) and the optional entropy, ref_logprobs,
    rollout_logprobs, recomputed_logprobs are [bsz, L] CUDA tensors (fp32 but the mask); slices whose tokens are
    contiguous, e.g. log_probs[:, -L-1:-1], are read in place.  loss_agg: "token-mean", "seq-mean-token-sum" or
    "seq-mean-token-mean" (get_loss_agg_func's names), applied to the policy loss, policy_loss_abs, the entropy and
    the KL term.  kl_order "fsdp" computes kl_penalty(ref_logprobs, logprobs), "megatron" kl_penalty(logprobs,
    ref_logprobs); the KL term is added when kl_beta > 0.  importance_sampling_fix multiplies the advantages by
    min(exp(recomputed - rollout), importance_sampling_clip).  fast_path_zero_loss_mask: an empty first row zeroes the
    policy part and its metrics, decided on the device.

    Returns (loss, metrics): loss = policy - entropy_bonus * entropy_loss + kl_beta * kl_loss as a 0-dim tensor,
    differentiable w.r.t. logprobs and entropy (only the gradients that are needed are computed); metrics maps the
    workers' keys (actor/policy_loss ... actor/clip_fraction, actor/entropy_loss, actor/kl_loss, actor/final_loss,
    and actor/rollout_train_kl when both rollout and recomputed log-probs are given) to 0-dim device tensors.  No host sync.
    """
    ins, hp = _token_loss_cfg(logprobs, old_logprobs, advantages, loss_mask, entropy, ref_logprobs, rollout_logprobs,
                              recomputed_logprobs, loss_agg, clip_ratio_low, clip_ratio_high, clip_ratio_c,
                              clip_log_ratio_min, clip_log_ratio_max, entropy_bonus, kl_beta, kl_penalty, kl_order,
                              importance_sampling_fix, importance_sampling_clip, fast_path_zero_loss_mask)
    lp, _ = ins["logprobs"]
    ent, _ = ins["entropy"]
    needs = torch.is_grad_enabled() and (logprobs.requires_grad or (entropy is not None and entropy.requires_grad))
    if needs:
        loss, metrics = _TokenPolicyLoss.apply(lp, ent, ins, hp)
    else:
        loss, metrics, _, _ = _token_loss_launch(lp, ent, ins, hp, False, False)
    with_rr = rollout_logprobs is not None and recomputed_logprobs is not None
    keys = {s: k for s, k in L.TM_KEYS.items() if k != "actor/rollout_train_kl" or with_rr}
    return loss, {k: metrics[s] for s, k in keys.items()}


def masked_stats(x, mask=None, mask_div=1):
    """{count, sum, min, max} (float64[4], device) of x over mask (mask index = flat index // mask_div)."""
    lib = L.load()
    xs = L.to_device(x, dtype=torch.float32).contiguous()
    m = L.as_u8(L.to_device(mask, xs.device))
    out = torch.empty(4, dtype=torch.float64, device=xs.device)
    L.check(lib.rb200_masked_stats(L.ptr(xs), L.ptr(m.contiguous() if m is not None else None), xs.numel(),
                                   int(mask_div), L.ptr(out), L.stream_ptr()), "masked_stats")
    return out


# ---- SURVEY 8(f) rank 4: remaining advantage estimators, fp64 masked normalisations -----------------------------------
def masked_moments(x, mask=None) -> torch.Tensor:
    """{count, sum, sumsq} (float64[3], device) of x over mask - masked_stats (rlinf/utils/distributed.py:942-954)."""
    lib = L.load()
    xs = L.to_device(x, dtype=torch.float32).contiguous()
    m = L.as_u8(L.to_device(mask, xs.device))
    if m is not None:
        if m.shape != xs.shape:
            raise AssertionError((tuple(m.shape), tuple(xs.shape)))
        m = m.contiguous()
    out = torch.empty(3, dtype=torch.float64, device=xs.device)
    L.check(lib.rb200_masked_moments(L.ptr(xs), L.ptr(m), xs.numel(), L.ptr(out), L.stream_ptr()), "masked_moments")
    return out


def masked_normalize(x, stats3, mask=None, mode=0, eps=1e-5, unbiased=False) -> torch.Tensor:
    """Apply half of the fp64 normalisations (mode 0 masked_normalization, 1 normalize_from_stats, 2 whitening)."""
    lib = L.load()
    xs = L.to_device(x, dtype=torch.float32).contiguous()
    m = L.as_u8(L.to_device(mask, xs.device))
    m = m.contiguous() if m is not None else None
    out = torch.empty_like(xs)
    st = L.to_device(stats3, xs.device, torch.float64)
    L.check(lib.rb200_masked_normalize(L.ptr(xs), L.ptr(m), L.ptr(out), xs.numel(), L.ptr(st), int(mode), float(eps),
                                       int(bool(unbiased)), L.stream_ptr()), "masked_normalize")
    return out


def raw_advantages(scores, loss_mask, want_stats=False):
    lib = L.load()
    s = L.to_device(scores, dtype=torch.float32).reshape(-1).contiguous()
    m = L.as_u8(L.to_device(loss_mask, s.device)).contiguous()
    Ln, B = m.shape
    if s.numel() != B:
        raise RuntimeError(f"{s.numel()} scores for a loss_mask of {tuple(m.shape)}")
    adv = torch.empty((Ln, B), dtype=torch.float32, device=s.device)
    stats = torch.empty(3, dtype=torch.float64, device=s.device) if want_stats else None
    L.check(lib.rb200_raw_advantages(L.ptr(s), L.ptr(m), L.ptr(adv), Ln, B, L.ptr(stats), L.stream_ptr()), "raw_advantages")
    return adv, stats


def reinpp_returns(rewards, loss_mask, kl_beta=0.0, logprob=None, ref_logprob=None, kl_kind="k1"):
    lib = L.load()
    r = L.to_device(rewards, dtype=torch.float32).reshape(-1).contiguous()
    m = L.as_u8(L.to_device(loss_mask, r.device)).contiguous()
    Ln, B = m.shape
    if r.numel() != B:
        raise RuntimeError(f"{r.numel()} rewards for a loss_mask of {tuple(m.shape)}")
    lp = rlp = None
    if kl_beta > 0:
        if kl_kind not in _KL_MODES:
            raise NotImplementedError(kl_kind)
        lp = L.to_device(logprob, r.device, torch.float32).contiguous()
        rlp = L.to_device(ref_logprob, r.device, torch.float32).contiguous()
        if lp.shape != m.shape or rlp.shape != m.shape:
            raise RuntimeError("logprob / ref_logprob must be [L, B] like loss_mask")
    ret = torch.empty((Ln, B), dtype=torch.float32, device=r.device)
    stats = torch.empty(3, dtype=torch.float64, device=r.device)
    L.check(lib.rb200_reinpp_returns(L.ptr(r), L.ptr(m), L.ptr(lp), L.ptr(rlp), L.ptr(ret), Ln, B, float(kl_beta),
                                     _KL_MODES.get(kl_kind, 0), L.ptr(stats), L.stream_ptr()), "reinpp_returns")
    return ret, stats


def grpo_video_advantages(rewards, loss_mask, group_size, mode):
    lib = L.load()
    r = L.to_device(rewards, dtype=torch.float32).contiguous()
    S, B = r.shape
    mf = m8 = None
    if loss_mask is not None:
        lm = L.to_device(loss_mask, r.device)
        if lm.dtype in (torch.bool, torch.uint8):
            m8 = L.as_u8(lm).contiguous()
        else:
            mf = lm.to(torch.float32).contiguous()
    adv = torch.empty_like(r)
    L.check(lib.rb200_grpo_video_advantages(L.ptr(r), L.ptr(mf), L.ptr(m8), L.ptr(adv), S, B, int(group_size),
                                            {"frame": 0, "video": 1}[mode], 1e-6, L.stream_ptr()), "grpo_video")
    return adv


def grpo_dynamic_turn_advantages(rewards, idx_to_traj, group_size, mode):
    lib = L.load()
    r = L.to_device(rewards, dtype=torch.float32).reshape(-1).contiguous()
    idx = torch.as_tensor(idx_to_traj, dtype=torch.int32).to(r.device)
    n = idx.numel()
    n_traj = int(max(idx_to_traj)) + 1
    out = torch.zeros(n, dtype=torch.float32, device=r.device)
    L.check(lib.rb200_grpo_dynamic_turn_advantages(L.ptr(r), L.ptr(idx), L.ptr(out), n, n_traj, int(group_size),
                                                   {"trajectory": 0, "turn": 1}[mode], 1e-6, L.stream_ptr()),
            "grpo_dynamic")
    return out


def sub(a, b) -> torch.Tensor:
    lib = L.load()
    x = L.to_device(a, dtype=torch.float32).contiguous()
    y = L.to_device(b, x.device, torch.float32).contiguous()
    out = torch.empty_like(x)
    L.check(lib.rb200_sub(L.ptr(x), L.ptr(y), L.ptr(out), x.numel(), L.stream_ptr()), "sub")
    return out


# ---------------------------------------------------------------------------------------------------------------
# SURVEY 8(f)3: log-probabilities / entropies from logits (csrc/logits.cu)
# ---------------------------------------------------------------------------------------------------------------
def _logits_geometry(logits: torch.Tensor):
    """(tensor, N, L, batch_stride, row_stride, V) of a [..., V] tensor whose last dim is contiguous; [bsz, L, V] slices
    such as `logits[:, -L-1:-1, :]` are addressed in place (no copy), anything else is made contiguous first."""
    V = logits.shape[-1]
    if logits.dim() == 3 and logits.stride(2) == 1 and logits.is_cuda:
        bsz, Lr, _ = logits.shape
        return logits, bsz * Lr, Lr, logits.stride(0), logits.stride(1), V
    x = L.to_device(logits).reshape(-1, V).contiguous()
    return x, x.shape[0], x.shape[0], 0, V, V


def _raw_ptr(t: torch.Tensor):
    return C.c_void_p(t.data_ptr())


class _LogitsLogprobEntropy(torch.autograd.Function):
    @staticmethod
    def forward(ctx, logits, target, temperature, window, want_entropy):
        lib = L.load()
        if logits.dtype not in (torch.float32, torch.bfloat16):
            raise ValueError(f"logits must be float32 or bfloat16, got {logits.dtype}")
        x, N, Lr, bs, rs, V = _logits_geometry(logits)
        tgt = L.to_device(target, x.device, torch.int64).reshape(-1).contiguous()
        if tgt.numel() != N:
            raise ValueError(f"target has {tgt.numel()} entries for {N} logit rows")
        lo, hi = (0, V) if window is None else (int(window[0]), int(window[1]))
        lp = torch.empty(N, dtype=torch.float32, device=x.device)
        ent = torch.empty(N, dtype=torch.float32, device=x.device) if want_entropy else None
        lse = torch.empty(N, dtype=torch.float32, device=x.device)
        dt = 0 if x.dtype == torch.float32 else 1
        L.check(lib.rb200_logits_logprob_entropy_fwd(_raw_ptr(x), dt, L.ptr(tgt), N, Lr, bs, rs, V, lo, hi,
                                                     1.0 / float(temperature), L.ptr(lp), L.ptr(ent), L.ptr(lse),
                                                     L.stream_ptr(x.device)), "logits_logprob_entropy_fwd")
        ctx.save_for_backward(x, tgt, lse, ent if want_entropy else lse)
        ctx.meta = (N, Lr, bs, rs, V, lo, hi, float(temperature), dt, want_entropy, tuple(logits.shape))
        shape = logits.shape[:-1]
        if want_entropy:
            return lp.view(shape), ent.view(shape)
        none = lp.new_zeros(())
        ctx.mark_non_differentiable(none)
        return lp.view(shape), none

    @staticmethod
    def backward(ctx, g_lp, g_ent):
        lib = L.load()
        x, tgt, lse, ent = ctx.saved_tensors
        N, Lr, bs, rs, V, lo, hi, temp, dt, want_entropy, shape = ctx.meta
        glp = g_lp.reshape(-1).float().contiguous() if g_lp is not None else None
        gh = g_ent.reshape(-1).float().contiguous() if (want_entropy and g_ent is not None) else None
        dx = torch.empty((N, V), dtype=x.dtype, device=x.device)  # contiguous gradient, whatever the logits' strides
        L.check(lib.rb200_logits_logprob_entropy_bwd(_raw_ptr(x), dt, L.ptr(tgt), N, Lr, bs, rs, V, lo, hi, 1.0 / temp,
                                                     L.ptr(lse), L.ptr(ent) if gh is not None else None, L.ptr(glp),
                                                     L.ptr(gh), L.ptr(dx), Lr * V, V, L.stream_ptr(x.device)),
                "logits_logprob_entropy_bwd")
        return dx.view(shape), None, None, None, None


def logprobs_entropy_from_logits(logits, target, temperature: float = 1.0, window=None, compute_entropy: bool = True):
    """compute_logprobs_from_logits + compute_entropy_from_logits (rlinf/utils/utils.py:454-512) of `logits / temperature`
    (fsdp_actor_worker.py:478) restricted to the vocabulary window [lo, hi) (OpenVLA action bins,
    openvla_oft_action_model.py:546-551) in ONE pass over the logits, differentiable w.r.t. the raw logits.
    Returns (logprobs [...], entropy [...] or None), fp32."""
    lp, ent = _LogitsLogprobEntropy.apply(logits, target, temperature, window, bool(compute_entropy))
    return lp, (ent if compute_entropy else None)


def compute_logprobs_from_logits(logits, target, op_type: str = "torch"):
    """Drop-in for rlinf.utils.utils.compute_logprobs_from_logits (:454-492); `op_type` is accepted and ignored (the
    reference's flash_attn / liger variants compute the same quantity)."""
    return logprobs_entropy_from_logits(logits, target, compute_entropy=False)[0]


def compute_entropy_from_logits(logits, dim: int = -1):
    """Drop-in for rlinf.utils.utils.compute_entropy_from_logits (:495-512), last-dim only."""
    if dim not in (-1, logits.dim() - 1):
        raise ValueError("compute_entropy_from_logits: only the last (vocabulary) dimension is supported")
    tgt = torch.zeros(logits.shape[:-1], dtype=torch.int64, device=logits.device)
    return logprobs_entropy_from_logits(logits, tgt, compute_entropy=True)[1]


# ---------------------------------------------------------------------------------------------------------------
# The same, fused into the LM-head GEMM: hidden states and lm_head.weight in, no logits tensor (csrc/lmhead.cu)
# ---------------------------------------------------------------------------------------------------------------
LMHEAD_DZ_BUDGET = 1 << 30  # bytes of the backward's bf16 dZ chunk [N, Vc]


def _lmhead_check(hidden: torch.Tensor, weight: torch.Tensor):
    if hidden.dtype != torch.bfloat16 or weight.dtype != torch.bfloat16:
        raise ValueError(f"linear_logprobs_entropy: hidden and weight must be bfloat16, got {hidden.dtype} / {weight.dtype}")
    if weight.dim() != 2:
        raise ValueError(f"linear_logprobs_entropy: weight must be [V, H], got shape {tuple(weight.shape)}")
    H = weight.shape[1]
    if hidden.shape[-1] != H:
        raise ValueError(f"linear_logprobs_entropy: hidden size {hidden.shape[-1]} != weight's {H}")
    if H % 64 != 0 or not 64 <= H <= 8192:
        raise ValueError(f"linear_logprobs_entropy: needs H % 64 == 0 and 64 <= H <= 8192, got H = {H}")
    if not (hidden.is_cuda and weight.is_cuda):
        raise L.Rb200Error("rlinf_b200 kernels take CUDA tensors; move inputs with to_device() first")


def _lmhead_geometry(hidden: torch.Tensor):
    """(tensor, N, L, batch_stride, row_stride) of [N, H] or [bsz, L, H] hidden states: addressed in place when the last
    dim is contiguous, the other strides are multiples of 8 elements and the base is 16-byte aligned (e.g. the slice
    `hidden[:, -L-1:-1, :]`); anything else is made contiguous first."""
    H = hidden.shape[-1]
    if hidden.dim() in (2, 3) and hidden.stride(-1) == 1 and hidden.data_ptr() % 16 == 0:
        if hidden.dim() == 2 and hidden.stride(0) % 8 == 0 and hidden.stride(0) >= H:
            return hidden, hidden.shape[0], hidden.shape[0], hidden.shape[0] * hidden.stride(0), hidden.stride(0)
        if hidden.dim() == 3 and hidden.stride(1) % 8 == 0 and hidden.stride(1) >= H and hidden.stride(0) % 8 == 0:
            bsz, Lr, _ = hidden.shape
            return hidden, bsz * Lr, Lr, hidden.stride(0), hidden.stride(1)
    x = hidden.reshape(-1, H).contiguous()
    return x, x.shape[0], x.shape[0], x.shape[0] * H, H


def lmhead_workspace_bytes(N: int, L_rows: int, H: int, V: int, lo: int, hi: int, vocab_chunk: int = 0) -> int:
    """Workspace of the fused LM-head log-prob kernels (forward, and a backward in chunks of vocab_chunk columns;
    0 = the whole window)."""
    n = L.load().rb200_lmhead_workspace_bytes(N, L_rows, H, V, lo, hi, vocab_chunk)
    if n < 0:
        raise ValueError(f"linear_logprobs_entropy: unsupported shape N={N} L={L_rows} H={H} V={V} window=[{lo}, {hi})")
    return int(n)


def _lmhead_chunk(N: int, lo: int, hi: int) -> int:
    """dZ chunk width under LMHEAD_DZ_BUDGET: the whole window if it fits, multiples of 256 columns otherwise."""
    whole = -(-(hi - lo) // 256) * 256
    fit = max(256, LMHEAD_DZ_BUDGET // (2 * N) // 256 * 256)
    return min(whole, fit)


class _LinearLogprobEntropy(torch.autograd.Function):
    @staticmethod
    def forward(ctx, hidden, weight, target, temperature, window, want_entropy):
        _lmhead_check(hidden, weight)
        lib = L.load()
        x, N, Lr, bs, rs = _lmhead_geometry(hidden)
        w = weight.contiguous()
        V, H = w.shape
        tgt = L.to_device(target, x.device, torch.int64).reshape(-1).contiguous()
        if tgt.numel() != N:
            raise ValueError(f"target has {tgt.numel()} entries for {N} hidden rows")
        lo, hi = (0, V) if window is None else (int(window[0]), int(window[1]))
        if not 0 <= lo < hi <= V:
            raise ValueError(f"linear_logprobs_entropy: window [{lo}, {hi}) must lie inside [0, {V}) and be non-empty")
        vc = _lmhead_chunk(N, lo, hi)
        wsb = lmhead_workspace_bytes(N, Lr, H, V, lo, hi, vc)
        ws = torch.empty(wsb, dtype=torch.uint8, device=x.device)
        lp = torch.empty(N, dtype=torch.float32, device=x.device)
        ent = torch.empty(N, dtype=torch.float32, device=x.device) if want_entropy else None
        lse = torch.empty(N, dtype=torch.float32, device=x.device)
        L.check(lib.rb200_lmhead_logprob_entropy_fwd(_raw_ptr(x), L.ptr(w), L.ptr(tgt), N, Lr, bs, rs, H, V, lo, hi,
                                                     1.0 / float(temperature), L.ptr(lp), L.ptr(ent), L.ptr(lse),
                                                     L.ptr(ws), wsb, L.stream_ptr(x.device)),
                "lmhead_logprob_entropy_fwd")
        del ws
        ctx.save_for_backward(x, w, tgt, lse, ent if want_entropy else lse)
        ctx.meta = (N, Lr, bs, rs, H, V, lo, hi, vc, float(temperature), want_entropy, tuple(hidden.shape))
        shape = hidden.shape[:-1]
        if want_entropy:
            return lp.view(shape), ent.view(shape)
        none = lp.new_zeros(())
        ctx.mark_non_differentiable(none)
        return lp.view(shape), none

    @staticmethod
    def backward(ctx, g_lp, g_ent):
        lib = L.load()
        x, w, tgt, lse, ent = ctx.saved_tensors
        N, Lr, bs, rs, H, V, lo, hi, vc, temp, want_entropy, shape = ctx.meta
        need_x, need_w = ctx.needs_input_grad[0], ctx.needs_input_grad[1]
        if not (need_x or need_w):
            return None, None, None, None, None, None
        glp = g_lp.reshape(-1).float().contiguous() if g_lp is not None else None
        gh = g_ent.reshape(-1).float().contiguous() if (want_entropy and g_ent is not None) else None
        dx = torch.empty((N, H), dtype=torch.bfloat16, device=x.device) if need_x else None
        dw = torch.empty((V, H), dtype=torch.bfloat16, device=x.device) if need_w else None
        wsb = lmhead_workspace_bytes(N, Lr, H, V, lo, hi, vc)
        ws = torch.empty(wsb, dtype=torch.uint8, device=x.device)
        L.check(lib.rb200_lmhead_logprob_entropy_bwd(_raw_ptr(x), L.ptr(w), L.ptr(tgt), N, Lr, bs, rs, H, V, lo, hi,
                                                     1.0 / temp, L.ptr(lse), L.ptr(ent) if gh is not None else None,
                                                     L.ptr(glp), L.ptr(gh), L.ptr(dx), L.ptr(dw), L.ptr(ws), wsb,
                                                     L.stream_ptr(x.device)),
                "lmhead_logprob_entropy_bwd")
        return (dx.view(shape) if need_x else None), dw, None, None, None, None


def linear_logprobs_entropy(hidden, weight, target, temperature: float = 1.0, window=None, compute_entropy: bool = True):
    """logprobs_entropy_from_logits(hidden @ weight.T, ...) without the logits tensor: `hidden` [N, H] or [bsz, L, H]
    (e.g. the last hidden state's `[:, -L-1:-1, :]` slice, read in place) and `weight` = lm_head.weight [V, H], both
    bf16, H % 64 == 0.  Temperature and the vocabulary window [lo, hi) act as in logprobs_entropy_from_logits.
    Differentiable w.r.t. hidden and weight (only the gradients whose inputs require them are computed).
    Returns (logprobs [...], entropy [...] or None), fp32."""
    lp, ent = _LinearLogprobEntropy.apply(hidden, weight, target, temperature, window, bool(compute_entropy))
    return lp, (ent if compute_entropy else None)


# ---------------------------------------------------------------------------------------------------------------
# Vocabulary-parallel (tensor-parallel) variants: each rank holds one equal shard of the vocabulary (Megatron's
# VocabUtility, parallel_output=True), reduces it to one 16-byte record per row, and ONE all-gather of the records
# gives every rank the rows' log-probs / entropies (csrc/vocab_parallel.cu)
# ---------------------------------------------------------------------------------------------------------------
def _vp_group(group, what: str):
    """(group, P, rank) of the tensor-parallel group the vocabulary is split over.  group=None resolves to Megatron's
    tensor-parallel group when megatron.core's model parallelism is initialised (as the reference's functions use), to
    one rank when torch.distributed is not initialised or its world has one rank, and is an error otherwise: the world
    group of a data- or pipeline-parallel job is not the group the vocabulary is split over."""
    import torch.distributed as dist

    if not (dist.is_available() and dist.is_initialized()):
        return None, 1, 0
    if group is None:
        try:
            from megatron.core import parallel_state
        except ImportError:
            parallel_state = None
        if parallel_state is not None and parallel_state.model_parallel_is_initialized():
            group = parallel_state.get_tensor_model_parallel_group()
        elif dist.get_world_size() > 1:
            raise ValueError(f"{what}: torch.distributed has {dist.get_world_size()} ranks and Megatron's model "
                             "parallelism is not initialised; pass the tensor-parallel group as group=")
    return group, dist.get_world_size(group), dist.get_rank(group)


def _vp_window(window, Vs: int, world_size: int, what: str, vocab_size=None):
    V = Vs * world_size
    if vocab_size is not None and int(vocab_size) != V:
        raise ValueError(f"{what}: shards must be equal, but vocab_size {vocab_size} != P * Vs = {world_size} * {Vs}")
    lo, hi = (0, V) if window is None else (int(window[0]), int(window[1]))
    if not 0 <= lo < hi <= V:
        raise ValueError(f"{what}: window [{lo}, {hi}) must lie inside [0, {V}) (P = {world_size} shards of {Vs}) "
                         "and be non-empty")
    return lo, hi


def _vp_rank(rank: int, world_size: int, what: str):
    if not 0 <= rank < world_size:
        raise ValueError(f"{what}: rank {rank} outside [0, {world_size})")


def _vp_target(target, device, N: int):
    tgt = L.to_device(target, device, torch.int64).reshape(-1).contiguous()
    if tgt.numel() != N:
        raise ValueError(f"target has {tgt.numel()} entries for {N} rows")
    return tgt


def lmhead_vp_workspace_bytes(N: int, L_rows: int, H: int, Vs: int, vocab_start: int, lo: int, hi: int,
                              vocab_chunk: int = 0) -> int:
    """Workspace of the shard's fused forward and of a backward in chunks of vocab_chunk columns (0 = the shard's
    whole part of the window; < 0 = the forward only)."""
    n = L.load().rb200_lmhead_vp_workspace_bytes(N, L_rows, H, Vs, vocab_start, lo, hi, vocab_chunk)
    if n < 0:
        raise ValueError(f"vocab_parallel_linear_logprobs_entropy: unsupported shape N={N} L={L_rows} H={H} Vs={Vs} "
                         f"vocab_start={vocab_start} window=[{lo}, {hi})")
    return int(n)


def _lmhead_vp_fwd(x, N, Lr, bs, rs, w, tgt, rank, lo, hi, temperature):
    Vs, H = w.shape
    vs = rank * Vs
    wsb = lmhead_vp_workspace_bytes(N, Lr, H, Vs, vs, lo, hi, -1)  # the forward's workspace only
    ws = torch.empty(wsb, dtype=torch.uint8, device=x.device)
    rec = torch.empty(N, 4, dtype=torch.float32, device=x.device)
    L.check(L.load().rb200_lmhead_vp_partials_fwd(_raw_ptr(x), L.ptr(w), L.ptr(tgt), N, Lr, bs, rs, H, Vs, vs, lo, hi,
                                                  1.0 / float(temperature), L.ptr(rec), L.ptr(ws), wsb,
                                                  L.stream_ptr(x.device)), "lmhead_vp_partials_fwd")
    return rec


def _lmhead_vp_bwd(x, N, Lr, bs, rs, w, tgt, rank, lo, hi, temperature, lse, ent, glp, gh, need_x, need_w):
    Vs, H = w.shape
    vs = rank * Vs
    slo, shi = min(max(lo - vs, 0), Vs), min(max(hi - vs, 0), Vs)
    vc = _lmhead_chunk(N, slo, shi) if slo < shi else 0
    wsb = lmhead_vp_workspace_bytes(N, Lr, H, Vs, vs, lo, hi, vc)
    ws = torch.empty(wsb, dtype=torch.uint8, device=x.device)
    dx = torch.empty((N, H), dtype=torch.float32, device=x.device) if need_x else None
    dw = torch.empty((Vs, H), dtype=torch.bfloat16, device=x.device) if need_w else None
    L.check(L.load().rb200_lmhead_vp_logprob_entropy_bwd(_raw_ptr(x), L.ptr(w), L.ptr(tgt), N, Lr, bs, rs, H, Vs, vs,
                                                         lo, hi, 1.0 / float(temperature), L.ptr(lse),
                                                         L.ptr(ent) if gh is not None else None, L.ptr(glp), L.ptr(gh),
                                                         L.ptr(dx), L.ptr(dw), L.ptr(ws), wsb, L.stream_ptr(x.device)),
            "lmhead_vp_logprob_entropy_bwd")
    return dx, dw


def lmhead_vp_partials(hidden, weight_shard, target, rank: int, world_size: int, temperature: float = 1.0,
                       window=None, vocab_size=None) -> torch.Tensor:
    """Rank `rank`'s records [N, 4] fp32 {m, s, t, z_t} of hidden @ weight_shard.T, weight_shard = rows
    [rank * Vs, (rank + 1) * Vs) of lm_head.weight; global targets and window.  No communication: with vp_combine
    this emulates `world_size` ranks on one device.  vocab_size, when given, must be world_size * Vs."""
    what = "vocab_parallel_linear_logprobs_entropy"
    _vp_rank(rank, world_size, what)
    lo, hi = _vp_window(window, weight_shard.shape[0], world_size, what, vocab_size)
    _lmhead_check(hidden, weight_shard)
    x, N, Lr, bs, rs = _lmhead_geometry(hidden)
    w = weight_shard.contiguous()
    return _lmhead_vp_fwd(x, N, Lr, bs, rs, w, _vp_target(target, x.device, N), rank, lo, hi, temperature)


def lmhead_vp_backward(hidden, weight_shard, target, rank: int, world_size: int, lse, entropy, grad_logprob,
                       grad_entropy, temperature: float = 1.0, window=None, need_hidden=True, need_weight=True):
    """Rank `rank`'s share of the backward given the combined lse / entropy: (dX partial [N, H] fp32 to be summed over
    ranks, or None; d_weight_shard [Vs, H] bf16, or None)."""
    what = "vocab_parallel_linear_logprobs_entropy"
    _vp_rank(rank, world_size, what)
    lo, hi = _vp_window(window, weight_shard.shape[0], world_size, what)
    _lmhead_check(hidden, weight_shard)
    x, N, Lr, bs, rs = _lmhead_geometry(hidden)
    w = weight_shard.contiguous()
    glp = grad_logprob.reshape(-1).float().contiguous() if grad_logprob is not None else None
    gh = grad_entropy.reshape(-1).float().contiguous() if grad_entropy is not None else None
    return _lmhead_vp_bwd(x, N, Lr, bs, rs, w, _vp_target(target, x.device, N), rank, lo, hi, temperature,
                          lse.contiguous(), entropy.contiguous() if entropy is not None else None, glp, gh,
                          need_hidden, need_weight)


def logits_vp_partials(logits_shard, target, rank: int, world_size: int, temperature: float = 1.0,
                       window=None, vocab_size=None) -> torch.Tensor:
    """Rank `rank`'s records [N, 4] fp32 {m, s, t, z_t} of a [..., Vs] logits shard (fp32 or bf16, the `[:, -L-1:-1, :]`
    slice read in place), global targets and window."""
    what = "vocab_parallel_entropy_and_log_probs"
    if logits_shard.dtype not in (torch.float32, torch.bfloat16):
        raise ValueError(f"{what}: logits must be float32 or bfloat16, got {logits_shard.dtype}")
    _vp_rank(rank, world_size, what)
    lo, hi = _vp_window(window, logits_shard.shape[-1], world_size, what, vocab_size)
    x, N, Lr, bs, rs, Vs = _logits_geometry(logits_shard)
    tgt = _vp_target(target, x.device, N)
    rec = torch.empty(N, 4, dtype=torch.float32, device=x.device)
    L.check(L.load().rb200_logits_vp_partials_fwd(_raw_ptr(x), 0 if x.dtype == torch.float32 else 1, L.ptr(tgt), N, Lr,
                                                  bs, rs, Vs, rank * Vs, lo, hi, 1.0 / float(temperature), L.ptr(rec),
                                                  L.stream_ptr(x.device)), "logits_vp_partials_fwd")
    return rec


def vp_combine(records, target, vocab_shard: int, window=None, compute_entropy: bool = True):
    """records [P, N, 4] gathered in rank order -> (logprob [N], entropy [N] or None, lse [N]), fp32."""
    P, N = records.shape[0], records.shape[1]
    if records.dtype != torch.float32 or records.shape[2] != 4:
        raise ValueError(f"vp_combine: records must be [P, N, 4] float32, got {tuple(records.shape)} {records.dtype}")
    rec = records.contiguous()
    lo, hi = _vp_window(window, vocab_shard, P, "vp_combine")
    tgt = _vp_target(target, rec.device, N)
    lp = torch.empty(N, dtype=torch.float32, device=rec.device)
    ent = torch.empty(N, dtype=torch.float32, device=rec.device) if compute_entropy else None
    lse = torch.empty(N, dtype=torch.float32, device=rec.device)
    L.check(L.load().rb200_vp_combine(L.ptr(rec), P, N, L.ptr(tgt), vocab_shard, lo, hi, L.ptr(lp), L.ptr(ent),
                                      L.ptr(lse), L.stream_ptr(rec.device)), "vp_combine")
    return lp, ent, lse


def _vp_gather(rec: torch.Tensor, group, P: int) -> torch.Tensor:
    """[N, 4] -> [P, N, 4]: the one collective of the forward."""
    if P == 1:
        return rec[None]
    import torch.distributed as dist

    out = torch.empty((P, *rec.shape), dtype=rec.dtype, device=rec.device)
    dist.all_gather_into_tensor(out, rec, group=group)
    return out


class _VPLinearLogprobEntropy(torch.autograd.Function):
    @staticmethod
    def forward(ctx, hidden, weight_shard, target, group, temperature, window, want_entropy, reduce_hidden_grad,
                vocab_size):
        what = "vocab_parallel_linear_logprobs_entropy"
        group, P, k = _vp_group(group, what)
        Vs = weight_shard.shape[0]
        lo, hi = _vp_window(window, Vs, P, what, vocab_size)
        _lmhead_check(hidden, weight_shard)
        x, N, Lr, bs, rs = _lmhead_geometry(hidden)
        w = weight_shard.contiguous()
        tgt = _vp_target(target, x.device, N)
        rec = _lmhead_vp_fwd(x, N, Lr, bs, rs, w, tgt, k, lo, hi, temperature)
        lp, ent, lse = vp_combine(_vp_gather(rec, group, P), tgt, Vs, (lo, hi), want_entropy)
        ctx.save_for_backward(x, w, tgt, lse, ent if want_entropy else lse)
        ctx.meta = (group, P, k, N, Lr, bs, rs, lo, hi, float(temperature), want_entropy, reduce_hidden_grad,
                    tuple(hidden.shape))
        shape = hidden.shape[:-1]
        if want_entropy:
            return lp.view(shape), ent.view(shape)
        none = lp.new_zeros(())
        ctx.mark_non_differentiable(none)
        return lp.view(shape), none

    @staticmethod
    def backward(ctx, g_lp, g_ent):
        x, w, tgt, lse, ent = ctx.saved_tensors
        group, P, k, N, Lr, bs, rs, lo, hi, temp, want_entropy, reduce_hidden_grad, shape = ctx.meta
        need_x, need_w = ctx.needs_input_grad[0], ctx.needs_input_grad[1]
        if not (need_x or need_w):
            return (None,) * 9
        glp = g_lp.reshape(-1).float().contiguous() if g_lp is not None else None
        gh = g_ent.reshape(-1).float().contiguous() if (want_entropy and g_ent is not None) else None
        dx32, dw = _lmhead_vp_bwd(x, N, Lr, bs, rs, w, tgt, k, lo, hi, temp, lse, ent, glp, gh, need_x, need_w)
        dx = None
        if need_x:
            if P > 1 and reduce_hidden_grad:
                import torch.distributed as dist

                dist.all_reduce(dx32, group=group)  # fp32: the rank sum rounds to bf16 once, below
            dx = dx32.to(torch.bfloat16).view(shape)
        return dx, dw, None, None, None, None, None, None, None


def vocab_parallel_linear_logprobs_entropy(hidden, weight_shard, target, group=None, temperature: float = 1.0,
                                           window=None, compute_entropy: bool = True, reduce_hidden_grad: bool = True,
                                           vocab_size=None):
    """linear_logprobs_entropy with the vocabulary split over the ranks of `group` (tensor parallelism): rank k holds
    weight_shard = lm_head.weight[k * Vs:(k + 1) * Vs] (equal shards, as Megatron pads the vocabulary), `hidden` is the
    full [N, H] / [bsz, L, H] input on every rank, `target` and `window` are global.  `group` is the tensor-parallel group; None resolves to Megatron's
    tensor-parallel group when megatron.core's model parallelism is initialised, to one rank without torch.distributed
    (or with a one-rank world), and raises ValueError in any other multi-rank job.
    The forward does one all-gather of N x 16 bytes and returns the same log-probs / entropies on every rank; the
    backward returns d_weight_shard and all-reduces dX in fp32 (reduce_hidden_grad=False leaves the rank's fp32 share
    un-summed, cast to bf16, for callers that reduce-scatter it themselves).  Shard widths are not compared across
    ranks (that would cost a collective per call): vocab_size, when given, is checked against P * Vs and is the only
    guard against unequal shards.  Without an initialised torch.distributed, P = 1 and the results are bit-identical
    to linear_logprobs_entropy.  Returns (logprobs [...], entropy [...] or None), fp32."""
    lp, ent = _VPLinearLogprobEntropy.apply(hidden, weight_shard, target, group, temperature, window,
                                            bool(compute_entropy), bool(reduce_hidden_grad), vocab_size)
    return lp, (ent if compute_entropy else None)


class _VPLogitsLogprobEntropy(torch.autograd.Function):
    @staticmethod
    def forward(ctx, logits, target, group, want_entropy, entropy_grad):
        what = "vocab_parallel_entropy_and_log_probs"
        if logits.dtype not in (torch.float32, torch.bfloat16):
            raise ValueError(f"{what}: logits must be float32 or bfloat16, got {logits.dtype}")
        group, P, k = _vp_group(group, what)
        x, N, Lr, bs, rs, Vs = _logits_geometry(logits)
        tgt = _vp_target(target, x.device, N)
        rec = torch.empty(N, 4, dtype=torch.float32, device=x.device)
        L.check(L.load().rb200_logits_vp_partials_fwd(_raw_ptr(x), 0 if x.dtype == torch.float32 else 1, L.ptr(tgt),
                                                      N, Lr, bs, rs, Vs, k * Vs, 0, P * Vs, 1.0, L.ptr(rec),
                                                      L.stream_ptr(x.device)), "logits_vp_partials_fwd")
        lp, ent, lse = vp_combine(_vp_gather(rec, group, P), tgt, Vs, None, want_entropy)
        ctx.save_for_backward(x, tgt - k * Vs, lse, ent if want_entropy else lse)  # shard-local targets
        ctx.meta = (N, Lr, bs, rs, Vs, entropy_grad, tuple(logits.shape))
        shape = logits.shape[:-1]
        ent = ent.view(shape) if want_entropy else lp.new_zeros(())
        if not entropy_grad:
            ctx.mark_non_differentiable(ent)
        return lp.view(shape), ent

    @staticmethod
    def backward(ctx, g_lp, g_ent):
        x, tgt_local, lse, ent = ctx.saved_tensors
        N, Lr, bs, rs, Vs, entropy_grad, shape = ctx.meta
        glp = g_lp.reshape(-1).float().contiguous() if g_lp is not None else None
        gh = g_ent.reshape(-1).float().contiguous() if (entropy_grad and g_ent is not None) else None
        return _logits_vp_bwd(x, N, Lr, bs, rs, Vs, tgt_local, lse, ent, glp, gh).view(shape), None, None, None, None


def _logits_vp_bwd(x, N, Lr, bs, rs, Vs, tgt_local, lse, ent, glp, gh):
    """dlogits [N, Vs] of the shard: the single-GPU backward with the global lse / entropy and shard-local targets
    (ids outside [0, Vs) get no target term)."""
    dx = torch.empty((N, Vs), dtype=x.dtype, device=x.device)
    L.check(L.load().rb200_logits_logprob_entropy_bwd(_raw_ptr(x), 0 if x.dtype == torch.float32 else 1,
                                                      L.ptr(tgt_local), N, Lr, bs, rs, Vs, 0, Vs, 1.0, L.ptr(lse),
                                                      L.ptr(ent) if gh is not None else None, L.ptr(glp), L.ptr(gh),
                                                      L.ptr(dx), Lr * Vs, Vs, L.stream_ptr(x.device)),
            "logits_logprob_entropy_bwd")
    return dx


def logits_vp_backward(logits_shard, target, rank: int, lse, entropy, grad_logprob, grad_entropy) -> torch.Tensor:
    """Rank `rank`'s dlogits [N, Vs] (the shard's dtype) given the combined lse / entropy and global targets."""
    x, N, Lr, bs, rs, Vs = _logits_geometry(logits_shard)
    tgt = _vp_target(target, x.device, N) - rank * Vs
    glp = grad_logprob.reshape(-1).float().contiguous() if grad_logprob is not None else None
    gh = grad_entropy.reshape(-1).float().contiguous() if grad_entropy is not None else None
    return _logits_vp_bwd(x, N, Lr, bs, rs, Vs, tgt, lse.contiguous(),
                          entropy.contiguous() if entropy is not None else None, glp, gh)


def vocab_parallel_entropy_and_log_probs(vocab_parallel_logits, target, label_smoothing: float = 0.0,
                                         calculate_entropy_loss: bool = True, group=None):
    """Drop-in for rlinf.utils.distributed.vocab_parallel_entropy_and_log_probs (:1230-1242): the rank's logits shard
    [..., Vs] (fp32 or bf16, Megatron's parallel_output=True; its padded vocabulary makes the shards equal), global
    targets, over the ranks of `group`.  `group` is the tensor-parallel group; None resolves to Megatron's
    tensor-parallel group when megatron.core's model parallelism is initialised, to one rank without torch.distributed
    (or with a one-rank world), and raises ValueError in any other multi-rank job.  One all-gather of N x 16 bytes
    per call; nothing [N, Vs] is saved for the backward beyond the logits themselves.  Returns (entropy, log_probs),
    fp32.  The entropy gradient is the mathematical one, which the reference's is not (DESIGN.md §2); with
    calculate_entropy_loss=False the entropy is returned without a gradient, as in the reference."""
    if label_smoothing != 0.0:
        raise ValueError("vocab_parallel_entropy_and_log_probs: label_smoothing != 0 is not supported")
    lp, ent = _VPLogitsLogprobEntropy.apply(vocab_parallel_logits, target, group, True, bool(calculate_entropy_loss))
    return ent, lp


def vocab_parallel_log_probs_from_logits(logits, labels, group=None):
    """Drop-in for rlinf.utils.distributed.vocab_parallel_log_probs_from_logits (:1245-1250, = -Megatron's
    vocab_parallel_cross_entropy) from the rank's logits shard; fp32 log-probs.  `group` as in
    vocab_parallel_entropy_and_log_probs."""
    return _VPLogitsLogprobEntropy.apply(logits, labels, group, False, False)[0]


# ---------------------------------------------------------------------------------------------------------------
# Response rows only: the LM-head log-probs / entropies of the rows a reasoning loss reads, for padded and packed
# batches, written straight into [bsz, response_len] (response_rows.py, csrc/response_rows.cu)
# ---------------------------------------------------------------------------------------------------------------
class _GatherRows(torch.autograd.Function):
    """hidden [T, H] -> the plan's compact rows [R, H]; the backward scatters dX back through the plan's inverse map
    (every row written once, zeros outside the responses)."""

    @staticmethod
    def forward(ctx, x, rows, hidden_map):
        ctx.save_for_backward(hidden_map)
        return gather_rows(x, rows)

    @staticmethod
    def backward(ctx, g):
        (hidden_map,) = ctx.saved_tensors
        ext = torch.cat([g.contiguous(), g.new_zeros(1, g.shape[1])])  # row R: the -1 sentinel's zero row
        return gather_rows(ext, hidden_map), None, None


class _ToCells(torch.autograd.Function):
    """Compact values [R] -> [bsz, L] (zeros past r_b); the backward gathers the cells' gradients back to compact rows.
    shift 1 reads each cell one compact row later (the FSDP-packed entropy alignment)."""

    @staticmethod
    def forward(ctx, v, cell_map, back_idx, shift, shape):
        ctx.save_for_backward(back_idx)
        ext = torch.cat([v, v.new_zeros(1)])
        return gather_rows(ext[shift:], cell_map).view(shape)

    @staticmethod
    def backward(ctx, g):
        (back_idx,) = ctx.saved_tensors
        ext = torch.cat([g.reshape(-1).float(), g.new_zeros(1, dtype=torch.float32)])
        return gather_rows(ext, back_idx), None, None, None, None


def response_logprobs_entropy(hidden, weight, tokens, plan, *, temperature: float = 1.0, compute_entropy: bool = True,
                              group=None):
    """Log-probabilities and entropies of `hidden @ weight.T / temperature` at the response tokens of a padded or
    packed batch, computed on the plan's rows only and returned as (logprobs [bsz, response_len], entropy
    [bsz, response_len] or None), fp32, zeros at j >= r_b - the layout reasoning_actor_loss reads.
    hidden: [T, H], [1, T, H], [T, 1, H] (Megatron's sequence-first output) or [bsz, S, H], bf16; tokens: the
    matching token ids (targets are read from them).  plan: a response_rows.padded / fsdp_packed / megatron_thd plan.
    weight is lm_head.weight [V, H] on one rank, or the rank's vocabulary shard when `group` (resolved as in
    vocab_parallel_linear_logprobs_entropy) has more than one rank; the all-gather then covers the plan's R rows.
    Differentiable w.r.t. hidden and weight (only where required); dX is zero on rows outside every response.
    Host syncs: none with host lengths; one device-to-host copy of R and the plan's verdict with device lengths;
    none in the backward.  With R = 0 the outputs are constant zeros."""
    what = "response_logprobs_entropy"
    if hidden.dim() not in (2, 3):
        raise ValueError(f"{what}: hidden must be [T, H], [1, T, H], [T, 1, H] or [bsz, S, H], got "
                         f"{tuple(hidden.shape)}")
    _lmhead_check(hidden, weight)
    group, P, _ = _vp_group(group, what)
    x = hidden.reshape(-1, hidden.shape[-1])
    T = x.shape[0]
    tok = L.to_device(tokens, x.device, torch.int64).reshape(-1)
    if tok.numel() != T:
        raise ValueError(f"{what}: {tok.numel()} token ids for {T} hidden rows")
    idx = plan.index(tok, T)
    shape = (plan.bsz, plan.response_len)
    if idx.R == 0:
        z = torch.zeros(shape, dtype=torch.float32, device=x.device)
        return z, (torch.zeros_like(z) if compute_entropy else None)
    hc = _GatherRows.apply(x, idx.rows, idx.hidden_map)
    if P == 1:
        lp, ent = linear_logprobs_entropy(hc, weight, idx.targets, temperature, None, compute_entropy)
    else:
        lp, ent = vocab_parallel_linear_logprobs_entropy(hc, weight, idx.targets, group=group, temperature=temperature,
                                                         compute_entropy=compute_entropy)
    s = plan.entropy_shift
    lp = _ToCells.apply(lp, idx.cell_map, idx.cells[1:], 0, shape)
    if compute_entropy:
        ent = _ToCells.apply(ent, idx.cell_map, idx.cells[1 - s:1 - s + idx.R], s, shape)
    return lp, ent


# ---------------------------------------------------------------------------------------------------------------
# Response rows under Megatron sequence and context parallelism: each rank passes its hidden-state shard, only the
# response rows cross the tensor-parallel group (response_rows.megatron_parallel, csrc/response_rows_mp.cu).  The
# stages below are one rank's work between collectives; megatron_response_logprobs_entropy runs them with
# torch.distributed, and a test can run them rank by rank with each collective replaced by a concatenation or a sum.
# ---------------------------------------------------------------------------------------------------------------
def mp_pack(hidden_shard, idx):
    """The rank's response rows: [Rmax_k, H] (SP; pad rows repeat a row of the shard and are dropped by mp_unpad),
    or the CP rank's compact rows [R_c, H] without SP."""
    x = hidden_shard.reshape(-1, hidden_shard.shape[-1])
    return gather_rows(x, idx.send if idx.sp else idx.rows)


def mp_unpad(gathered, idx):
    """TP-gathered rows [tp, Rmax_k, H] -> the CP rank's compact rows [R_c, H] (SP)."""
    return gather_rows(gathered.reshape(-1, gathered.shape[-1]), idx.unpad)


def mp_values(logprob, entropy, idx):
    """Compact log-probs / entropies [R_c] -> the [Rmax_c, 2] fp32 buffer of the CP all-gather (zero pad rows)."""
    vals = torch.zeros((idx.Rmax_c, 2), dtype=torch.float32, device=idx.cell_map.device)
    if idx.R:
        vals[:idx.R, 0] = logprob
        if entropy is not None:
            vals[:idx.R, 1] = entropy
    return vals


def mp_to_cells(gathered, idx, shape, compute_entropy=True):
    """CP-gathered values [cp, Rmax_c, 2] -> (logprobs [bsz, L], entropy [bsz, L] or None), zeros at j >= r_b."""
    ext = torch.cat([gathered.reshape(-1, 2), gathered.new_zeros(1, 2)])  # row cp * Rmax_c: the -1 sentinel's zeros
    out = gather_rows(ext, idx.cell_map)
    lp = out[:, 0].reshape(shape).contiguous()
    return lp, (out[:, 1].reshape(shape).contiguous() if compute_entropy else None)


def mp_cell_grads(grad_logprob, grad_entropy, idx):
    """Gradients of the [bsz, L] outputs -> the CP rank's compact rows [R_c] (other CP ranks' cells are dropped)."""
    def one(g):
        return None if g is None else gather_rows(g.reshape(-1).float().contiguous(), idx.cells)
    return one(grad_logprob), one(grad_entropy)


def mp_pack_grad(dx32, idx):
    """The rank's fp32 dX share of the compact rows [R_c, H] -> bf16, rounded once: the [tp, Rmax_k, H]
    reduce-scatter send layout (SP, zero pad rows), or, without SP, dX of the whole [T_c, H] input (zeros off the
    response rows; dx32 is then already summed over the TP ranks)."""
    H = dx32.shape[-1]
    m = idx.slot_map if idx.sp else idx.hidden_map
    out = torch.empty((m.numel(), H), dtype=torch.bfloat16, device=m.device)
    if idx.R == 0:  # a rank without prediction rows sends zeros
        out.zero_()
    else:
        L.check(L.load().rb200_response_rows_mp_pack_grad(L.ptr(dx32), L.ptr(m), L.ptr(out), m.numel(), H,
                                                          L.stream_ptr(m.device)), "response_rows_mp_pack_grad")
    return out.view(idx.tp, idx.Rmax_k, H) if idx.sp else out


def mp_grad_buffer(idx, H: int):
    """[Rmax_k + 1, H] bf16 receive buffer of the reduce-scatter (SP): rows [:Rmax_k] are written by the collective,
    the last row is the zero row of the -1 sentinel."""
    buf = torch.empty((idx.Rmax_k + 1, H), dtype=torch.bfloat16, device=idx.cell_map.device)
    buf[-1].zero_()
    return buf


def mp_unpack_grad(buf, idx):
    """Reduce-scattered rows (mp_grad_buffer) -> dX of the rank's hidden shard [T_c / tp, H], zeros elsewhere."""
    return gather_rows(buf, idx.hidden_map)


def _mp_group(group, kind: str, size: int, what: str):
    """(group, size, rank) of Megatron's tensor- or context-parallel group: group=None resolves to Megatron's group
    when megatron.core's model parallelism is initialised, to one rank when torch.distributed is not initialised or the
    plan has one rank along this dimension, and is an error otherwise."""
    import torch.distributed as dist

    if not (dist.is_available() and dist.is_initialized()):
        got = (None, 1, 0)
    else:
        if group is None:
            try:
                from megatron.core import parallel_state
            except ImportError:
                parallel_state = None
            if parallel_state is not None and parallel_state.model_parallel_is_initialized():
                group = (parallel_state.get_tensor_model_parallel_group() if kind == "tp"
                         else parallel_state.get_context_parallel_group())
            elif size > 1:
                raise ValueError(f"{what}: the plan has {kind}_size {size} and Megatron's model parallelism is not "
                                 f"initialised; pass the {kind} group as {kind}_group=")
        got = (None, 1, 0) if group is None else (group, dist.get_world_size(group), dist.get_rank(group))
    if got[1] != size:
        raise ValueError(f"{what}: the {kind} group has {got[1]} ranks, the plan {kind}_size {size}")
    return got


class _MegatronResponseRows(torch.autograd.Function):
    @staticmethod
    def forward(ctx, hidden, weight_shard, idx, tp_group, cp_group, temperature, want_entropy, shape):
        import torch.distributed as dist

        H = hidden.shape[-1]
        tp, cp, k = idx.tp, idx.cp, idx.k
        if idx.sp:
            send = mp_pack(hidden, idx)
            if tp > 1:
                gathered = torch.empty((tp, idx.Rmax_k, H), dtype=send.dtype, device=send.device)
                dist.all_gather_into_tensor(gathered, send, group=tp_group)
            else:
                gathered = send[None]
            hc = mp_unpad(gathered, idx)
        else:
            hc = mp_pack(hidden, idx)
        w = weight_shard.contiguous()
        Vs = w.shape[0]
        if idx.R:
            rec = _lmhead_vp_fwd(hc, idx.R, idx.R, idx.R * H, H, w, idx.targets, k, 0, tp * Vs, temperature)
        else:
            rec = torch.empty((0, 4), dtype=torch.float32, device=hc.device)
        recs = _vp_gather(rec, tp_group, tp)
        if idx.R:
            lp, ent, lse = vp_combine(recs, idx.targets, Vs, None, want_entropy)
        else:
            lp = ent = lse = rec[:, 0]
        vals = mp_values(lp, ent, idx)
        if cp > 1:
            allv = torch.empty((cp, *vals.shape), dtype=vals.dtype, device=vals.device)
            dist.all_gather_into_tensor(allv, vals, group=cp_group)
        else:
            allv = vals[None]
        out_lp, out_ent = mp_to_cells(allv, idx, shape, want_entropy)
        ctx.save_for_backward(hc, w, lse, ent if want_entropy else lse)
        ctx.meta = (idx, tp_group, float(temperature), want_entropy, tuple(hidden.shape))
        if want_entropy:
            return out_lp, out_ent
        none = out_lp.new_zeros(())
        ctx.mark_non_differentiable(none)
        return out_lp, none

    @staticmethod
    def backward(ctx, g_lp, g_ent):
        import torch.distributed as dist

        hc, w, lse, ent = ctx.saved_tensors
        idx, tp_group, temp, want_entropy, shape = ctx.meta
        need_x, need_w = ctx.needs_input_grad[0], ctx.needs_input_grad[1]
        if not (need_x or need_w):
            return (None,) * 8
        H, Vs, tp = hc.shape[1], w.shape[0], idx.tp
        glp, gh = mp_cell_grads(g_lp, g_ent if want_entropy else None, idx)
        if idx.R:
            dx32, dw = _lmhead_vp_bwd(hc, idx.R, idx.R, idx.R * H, H, w, idx.targets, idx.k, 0, tp * Vs, temp, lse,
                                      ent, glp, gh, need_x, need_w)
        else:
            dx32 = hc.new_zeros((0, H), dtype=torch.float32) if need_x else None
            dw = torch.zeros_like(w) if need_w else None
        dx = None
        if need_x:
            if idx.sp:
                send = mp_pack_grad(dx32, idx)
                buf = mp_grad_buffer(idx, H)
                if tp > 1:
                    dist.reduce_scatter_tensor(buf[:-1], send.reshape(-1, H), group=tp_group)  # bf16, as Megatron
                else:
                    buf[:-1].copy_(send[0])
                dx = mp_unpack_grad(buf, idx)
            else:
                if tp > 1:
                    dist.all_reduce(dx32, group=tp_group)  # fp32: the rank sum rounds to bf16 once, below
                dx = mp_pack_grad(dx32, idx)
            dx = dx.view(shape)
        return dx, dw, None, None, None, None, None, None


def megatron_response_logprobs_entropy(hidden_shard, weight_shard, responses, plan, *, temperature: float = 1.0,
                                       compute_entropy: bool = True, tp_group=None, cp_group=None):
    """response_logprobs_entropy for Megatron's packed THD batches under tensor, sequence and context parallelism, from
    each rank's own hidden-state shard: hidden_shard is the decoder output [T_c / tp, 1, H] or [T_c / tp, H] under
    sequence parallelism, [T_c, 1, H] or [T_c, H] without it (T_c = the CP rank's packed rows), bf16; weight_shard is
    the rank's vocabulary shard of the output layer; responses = input_ids[:, -response_len:] [bsz, response_len], the
    targets; plan = response_rows.megatron_parallel(...).  Returns (logprobs [bsz, response_len], entropy or None),
    fp32, the same on every rank, zeros at j >= r_b - what the reference's loss reads from log_probs[:, -L-1:-1].
    tp_group / cp_group: None resolves to Megatron's tensor- / context-parallel group when megatron.core's model
    parallelism is initialised, to one rank when the plan has one rank along that dimension (or without
    torch.distributed); sizes that disagree with the plan raise ValueError.
    Collectives: forward, under SP one all-gather of the rank's padded response rows [Rmax_k, H] bf16 over TP, one
    all-gather of the [R_c, 4] records over TP, one all-gather of [Rmax_c, 2] fp32 values over CP; backward, one bf16
    reduce-scatter over TP under SP, or an fp32 all-reduce of [R_c, H] without it, and nothing over CP.  As in the
    reference's postprocess_packed_seqs, other CP ranks' cells arrive detached: a rank's dX comes only from the cells
    whose rows it holds, its d_weight_shard from all of its CP rank's rows.  Host syncs: none with host lengths; one
    device-to-host copy of the counts and the plan's verdict with device lengths."""
    what = "megatron_response_logprobs_entropy"
    if hidden_shard.dim() not in (2, 3) or (hidden_shard.dim() == 3 and hidden_shard.shape[1] != 1):
        raise ValueError(f"{what}: hidden_shard must be [rows, H] or [rows, 1, H], got {tuple(hidden_shard.shape)}")
    _lmhead_check(hidden_shard, weight_shard)
    tp_group, tp, k = _mp_group(tp_group, "tp", plan.tp_size, what)
    cp_group, cp, c = _mp_group(cp_group, "cp", plan.cp_size, what)
    x = hidden_shard.reshape(-1, hidden_shard.shape[-1])
    resp = L.to_device(responses, x.device, torch.int64)
    idx = plan.index(resp, x.shape[0], k, c)
    shape = (plan.bsz, plan.response_len)
    if all(sum(r) == 0 for r in idx.counts):  # no response row on any rank: no collective on any rank
        z = torch.zeros(shape, dtype=torch.float32, device=x.device)
        return z, (torch.zeros_like(z) if compute_entropy else None)
    lp, ent = _MegatronResponseRows.apply(hidden_shard, weight_shard, idx, tp_group, cp_group, temperature,
                                          bool(compute_entropy), shape)
    return lp, (ent if compute_entropy else None)


# ---------------------------------------------------------------------------------------------------------------
# Reasoning PPO critic: the value head on the response rows of Megatron packed batches under TP / SP / CP
# (csrc/value_head.cu) and the token-level critic loss (csrc/token_critic_loss.cu)
# ---------------------------------------------------------------------------------------------------------------
def _value_head_check(hidden: torch.Tensor, weight: torch.Tensor, what: str):
    if hidden.dtype != torch.bfloat16 or weight.dtype != torch.bfloat16:
        raise ValueError(f"{what}: hidden and value weight must be bfloat16, got {hidden.dtype} / {weight.dtype}")
    if weight.dim() != 2 or weight.shape[0] != 1:
        raise ValueError(f"{what}: the value weight must be [1, H], got shape {tuple(weight.shape)}")
    H = weight.shape[1]
    if hidden.shape[-1] != H:
        raise ValueError(f"{what}: hidden size {hidden.shape[-1]} != the value weight's {H}")
    if H % 64 != 0 or not 64 <= H <= 8192:
        raise ValueError(f"{what}: needs H % 64 == 0 and 64 <= H <= 8192, got H = {H}")


def _value_head_rows(x: torch.Tensor):
    """(tensor, row stride) of [rows, H] hidden states: read in place when rows are 16-byte aligned."""
    if x.stride(-1) == 1 and x.stride(0) % 8 == 0 and x.stride(0) >= x.shape[1] and x.data_ptr() % 16 == 0:
        return x, x.stride(0)
    x = x.contiguous()
    return x, x.shape[1]


def value_head_rows(x: torch.Tensor, rows: torch.Tensor, weight: torch.Tensor) -> torch.Tensor:
    """v [n] fp32 = float(bf16(x[rows] @ weight[0])) on rows of x [T, H] bf16 read in place; 0 where rows == -1."""
    x, rs = _value_head_rows(x)
    H = x.shape[1]
    v = torch.empty(rows.numel(), dtype=torch.float32, device=x.device)
    if rows.numel():
        w = weight.contiguous()
        L.check(L.load().rb200_value_head_fwd(L.ptr(x), rs, L.ptr(rows), rows.numel(), H, L.ptr(w), L.ptr(v),
                                              L.stream_ptr(x.device)), "value_head_fwd")
    return v


def value_head_backward(x, rows, grad, weight, inv_map, need_x: bool, need_w: bool):
    """Backward of value_head_rows for grad [n] fp32 (rounded to bf16 first): dX [inv_map.numel(), H] bf16 =
    bf16(grad[inv_map[t]] * weight), zeros where inv_map == -1, and dW [1, H] bf16 = bf16(sum_i grad[i] x[rows[i]]);
    either is None when not needed."""
    x, rs = _value_head_rows(x)
    H, n, T = x.shape[1], rows.numel(), inv_map.numel()
    dev = x.device
    w = weight.contiguous()
    if n == 0 or T == 0:  # no row: every inv_map entry is -1, and dW is an empty sum
        return (torch.zeros((T, H), dtype=torch.bfloat16, device=dev) if need_x else None,
                torch.zeros((1, H), dtype=torch.bfloat16, device=dev) if need_w else None)
    dx = torch.empty((T, H), dtype=torch.bfloat16, device=dev) if need_x else None
    dw = torch.empty((1, H), dtype=torch.bfloat16, device=dev) if need_w else None
    if not (need_x or need_w):
        return dx, dw
    wsb = L.load().rb200_value_head_workspace_bytes(n, H) if need_w else 0
    ws = torch.empty(wsb, dtype=torch.uint8, device=dev) if need_w else None
    g = grad.reshape(-1).float().contiguous()
    L.check(L.load().rb200_value_head_bwd(L.ptr(x), rs, L.ptr(rows), n, H, L.ptr(g), L.ptr(w), L.ptr(inv_map), T,
                                          L.ptr(dx), L.ptr(dw), L.ptr(ws), wsb, L.stream_ptr(dev)), "value_head_bwd")
    return dx, dw


def mp_value_head(hidden_shard, value_weight, idx):
    """One rank's values: under SP [Rmax_k] fp32 for its own response rows in pad-slot order (the buffer of the TP
    all-gather, zeros in pad slots); without SP [R_c], its CP rank's compact rows."""
    x = hidden_shard.reshape(-1, hidden_shard.shape[-1])
    return value_head_rows(x, idx.send if idx.sp else idx.rows, value_weight)


def mp_value_unpad(gathered, idx):
    """TP-gathered values [tp, Rmax_k] -> the CP rank's compact values [R_c] (SP)."""
    return mp_unpad(gathered.reshape(-1, 1), idx).reshape(-1)


def mp_value_head_backward(grad, hidden_shard, value_weight, idx, need_x: bool = True, need_w: bool = True):
    """One rank's backward from the gradients of its CP rank's compact values [R_c] (mp_cell_grads): (dX of the hidden
    shard, in its shape, or None; d value_weight [1, H] or None).  Under SP the rank takes its own slots' gradients
    and its dW is its share of the TP sum; without SP every TP rank computes the full dW and the full dX."""
    x = hidden_shard.reshape(-1, hidden_shard.shape[-1])
    if idx.sp:
        ext = torch.cat([grad.reshape(-1).float(), grad.new_zeros(1, dtype=torch.float32)])  # -1: the zero slot
        own = idx.slot_map[idx.k * idx.Rmax_k:(idx.k + 1) * idx.Rmax_k]
        g, rows = gather_rows(ext, own), idx.send
    else:
        g, rows = grad, idx.rows
    dx, dw = value_head_backward(x, rows, g, value_weight, idx.hidden_map, need_x, need_w)
    return (None if dx is None else dx.view(hidden_shard.shape)), dw


class _MegatronResponseValues(torch.autograd.Function):
    @staticmethod
    def forward(ctx, hidden, value_weight, idx, tp_group, cp_group, shape):
        import torch.distributed as dist

        v = mp_value_head(hidden, value_weight, idx)
        if idx.sp:
            if idx.tp > 1:
                gathered = torch.empty((idx.tp, idx.Rmax_k), dtype=v.dtype, device=v.device)
                dist.all_gather_into_tensor(gathered, v, group=tp_group)
            else:
                gathered = v[None]
            v = mp_value_unpad(gathered, idx)
        vals = mp_values(v, None, idx)
        if idx.cp > 1:
            allv = torch.empty((idx.cp, *vals.shape), dtype=vals.dtype, device=vals.device)
            dist.all_gather_into_tensor(allv, vals, group=cp_group)
        else:
            allv = vals[None]
        out, _ = mp_to_cells(allv, idx, shape, False)
        ctx.save_for_backward(hidden, value_weight)
        ctx.idx = idx
        return out

    @staticmethod
    def backward(ctx, g):
        hidden, w = ctx.saved_tensors
        idx, ctx.idx = ctx.idx, None
        need_x, need_w = ctx.needs_input_grad[0], ctx.needs_input_grad[1]
        if not (need_x or need_w):
            return (None,) * 6
        grad, _ = mp_cell_grads(g, None, idx)
        dx, dw = mp_value_head_backward(grad, hidden, w, idx, need_x, need_w)
        return dx, dw, None, None, None, None


def megatron_response_values(hidden_shard, value_weight, plan, *, tp_group=None, cp_group=None):
    """The reasoning critic's values at the response tokens of a Megatron packed batch, from each rank's own
    hidden-state shard: the reference's LinearForLastLayer(H, 1) value head (a bf16 Linear without bias, cast with
    .float()) read at log_probs[:, -L-1:-1], computed on the response rows only.  hidden_shard is the decoder output
    without the output layer, [T_c / tp, 1, H] or [T_c / tp, H] under sequence parallelism, [T_c, 1, H] or [T_c, H]
    without it, bf16; value_weight is output_layer.weight [1, H] bf16; plan = response_rows.megatron_parallel(...)
    (tp = cp = 1 is the megatron_thd layout).  Returns values [bsz, response_len] fp32, the same on every rank, zeros
    at j >= r_b: the reference's inference output vpreds * mask, and the vpreds its loss reads.  Differentiable w.r.t.
    hidden_shard and value_weight (only where required).
    tp_group / cp_group resolve as in megatron_response_logprobs_entropy.  Collectives: forward, under SP one
    all-gather of [Rmax_k] fp32 values over TP, and one all-gather of [Rmax_c, 2] fp32 over CP; backward none.  Under
    SP a rank's dX comes from its own rows and its d value_weight is its share, which Megatron sums over TP (the weight
    carries sequence_parallel); without SP every TP rank computes the full, identical d value_weight.  Other CP ranks'
    cells arrive detached, as in postprocess_packed_seqs.  No response row on any rank: zeros and no collective.
    Host syncs: none with host lengths; one device-to-host copy of the counts and the plan's verdict with device
    lengths."""
    from .response_rows import MegatronParallelPlan

    what = "megatron_response_values"
    if not isinstance(plan, MegatronParallelPlan):
        raise ValueError(f"{what}: plan must be a response_rows.megatron_parallel plan, got {type(plan).__name__}")
    if hidden_shard.dim() not in (2, 3) or (hidden_shard.dim() == 3 and hidden_shard.shape[1] != 1):
        raise ValueError(f"{what}: hidden_shard must be [rows, H] or [rows, 1, H], got {tuple(hidden_shard.shape)}")
    _value_head_check(hidden_shard, value_weight, what)
    tp_group, tp, k = _mp_group(tp_group, "tp", plan.tp_size, what)
    cp_group, cp, c = _mp_group(cp_group, "cp", plan.cp_size, what)
    if not (hidden_shard.is_cuda and value_weight.is_cuda):
        raise L.Rb200Error("rlinf_b200 kernels take CUDA tensors; move inputs with to_device() first")
    rows = hidden_shard.shape[0]
    no_targets = torch.zeros((plan.bsz, plan.response_len), dtype=torch.int64, device=hidden_shard.device)
    idx = plan.index(no_targets, rows, k, c)
    shape = (plan.bsz, plan.response_len)
    if all(sum(r) == 0 for r in idx.counts):  # no response row on any rank: no collective on any rank
        return torch.zeros(shape, dtype=torch.float32, device=hidden_shard.device)
    return _MegatronResponseValues.apply(hidden_shard, value_weight, idx, tp_group, cp_group, shape)


def _critic_rows(t, name, shape, dev, dtype):
    if t is None or tuple(t.shape) != shape:
        raise ValueError(f"token_critic_loss: {name} has shape {None if t is None else tuple(t.shape)}, expected "
                         f"{shape} (that of values)")
    if t.dtype != dtype:
        raise ValueError(f"token_critic_loss: {name} must be {dtype}, got {t.dtype}")
    if t.device != dev:
        raise ValueError(f"token_critic_loss: {name} is on {t.device}, values on {dev}")
    if t.stride(1) != 1 or t.stride(0) < shape[1]:
        t = t.contiguous()
    return t


def _token_critic_launch(v, ins, value_clip, huber_delta, want_d):
    lib = L.load()
    dev = v.device
    bsz, Ln = v.shape
    a = L.TokenCriticLossArgs()
    a.bsz, a.L = bsz, Ln
    for name, t in (("values", v), *ins.items()):
        setattr(a, name, C.c_void_p(t.data_ptr()))
        setattr(a, name + "_stride", t.stride(0))
    a.value_clip, a.huber_delta = float(value_clip), float(huber_delta)
    wsb = lib.rb200_token_loss_workspace_bytes(bsz, Ln)
    if wsb < 0:
        raise ValueError(f"token_critic_loss: unsupported shape bsz={bsz} L={Ln} (bsz <= 65535)")
    ws = torch.empty(wsb, dtype=torch.uint8, device=dev)
    loss = torch.empty(1, dtype=torch.float32, device=dev)
    metrics = torch.empty(L.CM_NUM, dtype=torch.float32, device=dev)
    d_v = torch.empty((bsz, Ln), dtype=torch.float32, device=dev) if want_d else None
    a.workspace, a.workspace_bytes = L.ptr(ws), wsb
    a.loss, a.metrics, a.d_values = L.ptr(loss), L.ptr(metrics), L.ptr(d_v)
    L.check(lib.rb200_token_critic_loss(C.byref(a), L.stream_ptr(dev)), "token_critic_loss")
    return loss.reshape(()), metrics, d_v


class _TokenCriticLoss(torch.autograd.Function):
    """forward: one launch group writes the loss, the metrics and d values; backward: d values times the upstream
    scalar, read on the device."""

    @staticmethod
    def forward(ctx, values, ins, value_clip, huber_delta):
        loss, metrics, d_v = _token_critic_launch(values.detach(), ins, value_clip, huber_delta, True)
        ctx.grad = d_v
        ctx.mark_non_differentiable(metrics)
        return loss, metrics

    @staticmethod
    def backward(ctx, g_loss, _g_metrics):
        d_v, ctx.grad = ctx.grad, None
        return scale_by_(d_v, g_loss), None, None, None


def token_critic_loss(values, returns, prev_values, loss_mask, *, value_clip: float, huber_delta: float = 10000.0):
    """Token-level PPO critic loss of the reasoning critic, in one device pass: compute_ppo_critic_loss as
    MegatronCritic's loss_func calls it.  values, returns, prev_values (fp32) and loss_mask (bool / uint8) are
    [bsz, L] CUDA tensors; slices whose tokens are contiguous are read in place.  The aggregation is masked_mean, as
    in the reference whatever the worker's loss_agg_func (an all-masked batch gives 0).
    Returns (loss, metrics): loss as a 0-dim tensor, differentiable w.r.t. values; metrics maps critic/value_loss,
    critic/value_clip_ratio (unmasked mean over all cells), the five __sum__/_critic_explained_variance/* sums (masked
    cells) and critic/final_value_loss to 0-dim device tensors.  Four launches, no host sync."""
    if values.dim() != 2:
        raise ValueError(f"token_critic_loss: values must be [bsz, L], got {tuple(values.shape)}")
    shape, dev = tuple(values.shape), values.device
    if 0 in shape:
        raise ValueError(f"token_critic_loss: empty values {shape}")
    if loss_mask is not None and loss_mask.dtype not in (torch.bool, torch.uint8):
        raise ValueError(f"token_critic_loss: loss_mask must be bool or uint8, got {loss_mask.dtype}")
    if value_clip is None:
        raise ValueError("token_critic_loss: value_clip is required")
    v = _critic_rows(values, "values", shape, dev, torch.float32)
    ins = {"returns": _critic_rows(returns, "returns", shape, dev, torch.float32),
           "prev_values": _critic_rows(prev_values, "prev_values", shape, dev, torch.float32),
           "loss_mask": _critic_rows(L.as_u8(loss_mask), "loss_mask", shape, dev, torch.uint8)}
    if not values.is_cuda:
        raise L.Rb200Error("token_critic_loss takes CUDA tensors; there is no CPU path")
    if torch.is_grad_enabled() and values.requires_grad:
        loss, metrics = _TokenCriticLoss.apply(v, ins, value_clip, huber_delta)
    else:
        loss, metrics, _ = _token_critic_launch(v, ins, value_clip, huber_delta, False)
    return loss, {k: metrics[s] for s, k in L.CM_KEYS.items()}


# ---- reasoning step bookkeeping (csrc/reasoning_stats.cu) ----------------------------------------------------------

def _cells(t, name, shape, dev, dtype):
    """A [bsz, L] operand read in place through its row stride when its tokens are contiguous."""
    if tuple(t.shape) != shape:
        raise ValueError(f"reasoning rollout metrics: {name} has shape {tuple(t.shape)}, expected {shape}")
    t = L.to_device(t, dev) if t.device != dev else t
    if t.dtype != dtype:
        t = t.to(dtype)
    if t.stride(1) != 1 or t.stride(0) < shape[1]:
        t = t.contiguous()
    return t


def _per_seq(t, name, bsz, dev, dtype):
    t = t.reshape(-1)
    if t.numel() != bsz:
        raise ValueError(f"reasoning rollout metrics: {name} has {t.numel()} entries, expected {bsz}")
    return L.to_device(t, dev, dtype)


def reasoning_rollout_record(advantages, response_mask, prompt_lengths, response_lengths, rewards, is_end, *,
                             values=None, idx_to_traj=None) -> torch.Tensor:
    """This rank's fixed-layout record, float64 [RR_NUM] on the device, for compute_rollout_metrics(_dynamic):
    advantages / response_mask / values are [bsz, L] (the mask read in place, e.g. response_mask[:, -L:]),
    prompt / response lengths, rewards and is_end [bsz]; idx_to_traj [bsz] (list or tensor) selects the multi-turn
    fields.  Two launches, no host sync."""
    if advantages.dim() != 2 or 0 in advantages.shape:
        raise ValueError(f"reasoning rollout metrics: advantages must be a non-empty [bsz, L], got "
                         f"{tuple(advantages.shape)}")
    dev = advantages.device if advantages.is_cuda else L.default_device()
    shape = tuple(advantages.shape)
    bsz, Ln = shape
    adv = _cells(advantages, "advantages", shape, dev, torch.float32)
    mask = _cells(L.as_u8(response_mask), "response_mask", shape, dev, torch.uint8)
    val = None if values is None else _cells(values, "values", shape, dev, torch.float32)
    a = L.ReasoningRecordArgs()
    a.bsz, a.L = bsz, Ln
    keep = [adv, mask, val]
    for name, t in (("advantages", adv), ("mask", mask), ("values", val)):
        setattr(a, name, None if t is None else C.c_void_p(t.data_ptr()))
        setattr(a, name + "_stride", 0 if t is None else t.stride(0))
    seq = {"prompt_lengths": _per_seq(prompt_lengths, "prompt_lengths", bsz, dev, torch.int64),
           "response_lengths": _per_seq(response_lengths, "response_lengths", bsz, dev, torch.int64),
           "rewards": _per_seq(rewards, "rewards", bsz, dev, torch.float32),
           "is_end": _per_seq(L.as_u8(torch.as_tensor(is_end)), "is_end", bsz, dev, torch.uint8)}
    if idx_to_traj is not None:
        seq["idx_to_traj"] = _per_seq(torch.as_tensor(idx_to_traj, dtype=torch.int64), "idx_to_traj", bsz, dev,
                                      torch.int64)
    for name, t in seq.items():
        setattr(a, name, L.ptr(t))
    keep.append(seq)
    lib = L.load()
    wsb = lib.rb200_reasoning_record_workspace_bytes(bsz, Ln)
    if wsb < 0:
        raise ValueError(f"reasoning rollout metrics: unsupported shape bsz={bsz} L={Ln} (bsz <= 65535)")
    ws = torch.empty(wsb, dtype=torch.uint8, device=dev)
    rec = torch.empty(L.RR_NUM, dtype=torch.float64, device=dev)
    a.workspace, a.workspace_bytes, a.record = L.ptr(ws), wsb, L.ptr(rec)
    L.check(lib.rb200_reasoning_rollout_record(C.byref(a), L.stream_ptr(dev)), "reasoning_rollout_record")
    return rec


def reasoning_rollout_finish(records: torch.Tensor, values_world_sum: Optional[torch.Tensor] = None,
                             world_size: int = 0) -> torch.Tensor:
    """[P, RR_NUM] records in rank order -> float64 [RM_NUM + P]: the metric slots (L.RM_SLOTS), the verdict, the
    largest num_seq, then each rank's num_seq.  values_world_sum: fp32 [1] sum of RR_VALUES_MEAN over the default
    group of world_size ranks (None: the values mean is averaged over the P records).  One launch."""
    if records.dim() != 2 or records.shape[1] != L.RR_NUM or records.dtype != torch.float64:
        raise ValueError(f"reasoning_rollout_finish: records must be float64 [P, {L.RR_NUM}]")
    records = records.contiguous()
    P = records.shape[0]
    out = torch.empty(L.RM_NUM + P, dtype=torch.float64, device=records.device)
    ws = None if values_world_sum is None else values_world_sum.contiguous()
    L.check(L.load().rb200_reasoning_rollout_finish(L.ptr(records), P, L.ptr(ws), int(world_size), L.ptr(out),
                                                    L.stream_ptr(records.device)), "reasoning_rollout_finish")
    return out


def mask_count_f32(mask: torch.Tensor) -> torch.Tensor:
    """mask.to(float32).sum() as a 0-dim fp32 device tensor (the exact count rounded once); mask [bsz, L] bool /
    uint8, read in place when its tokens are contiguous.  Three launches, no host sync."""
    if mask.dim() != 2 or 0 in mask.shape:
        raise ValueError(f"mask_count_f32: mask must be a non-empty [bsz, L], got {tuple(mask.shape)}")
    dev = mask.device if mask.is_cuda else L.default_device()
    m = _cells(L.as_u8(mask), "mask", tuple(mask.shape), dev, torch.uint8)
    lib = L.load()
    wsb = lib.rb200_token_loss_workspace_bytes(*m.shape)
    if wsb < 0:
        raise ValueError(f"mask_count_f32: unsupported shape {tuple(m.shape)} (bsz <= 65535)")
    ws = torch.empty(wsb, dtype=torch.uint8, device=dev)
    out = torch.empty(1, dtype=torch.float32, device=dev)
    L.check(lib.rb200_mask_count_f32(L.ptr(m) if m.is_contiguous() else C.c_void_p(m.data_ptr()), m.stride(0),
                                     m.shape[0], m.shape[1], L.ptr(ws), wsb, L.ptr(out), L.stream_ptr(dev)),
            "mask_count_f32")
    return out.reshape(())


def mb_epilogue_pack(args, stream_dev) -> None:
    """rb200_mb_epilogue_pack on a filled L.MbEpilogueArgs (see algorithms.MegatronLossEpilogue)."""
    L.check(L.load().rb200_mb_epilogue_pack(C.byref(args), L.stream_ptr(stream_dev)), "mb_epilogue_pack")


def mb_epilogue_apply(args, stream_dev) -> None:
    L.check(L.load().rb200_mb_epilogue_apply(C.byref(args), L.stream_ptr(stream_dev)), "mb_epilogue_apply")


def step_metrics_finish(step_acc: torch.Tensor, n_avg: int, n_sum: int) -> torch.Tensor:
    """[n_mb, n_avg + n_sum] fp32 per-micro-batch metrics -> fp32 [n_avg + n_sum + 1]: means over micro-batches in
    index order, sums of the SUM keys, and (n_sum == 5) the explained variance.  One launch."""
    if step_acc.dim() != 2 or step_acc.shape[1] != n_avg + n_sum or step_acc.dtype != torch.float32:
        raise ValueError("step_metrics_finish: step_acc must be fp32 [n_mb, n_avg + n_sum]")
    out = torch.empty(n_avg + n_sum + 1, dtype=torch.float32, device=step_acc.device)
    L.check(L.load().rb200_step_metrics_finish(L.ptr(step_acc.contiguous()), step_acc.shape[0], n_avg, n_sum,
                                               L.ptr(out), L.stream_ptr(step_acc.device)), "step_metrics_finish")
    return out
