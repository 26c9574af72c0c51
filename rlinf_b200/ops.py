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
