"""The composed MLP policy kernels (csrc/mlp.cu) against an fp64 restatement, over the shapes its dispatch branches on.

Every case drives MLPPolicy on the device and compares it with oracle.rl_oracle.mlp_forward in fp64 plus autograd on the
host.  A plain fp32 CPU run of the same restatement is computed as well; it only reports how the kernel's error
compares with fp32.

Dispatch branches covered (obs -> layer 0):
  7, 42     SIMT forward and weight gradient, scalar loads (obs % 4 != 0)
  12        SIMT, vector loads
  32, 96    tensor-core forward, tensor-core wgrad<128>
  160, 256  tensor-core forward, tensor-core wgrad<256>
  288       tensor-core forward with K > 256, SIMT weight gradient
and head layouts act / value_dim 1/1, 8/2 (register head backward), 9/1 and 6/3 (shared-memory head backward),
16/1 (chunk-level value), 32/8 (both maxima), 3/0 (no value head); n in {1, 7, 129, 4097, 20001}, rows taken as a
contiguous slice at an odd row offset of a larger buffer as the actor does (a subset also through the idx gather).

The bar is condition-aware, the measure of the GEMM tests: a weight gradient's error is divided by |dZ|^T.|H|, a bias
gradient's by sum|dZ|, both from the fp64 reference's own dZ and H; per-row outputs by the absolute-value propagation
through the head.  dZ = dH * (1 - H^2) carries a floor of |dH| * 2^-22: where tanh saturates, 1 - H^2 is below fp32's
resolution around 1 (it is exactly 0 in any fp32 evaluation), so only that much of it is defined.  The head's mean
error enters the log-prob gradients through x - mean, so their measures use |x - mean| + S_mean (S_mean = |W|.|H3| +
|b|, the mean's own condition) in place of |x - mean|.

A flat relative tolerance would not do: at n = 20001 a dropped row changes a weight gradient by ~5e-5 relative.
"""
import math

import pytest
import torch

from oracle import rl_oracle as O

pytestmark = pytest.mark.gpu

H = 256
HALF_LOG_2PI = 0.5 * math.log(2.0 * math.pi)
TANH_FLOOR = 2.0 ** -22
# About 4x the worst ratios measured over this file on an H100 80GB HBM3 SXM (700 W power limit): 2.2e-7 for the
# parameter gradients, 6.6e-7 for the per-row outputs (the fp32 CPU restatement: 8.6e-8 and 1.8e-7).
GRAD_BAR = 1e-6
OUT_BAR = 2.5e-6

# name: (action_dim, num_action_chunks, add_value_head, value_granularity) -> act = A * C, value_dim
HEADS = {
    "1/1": (1, 1, True, "action_level"),
    "8/2": (4, 2, True, "action_level"),
    "9/1": (9, 1, True, "action_level"),
    "6/3": (2, 3, True, "action_level"),
    "16/1": (8, 2, True, "chunk_level"),
    "32/8": (4, 8, True, "action_level"),
    "3/0": (3, 1, False, "action_level"),
}

# (obs, head, n, variant, with_idx).  variant: "full" | "no_d_entropy" (entropy computed, no gradient through it) |
# "no_entropy" (compute_entropy=False) | "no_values" (compute_values=False, d_values=None)
CASES = [
    (7, "1/1", 129, "full", True),
    (7, "16/1", 20001, "no_d_entropy", False),
    (42, "9/1", 4097, "full", True),
    (42, "8/2", 20001, "full", False),
    (12, "8/2", 7, "no_entropy", True),
    (12, "3/0", 4097, "full", False),
    (32, "6/3", 129, "full", True),
    (32, "1/1", 20001, "no_values", False),
    (96, "16/1", 4097, "full", False),
    (96, "3/0", 1, "full", False),
    (160, "32/8", 1, "full", False),
    (160, "9/1", 7, "no_d_entropy", True),
    (256, "3/0", 20001, "full", False),
    (256, "6/3", 4097, "no_values", False),
    (288, "8/2", 20001, "full", True),
    (288, "32/8", 129, "no_entropy", False),
]

WORST: dict = {}  # tensor / output name -> [kernel ratio, fp32 CPU ratio] over the file


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    if WORST:
        print("\nworst error / condition per tensor over the file (kernel | fp32 CPU restatement):")
        for k in sorted(WORST):
            print(f"  {k:28s} {WORST[k][0]:.2e} | {WORST[k][1]:.2e}")


def _note(name, kern, cpu):
    w = WORST.setdefault(name, [0.0, 0.0])
    w[0], w[1] = max(w[0], kern), max(w[1], cpu)


def _policy(obs, head):
    from rlinf_b200.policy import MLPPolicy

    A, Cn, vh, gran = HEADS[head]
    return MLPPolicy(obs, A, Cn, add_value_head=vh, value_granularity=gran)


def _randomise(pol, seed):
    """Every parameter random (not the default init, whose zero biases and tiny heads hide epilogue bugs)."""
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for name, p in pol.named_parameters():
        shape = tuple(p.shape)
        if name == "actor_logstd":  # a different std in every dimension
            v = torch.rand(shape, generator=g) * 2.5 - 2.0
        elif name.endswith("bias"):
            v = torch.rand(shape, generator=g) - 0.5
        elif name in ("actor_mean.weight", "value_head.mlp.6.weight"):
            v = torch.randn(shape, generator=g) * 0.3
        else:  # about the default init's scale
            v = torch.randn(shape, generator=g) * (1.4 / math.sqrt(shape[1]))
        sd[name] = v
    pol.load_state_dict(sd)
    pol.mark_params_changed()
    return sd


def _row_spread(g, n, cols):
    """Random upstream gradient whose rows differ in scale by up to e^+-3 (the operand scaling sees it)."""
    return torch.randn(n, cols, generator=g, dtype=torch.float64) * torch.exp(
        6.0 * torch.rand(n, 1, generator=g, dtype=torch.float64) - 3.0)


def _restatement(sd, X, action, dlp, dent, dv, want_ent, want_v, dtype):
    P = {k: v.to(dtype).clone().requires_grad_(True) for k, v in sd.items()}
    out = O.mlp_forward(P, X.to(dtype), action.to(dtype), want_entropy=want_ent, want_values=want_v)
    loss = (out["logprobs"] * dlp.to(dtype)).sum()
    if dent is not None:
        loss = loss + (out["entropy"] * dent.to(dtype)).sum()
    if dv is not None:
        loss = loss + (out["values"] * dv.to(dtype)).sum()
    loss.backward()
    return {k: v.detach() for k, v in out.items()}, {k: P[k].grad for k in P}


def _rss(e, W):
    """Root-sum-square propagation of independent per-element errors e through x -> x . W^T."""
    return torch.sqrt((e * e) @ (W * W).t())


def _conditions(sd, X, action, dlp, dent, dv, want_v):
    """fp64 per-element condition measures c of every gradient and output, such that the error of an fp32-level
    computation is a small multiple of 2^-24 * c: a first-order error analysis in which every GEMM step carries the
    |A|.|B| measure of the GEMM tests and errors carried in from earlier steps propagate root-sum-square (they are
    independent roundings)."""
    P = {k: v.double() for k, v in sd.items()}
    X = X.double()

    def tower(prefix):  # activations H_l, pre-activation conditions c_Z, activation error conditions e_H
        hs, cz, eh = [X], [None], [torch.zeros_like(X)]
        for i in (0, 2, 4):
            W, b = P[f"{prefix}{i}.weight"], P[f"{prefix}{i}.bias"]
            c = hs[-1].abs() @ W.abs().t() + b.abs() + _rss(eh[-1], W)
            h = torch.tanh(hs[-1] @ W.t() + b)
            hs.append(h)
            cz.append(c)
            eh.append((1 - h * h) * c + h.abs())
        return hs, cz, eh

    def down(t, prefix, dh, e_dh, cond):  # layers 2, 1, 0 (backward order)
        hs, cz, eh = t
        for li, i in zip((3, 2, 1), (4, 2, 0)):
            h = hs[li]
            gt = 1 - h * h
            dz = dh * gt
            # error of dH, of tanh' = 1 - H^2 from an H that carries the forward's error, and fp32's resolution of
            # 1 - H^2 where tanh saturates (2^-22 = 4 * 2^-24: exactly 0 in fp32, tiny in fp64)
            e_dz = e_dh * gt + dh.abs() * (2 * h.abs() * gt * cz[li] + 4.0) + dz.abs()
            W = P[f"{prefix}{i}.weight"]
            cond[f"{prefix}{i}.weight"] = e_dz.t() @ hs[li - 1].abs() + torch.sqrt((dz * dz).t() @ (eh[li - 1] ** 2))
            cond[f"{prefix}{i}.bias"] = e_dz.sum(0)
            e_dh = dz.abs() @ W.abs() + _rss(e_dz, W.t())
            dh = dz @ W

    cond = {}
    tb = tower("backbone.")
    hb, eb = tb[0], tb[2]
    Wm, bm, ls = P["actor_mean.weight"], P["actor_mean.bias"], P["actor_logstd"].reshape(-1)
    mean = hb[3] @ Wm.t() + bm
    c_mu = hb[3].abs() @ Wm.abs().t() + bm.abs() + _rss(eb[3], Wm)
    var = torch.exp(2 * ls)
    d = action.double() - mean
    dlp = dlp.double()
    cond["mean"] = c_mu
    cond["logprobs"] = d.abs() / var * c_mu + d * d / (2 * var) + ls.abs() + HALF_LOG_2PI
    cond["entropy"] = (0.5 + HALF_LOG_2PI + ls.abs()).expand_as(mean)
    dmu = dlp * d / var
    e_dmu = dlp.abs() * (d.abs() + c_mu) / var  # the mean's error enters through x - mean
    cond["actor_mean.weight"] = e_dmu.t() @ hb[3].abs() + torch.sqrt((dmu * dmu).t() @ (eb[3] ** 2))
    cond["actor_mean.bias"] = e_dmu.sum(0)
    c_ls = dlp.abs() * ((d * d + 2 * d.abs() * c_mu) / var + 1)
    if dent is not None:
        c_ls = c_ls + dent.double().abs()
    cond["actor_logstd"] = c_ls.sum(0).reshape(1, -1)
    down(tb, "backbone.", dmu @ Wm, dmu.abs() @ Wm.abs() + _rss(e_dmu, Wm.t()), cond)
    if want_v:
        tv = tower("value_head.mlp.")
        hv, ev = tv[0], tv[2]
        Wv = P["value_head.mlp.6.weight"]
        cond["values"] = hv[3].abs() @ Wv.abs().t() + _rss(ev[3], Wv)
        if dv is not None:
            dv = dv.double()
            cond["value_head.mlp.6.weight"] = dv.abs().t() @ hv[3].abs() + torch.sqrt((dv * dv).t() @ (ev[3] ** 2))
            down(tv, "value_head.mlp.", dv @ Wv, dv.abs() @ Wv.abs(), cond)
    return cond, mean, c_mu


def _ratio(got, ref, cond):
    err = (got.double().cpu() - ref.double()).abs()
    return (err / cond.clamp_min(1e-300)).max().item()


def _check(name, got, ref, ref32, cond, bar, tag):
    assert torch.isfinite(got).all(), f"{tag} {name}: non-finite values"
    kern = _ratio(got, ref, cond)
    cpu = _ratio(ref32, ref, cond)
    _note(name, kern, cpu)
    assert kern < bar, f"{tag} {name}: error / condition {kern:.2e} >= {bar:.0e} (fp32 CPU {cpu:.2e})"
    return kern


def _segments(pol):
    import math as _m

    return [(name, off, _m.prod(shape), shape) for name, off, shape in pol._spec]


def _pattern(pol, ref_grads, conds, g):
    """Known nonzero gradient-buffer contents: per tensor 0.5 * its gradient plus 0.1 * its condition with random sign
    (so a kernel that overwrites instead of accumulating is off by half a gradient), pads set to 1.5."""
    total = pol.flat_grads.numel()
    pat = torch.full((total,), 1.5, dtype=torch.float32)
    covered = torch.zeros(total, dtype=torch.bool)
    for name, off, numel, shape in _segments(pol):
        ref = ref_grads[name]
        if ref is None:  # receives no gradient in this case: must stay as it is
            v = torch.randn(numel, generator=g, dtype=torch.float64)
        else:
            sign = torch.randint(0, 2, (numel,), generator=g).double() * 2 - 1
            v = 0.5 * ref.reshape(-1) + 0.1 * conds[name].reshape(-1) * sign
        pat[off: off + numel] = v.float()
        covered[off: off + numel] = True
    return pat, ~covered


def _run_case(obs, head, n, variant, with_idx, seed, state_scale=None):
    pol = _policy(obs, head)
    sd = _randomise(pol, seed)
    act, vdim = pol.act_dim, pol.value_dim
    g = torch.Generator().manual_seed(seed + 1)
    lo = 37  # odd row offset of the micro-batch inside a larger buffer
    N = lo + n + 5
    Xbig = torch.randn(N, obs, generator=g)
    if state_scale is not None:
        Xbig = state_scale(Xbig)
    Abig = torch.randn(N, act, generator=g) * 3.0
    X, action = Xbig[lo: lo + n], Abig[lo: lo + n]
    want_ent = variant != "no_entropy"
    want_v = vdim > 0 and variant != "no_values"
    dlp = _row_spread(g, n, act)
    dent = _row_spread(g, n, act) if variant not in ("no_entropy", "no_d_entropy") else None
    dv = _row_spread(g, n, vdim) if want_v else None
    noise = torch.randn(n, act, generator=g)

    out64, grads64 = _restatement(sd, X, action, dlp, dent, dv, want_ent, want_v, torch.float64)
    out32, grads32 = _restatement(sd, X, action, dlp, dent, dv, want_ent, want_v, torch.float32)
    conds, _, _ = _conditions(sd, X, action, dlp, dent, dv, want_v)
    tag = f"obs={obs} head={head} n={n} {variant}"

    Xg, Ag = Xbig.cuda()[lo: lo + n], Abig.cuda()[lo: lo + n]
    dlp_g = dlp.float().cuda()
    dent_g = None if dent is None else dent.float().cuda()
    dv_g = None if dv is None else dv.float().cuda()

    # ---- training forward --------------------------------------------------------------------------------------
    out = pol.forward_train(Xg, Ag, compute_entropy=want_ent, compute_values=want_v)
    assert ("entropy" in out) == want_ent and ("values" in out) == want_v
    worst = {}
    for k in ("logprobs", "entropy", "values"):
        if k in out:
            worst[k] = _check(k, out[k], out64[k], out32[k], conds[k], OUT_BAR, tag)

    # ---- backward: accumulates into a known pattern, leaves pads and untouched tensors alone, is reproducible -----
    pat, pads = _pattern(pol, grads64, conds, g)
    pat_g = pat.cuda()
    pol.flat_grads.copy_(pat_g)
    pol.backward(dlp_g, dv_g, dent_g)
    first = pol.flat_grads.clone()
    pol.flat_grads.copy_(pat_g)
    pol.backward(dlp_g, dv_g, dent_g)
    assert torch.equal(first, pol.flat_grads), f"{tag}: two identical backward calls differ"
    res = first.cpu()
    assert torch.equal(res[pads], pat[pads]), f"{tag}: pad floats between gradient tensors were written"
    for name, off, numel, shape in _segments(pol):
        got = res[off: off + numel]
        ref = grads64[name]
        if ref is None:
            assert torch.equal(got, pat[off: off + numel]), f"{tag} {name}: gradient written though it gets none"
            continue
        delta = got.double() - pat[off: off + numel].double()
        r = _check(name, delta.reshape(shape), ref, grads32[name], conds[name], GRAD_BAR, tag)
        worst[name] = r

    # ---- inference entries at the same rows ---------------------------------------------------------------------
    ref_mean = out64["mean"]
    a_mean, lp_mean, v_mean = pol.mean(Xg, calculate_values=vdim > 0)
    _check("mean", a_mean, ref_mean, out32["mean"], conds["mean"], OUT_BAR, tag + " mean()")
    ls = sd["actor_logstd"].double().reshape(-1)
    lp_ref = (-ls - HALF_LOG_2PI).expand_as(ref_mean)
    _check("logprobs", lp_mean, lp_ref, lp_ref.float(), (ls.abs() + HALF_LOG_2PI).expand_as(ref_mean), OUT_BAR,
           tag + " mean()")
    sd_ = torch.exp(ls)
    x_ref = ref_mean + sd_ * noise.double()
    x_cond = conds["mean"] + sd_ * noise.double().abs()
    a_s, lp_s, v_s = pol.sample(Xg, noise=noise.cuda(), calculate_values=vdim > 0)
    _check("sample.action", a_s, x_ref, x_ref.float(), x_cond, OUT_BAR, tag + " sample()")
    z2 = noise.double() ** 2
    lps_ref = -z2 / 2 - ls - HALF_LOG_2PI
    d = (x_ref - ref_mean).abs()
    lps_cond = d / sd_ ** 2 * (conds["mean"] + x_ref.abs()) + z2 / 2 + ls.abs() + HALF_LOG_2PI
    _check("sample.logprobs", lp_s, lps_ref, lps_ref.float(), lps_cond, OUT_BAR, tag + " sample()")
    if vdim > 0:
        vref = out64["values"] if want_v else O.mlp_forward({k: v.double() for k, v in sd.items()}, X.double(),
                                                           want_entropy=False)["values"]
        vcond = conds["values"] if want_v else _conditions(sd, X, action, dlp, dent, None, True)[0]["values"]
        for what, v in (("mean()", v_mean), ("sample()", v_s), ("value()", pol.value(Xg))):
            _check("values", v, vref, vref.float(), vcond, OUT_BAR, f"{tag} {what}")

    # ---- the idx gather route at the same rows ------------------------------------------------------------------
    if with_idx:
        idx = torch.arange(lo, lo + n, dtype=torch.int64, device="cuda")
        out_i = pol.forward_train(Xbig.cuda(), Abig.cuda(), idx=idx, compute_entropy=want_ent, compute_values=want_v)
        for k in out_i:
            _check(k, out_i[k], out64[k], out32[k], conds[k], OUT_BAR, tag + " idx")
            assert _ratio(out_i[k], out[k].double().cpu(), conds[k]) < OUT_BAR, f"{tag} {k}: idx and slice routes differ"
        pol.flat_grads.copy_(pat_g)
        pol.backward(dlp_g, dv_g, dent_g)
        res_i = pol.flat_grads.cpu()
        for name, off, numel, shape in _segments(pol):
            if grads64[name] is None:
                continue
            delta = (res_i[off: off + numel].double() - pat[off: off + numel].double()).reshape(shape)
            _check(name, delta, grads64[name], grads32[name], conds[name], GRAD_BAR, tag + " idx")
            got = (res[off: off + numel].double() - pat[off: off + numel].double()).reshape(shape)
            assert _ratio(delta, got, conds[name]) < GRAD_BAR, f"{tag} {name}: idx and slice routes differ"
    print(f"{tag}: " + ", ".join(f"{k} {v:.1e}" for k, v in sorted(worst.items())))


@pytest.mark.parametrize("obs,head,n,variant,with_idx", CASES,
                         ids=[f"obs{c[0]}-{c[1].replace('/', 'x')}-n{c[2]}-{c[3]}" for c in CASES])
def test_mlp_matches_fp64(obs, head, n, variant, with_idx):
    _run_case(obs, head, n, variant, with_idx, seed=1000 * obs + n)


def _scaled(k):
    return lambda x: x * 2.0 ** k


def _scaled_with_huge_column(x):
    x = x * 2.0 ** 12
    x[:, 3] = x[:, 3].sign() * 2.0 ** 17  # past fp16's largest finite value (65504)
    return x


@pytest.mark.parametrize("obs", [128, 288])
@pytest.mark.parametrize("scale", ["2^-8", "2^12", "2^12+2^17"])
def test_mlp_input_magnitudes(obs, scale):
    """Observations are not normalised by this library: tiny and huge states reach layer 0 as they are.  Tensor-core
    layer 0 (obs 128: forward and wgrad; obs 288: forward) must keep fp32-level accuracy and finite outputs: 2^-8 and
    2^17 need the operand scaling, 2^12 (max|X| just below 2^15) is the top of the range split unscaled."""
    fn = {"2^-8": _scaled(-8), "2^12": _scaled(12), "2^12+2^17": _scaled_with_huge_column}[scale]
    _run_case(obs, "8/2", 4097, "full", False, seed=77 + obs, state_scale=fn)


@pytest.mark.parametrize("K", [288, 512])
@pytest.mark.parametrize("grad_like", [False, True])
def test_tc_gemm_h_forward_long_k(K, grad_like):
    """rb200_tc_gemm_h forward past K = 256 (layer 0 of observations wider than 256), vs fp64 at the GEMM tests' bar."""
    from rlinf_b200 import _lib as L

    lib = L.load()
    M = 5000
    g = torch.Generator(device="cuda").manual_seed(K + grad_like)
    A = torch.randn(M, K, device="cuda", generator=g)
    if grad_like:
        A = A * 3e-7 * torch.exp(2 * torch.randn(M, 1, device="cuda", generator=g))
    B = torch.randn(256, K, device="cuda", generator=g) / K ** 0.5
    C = torch.empty(M, 256, device="cuda")
    work = torch.empty(512 * K, device="cuda")
    amax = A.abs().max().reshape(1) if grad_like else None
    L.check(lib.rb200_tc_gemm_h(L.ptr(A), L.ptr(B), L.ptr(C), M, K, 0, L.ptr(amax), L.ptr(work), L.stream_ptr()),
            "tc_gemm_h")
    ref = A.double() @ B.double().t()
    scale = (A.double().abs() @ B.double().abs().t()).clamp_min(1e-300)
    if grad_like:  # as in test_gpu_tc_gemm.py: elements below amax * 2^-16 keep fewer than 22 bits
        scale = scale + (amax.double() * 2.0 ** -16) * B.double().abs().sum(dim=1)
    err = ((C.double() - ref).abs() / scale).max().item()
    print(f"tc_gemm_h forward M={M} K={K} grad_like={grad_like}: max |err| / (|A|.|B|) = {err:.2e}")
    assert err < 2e-6, err


def test_mlp_entries_require_the_weight_cache():
    """Every MLP entry returns RB200_E_NULL for wsplit = NULL: the towers run only with the tensor-core weight cache.
    The buffers are real and sized as the entries require (the same calls with the cache succeed), so an entry that
    lacks the check launches on valid memory and fails the assertion instead."""
    import ctypes as C

    from rlinf_b200 import _lib as L

    lib = L.load()
    pol = _policy(42, "8/2")
    n = 129
    lay = C.byref(pol.layout)
    nscr = lib.rb200_mlp_fwd_scratch_floats(lay, n)

    def zeros(*shape):
        return torch.zeros(*shape, device="cuda")

    states, action, noise = zeros(n, pol.obs_dim), zeros(n, pol.act_dim), zeros(n, pol.act_dim)
    logp, ent, vals = zeros(n, pol.act_dim), zeros(n, pol.act_dim), zeros(n, pol.value_dim)
    acts, work = zeros(nscr), zeros(nscr)
    P, G, st = L.ptr(pol.flat_params), L.ptr(pol.flat_grads), L.stream_ptr()
    X, A, lp, en, v = L.ptr(states), L.ptr(action), L.ptr(logp), L.ptr(ent), L.ptr(vals)
    calls = {  # in this order with the cache: the backward reads the forward's activations
        "forward": lambda ws: lib.rb200_mlp_forward(lay, P, ws, X, A, None, n, lp, en, v, L.ptr(acts), L.ptr(work), None,
                                                    st),
        "backward": lambda ws: lib.rb200_mlp_backward(lay, P, ws, X, A, None, n, lp, en, v, L.ptr(acts), L.ptr(work), G,
                                                      st),
        "sample": lambda ws: lib.rb200_mlp_sample(lay, P, ws, X, L.ptr(noise), 0, 0, None, n, A, lp, v, L.ptr(work), st),
        "value": lambda ws: lib.rb200_mlp_value(lay, P, ws, X, n, v, L.ptr(work), st),
        "mean": lambda ws: lib.rb200_mlp_mean(lay, P, ws, X, n, A, lp, v, L.ptr(work), st),
    }
    for name, call in calls.items():
        assert call(None) == -1, f"rb200_mlp_{name} with wsplit = NULL"  # RB200_E_NULL
    for name, call in calls.items():
        assert call(pol._ws()) == 0, f"rb200_mlp_{name} with the weight cache"
    torch.cuda.synchronize()


def test_runner_update_is_bit_reproducible_simt_layer0():
    """obs 42 keeps layer 0 on the SIMT kernels; one micro-batch of 16384 rows.  Two identical runners must end one
    iteration with identical parameters and Adam moments.  clip_grad is far above the gradient norm, so the clip
    coefficient is exactly 1 and the fp64-atomic norm cannot reach the parameters."""
    from rlinf_b200.config import synthetic_ppo_config
    from rlinf_b200.runner import EmbodiedRunner

    def make():
        cfg = synthetic_ppo_config(B=2048, T=8, obs_dim=42, action_dim=3, update_epoch=2, num_minibatches=1,
                                   **{"actor.optim.clip_grad": 1.0e30})
        return EmbodiedRunner(cfg)

    states = []
    for _ in range(2):
        run = make()
        assert run.actor.cfg.actor.micro_batch_size >= 8192
        run.run(1)
        torch.cuda.synchronize()
        opt = run.actor.optimizer
        assert opt.state[2].item() == 1.0  # clip coefficient
        states.append({"params": run.actor.model.flat_params.cpu().clone(), "exp_avg": opt.exp_avg.cpu().clone(),
                       "exp_avg_sq": opt.exp_avg_sq.cpu().clone()})
        del run
    for k in states[0]:
        assert torch.equal(states[0][k], states[1][k]), k
