"""ops.linear_logprobs_entropy / rb200_lmhead_logprob_entropy_* (csrc/lmhead.cu) against fp64 torch on the same bf16
operands: log-probs, entropies and the gradients w.r.t. the hidden states and the LM-head weight, without a logits
tensor."""
import ctypes as C

import pytest
import torch

pytestmark = pytest.mark.gpu

OPENVLA_WINDOW = (32000 - 256, 32000)  # 256 action bins below the 32000-token vocabulary, padded to V = 32064


def _inputs(N, H, V, seed, shape=None):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(shape or (N, H), generator=g, device="cuda").to(torch.bfloat16)
    w = (torch.randn(V, H, generator=g, device="cuda") * (2.0 / H ** 0.5)).to(torch.bfloat16)
    return x, w


def _ref(x, w, tgt, temp, lo, hi, glp, gh):
    """fp64 log-probs, entropies, lse and (dX, dW) of the same bf16 operands."""
    H = w.shape[1]
    X = x.reshape(-1, H).double()
    W = w.double()
    z = (X @ W.T) * (1.0 / temp)
    z[:, :lo] = -float("inf")
    z[:, hi:] = -float("inf")
    lse = torch.logsumexp(z, -1)
    logp = z - lse[:, None]
    p = torch.exp(logp)
    plogp = torch.where(p > 0, p * logp, torch.zeros_like(p))
    ent = -plogp.sum(-1)
    t = tgt.reshape(-1)
    t_in = (t >= lo) & (t < hi)
    lp = torch.where(t_in, logp.gather(1, t.clamp(0, w.shape[0] - 1)[:, None])[:, 0], torch.full_like(lse, -float("inf")))
    dz = -glp.double()[:, None] * p - torch.where(p > 0, gh.double()[:, None] * p * (logp + ent[:, None]),
                                                   torch.zeros_like(p))
    rows = torch.nonzero(t_in)[:, 0]
    dz[rows, t[rows]] += glp.double()[rows]
    dz = dz / temp
    # magnitudes of the summed terms: the kernels round dZ to bf16, an error of up to 2^-9 of each term
    return lp, ent, lse, (dz @ W, dz.abs() @ W.abs()), (dz.T @ X, dz.abs().T @ X.abs())


def _close_fp32(got, want, what):
    fin = torch.isfinite(want)
    assert torch.equal(torch.isfinite(got), fin), what
    torch.testing.assert_close(got[fin].double(), want[fin], rtol=1e-4, atol=1e-4, msg=what)


def _close_bf16_grad(got, ref, what):
    """One bf16 rounding (2^-8 relative) of the output plus one of dZ, plus 1e-3 max |ref|.  dZ is rounded to bf16
    before the gradient GEMMs, so its rounding is relative to the magnitude of the summed terms, not of their sum."""
    want, mag = ref
    err = (got.double() - want).abs()
    bound = 2.0 ** -8 * (want.abs() + mag) + 1e-3 * want.abs().max()
    worst = (err - bound).max().item()
    assert worst <= 0, f"{what}: max excess {worst:.3e} (max |ref| {want.abs().max().item():.3e})"


CASES = {
    # name: (N or (bsz, S, L), H, V, temperature, window)
    "h64_vtail": (333, 64, 32003, 0.7, None),
    "h1536_v32064": (333, 1536, 32064, 0.7, None),
    "h1536_vtail": (333, 1536, 32003, 1.0, None),
    "openvla_window": (333, 1536, 32064, 1.0, OPENVLA_WINDOW),
    "slice3d": ((3, 120, 111), 1536, 32003, 0.7, None),
}


def _case(name, seed=0):
    n, H, V, temp, window = CASES[name]
    if isinstance(n, tuple):
        bsz, S, Lr = n
        full, w = _inputs(None, H, V, seed, shape=(bsz, S, H))
        x = full[:, -Lr - 1:-1, :]  # the caller's response slice, read in place
        N = bsz * Lr
    else:
        x, w = _inputs(n, H, V, seed)
        N = n
    lo, hi = window or (0, V)
    g = torch.Generator(device="cuda").manual_seed(seed + 1)
    tgt = torch.randint(lo, hi, (N,), generator=g, device="cuda")
    tgt[::7] = torch.randint(0, V, (tgt[::7].numel(),), generator=g, device="cuda")  # some outside a window
    tgt = tgt.reshape(x.shape[:-1])
    glp = torch.randn(N, generator=g, device="cuda")
    gh = torch.randn(N, generator=g, device="cuda")
    t = tgt.reshape(-1)
    glp = torch.where((t >= lo) & (t < hi), glp, torch.zeros_like(glp))  # a -inf log-prob gets no gradient
    return x, w, tgt, temp, window, lo, hi, glp, gh


@pytest.mark.parametrize("name", list(CASES))
def test_lmhead_forward_backward_vs_fp64(name):
    from rlinf_b200 import ops

    x, w, tgt, temp, window, lo, hi, glp, gh = _case(name)
    if x.dim() == 3:
        assert ops._lmhead_geometry(x)[0] is x  # strided slice, no copy
    rlp, rent, _, rdx, rdw = _ref(x, w, tgt, temp, lo, hi, glp, gh)
    shape = x.shape[:-1]
    for mode in ("both", "hidden_frozen", "weight_frozen", "no_entropy"):
        xx = x.detach().clone().requires_grad_(mode != "hidden_frozen") if x.dim() == 2 else x.detach()
        if x.dim() == 3:  # keep the strided view: differentiate through a leaf of the full tensor
            base = x._base.detach().clone().requires_grad_(mode != "hidden_frozen")
            xx = base[:, -x.shape[1] - 1:-1, :]
        ww = w.detach().clone().requires_grad_(mode != "weight_frozen")
        lp, ent = ops.linear_logprobs_entropy(xx, ww, tgt, temperature=temp, window=window,
                                              compute_entropy=mode != "no_entropy")
        assert lp.shape == shape and lp.dtype == torch.float32
        _close_fp32(lp.reshape(-1), rlp, f"{name}/{mode} logprob")
        loss = (lp.reshape(-1).masked_fill(~torch.isfinite(lp.reshape(-1)), 0) * glp).sum()
        if mode == "no_entropy":
            assert ent is None
            want_dx, want_dw = _ref(x, w, tgt, temp, lo, hi, glp, torch.zeros_like(gh))[3:]
        else:
            _close_fp32(ent.reshape(-1), rent, f"{name}/{mode} entropy")
            loss = loss + (ent.reshape(-1) * gh).sum()
            want_dx, want_dw = rdx, rdw
        loss.backward()
        if mode != "hidden_frozen":
            leaf = xx if x.dim() == 2 else base
            got = leaf.grad if x.dim() == 2 else leaf.grad[:, -x.shape[1] - 1:-1, :]
            _close_bf16_grad(got.reshape(-1, w.shape[1]), want_dx, f"{name}/{mode} dX")
            if x.dim() == 3:
                assert (base.grad[:, -1, :] == 0).all() and (base.grad[:, :-x.shape[1] - 1, :] == 0).all()
        if mode != "weight_frozen":
            assert ww.grad.dtype == torch.bfloat16
            _close_bf16_grad(ww.grad, want_dw, f"{name}/{mode} dW")
            assert (ww.grad[:lo] == 0).all() and (ww.grad[hi:] == 0).all(), "dW rows outside the window"


def test_lmhead_equals_materialised_logits_at_vocabulary_scale():
    from rlinf_b200 import ops

    N, H, V, temp = 512, 1536, 151936, 0.7
    x, w = _inputs(N, H, V, 3)
    tgt = torch.randint(0, V, (N,), device="cuda")
    lp, ent = ops.linear_logprobs_entropy(x, w, tgt, temperature=temp)
    logits = x.float() @ w.float().T
    wlp, went = ops.logprobs_entropy_from_logits(logits, tgt, temperature=temp)
    torch.testing.assert_close(lp, wlp, rtol=1e-4, atol=1e-4)
    torch.testing.assert_close(ent, went, rtol=1e-4, atol=1e-4)


def _abi_backward(x, w, tgt, temp, lo, hi, lse, ent, glp, gh, chunk):
    """rb200_lmhead_logprob_entropy_bwd with a workspace sized for `chunk` vocabulary columns."""
    from rlinf_b200 import _lib as L
    from rlinf_b200 import ops

    lib = L.load()
    xx, N, Lr, bs, rs = ops._lmhead_geometry(x)
    V, H = w.shape
    wsb = ops.lmhead_workspace_bytes(N, Lr, H, V, lo, hi, chunk)
    ws = torch.empty(wsb, dtype=torch.uint8, device="cuda")
    dx = torch.empty(N, H, dtype=torch.bfloat16, device="cuda")
    dw = torch.empty(V, H, dtype=torch.bfloat16, device="cuda")
    L.check(lib.rb200_lmhead_logprob_entropy_bwd(C.c_void_p(xx.data_ptr()), L.ptr(w), L.ptr(tgt.reshape(-1).contiguous()),
                                                 N, Lr, bs, rs, H, V, lo, hi, 1.0 / temp, L.ptr(lse), L.ptr(ent),
                                                 L.ptr(glp), L.ptr(gh), L.ptr(dx), L.ptr(dw), L.ptr(ws), wsb,
                                                 L.stream_ptr()), "lmhead bwd")
    return dx, dw


def _abi_forward(x, w, tgt, temp, lo, hi):
    from rlinf_b200 import _lib as L
    from rlinf_b200 import ops

    lib = L.load()
    xx, N, Lr, bs, rs = ops._lmhead_geometry(x)
    V, H = w.shape
    wsb = ops.lmhead_workspace_bytes(N, Lr, H, V, lo, hi, 0)
    ws = torch.empty(wsb, dtype=torch.uint8, device="cuda")
    lp, ent, lse = (torch.empty(N, device="cuda") for _ in range(3))
    L.check(lib.rb200_lmhead_logprob_entropy_fwd(C.c_void_p(xx.data_ptr()), L.ptr(w), L.ptr(tgt.reshape(-1).contiguous()),
                                                 N, Lr, bs, rs, H, V, lo, hi, 1.0 / temp, L.ptr(lp), L.ptr(ent),
                                                 L.ptr(lse), L.ptr(ws), wsb, L.stream_ptr()), "lmhead fwd")
    return lp, ent, lse


@pytest.mark.parametrize("name", ["h1536_vtail", "slice3d"])
def test_lmhead_forced_vocabulary_chunks_and_determinism(name):
    x, w, tgt, temp, window, lo, hi, glp, gh = _case(name, seed=5)
    chunk = 8192  # 4 chunks of the 32003-column window
    assert -(-(hi - lo) // chunk) >= 3
    lp, ent, lse = _abi_forward(x, w, tgt, temp, lo, hi)
    dx, dw = _abi_backward(x, w, tgt, temp, lo, hi, lse, ent, glp, gh, chunk)
    _, _, _, rdx, rdw = _ref(x, w, tgt, temp, lo, hi, glp, gh)
    _close_bf16_grad(dx, rdx, f"{name} dX, {chunk}-column chunks")
    _close_bf16_grad(dw, rdw, f"{name} dW, {chunk}-column chunks")
    # two identical calls: bit-identical (several vocabulary ranges in the forward, several chunks in the backward)
    lp2, ent2, lse2 = _abi_forward(x, w, tgt, temp, lo, hi)
    dx2, dw2 = _abi_backward(x, w, tgt, temp, lo, hi, lse2, ent2, glp, gh, chunk)
    for a, b in ((lp, lp2), (ent, ent2), (lse, lse2), (dx, dx2), (dw, dw2)):
        assert torch.equal(a, b)
    # the whole window in one chunk gives the same gradient up to the fp32 accumulation order of dX
    dx1, dw1 = _abi_backward(x, w, tgt, temp, lo, hi, lse, ent, glp, gh, 0)
    assert torch.equal(dw1, dw)
    _close_bf16_grad(dx1, rdx, f"{name} dX, one chunk")


def test_lmhead_memory_stays_below_one_logits_tensor():
    from rlinf_b200 import ops

    N, H, V = 8192, 1536, 151936
    x, w = _inputs(N, H, V, 7)
    x.requires_grad_(True)
    w.requires_grad_(True)
    tgt = torch.randint(0, V, (N,), device="cuda")
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    lp, ent = ops.linear_logprobs_entropy(x, w, tgt)
    (lp.sum() + 0.1 * ent.sum()).backward()
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    vc = ops._lmhead_chunk(N, 0, V)
    ws = ops.lmhead_workspace_bytes(N, N, H, V, 0, V, vc)
    outputs = x.grad.numel() * 2 + w.grad.numel() * 2 + 8 * N * 4  # gradients + per-row vectors
    assert peak <= ws + outputs + (2 << 20), (peak, ws, outputs)
    assert peak < N * V * 2, (peak, N * V * 2)
