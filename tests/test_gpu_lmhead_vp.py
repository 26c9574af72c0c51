"""Vocabulary-parallel log-probs / entropies (ops.vocab_parallel_*, csrc/vocab_parallel.cu) with P ranks emulated on one
device: each rank's records from its shard, combined in rank order, and each rank's backward share, against fp64 torch on
the full materialised logits of the same bf16 operands.  P = 1 must be bit-identical to the single-GPU ops."""
import pytest
import torch

pytestmark = pytest.mark.gpu

OPENVLA_WINDOW = (32000 - 256, 32000)


def _inputs(N, H, V, seed, shape=None):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(shape or (N, H), generator=g, device="cuda").to(torch.bfloat16)
    w = (torch.randn(V, H, generator=g, device="cuda") * (2.0 / H ** 0.5)).to(torch.bfloat16)
    return x, w


def _ref(x, w, tgt, temp, lo, hi, glp, gh):
    """fp64 log-probs, entropies, lse and (dX, dW) of the same bf16 operands, each gradient with the magnitude of its
    summed terms."""
    H = w.shape[1]
    X = x.reshape(-1, H).double()
    W = w.double()
    z = (X @ W.T) * (1.0 / temp)
    z[:, :lo] = -float("inf")
    z[:, hi:] = -float("inf")
    lse = torch.logsumexp(z, -1)
    logp = z - lse[:, None]
    p = torch.exp(logp)
    ent = -torch.where(p > 0, p * logp, torch.zeros_like(p)).sum(-1)
    t = tgt.reshape(-1)
    t_in = (t >= lo) & (t < hi)
    lp = torch.where(t_in, logp.gather(1, t.clamp(0, w.shape[0] - 1)[:, None])[:, 0], torch.full_like(lse, -float("inf")))
    dz = -glp.double()[:, None] * p - torch.where(p > 0, gh.double()[:, None] * p * (logp + ent[:, None]),
                                                   torch.zeros_like(p))
    rows = torch.nonzero(t_in)[:, 0]
    dz[rows, t[rows]] += glp.double()[rows]
    dz = dz / temp
    return lp, ent, lse, (dz @ W, dz.abs() @ W.abs()), (dz.T @ X, dz.abs().T @ X.abs()), dz


def _close_fp32(got, want, what):
    fin = torch.isfinite(want)
    assert torch.equal(torch.isfinite(got), fin), what
    torch.testing.assert_close(got[fin].double(), want[fin], rtol=1e-4, atol=1e-4, msg=what)


def _close_bf16_grad(got, ref, what):
    """Two bf16 roundings (dZ before the gradient GEMMs, the bf16 output), each 2^-9 relative to the magnitude of the
    summed terms, plus 1e-3 max |ref| (test_gpu_lmhead.py's bound)."""
    want, mag = ref
    err = (got.double() - want).abs()
    bound = 2.0 ** -8 * (want.abs() + mag) + 1e-3 * want.abs().max()
    worst = (err - bound).max().item()
    assert worst <= 0, f"{what}: max excess {worst:.3e} (max |ref| {want.abs().max().item():.3e})"


CASES = {
    # name: (N or (bsz, S, L), H, V, P, temperature, window)
    "p1_v151936": (333, 256, 151936, 1, 0.7, None),
    "p2_v151936": (333, 256, 151936, 2, 1.0, None),
    "p4_v151936": (333, 256, 151936, 4, 0.7, None),
    "p8_v151936": (333, 256, 151936, 8, 0.7, None),  # shards of 18,992 columns: not a multiple of 256
    "p4_window": (333, 1536, 32064, 4, 1.0, OPENVLA_WINDOW),  # the window lies in shard 3 only
    "p2_window_straddles": (333, 512, 32064, 2, 0.7, (15000, 17500)),
    "p2_slice3d": ((3, 120, 111), 1536, 32064, 2, 0.7, None),
}


def _case(name, seed=0):
    n, H, V, P, temp, window = CASES[name]
    if isinstance(n, tuple):
        bsz, S, Lr = n
        full, w = _inputs(None, H, V, seed, shape=(bsz, S, H))
        x = full[:, -Lr - 1:-1, :]
        N = bsz * Lr
    else:
        x, w = _inputs(n, H, V, seed)
        N = n
    lo, hi = window or (0, V)
    g = torch.Generator(device="cuda").manual_seed(seed + 1)
    tgt = torch.randint(lo, hi, (N,), generator=g, device="cuda")
    tgt[::5] = torch.randint(0, V, (tgt[::5].numel(),), generator=g, device="cuda")  # every shard, and outside a window
    tgt = tgt.reshape(x.shape[:-1])
    glp = torch.randn(N, generator=g, device="cuda")
    gh = torch.randn(N, generator=g, device="cuda")
    t = tgt.reshape(-1)
    glp = torch.where((t >= lo) & (t < hi), glp, torch.zeros_like(glp))
    return x, w, tgt, P, temp, window, lo, hi, glp, gh


def _emulate(x, w, tgt, P, temp, window, glp, gh, want_entropy=True, need_x=True, need_w=True):
    """P ranks on one device: records -> combine -> each rank's backward, dX shares summed in fp32 in rank order."""
    from rlinf_b200 import ops

    Vs = w.shape[0] // P
    shards = [w[k * Vs:(k + 1) * Vs] for k in range(P)]
    rec = torch.stack([ops.lmhead_vp_partials(x, shards[k], tgt, k, P, temp, window) for k in range(P)])
    lp, ent, lse = ops.vp_combine(rec, tgt, Vs, window, want_entropy)
    parts = [ops.lmhead_vp_backward(x, shards[k], tgt, k, P, lse, ent, glp, gh if want_entropy else None, temp, window,
                                    need_x, need_w) for k in range(P)]
    dx = None
    if need_x:
        dx = parts[0][0]
        for k in range(1, P):
            dx = dx + parts[k][0]
        dx = dx.to(torch.bfloat16)
    dw = torch.cat([p[1] for p in parts]) if need_w else None
    return rec, lp, ent, lse, dx, dw


@pytest.mark.parametrize("name", list(CASES))
def test_vp_emulated_ranks_vs_fp64(name):
    x, w, tgt, P, temp, window, lo, hi, glp, gh = _case(name)
    rlp, rent, rlse, rdx, rdw, _ = _ref(x, w, tgt, temp, lo, hi, glp, gh)
    _, _, _, rdx0, rdw0, _ = _ref(x, w, tgt, temp, lo, hi, glp, torch.zeros_like(gh))
    Vs = w.shape[0] // P
    for mode in ("both", "hidden_frozen", "weight_frozen", "no_entropy"):
        rec, lp, ent, lse, dx, dw = _emulate(x, w, tgt, P, temp, window, glp, gh, want_entropy=mode != "no_entropy",
                                             need_x=mode != "hidden_frozen", need_w=mode != "weight_frozen")
        _close_fp32(lp, rlp, f"{name}/{mode} logprob")
        _close_fp32(lse, rlse, f"{name}/{mode} lse")
        if mode == "no_entropy":
            assert ent is None
        else:
            _close_fp32(ent, rent, f"{name}/{mode} entropy")
        wdx, wdw = (rdx0, rdw0) if mode == "no_entropy" else (rdx, rdw)
        if mode == "hidden_frozen":
            assert dx is None
        else:
            _close_bf16_grad(dx, wdx, f"{name}/{mode} dX")
        if mode == "weight_frozen":
            assert dw is None
        else:
            _close_bf16_grad(dw, wdw, f"{name}/{mode} dW")
            assert (dw[:lo] == 0).all() and (dw[hi:] == 0).all(), "dW rows outside the window"
    # ranks whose shard misses the window contribute the empty record
    for k in range(P):
        if (k + 1) * Vs <= lo or k * Vs >= hi:
            assert (rec[k, :, 0] == -float("inf")).all() and (rec[k, :, 1:] == 0).all()


@pytest.mark.parametrize("name", ["p1_v151936", "p2_slice3d", "p4_window"])
def test_vp_single_rank_bit_identical_to_linear_logprobs_entropy(name):
    """P = 1 (no process group) runs the same kernels in the same order: log-prob, entropy, lse, dX and dW bit-equal."""
    from rlinf_b200 import ops

    x, w, tgt, _, temp, window, lo, hi, glp, gh = _case(name, seed=3)
    outs = []
    for fn in (ops.linear_logprobs_entropy, ops.vocab_parallel_linear_logprobs_entropy):
        if x.dim() == 3:
            base = x._base.detach().clone().requires_grad_(True)
            xx = base[:, -x.shape[1] - 1:-1, :]
        else:
            base = xx = x.detach().clone().requires_grad_(True)
        ww = w.detach().clone().requires_grad_(True)
        lp, ent = fn(xx, ww, tgt, temperature=temp, window=window)
        (lp.reshape(-1).masked_fill(~torch.isfinite(lp.reshape(-1)), 0) * glp + ent.reshape(-1) * gh).sum().backward()
        outs.append((lp, ent, base.grad, ww.grad))
    for a, b, what in zip(outs[0], outs[1], ("logprob", "entropy", "dX", "dW")):
        assert torch.equal(a, b), f"{name}: {what}"
    _, _, lse = ops.vp_combine(ops.lmhead_vp_partials(x, w, tgt, 0, 1, temp, window)[None], tgt, w.shape[0], window)
    assert torch.equal(lse, _single_gpu_lse(x, w, tgt, temp, lo, hi))


@pytest.mark.parametrize("mode", ["hidden_frozen", "weight_frozen", "no_entropy", "no_hidden_reduce"])
def test_vp_autograd_single_rank_frozen_inputs_and_flags(mode):
    """The autograd path's input freezing, entropy off and reduce_hidden_grad=False (a no-op with one rank), each
    bit-identical to linear_logprobs_entropy with the same inputs frozen."""
    from rlinf_b200 import ops

    x, w, tgt, _, temp, window, lo, hi, glp, gh = _case("p2_slice3d", seed=4)
    outs = []
    for vp in (False, True):
        base = x._base.detach().clone().requires_grad_(mode != "hidden_frozen")
        xx = base[:, -x.shape[1] - 1:-1, :]
        ww = w.detach().clone().requires_grad_(mode != "weight_frozen")
        kw = dict(temperature=temp, window=window, compute_entropy=mode != "no_entropy")
        if vp:
            kw["reduce_hidden_grad"] = mode != "no_hidden_reduce"
            lp, ent = ops.vocab_parallel_linear_logprobs_entropy(xx, ww, tgt, **kw)
        else:
            lp, ent = ops.linear_logprobs_entropy(xx, ww, tgt, **kw)
        loss = (lp.reshape(-1).masked_fill(~torch.isfinite(lp.reshape(-1)), 0) * glp).sum()
        if mode == "no_entropy":
            assert ent is None
        else:
            loss = loss + (ent.reshape(-1) * gh).sum()
        loss.backward()
        outs.append((lp, ent, base.grad, ww.grad))
    assert (outs[1][2] is None) == (mode == "hidden_frozen")
    assert (outs[1][3] is None) == (mode == "weight_frozen")
    for a, b, what in zip(outs[0], outs[1], ("logprob", "entropy", "dX", "dW")):
        assert (a is None and b is None) or torch.equal(a, b), f"{mode}: {what}"


def test_vp_sequence_first_hidden_read_in_place():
    """Megatron's decoder output is [S, bsz, H]: its transposed response slice is addressed in place and gives the
    bits of the same rows made contiguous."""
    from rlinf_b200 import ops

    S, bsz, H, V, Lr = 130, 3, 512, 32064, 111
    g = torch.Generator(device="cuda").manual_seed(21)
    dec = torch.randn(S, bsz, H, generator=g, device="cuda").to(torch.bfloat16)
    w = (torch.randn(V, H, generator=g, device="cuda") * (2.0 / H ** 0.5)).to(torch.bfloat16)
    tgt = torch.randint(0, V, (bsz, Lr), generator=g, device="cuda")
    outs = []
    for in_place in (True, False):
        base = dec.detach().clone().requires_grad_(True)
        x = base.transpose(0, 1)[:, -Lr - 1:-1, :]
        if in_place:
            assert ops._lmhead_geometry(x)[0] is x
        else:
            x = x.contiguous()
        ww = w.detach().clone().requires_grad_(True)
        lp, ent = ops.vocab_parallel_linear_logprobs_entropy(x, ww, tgt, temperature=0.7)
        (lp.sum() + 0.3 * ent.sum()).backward()
        outs.append((lp, ent, base.grad, ww.grad))
    for a, b, what in zip(outs[0], outs[1], ("logprob", "entropy", "dX", "dW")):
        assert torch.equal(a, b), what


def _single_gpu_lse(x, w, tgt, temp, lo, hi):
    import ctypes as C

    from rlinf_b200 import _lib as L
    from rlinf_b200 import ops

    xx, N, Lr, bs, rs = ops._lmhead_geometry(x)
    V, H = w.shape
    wsb = ops.lmhead_workspace_bytes(N, Lr, H, V, lo, hi, 0)
    ws = torch.empty(wsb, dtype=torch.uint8, device="cuda")
    lp, ent, lse = (torch.empty(N, device="cuda") for _ in range(3))
    L.check(L.load().rb200_lmhead_logprob_entropy_fwd(C.c_void_p(xx.data_ptr()), L.ptr(w),
                                                      L.ptr(tgt.reshape(-1).contiguous()), N, Lr, bs, rs, H, V, lo, hi,
                                                      1.0 / temp, L.ptr(lp), L.ptr(ent), L.ptr(lse), L.ptr(ws), wsb,
                                                      L.stream_ptr()), "lmhead fwd")
    return lse


def test_vp_logits_dropins_single_rank_bit_identical():
    from rlinf_b200 import ops

    g = torch.Generator(device="cuda").manual_seed(11)
    full = torch.randn(2, 70, 32064, generator=g, device="cuda") * 3
    for dtype in (torch.float32, torch.bfloat16):
        outs = []
        for which in ("single", "vp"):
            base = full.to(dtype).detach().clone().requires_grad_(True)
            logits = base[:, -65:-1, :]
            tgt = torch.randint(0, 32064, logits.shape[:-1], generator=g.manual_seed(12), device="cuda")
            if which == "single":
                lp, ent = ops.logprobs_entropy_from_logits(logits, tgt)
            else:
                ent, lp = ops.vocab_parallel_entropy_and_log_probs(logits, tgt)
            gw = torch.randn(lp.shape, generator=g.manual_seed(13), device="cuda")
            (lp * gw + 0.5 * ent * gw.flip(-1)).sum().backward()
            outs.append((lp, ent, base.grad))
        for a, b, what in zip(outs[0], outs[1], ("logprob", "entropy", "dlogits")):
            assert torch.equal(a, b), f"{dtype}: {what}"
        lp1 = ops.vocab_parallel_log_probs_from_logits(full.to(dtype)[:, -65:-1, :], tgt)
        assert torch.equal(lp1, outs[0][0])
    # calculate_entropy_loss=False: the entropy is returned without a gradient
    ent, lp = ops.vocab_parallel_entropy_and_log_probs(full[:, :4].clone().requires_grad_(True), tgt[:, :4],
                                                       calculate_entropy_loss=False)
    assert lp.requires_grad and not ent.requires_grad


@pytest.mark.parametrize("P", [2, 4])
def test_vp_logits_shards_agree_with_fused_and_fp64(P):
    """The logits-level records / backward of each rank's [..., Vs] shard of x @ W^T give what the fused op gives on the
    same shards, and the fp64 gradient of the full logits (targets outside a shard get no target term there)."""
    from rlinf_b200 import ops

    x, w, tgt, _, temp, window, lo, hi, glp, gh = _case("p2_window_straddles", seed=7)
    _, lp_f, ent_f, lse_f, _, _ = _emulate(x, w, tgt, P, temp, window, glp, gh)
    logits = (x.float() @ w.float().T)
    Vs = w.shape[0] // P
    rec = torch.stack([ops.logits_vp_partials(logits[:, k * Vs:(k + 1) * Vs], tgt, k, P, temp, window)
                       for k in range(P)])
    lp, ent, lse = ops.vp_combine(rec, tgt, Vs, window)
    for a, b, what in ((lp, lp_f, "logprob"), (ent, ent_f, "entropy"), (lse, lse_f, "lse")):
        _close_fp32(a, b.double(), what)
    rlp, rent, _, _, _, rdz = _ref(x, w, tgt, temp, lo, hi, glp, gh)
    _close_fp32(lp, rlp, "logprob vs fp64")
    _close_fp32(ent, rent, "entropy vs fp64")
    # the backward over the whole vocabulary, temperature folded into the logits (d(logits / T) = dz * T)
    V = w.shape[0]
    _, _, _, _, _, rdz = _ref(x, w, tgt, temp, 0, V, glp, gh)
    scaled = logits / temp
    rec = torch.stack([ops.logits_vp_partials(scaled[:, k * Vs:(k + 1) * Vs], tgt, k, P) for k in range(P)])
    lp, ent, lse = ops.vp_combine(rec, tgt, Vs)
    # shard-local targets run negative and past the end on the ranks that do not own them: no target term there
    dl = torch.cat([ops.logits_vp_backward(scaled[:, k * Vs:(k + 1) * Vs], tgt, k, lse, ent, glp, gh)
                    for k in range(P)], dim=1)
    torch.testing.assert_close(dl.double(), rdz * temp, rtol=1e-4, atol=1e-6)


def test_vp_repeat_calls_bit_identical():
    x, w, tgt, P, temp, window, lo, hi, glp, gh = _case("p8_v151936", seed=9)
    a = _emulate(x, w, tgt, P, temp, window, glp, gh)
    b = _emulate(x, w, tgt, P, temp, window, glp, gh)
    for u, v in zip(a, b):
        assert torch.equal(u, v)


def test_vp_two_rank_nccl_matches_emulation(tmp_path):
    import json
    import os
    import socket
    import subprocess
    import sys

    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    outp = tmp_path / "vp.json"
    env = dict(os.environ, RB200_DIST_OUT=str(outp))
    worker = os.path.join(os.path.dirname(os.path.abspath(__file__)), "dist_lmhead_vp_worker.py")
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2",
                        "--master-addr", "127.0.0.1", "--master-port", str(port), worker], env=env, capture_output=True,
                       text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    res = json.loads(outp.read_text())
    assert res["ok"], res
