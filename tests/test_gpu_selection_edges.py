"""The top-k and action-token selections where they break (csrc/topk.cu, csrc/lmhead_topk.cu, csrc/action_sample.cu,
csrc/lmhead_sample.cu), against the fp64 oracles (tests/topk_oracle.py, tests/action_sample_oracle.py) on the same
rounded inputs:
  - vocabularies on both sides of the forward's shared-memory staging limit and LM-sized ones, so that the radix select
    also runs from global memory, with rows at every 16-byte phase; bit identity of the staged and the global-memory
    select on the same row; the fused LM head at V = 151936 over several row blocks with padding rows;
  - -inf columns (k past the finite count, so the k-th value is -inf), thousands of ties at the k-th value, all-equal
    rows and signed zeros at the k-th value (tests/selection_rows.py), for the top-k op and the sampler's top-k;
  - greedy ties across lanes and column groups, lowest index first, at every window-width regime of the sampler;
  - draws of a zero-probability column: -inf logits without a top-k filter and exp underflow at a low temperature."""
from __future__ import annotations

import os
import re

import pytest
import torch

import action_sample_oracle as A
import selection_rows as S
import topk_oracle as O

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
V_VLA = 32064
WIN_VLA = (32000 - 256, 32000)
V_LM = 151936
NEG = float("-inf")


def _ops():
    from rlinf_b200 import ops

    return ops


def _bits(t):
    return t.view(torch.int16 if t.dtype == torch.bfloat16 else torch.int32)


# --- the forward's staging limit (topk.cu launch_fwd: stage iff sizeof(Shared) + V * sizeof(T) + 16 <= kMaxSmem) ---
def _stage_geometry():
    """(sizeof(Shared), kMaxSmem) from topk.cu's constants; the layout of Shared is pinned so that a change to it fails
    here instead of moving the limit away from the tested V."""
    src = open(os.path.join(ROOT, "rlinf_b200", "csrc", "topk.cu")).read()
    c = {n: int(re.search(rf"constexpr int {n} = (\d+);", src).group(1)) for n in ("kThreads", "kDigit", "kMaxSmem")}
    body = re.search(r"struct __align__\(16\) Shared \{(.*?)\};", src, flags=re.S).group(1)
    members = [line.split("//")[0].strip() for line in body.strip().splitlines()]
    assert members == ["uint32_t hist[kBins];", "uint32_t wsum[kWarps];", "uint32_t sel_digit, sel_below;",
                       "Acc part[kWarps];"], members
    acc = open(os.path.join(ROOT, "rlinf_b200", "csrc", "softmax_acc.cuh")).read()
    assert re.search(r"struct Acc \{\s*float m, s, t;\s*\};", acc)
    warps = c["kThreads"] // 32
    size = 4 * (1 << c["kDigit"]) + 4 * warps + 8 + 12 * warps
    return (size + 15) // 16 * 16, c["kMaxSmem"]


SHARED, MAX_SMEM = _stage_geometry()


def _staged(V, item):
    return SHARED + V * item + 16 <= MAX_SMEM


def _largest_staged(item):
    return (MAX_SMEM - SHARED - 16) // item


LIM = {torch.float32: _largest_staged(4), torch.bfloat16: _largest_staged(2)}
WIDE = [(torch.float32, LIM[torch.float32]), (torch.float32, LIM[torch.float32] + 1), (torch.float32, 65536),
        (torch.float32, V_LM), (torch.bfloat16, 65536), (torch.bfloat16, LIM[torch.bfloat16]),
        (torch.bfloat16, LIM[torch.bfloat16] + 1), (torch.bfloat16, V_LM)]


def test_stage_limit_pairs_straddle_the_threshold():
    for dtype, item in ((torch.float32, 4), (torch.bfloat16, 2)):
        v = LIM[dtype]
        assert _staged(v, item) and not _staged(v + 1, item)
        assert v * item % 16 == 0  # 16-byte rows at the largest staged V (the bit-identity test)
        assert not _staged(V_LM, item)
    assert not _staged(65536, 4) and _staged(65536, 2)


def _check(lp, ent, dg, o, dtype, tgt):
    """lp / entropy / gradient of the op against the oracle's: the same NaN and -inf rows, finite entropies and
    gradients, no gradient off the kept set."""
    got_lp, got_ent = lp.detach().double(), ent.detach().double()
    assert torch.equal(torch.isnan(got_lp), torch.isnan(o["lp"]))
    assert torch.equal(torch.isneginf(got_lp), torch.isneginf(o["lp"]))
    fin = torch.isfinite(o["lp"])
    torch.testing.assert_close(got_lp[fin], o["lp"][fin], rtol=1e-4, atol=1e-5)
    assert torch.isfinite(got_ent).all()
    torch.testing.assert_close(got_ent, o["ent"], rtol=1e-4, atol=1e-5)
    dg = dg.double()
    assert torch.isfinite(dg).all()
    assert (dg[~o["kept"]] == 0).all()
    tol = 1e-4 if dtype == torch.float32 else 8e-3  # bf16 gradient: one rounding of each element
    t = torch.nn.functional.one_hot(tgt, dg.shape[-1]).bool()
    torch.testing.assert_close(dg[~t], o["grad"][~t], rtol=tol, atol=1e-6)
    # at the target g_lp (1 - p) cancels when p is near 1 (k = 1 on the argmax: exactly 0 in fp64); the kernel's
    # log-prob there is exact to about an ulp of z, which leaves |g| |z| 2^-24, a few 1e-6 at these logits
    torch.testing.assert_close(dg[t], o["grad"][t], rtol=tol, atol=1e-5)
    return fin


def _wide_logits(dtype, V, win, seed, bsz=3, L=11):
    """[bsz, L, V + 1] logits whose [:, :, 1:] slice holds the rows; the window is lifted by 0 ... 14 across the rows,
    so that rows with and without kept window columns both occur at small k.  Half the targets are the window's
    argmax, so that finite log-probs occur at every k."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    full = torch.randn(bsz, L, V + 1, device="cuda", generator=g) * 2.5
    lo, hi = win
    full[..., 1 + lo:1 + hi] += torch.linspace(0.0, 14.0, bsz * L, device="cuda").view(bsz, L, 1)
    full = full.to(dtype)
    tgt = torch.randint(lo, hi, (bsz, L), device="cuda", generator=g)
    tgt[:, ::2] = full[:, ::2, 1 + lo:1 + hi].float().argmax(-1) + lo  # kept whenever the row keeps a window column
    return full, tgt


@pytest.mark.parametrize("win", ["top", "all"])
@pytest.mark.parametrize("k_of", [1, 50, 4096, -1])  # -1: V - 1
@pytest.mark.parametrize("dtype,V", WIDE, ids=[f"{str(d)[6:]}-{v}" for d, v in WIDE])
def test_wide_vocab_against_fp64(dtype, V, k_of, win):
    ops = _ops()
    k = V - 1 if k_of < 0 else k_of
    lo, hi = (V - 256, V) if win == "top" else (0, V)
    full, tgt = _wide_logits(dtype, V, (lo, hi), seed=V + k)
    full.requires_grad_(True)
    sl = full[:, :, 1:]  # read in place: row starts at every 16-byte phase
    lp, ent = ops.logprobs_entropy_from_logits(sl, tgt, 1.3, (lo, hi), top_k=k)
    g = torch.Generator(device="cuda").manual_seed(7)
    g_lp = torch.randn(tgt.shape, device="cuda", generator=g)
    g_h = torch.randn(tgt.shape, device="cuda", generator=g)
    (d,) = torch.autograd.grad((lp, ent), full, grad_outputs=(g_lp, g_h))
    o = O.topk_logprobs_entropy(sl.detach(), tgt, 1.3, (lo, hi), k, g_lp=g_lp, g_h=g_h)
    fin = _check(lp, ent, d[:, :, 1:], o, dtype, tgt)
    assert (d[:, :, 0] == 0).all()
    assert int(fin.sum()) > 0


@pytest.mark.parametrize("k_of", [50, -1])  # -1: V - 1 of the staged row, below its finite count
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_staged_and_global_select_are_bit_identical(dtype, k_of):
    """The same rows at the largest staged V and padded with -inf to an unstaged V: the kept set and every vector split
    are the same, so only the staging differs and every output bit must match."""
    ops = _ops()
    item = torch.finfo(dtype).bits // 8
    Vs = LIM[dtype]
    Vu = Vs + 16 // item
    assert _staged(Vs, item) and not _staged(Vu, item) and Vs * item % 16 == 0 and Vu * item % 16 == 0
    k = Vs - 1 if k_of < 0 else k_of
    N, win = 64, (Vs - 777, Vs - 3)
    g = torch.Generator(device="cuda").manual_seed(Vs + k)
    xs = torch.randn(N, Vs, device="cuda", generator=g) * 2.5
    xs[:, win[0]:win[1]] += torch.linspace(0.0, 14.0, N, device="cuda").view(N, 1)
    xs = xs.to(dtype)
    xu = torch.cat([xs, torch.full((N, Vu - Vs), NEG, device="cuda", dtype=dtype)], 1)
    tgt = torch.randint(win[0], win[1], (N,), device="cuda", generator=g)
    g_lp, g_h = torch.randn(N, device="cuda", generator=g), torch.randn(N, device="cuda", generator=g)

    def run(x):
        xg = x.clone().requires_grad_(True)
        lp, ent = ops.logprobs_entropy_from_logits(xg, tgt, 1.3, win, top_k=k)
        (d,) = torch.autograd.grad((lp, ent), xg, grad_outputs=(g_lp, g_h))
        return lp.detach(), ent.detach(), d

    a, b = run(xs), run(xu)
    assert torch.equal(_bits(a[0]), _bits(b[0])) and torch.equal(_bits(a[1]), _bits(b[1]))
    assert torch.equal(_bits(a[2]), _bits(b[2][:, :Vs])) and (b[2][:, Vs:] == 0).all()
    assert torch.isfinite(a[0]).any()


def _separated(z, k, gap=1e-5):
    """rows whose k-th and (k+1)-th largest logits are more than gap apart: the kept set does not depend on rounding"""
    v = torch.topk(z, k + 1, dim=-1).values
    return (v[:, k - 1] - v[:, k]) > gap


@pytest.mark.parametrize("k", [50, 4096])
def test_fused_lm_vocab_over_row_blocks(monkeypatch, k):
    """V = 151936 (the select runs from global memory) with N not a multiple of 128 and one-tile row blocks: four
    blocks, the last with padding rows."""
    ops = _ops()
    monkeypatch.setattr(ops, "LMHEAD_TOPK_ROW_BLOCK", 128)
    N, H, win = 3 * 128 + 45, 256, (V_LM - 256, V_LM)
    g = torch.Generator(device="cuda").manual_seed(k)
    x = torch.randn(N, H, generator=g, device="cuda").to(torch.bfloat16)
    w = torch.randn(V_LM, H, generator=g, device="cuda") * H ** -0.5
    w[win[0]:win[1]] *= 1.5
    w = w.to(torch.bfloat16)
    tgt = torch.randint(win[0], win[1], (N,), generator=g, device="cuda")
    xg, wg = x.clone().requires_grad_(True), w.clone().requires_grad_(True)
    lp, ent = ops.linear_logprobs_entropy(xg, wg, tgt, 1.6, win, top_k=k)
    z32 = (x.float() @ w.float().T).requires_grad_(True)
    lp2, ent2 = ops.logprobs_entropy_from_logits(z32, tgt, 1.6, win, top_k=k)
    z64 = x.double() @ w.double().T
    o = O.topk_logprobs_entropy(z64, tgt, 1.6, win, k)
    ok = _separated(z64, k)
    assert ok.float().mean() > 0.8  # at k = 4096 the sorted logits are about 3e-4 apart
    for a in (lp.detach(), lp2.detach()):
        assert torch.equal(torch.isnan(a)[ok], torch.isnan(o["lp"])[ok])
        assert torch.equal(torch.isneginf(a)[ok], torch.isneginf(o["lp"])[ok])
    fin = ok & torch.isfinite(o["lp"])
    assert int(fin.sum()) > 0
    torch.testing.assert_close(lp.detach()[fin].double(), o["lp"][fin], rtol=2e-3, atol=2e-3)
    torch.testing.assert_close(ent.detach()[ok].double(), o["ent"][ok], rtol=2e-3, atol=2e-3)
    torch.testing.assert_close(lp.detach()[fin], lp2.detach()[fin], rtol=1e-4, atol=1e-4)
    torch.testing.assert_close(ent.detach()[ok], ent2.detach()[ok], rtol=1e-4, atol=1e-4)
    gg = torch.Generator(device="cuda").manual_seed(5)
    g_lp, g_h = torch.randn(N, device="cuda", generator=gg), torch.randn(N, device="cuda", generator=gg)
    g_lp = torch.where(torch.isfinite(lp.detach()), g_lp, 0.0)
    (lp * g_lp).sum().add_((ent * g_h).sum()).backward()
    (dz,) = torch.autograd.grad((lp2 * g_lp).sum() + (ent2 * g_h).sum(), z32)
    dz = torch.where(ok.unsqueeze(-1), dz, 0.0)
    rows = ok.nonzero()[:, 0]
    torch.testing.assert_close(xg.grad[rows].float(), dz[rows] @ w.float(), rtol=3e-2, atol=3e-3)
    if bool(ok.all()):
        torch.testing.assert_close(wg.grad.float(), dz.T @ x.float(), rtol=3e-2, atol=3e-3)


# --- hard rows: -inf, ties, all-equal, signed zeros ---
@pytest.mark.parametrize("win", ["top", "all"])
@pytest.mark.parametrize("k_of", [1, 50, 4096, -1])  # -1: V - 1
@pytest.mark.parametrize("V", [V_VLA, V_LM])  # staged / from global memory, in both dtypes
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_topk_hard_rows_against_fp64(dtype, V, k_of, win):
    ops = _ops()
    k = V - 1 if k_of < 0 else k_of
    lo, hi = (V - 320, V - 64) if win == "top" else (0, V)
    rows, _ = S.hard_rows(V, lo, hi, k, seed=V + k)
    R = rows.shape[0]
    x = rows.to(dtype).cuda()  # exact in both dtypes
    g = torch.Generator().manual_seed(V + k)
    tgt = torch.randint(lo, hi, (R,), generator=g).cuda()
    g_lp, g_h = torch.randn(R, generator=g).cuda(), torch.randn(R, generator=g).cuda()
    T = 0.7
    xg = x.clone().requires_grad_(True)
    lp, ent = ops.logprobs_entropy_from_logits(xg, tgt, T, (lo, hi), top_k=k)
    # the kept set through the log-prob gradient: -p_i / T at every kept finite column, so nonzero exactly there
    # (and at the target, 1 - p_t, which is left out: a lone dominant column can round p_t to 1 in fp32)
    (d1,) = torch.autograd.grad(lp, xg, grad_outputs=torch.ones_like(lp), retain_graph=True)
    o1 = O.topk_logprobs_entropy(x, tgt, T, (lo, hi), k, g_lp=torch.ones(R, device="cuda"))
    nz, nz1 = d1 != 0, o1["grad"] != 0
    ar = torch.arange(R, device="cuda")
    nz[ar, tgt] = False
    nz1[ar, tgt] = False
    assert torch.equal(nz, nz1)
    (d,) = torch.autograd.grad((lp, ent), xg, grad_outputs=(g_lp, g_h))
    o = O.topk_logprobs_entropy(x, tgt, T, (lo, hi), k, g_lp=g_lp, g_h=g_h)
    _check(lp, ent, d, o, dtype, tgt)


@pytest.mark.parametrize("k_of", [0, 1, 16, -1])  # -1: W - 1
@pytest.mark.parametrize("W", [32, 257, 1024])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_sampler_topk_hard_rows(dtype, W, k_of):
    """2^14 draws of each hard row (a stride-0 batch): only columns of positive probability are drawn, with the fp64
    log-prob, and every column the oracle expects 30 or more times is drawn (ties at the k-th value are all kept)."""
    ops = _ops()
    k = W - 1 if k_of < 0 else k_of
    lo = 32000 - W
    rows, _ = S.hard_rows(W, 0, W, k, seed=W + k)
    R, D, T = rows.shape[0], 1 << 14, 0.7
    x = torch.full((R, V_VLA), float("nan"), dtype=dtype)
    x[:, lo:lo + W] = rows.to(dtype)
    xs = x.cuda().view(1, R, V_VLA).expand(D, R, V_VLA)
    tok, lp, _ = ops.sample_action_tokens(xs, (lo, lo + W), do_sample=True, temperature=T, top_k=k, seed=5, offset=W)
    logp = A.window_logprobs(rows.double(), 0, W, True, T, k)  # [R, W]
    col = (tok - lo).cpu()
    assert ((col >= 0) & (col < W)).all()
    at = logp[torch.arange(R).view(1, R), col]
    assert torch.isfinite(at).all()
    torch.testing.assert_close(lp.cpu().double(), at, rtol=1e-5, atol=1e-5)
    counts = torch.zeros(R, W, dtype=torch.int64).scatter_add_(1, col.T, torch.ones_like(col.T))
    assert (counts[logp.exp() * D >= 30] > 0).all()


def _tie_sets(W, R, g):
    """Column sets tied at the row maximum: fixed ones across lanes (31 / 32), column groups (7, 39, 71) and the
    NJ = 8 / 32 boundary (255 / 256), then random ones."""
    fixed = [(31, 32), (0, W - 1), (7, 39, 71), (32, 95), (255, 256), (1, 33, 65, 1023), (W - 2, W - 1),
             (W // 2, W // 2 + 32), (63, 64, 1000)]
    sets = [sorted({c for c in s if 0 <= c < W}) for s in fixed]
    sets = [s for s in sets if len(s) >= 2]
    while len(sets) < R and W >= 2:
        n = int(torch.randint(2, min(W, 6) + 1, (1,), generator=g))
        sets.append(sorted(torch.randperm(W, generator=g)[:n].tolist()))
    return sets[:R]


@pytest.mark.parametrize("W", [1, 31, 32, 33, 256, 257, 1024])
def test_greedy_ties_lowest_index(W):
    ops = _ops()
    lo, R = 32000 - W, 512
    g = torch.Generator().manual_seed(W)
    win = torch.randn(R, W, generator=g).to(torch.bfloat16)  # bf16 rows also tie by themselves
    sets = _tie_sets(W, R, g)
    for r, cols in enumerate(sets):
        win[r, cols] = 8.0
    x = torch.full((R, V_VLA), float("nan"), dtype=torch.bfloat16)
    x[:, lo:lo + W] = win
    tok, lp, _ = ops.sample_action_tokens(x.cuda().view(4, R // 4, V_VLA), (lo, lo + W), do_sample=False, seed=0,
                                          offset=0)
    tok, lp = tok.reshape(-1).cpu(), lp.reshape(-1).cpu()
    assert torch.equal(tok, A.greedy_tokens(x, lo, lo + W))
    assert [int(tok[r]) for r in range(len(sets))] == [lo + s[0] for s in sets]
    logp = A.window_logprobs(x.double(), lo, lo + W, False)
    torch.testing.assert_close(lp.double(), logp[torch.arange(R), tok - lo], rtol=1e-5, atol=1e-5)


@pytest.mark.parametrize("W", [1, 31, 32, 33, 256, 257, 1024])
def test_fused_greedy_ties_lowest_index(W):
    """Identical weight rows on a small-integer grid (exact fp32 logits) tie at the maximum of nearly every row; the fused
    sampler takes the lowest of them, bit for bit with the logits-level sampler."""
    ops = _ops()
    lo, N, H = 32000 - W, 2 * 128 + 37, 128
    g = torch.Generator(device="cuda").manual_seed(W)
    hidden = torch.randint(-2, 3, (N, H), device="cuda", generator=g).to(torch.bfloat16)
    hidden[:, :16] = 3
    w = torch.randint(-1, 2, (V_VLA, H), device="cuda", generator=g).to(torch.bfloat16)
    w[:, :16] = 0
    cols = sorted({c for c in (31, 32, 71, W // 2, W - 1) if c < W})
    tie = torch.randint(-1, 2, (H,), device="cuda", generator=g).to(torch.bfloat16)
    tie[:16] = 3  # +144 over the other columns
    w[[lo + c for c in cols]] = tie
    a = ops.linear_sample_action_tokens(hidden, w, (lo, lo + W), do_sample=False, seed=0, offset=0)
    z = hidden.double() @ w.double().T
    b = ops.sample_action_tokens(z.float().view(1, N, V_VLA), (lo, lo + W), do_sample=False, seed=0, offset=0)
    assert torch.equal(a[0], b[0].view(-1)) and torch.equal(_bits(a[1]), _bits(b[1].view(-1)))
    tok = a[0].cpu()
    assert torch.equal(tok, A.greedy_tokens(z.cpu(), lo, lo + W))
    assert (tok == lo + cols[0]).float().mean() > 0.99
    logp = A.window_logprobs(z.cpu(), lo, lo + W, False)
    torch.testing.assert_close(a[1].cpu().double(), logp[torch.arange(N), tok - lo], rtol=1e-5, atol=1e-5)


# --- zero-probability draws ---
# A draw lands on the first kept column whose inclusive prefix sum reaches u * total.  The shuffle scan sums each lane
# over its own tree, so a zero-weight column can carry a larger prefix than the positive column before it; a target
# between the two must not return the zero-weight column.  In an fp32 emulation of the scan about 90 % of these rows
# leave such a gap, 6e-8 to 9e-8 of the total on average: 2^30 draws expect several dozen hits if the kernel took those
# columns.  Only columns with z - m < -110 count, well clear of where exp(z - m) underflows.
ZP_ROWS, ZP_DRAWS = 64, 1 << 30


def _zero_weight_rows(case, g):
    """[64, 256] window values and the temperature: scattered -inf at T = 1, or at T = 0.02 half the columns within 0.3
    of the maximum and the rest 2.5 to 4 below it (z - m < -125: exp underflows to 0)."""
    if case == "neginf":
        w = torch.randn(ZP_ROWS, 256, generator=g) * 2
        w[torch.rand(ZP_ROWS, 256, generator=g) < 0.5] = NEG
        w[:, 0] = 0.5
        return w, 1.0
    near = torch.rand(ZP_ROWS, 256, generator=g) < 0.5
    near[:, 0] = True
    return torch.where(near, 1 - 0.3 * torch.rand(ZP_ROWS, 256, generator=g),
                       1 - 2.5 - 1.5 * torch.rand(ZP_ROWS, 256, generator=g)), 0.02


def _zero_weight(z, T):
    """columns of weight 0 with margin: -inf, or (z - max) / T < -110 (fp64)"""
    s = z.double() / T
    return torch.isneginf(z) | (s - s.max(-1, keepdim=True).values < -110)


@pytest.mark.parametrize("case", ["neginf", "low_T"])
def test_no_zero_probability_draws(case):
    ops = _ops()
    win, T = _zero_weight_rows(case, torch.Generator().manual_seed(11))
    bad = _zero_weight(win, T)
    assert bad.any(-1).all() and (~bad).sum(-1).min() > 1
    lo, hi = WIN_VLA
    x = torch.full((ZP_ROWS, V_VLA), float("nan"))
    x[:, lo:hi] = win
    D = 1 << 16
    xs = x.cuda().view(1, ZP_ROWS, V_VLA).expand(D, ZP_ROWS, V_VLA)
    bad = bad.cuda().reshape(-1)
    base = torch.arange(ZP_ROWS, device="cuda") * 256
    hits = torch.zeros((), dtype=torch.int64, device="cuda")
    neg = torch.zeros((), dtype=torch.int64, device="cuda")
    calls = ZP_DRAWS // (D * ZP_ROWS)
    for off in range(calls):
        tok, lp, _ = ops.sample_action_tokens(xs, WIN_VLA, do_sample=True, temperature=T, seed=2024, offset=off)
        hits += bad[base + (tok - lo)].sum()
        neg += torch.isneginf(lp).sum()
    hits, neg = int(hits), int(neg)
    assert hits == 0 and neg == 0, f"{hits} zero-weight draws and {neg} -inf log-probs in {calls * D * ZP_ROWS} draws"


def test_no_zero_probability_draws_fused():
    """The low-temperature case through the fused head: hidden states close to v, half the window's weight rows close to
    v and half close to -v, so the logits are about +1.5 and -1.5 and the second half underflows at T = 0.02."""
    ops = _ops()
    g = torch.Generator().manual_seed(12)
    H, T = 64, 0.02
    lo, hi = WIN_VLA
    v = torch.randn(H, generator=g)
    v /= v.norm()
    h = (1.5 * v + 0.03 * torch.randn(ZP_ROWS, H, generator=g)).to(torch.bfloat16)
    near = torch.rand(256, 1, generator=g) < 0.5
    near[0] = True
    w_win = (torch.where(near, v, -v) + 0.1 * torch.randn(256, H, generator=g)).to(torch.bfloat16)
    w = (0.1 * torch.randn(V_VLA, H, generator=g)).to(torch.bfloat16)
    w[lo:hi] = w_win
    bad = _zero_weight(h.double() @ w_win.double().T, T)
    assert bad.any(-1).all() and (~bad).sum(-1).min() > 1
    reps = 1 << 14  # 2^20 rows per call
    hidden = h.cuda().repeat(reps, 1)
    w = w.cuda()
    bad = bad.cuda().reshape(-1)
    base = (torch.arange(reps * ZP_ROWS, device="cuda") % ZP_ROWS) * 256
    hits = torch.zeros((), dtype=torch.int64, device="cuda")
    neg = torch.zeros((), dtype=torch.int64, device="cuda")
    calls = (ZP_DRAWS // 2) // (reps * ZP_ROWS)
    for off in range(calls):
        tok, lp, _ = ops.linear_sample_action_tokens(hidden, w, WIN_VLA, do_sample=True, temperature=T, seed=77,
                                                     offset=off)
        hits += bad[base + (tok - lo)].sum()
        neg += torch.isneginf(lp).sum()
    hits, neg = int(hits), int(neg)
    assert hits == 0 and neg == 0, f"{hits} zero-weight draws and {neg} -inf log-probs in {calls * reps * ZP_ROWS} draws"
