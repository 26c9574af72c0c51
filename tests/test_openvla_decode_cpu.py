"""Plain OpenVLA's generate step without a GPU: the restatement (tests/openvla_decode_oracle.py) against the
transformers-generate fixture (tests/golden/golden_openvla_decode.npz), HF's processor order, rb200_sample_step against
the header, the argument checks of the step and counter modes, and ptxas on the sampler objects (no spills, no
serialised wgmma)."""
from __future__ import annotations

import ctypes as C
import os
import re
import shutil
import subprocess
import sys

import numpy as np
import pytest
import torch

import action_sample_oracle as O
import openvla_decode_oracle as D
from rlinf_b200 import _lib, build

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_golden_openvla_decode as G  # noqa: E402

FIX = os.path.join(HERE, "golden", "golden_openvla_decode.npz")
SAMPLED = [n for n in G.CASES if "greedy" not in n]


@pytest.fixture(scope="module")
def g():
    return dict(np.load(FIX))


def _case(n):
    """(do_sample, T, k) of a case name."""
    if n.endswith("greedy"):
        return False, 1.0, 0
    m = re.search(r"T([0-9.]+)_k(\d+)$", n)
    return True, float(m.group(1)), int(m.group(2))


def _detok(g, tokens):
    return O.detokenize(tokens, G.VOCAB, g["bin_centers"], g["q01"], g["q99"], g["mask"])


@pytest.mark.parametrize("n", ["greedy", "tie_greedy"])
def test_restatement_reproduces_greedy_fixture(g, n):
    x = torch.from_numpy(g[f"{n}_logits"])
    tok = D.greedy_step(x, G.LO)
    assert np.array_equal(tok.numpy(), g[f"{n}_tokens"])
    lp = D.step_logprobs(x, False).gather(-1, tok.unsqueeze(-1) - G.LO).squeeze(-1)
    np.testing.assert_allclose(lp.numpy(), g[f"{n}_logprob"], rtol=1e-6, atol=2e-6)
    act = _detok(g, g[f"{n}_tokens"])
    assert act.dtype == np.float64 and np.array_equal(act, g[f"{n}_actions"])
    assert not g["mask"][G.MASK_OFF] and np.array_equal(act[:, G.MASK_OFF],
                                                        g["bin_centers"][G.VOCAB - g[f"{n}_tokens"][:, G.MASK_OFF] - 1])
    if n.startswith("tie"):  # the duplicated rows tie at the argmax somewhere, and the lowest index wins
        ties = (x == x.max(-1, keepdim=True).values).sum(-1) > 1
        assert ties.any()


@pytest.mark.parametrize("n", G.CASES)
def test_processed_scores_are_window_then_temperature_then_top_k(g, n):
    do_sample, T, k = _case(n)
    assert bool(g[f"{n}_outside_inf"])
    want = D.processed_scores(torch.from_numpy(g[f"{n}_logits"]), do_sample, T, k).numpy()
    assert np.array_equal(want.view(np.int32), g[f"{n}_scores"].view(np.int32))
    if 0 < k:  # ties at the k-th value are kept: some steps keep more than k columns
        assert (np.isfinite(g[f"{n}_scores"]).sum(-1) > k).any()


@pytest.mark.parametrize("n", SAMPLED)
def test_fixture_draws_and_logprobs(g, n):
    do_sample, T, k = _case(n)
    s = torch.from_numpy(g[f"{n}_scores"]).double()
    tok = g[f"{n}_tokens"]
    at = torch.log_softmax(s, -1).gather(-1, torch.from_numpy(tok - G.LO)[..., None])[..., 0].numpy()
    assert np.isfinite(at).all()
    np.testing.assert_allclose(g[f"{n}_logprob"], at, rtol=1e-6, atol=2e-6)
    assert np.array_equal(_detok(g, tok), g[f"{n}_actions"])
    # the sampler's kept set (top-k on the unscaled values) is HF's: no two bf16 logits merge when divided by T
    mine = D.step_logprobs(torch.from_numpy(g[f"{n}_logits"]), do_sample, T, k)
    assert torch.equal(torch.isneginf(mine), torch.isneginf(s))


def test_hidden_rows_and_window_weight_give_the_logits(g):
    for n in ("greedy", "tie_greedy"):
        w = torch.from_numpy(g[("tie_" if n.startswith("tie") else "") + "w_window"]).double()
        z = (torch.from_numpy(g[f"{n}_hidden"]).double() @ w.T).to(torch.bfloat16).float()
        torch.testing.assert_close(z, torch.from_numpy(g[f"{n}_logits"]), rtol=1e-2, atol=1e-2)


# ------------------------------------------------------------------ ABI
def test_sample_step_layout_matches_ctypes(tmp_path):
    cls, cname = _lib.SampleStep, "rb200_sample_step"
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
    assert got["sizeof"] == (C.sizeof(cls),) == (24,)
    for f in cls._fields_:
        d = getattr(cls, f[0])
        assert got[f[0]] == (d.offset, d.size), f[0]


def _lib_loaded():
    if not os.path.exists(_lib.LIB_PATH):
        build.build()
    return _lib.load()


def test_step_envelope_returns_invalid_argument():
    """The checks that fail before any launch: an output layout that does not hold the rows."""
    lib = _lib_loaded()
    p = _lib.c_void_p(1 << 20)
    f = lib.rb200_logits_sample_step

    def call(step, L=1, N=4):
        return f(p, 1, N, L, 320, 320, 320, 44, 300, 1, 1.0, 8, 1, 2, None, p, p, None, step, None)

    assert call(C.byref(_lib.SampleStep(None, 7, -1, 0))) == -2          # col0 < 0
    assert call(C.byref(_lib.SampleStep(None, 7, 7, 0))) == -2           # col0 + L past the row stride
    assert call(C.byref(_lib.SampleStep(None, 13, 7, 0)), L=7, N=14) == -2
    fused = lib.rb200_lmhead_sample_step

    def fcall(step, H=64):
        return fused(p, p, 256, 1, H, H, H, 320, 44, 300, 1, 1.0, 8, 1, 2, None, p, p, None, p, 1 << 30, step, None)

    assert fcall(C.byref(_lib.SampleStep(None, 7, 7, 0))) == -2
    assert fcall(C.byref(_lib.SampleStep(None, 7, 0, 0)), H=96) == -2   # H % 64


# ------------------------------------------------------------------ argument checks
def _out(bsz=4, A=7, bins=True, **over):
    o = dict(tok=torch.zeros(bsz, A, dtype=torch.int64), lp=torch.zeros(bsz, A), act=torch.zeros(bsz, A,
                                                                                                dtype=torch.float64))
    o.update(over)
    return o["tok"], o["lp"], (o["act"] if bins else None)


def _bins():
    from rlinf_b200 import ops

    return ops.ActionBins(32000, np.linspace(-1, 1, 255), np.zeros(7), np.ones(7))


def test_step_arguments_are_validated():
    from rlinf_b200 import ops

    x = torch.zeros(4, 1, 32064)
    win = (31744, 32000)
    kw = dict(do_sample=True, seed=0, offset=0, bins=_bins())
    f = ops.sample_action_tokens
    for j in (-1, 7, 100):
        with pytest.raises(ValueError, match="column"):
            f(x, win, out=_out(), column=j, **kw)
    for j in (1.0, True, "2"):
        with pytest.raises(ValueError, match="column must be an integer"):
            f(x, win, out=_out(), column=j, **kw)
    with pytest.raises(ValueError, match="go together"):
        f(x, win, out=_out(), **kw)
    with pytest.raises(ValueError, match="go together"):
        f(x, win, column=0, **kw)
    with pytest.raises(ValueError, match="out must be"):
        f(x, win, out=_out()[:2], column=0, **kw)
    bad = [dict(tok=torch.zeros(4, 7, dtype=torch.int32)), dict(lp=torch.zeros(4, 7, dtype=torch.float64)),
           dict(act=torch.zeros(4, 7)), dict(lp=torch.zeros(4, 7, 1)), dict(lp=torch.zeros(4, 8)),
           dict(act=torch.zeros(7, 4, dtype=torch.float64).T), dict(tok=torch.zeros(4, 14, dtype=torch.int64)[:, ::2])]
    for over in bad:
        with pytest.raises(ValueError, match="out's"):
            f(x, win, out=_out(**over), column=0, **kw)
    with pytest.raises(ValueError, match="actions buffer"):
        f(x, win, out=_out(bins=False), column=0, **kw)
    with pytest.raises(ValueError, match="actions buffer"):
        f(x, win, out=_out(), column=0, do_sample=True, seed=0, offset=0)
    for shape in ((4, 2, 32064), (5, 1, 32064), (3, 32064)):
        with pytest.raises(ValueError, match=r"\[bsz, 1, V\]"):
            f(torch.zeros(shape), win, out=_out(), column=0, **kw)
    for top_p in (0.9, 0.0, 1.1):
        with pytest.raises(ValueError, match="top_p"):
            f(x, win, out=_out(), column=0, top_p=top_p, **kw)
        with pytest.raises(ValueError, match="top_p"):
            f(x, win, top_p=top_p, **kw)


def test_offset_and_counter_are_exclusive_and_checked():
    from rlinf_b200 import ops

    x = torch.zeros(4, 1, 32064)
    win = (31744, 32000)
    for fn, args in ((ops.sample_action_tokens, (x, win)),
                     (ops.linear_sample_action_tokens, (torch.zeros(4, 64, dtype=torch.bfloat16),
                                                        torch.zeros(32064, 64, dtype=torch.bfloat16), win))):
        with pytest.raises(ValueError, match="exactly one of offset"):
            fn(*args, do_sample=True, seed=0)
        with pytest.raises(ValueError, match="exactly one of offset"):
            fn(*args, do_sample=True, seed=0, offset=0, counter=torch.zeros(1, dtype=torch.int64))
        with pytest.raises(ValueError, match="CUDA tensor"):
            fn(*args, do_sample=True, seed=0, counter=torch.zeros(1, dtype=torch.int64))
        for c in (torch.zeros(1, dtype=torch.int32), torch.zeros(1), torch.zeros(2, dtype=torch.int64), 3):
            with pytest.raises(ValueError, match="1-element int64"):
                fn(*args, do_sample=True, seed=0, counter=c)
        with pytest.raises(ValueError, match="column"):
            fn(*args, do_sample=True, seed=0, offset=0, out=_out(bins=False), column=7)


# ------------------------------------------------------------------ ptxas
def _ptxas_log(tmp_path, src):
    try:
        nvcc = build._nvcc()
    except RuntimeError:
        pytest.skip("nvcc not found")
    cmd = [nvcc, *build.NVCC_FLAGS, "-Xptxas", "-v", "-c", os.path.join(build.CSRC, src), "-o", str(tmp_path / "x.o")]
    out = subprocess.run(cmd, capture_output=True, text=True)
    log = out.stdout + out.stderr
    assert out.returncode == 0, log
    entries = re.findall(r"Compiling entry function '([^']+)'.*?(\d+) bytes spill stores, (\d+) bytes spill loads", log,
                         flags=re.S)
    return log, entries


def test_sampler_objects_no_spills_no_serialised_wgmma(tmp_path):
    log, entries = _ptxas_log(tmp_path, "action_sample.cu")
    assert len(entries) == 4 and all(e[1:] == ("0", "0") for e in entries), log
    log, entries = _ptxas_log(tmp_path, "lmhead_sample.cu")
    assert not re.search(r"C751[0-4]", log) and "serialized" not in log, log
    assert len(entries) == 1 and all(e[1:] == ("0", "0") for e in entries), log
