"""Action-token sampling of the OpenVLA-OFT rollout without a GPU: the fp64 oracle and the numpy de-tokeniser
(tests/action_sample_oracle.py) against the reference fixture (tests/golden/golden_action_sample.npz), argument
validation, the C envelope of both entries, their ctypes signatures and rb200_action_bins against the header, no spills
in csrc/action_sample.cu and csrc/lmhead_sample.cu and no serialised wgmma in the latter, and the SASS of logits.o,
lmhead.o and topk.o as at the parent commit (tests/golden/sass_digests_action_sample.json)."""
from __future__ import annotations

import ctypes as C
import hashlib
import json
import os
import re
import shutil
import subprocess
import sys

import numpy as np
import pytest
import torch

import action_sample_oracle as O
from rlinf_b200 import _lib, build

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_golden_action_sample as G  # noqa: E402

FIX = os.path.join(HERE, "golden", "golden_action_sample.npz")
DIGESTS = os.path.join(HERE, "golden", "sass_digests_action_sample.json")


@pytest.fixture(scope="module")
def g():
    return dict(np.load(FIX))


def _detok(g, tokens):
    return O.detokenize(tokens, G.VOCAB, g["bin_centers"], g["q01"], g["q99"], g["mask"])


@pytest.mark.parametrize("C", G.CHUNKS)
def test_oracle_reproduces_greedy_fixture(g, C):
    x = torch.from_numpy(g[f"c{C}_logits"])
    tok = O.greedy_tokens(x, G.LO, G.HI)
    want = g[f"c{C}_greedy_tokens"]
    assert np.array_equal(tok.numpy(), want)
    lp = O.window_logprobs(x, G.LO, G.HI, False).gather(-1, tok.unsqueeze(-1) - G.LO).squeeze(-1)
    np.testing.assert_allclose(lp.numpy(), g[f"c{C}_greedy_logprob"], rtol=1e-6, atol=1e-6)
    act = _detok(g, want)
    assert act.dtype == np.float64 and np.array_equal(act, g[f"c{C}_greedy_actions"])
    # the planted rows do what they are there for
    for b in range(want.shape[0]):
        assert G.LO <= want[b, 0] < G.HI and x[b, 0].argmax() >= G.HI           # the maximum is outside the window
        ties = (x[b, 1, G.LO:G.HI] == x[b, 1, G.LO:G.HI].max()).nonzero()[:, 0]
        assert len(ties) == 2 and want[b, 1] == G.LO + ties[0]                  # lowest index of the tie
        assert want[b, 5] == G.LO and want[b, 6] == G.HI - 1                    # both window edges
    assert (act[:, 5] == _detok(g, np.full_like(want, G.LO))[:, 5]).all()       # the bin clip at the low edge


@pytest.mark.parametrize("C,T,k", [(C, T, k) for C in G.CHUNKS for T, k in G.CASES])
def test_oracle_reproduces_sampling_fixture(g, C, T, k):
    x = torch.from_numpy(g[f"c{C}_logits"])
    n = G.case_name(C, T, k)
    table = g[f"{n}_table"]
    o = O.window_logprobs(x, G.LO, G.HI, True, T, k).numpy()
    assert np.array_equal(np.isneginf(o), np.isneginf(table))
    fin = np.isfinite(table)
    np.testing.assert_allclose(o[fin], table[fin], rtol=1e-6, atol=1e-6)
    tok = g[f"{n}_tokens"]
    at = np.take_along_axis(table, (tok - G.LO)[..., None], -1)[..., 0]
    assert np.isfinite(at).all()
    np.testing.assert_allclose(g[f"{n}_logprob"], at, rtol=1e-6, atol=1e-6)
    assert np.array_equal(_detok(g, tok), g[f"{n}_actions"])
    if 0 < k < G.HI - G.LO:
        kept = fin.sum(-1)
        assert (kept >= k).all()
        if k in G.TIE_KS:
            assert (kept[:, 2 + G.TIE_KS.index(k)] == k + 1).all()            # ties at the k-th value are all kept


def test_oracle_no_filter_is_the_window_softmax():
    gen = torch.Generator().manual_seed(5)
    x = torch.randn(4, 64, generator=gen, dtype=torch.float64)
    base = O.window_logprobs(x, 10, 50, True, 1.3, 0)
    for k in (-1, 40, 41):
        assert torch.equal(O.window_logprobs(x, 10, 50, True, 1.3, k), base)
    assert torch.allclose(base, torch.log_softmax(x[:, 10:50] / 1.3, -1))
    assert torch.equal(O.window_logprobs(x, 10, 50, False, 1.3, 5), torch.log_softmax(x[:, 10:50], -1))


def test_arguments_are_validated():
    from rlinf_b200 import ops

    x = torch.zeros(2, 7, 320)
    kw = dict(do_sample=True, seed=0, offset=0)
    for bad in (True, 2.0, "50", None):
        with pytest.raises(ValueError, match="top_k must be an integer"):
            ops.sample_action_tokens(x, (44, 300), top_k=bad, **kw)
    for T in (0.0, -1.0):
        with pytest.raises(ValueError, match="temperature"):
            ops.sample_action_tokens(x, (44, 300), temperature=T, **kw)
    for V, win in ((320, (-1, 300)), (320, (44, 321)), (320, (300, 44)), (320, (44, 44)), (2000, (0, 1025))):
        with pytest.raises(ValueError, match="window"):
            ops.sample_action_tokens(torch.zeros(2, 7, V), win, **kw)
    bins = ops.ActionBins(300, np.linspace(-1, 1, 255), np.zeros(7), np.ones(7))
    with pytest.raises(ValueError, match="whole actions"):
        ops.sample_action_tokens(torch.zeros(2, 8, 320), (44, 300), bins=bins, **kw)
    with pytest.raises(ValueError, match="same non-zero length"):
        ops.ActionBins(300, np.linspace(-1, 1, 255), np.zeros(7), np.ones(6))
    with pytest.raises(ValueError, match="seed"):
        ops.sample_action_tokens(x, (44, 300), do_sample=True, seed=-1, offset=0)


def _lib_loaded():
    if not os.path.exists(_lib.LIB_PATH):
        build.build()
    return _lib.load()


@pytest.mark.parametrize("name", ["rb200_logits_sample_step", "rb200_lmhead_sample_workspace_bytes",
                                  "rb200_lmhead_sample_step"])
def test_ctypes_signature_matches_header(name):
    src = open(os.path.join(ROOT, "include", "rlinf_b200.h")).read()
    m = re.search(rf"(int|int64_t) {name}\((.*?)\);", src, flags=re.S)
    params = [q.strip() for q in m.group(2).split(",")]
    ctype = {"int": _lib.c_int, "int64_t": _lib.c_int64, "uint64_t": _lib.c_uint64, "double": _lib.c_double}
    want = []
    for q in params:
        if q.startswith("const rb200_action_bins*"):
            want.append(C.POINTER(_lib.ActionBins))
        elif q.startswith("const rb200_sample_step*"):
            want.append(C.POINTER(_lib.SampleStep))
        elif "*" in q or q.startswith("rb200_stream_t"):
            want.append(_lib.c_void_p)
        else:
            want.append(ctype[q.rsplit(" ", 1)[0]])
    res, args = _lib.SIGNATURES[name]
    assert res is ctype[m.group(1)] and args == want


def test_struct_layout_matches_ctypes(tmp_path):
    cls, cname = _lib.ActionBins, "rb200_action_bins"
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
    assert got["sizeof"] == (C.sizeof(cls),)
    for f in cls._fields_:
        d = getattr(cls, f[0])
        assert got[f[0]] == (d.offset, d.size), f[0]


def test_c_envelope_returns_invalid_argument():
    lib = _lib_loaded()
    p = _lib.c_void_p(1 << 20)
    f = lib.rb200_logits_sample_step

    def call(lo=44, hi=300, V=320, do_sample=1, inv_t=1.0, bins=None, tok=p, lp=p, act=p, dtype=1, N=14, L=7):
        return f(p, dtype, N, L, 7 * V, V, V, lo, hi, do_sample, inv_t, 8, 1, 2, bins, tok, lp, act, None, None)

    assert call(lo=44, hi=44) == -2                          # W = 0
    assert call(lo=0, hi=1025, V=2000) == -2                 # W > 1024
    assert call(lo=-1) == -2 and call(hi=321) == -2          # outside [0, V)
    assert call(inv_t=0.0) == -3 and call(inv_t=-1.0) == -3  # T <= 0 when sampling
    assert call(N=13) == -2                                  # N % L
    assert call(dtype=2) == -5
    assert call(tok=None) == -1 and call(lp=None) == -1
    bad = _lib.ActionBins(None, 1 << 20, 1 << 20, 1 << 20, 300, 255, 7)
    assert call(bins=C.byref(bad)) == -1                     # a table without its bin centres
    good = _lib.ActionBins(1 << 20, 1 << 20, 1 << 20, 1 << 20, 300, 255, 7)
    assert call(bins=C.byref(good), act=None) == -1          # actions need an output
    ws = lib.rb200_lmhead_sample_workspace_bytes
    assert ws(256, 256, 1000, 320, 44, 300) == -1            # H % 64 != 0
    assert ws(256, 256, 64, 320, 44, 300) == 2 * 128 * 256 * 4
    assert ws(300, 300, 64, 320, 44, 301) == 3 * 128 * 260 * 4
    fused = lib.rb200_lmhead_sample_step

    def fcall(H=64, lo=44, hi=300, V=320, inv_t=1.0, wsb=1 << 30):
        return fused(p, p, 256, 256, 256 * H, H, H, V, lo, hi, 1, inv_t, 8, 1, 2, None, p, p, None, p, wsb, None, None)

    assert fcall(H=96) == -2 and fcall(H=8256) == -2          # H % 64, H > 8192
    assert fcall(lo=44, hi=44) == -2 and fcall(lo=0, hi=1025, V=2000) == -2 and fcall(hi=321) == -2
    assert fcall(inv_t=0.0) == -3
    assert fcall(wsb=2 * 128 * 256 * 4 - 16) == -3           # workspace below the window block


def _nvcc():
    try:
        return build._nvcc()
    except RuntimeError:
        pytest.skip("nvcc not found")


def _ptxas_log(tmp_path, src):
    cmd = [_nvcc(), *build.NVCC_FLAGS, "-Xptxas", "-v", "-c", os.path.join(build.CSRC, src), "-o", str(tmp_path / "x.o")]
    out = subprocess.run(cmd, capture_output=True, text=True)
    log = out.stdout + out.stderr
    assert out.returncode == 0, log
    entries = re.findall(r"Compiling entry function '([^']+)'.*?(\d+) bytes spill stores, (\d+) bytes spill loads", log,
                         flags=re.S)
    return log, entries


def test_sampler_kernels_do_not_spill(tmp_path):
    log, entries = _ptxas_log(tmp_path, "action_sample.cu")
    assert len(entries) == 4 and all(e[1:] == ("0", "0") for e in entries), log  # fp32 / bf16 x W <= 256 / <= 1024


def test_fused_sampler_not_serialised_and_no_spills(tmp_path):
    log, entries = _ptxas_log(tmp_path, "lmhead_sample.cu")
    assert "C7512" not in log and "C7514" not in log and "C7510" not in log and "serialized" not in log, log
    assert len(entries) == 1 and all(e[1:] == ("0", "0") for e in entries), log


def _sass(tmp_path, obj):
    nvcc = _nvcc()
    cuobjdump = shutil.which("cuobjdump") or os.path.join(os.path.dirname(nvcc), "cuobjdump")
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not found")
    o = tmp_path / obj
    subprocess.run([nvcc, *build.NVCC_FLAGS, "-c", os.path.join(build.CSRC, obj[:-2] + ".cu"), "-o", str(o)],
                   check=True, capture_output=True)
    text = subprocess.run([cuobjdump, "-sass", str(o)], check=True, capture_output=True, text=True).stdout
    text = re.sub(r"_GLOBAL__N__[0-9a-f]+_\d+_\w+?_cu_[0-9a-f]+", "_GLOBAL__N_", text)
    return "\n".join(line for line in text.splitlines() if not line.strip().startswith("identifier"))


def test_existing_objects_keep_their_sass(tmp_path):
    """The generalised ACC epilogue and the shared radix keys leave logits.o, lmhead.o and topk.o as they were."""
    out = {}
    for obj in ("logits.o", "lmhead.o", "topk.o"):
        parts = re.split(r"^\s*Function : (\S+)\s*$", _sass(tmp_path, obj), flags=re.M)
        out[obj] = {parts[i]: hashlib.sha256(parts[i + 1].encode()).hexdigest() for i in range(1, len(parts), 2)}
    assert out == json.load(open(DIGESTS))
