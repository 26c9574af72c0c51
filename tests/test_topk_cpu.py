"""Top-k filtered log-probabilities without a GPU: the fp64 oracle (tests/topk_oracle.py) against the reference fixture
(tests/golden/golden_topk.npz: the OpenVLA heads' training forward with TopKLogitsWarper), the C envelope of the new
entries (logits level and fused head), the ctypes signatures against the header, no spills in csrc/topk.cu and
csrc/lmhead_topk.cu and no serialised wgmma in the latter, and the SASS of logits.o and lmhead.o as at the parent commit
(tests/golden/sass_digests_topk.json)."""
from __future__ import annotations

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

import topk_oracle as O
from rlinf_b200 import _lib, build

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_golden_topk as G  # noqa: E402

FIX = os.path.join(HERE, "golden", "golden_topk.npz")
DIGESTS = os.path.join(HERE, "golden", "sass_digests_topk.json")
CASES = [(C, T, k) for C in G.CHUNKS for T, k in G.CASES]


@pytest.fixture(scope="module")
def g():
    return dict(np.load(FIX))


def _slice(g, C):
    x = torch.from_numpy(g[f"c{C}_logits"])
    R = G.ADIM * C
    return x[:, x.shape[1] - R - 1:-1], torch.from_numpy(g[f"c{C}_target"])


@pytest.mark.parametrize("C,T,k", CASES)
def test_oracle_reproduces_reference_fixture(g, C, T, k):
    x, tgt = _slice(g, C)
    n = G.case_name(C, T, k)
    glp = torch.from_numpy(g[f"c{C}_g_lp"])
    o = O.topk_logprobs_entropy(x, tgt, T, (G.LO, G.HI), k, g_lp=glp)
    lp, ent = g[f"{n}_logprob"], g[f"{n}_entropy"]
    ol, oe = o["lp"].numpy(), o["ent"].numpy()
    assert np.array_equal(np.isnan(ol), np.isnan(lp)) and np.array_equal(np.isneginf(ol), np.isneginf(lp))
    fin = np.isfinite(lp)
    np.testing.assert_allclose(ol[fin], lp[fin], rtol=1e-6, atol=1e-6)
    np.testing.assert_allclose(oe, ent, rtol=1e-6, atol=1e-6)
    assert np.array_equal(np.signbit(oe[np.isnan(ol)]), np.signbit(ent[np.isnan(lp)]))  # -0.0 on empty rows
    d = g[f"{n}_grad_lp"]
    np.testing.assert_allclose(o["grad"].numpy(), d, rtol=1e-5, atol=1e-6)
    assert np.array_equal(o["grad"].numpy() == 0, d == 0)
    if k < G.V:  # the planted rows do what they are there for
        assert np.isnan(lp[:, 0]).all() and np.isneginf(lp[:, 1]).all()
        assert (o["kept"].sum(-1) > 0).sum() >= lp.size - lp.shape[0]
        tie = 2 + G.TIE_KS.index(k) if k in G.TIE_KS else None
        if tie is not None:
            assert (o["kept"][:, tie].sum(-1) == k + 1).all()


@pytest.mark.parametrize("C", G.CHUNKS)
def test_reference_entropy_gradient_is_nan_where_the_closed_form_is_finite(g, C):
    """The deviation kept on purpose (DESIGN §2): autograd through the reference's entropy has NaNs on every row with a
    kept and a masked column, the op returns the finite closed form; on rows with no kept column both are 0."""
    x, tgt = _slice(g, C)
    for T, k in G.CASES:
        n = G.case_name(C, T, k)
        o = O.topk_logprobs_entropy(x, tgt, T, (G.LO, G.HI), k, g_lp=torch.from_numpy(g[f"c{C}_g_lp"]),
                                    g_h=torch.from_numpy(g[f"c{C}_g_h"]))
        d = g[f"{n}_grad_all"]
        nonempty = o["kept"].any(-1).numpy()
        assert np.isnan(d[nonempty]).any(-1).all() and torch.isfinite(o["grad"]).all()
        assert (d[~nonempty] == 0).all() and (o["grad"].numpy()[~nonempty] == 0).all()


def test_oracle_no_filter_is_the_window_op():
    gen = torch.Generator().manual_seed(3)
    x = torch.randn(5, 40, generator=gen, dtype=torch.float64)
    t = torch.randint(0, 40, (5,), generator=gen)
    base = O.topk_logprobs_entropy(x, t, 1.3, (4, 30), 0)
    for k in (-1, 40, 47):
        o = O.topk_logprobs_entropy(x, t, 1.3, (4, 30), k)
        assert torch.equal(o["lp"], base["lp"]) and torch.equal(o["ent"], base["ent"])
    ref = torch.log_softmax(x[:, 4:30] / 1.3, -1)
    tin = (t >= 4) & (t < 30)
    assert torch.allclose(base["lp"][tin], ref[tin.nonzero()[:, 0], t[tin] - 4])


@pytest.mark.parametrize("bad", [True, 2.0, "50", None])
def test_top_k_must_be_an_integer(bad):
    from rlinf_b200 import ops

    with pytest.raises(ValueError, match="top_k must be an integer"):
        ops.logprobs_entropy_from_logits(torch.zeros(2, 8), torch.zeros(2, dtype=torch.int64), top_k=bad)


def _lib_loaded():
    if not os.path.exists(_lib.LIB_PATH):
        build.build()
    return _lib.load()


@pytest.mark.parametrize("name", ["rb200_logits_topk_logprob_entropy_fwd", "rb200_logits_topk_logprob_entropy_bwd",
                                  "rb200_lmhead_topk_workspace_bytes", "rb200_lmhead_topk_logprob_entropy_fwd",
                                  "rb200_lmhead_topk_logprob_entropy_bwd"])
def test_ctypes_signature_matches_header(name):
    src = open(os.path.join(ROOT, "include", "rlinf_b200.h")).read()
    m = re.search(rf"(int|int64_t) {name}\((.*?)\);", src, flags=re.S)
    params = [q.strip() for q in m.group(2).split(",")]
    ctype = {"int": _lib.c_int, "int64_t": _lib.c_int64, "double": _lib.c_double}
    want = [_lib.c_void_p if ("*" in q or q.startswith("rb200_stream_t")) else ctype[q.rsplit(" ", 1)[0]]
            for q in params]
    res, args = _lib.SIGNATURES[name]
    assert res is ctype[m.group(1)] and args == want


def test_c_envelope_returns_invalid_argument():
    lib = _lib_loaded()
    p = _lib.c_void_p(1 << 20)
    fwd = lib.rb200_logits_topk_logprob_entropy_fwd
    for k in (0, -1, 320, 321):  # 1 <= top_k < V
        assert fwd(p, 1, p, 4, 4, 0, 320, 320, 44, 300, 1.0, k, p, p, p, p, None) == -3, k
    assert fwd(p, 1, p, 4, 4, 0, 320, 320, 44, 300, 1.0, 8, p, p, p, None, None) == -1  # threshold required
    assert fwd(p, 1, p, 4, 4, 0, 320, 320, 44, 300, 1.0, 8, None, p, p, p, None) == -1  # logprob required
    assert fwd(p, 2, p, 4, 4, 0, 320, 320, 44, 300, 1.0, 8, p, p, p, p, None) == -5  # dtype
    assert fwd(p, 1, p, 4, 4, 0, 320, 320, 300, 44, 1.0, 8, p, p, p, p, None) == -2  # empty window
    bwd = lib.rb200_logits_topk_logprob_entropy_bwd
    assert bwd(p, 1, p, 4, 4, 0, 320, 320, 44, 300, 1.0, None, p, p, p, p, p, 0, 320, None) == -1
    assert bwd(p, 1, p, 4, 4, 0, 320, 320, 44, 300, 1.0, p, p, None, p, p, p, 0, 320, None) == -1  # g_H without H


def test_lmhead_topk_envelope_returns_invalid_argument():
    lib = _lib_loaded()
    p = _lib.c_void_p(1 << 20)
    ws = lib.rb200_lmhead_topk_workspace_bytes
    assert ws(256, 256, 1000, 320, 44, 300, 0, 0) == -1  # H % 64 != 0
    assert ws(256, 256, 64, 320, 44, 300, 0, 0) > 0
    one_tile = 128 * 320 * 4
    assert ws(4096, 4096, 64, 320, 44, 300, 128, 0) >= one_tile
    fwd = lib.rb200_lmhead_topk_logprob_entropy_fwd
    big = 1 << 30
    for k in (0, -1, 320, 400):  # 1 <= top_k < V
        assert fwd(p, p, p, 256, 256, 256 * 64, 64, 64, 320, 44, 300, 1.0, k, p, p, p, p, p, big, None) == -3, k
    assert fwd(p, p, p, 256, 256, 256 * 96, 96, 96, 320, 44, 300, 1.0, 8, p, p, p, p, p, big, None) == -2  # H
    assert fwd(p, p, p, 256, 256, 256 * 64, 64, 64, 320, 44, 300, 1.0, 8, p, p, p, p, p, one_tile - 16, None) == -3
    assert fwd(p, p, p, 256, 256, 256 * 64, 64, 64, 320, 44, 300, 1.0, 8, p, p, p, None, p, big, None) == -1
    bwd = lib.rb200_lmhead_topk_logprob_entropy_bwd
    assert bwd(p, p, p, 256, 256, 256 * 64, 64, 64, 320, 44, 300, 1.0, None, p, p, p, p, p, p, p, big, None) == -1
    assert bwd(p, p, p, 256, 256, 256 * 64, 64, 64, 320, 44, 300, 1.0, p, p, p, p, p, p, p, p, 16, None) == -3


def test_lmhead_topk_kernels_not_serialised_and_no_spills(tmp_path):
    cmd = [_nvcc(), *build.NVCC_FLAGS, "-Xptxas", "-v", "-c", os.path.join(build.CSRC, "lmhead_topk.cu"), "-o",
           str(tmp_path / "x.o")]
    out = subprocess.run(cmd, capture_output=True, text=True)
    log = out.stdout + out.stderr
    assert out.returncode == 0, log
    assert "C7512" not in log and "C7514" not in log and "serialized" not in log, log
    entries = re.findall(r"Compiling entry function '([^']+)'.*?(\d+) bytes spill stores, (\d+) bytes spill loads", log,
                         flags=re.S)
    assert len(entries) == 2 and all(e[1:] == ("0", "0") for e in entries), log


def _nvcc():
    try:
        return build._nvcc()
    except RuntimeError:
        pytest.skip("nvcc not found")


def test_new_kernels_do_not_spill(tmp_path):
    cmd = [_nvcc(), *build.NVCC_FLAGS, "-Xptxas", "-v", "-c", os.path.join(build.CSRC, "topk.cu"), "-o",
           str(tmp_path / "x.o")]
    out = subprocess.run(cmd, capture_output=True, text=True)
    log = out.stdout + out.stderr
    assert out.returncode == 0, log
    entries = re.findall(r"Compiling entry function '([^']+)'.*?(\d+) bytes spill stores, (\d+) bytes spill loads", log,
                         flags=re.S)
    assert len(entries) == 4 and all(e[1:] == ("0", "0") for e in entries), log


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


def sass_digests(tmp_path):
    """{object: {kernel: sha256 of its SASS}} for the objects whose SASS this change keeps."""
    out = {}
    for obj in ("logits.o", "lmhead.o"):
        parts = re.split(r"^\s*Function : (\S+)\s*$", _sass(tmp_path, obj), flags=re.M)
        out[obj] = {parts[i]: hashlib.sha256(parts[i + 1].encode()).hexdigest() for i in range(1, len(parts), 2)}
    return out


def test_existing_objects_keep_their_sass(tmp_path):
    assert sass_digests(tmp_path) == json.load(open(DIGESTS))
