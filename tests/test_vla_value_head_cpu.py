"""The OpenVLA value head without a GPU: the fp64 oracle (tests/vla_value_head_oracle.py) against the reference fixture
(tests/golden/golden_vla_value_head.npz), the ValueError envelope of ops.vla_value_head, the C invalid-argument status,
the ctypes signatures against the header, no spills and no serialised wgmma in csrc/vla_value_head.cu, and the SASS of
the existing objects that include the same shared header as at the parent commit
(tests/golden/sass_digests_vla_value_head.json)."""
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

import vla_value_head_oracle as OR
from rlinf_b200 import _lib, build

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_golden_vla_value_head as G  # noqa: E402

DIGESTS = os.path.join(HERE, "golden", "sass_digests_vla_value_head.json")
NAMES = ("v", "dx", "dw0", "db0", "dw1", "db1", "dw2")


@pytest.fixture(scope="module")
def fix():
    return dict(np.load(G.OUT))


def _oracle(H, O, bf16):
    inp = G.make_inputs(H, O)
    v, saved = OR.forward(inp["x"], inp["w0"], inp["b0"], inp["w1"], inp["b1"], inp["w2"], bf16=bf16)
    out = OR.backward(inp["x"], inp["w0"], inp["w1"], inp["w2"], saved, inp["gv"], bf16=bf16)
    out["v"], out["dw0"], out["dw1"] = v, out["dw0"][G.W0_ROWS], out["dw1"][G.W1_ROWS]
    return out


@pytest.mark.parametrize("H,O", [(H, O) for H in G.HS for O in G.OS])
def test_oracle_reproduces_bf16_fixture(fix, H, O):
    """Every output is rounded to bf16 once from a sum the module forms in fp32 and the oracle in fp64, so the two can
    round to neighbouring bf16 values: an element may differ by one ulp (2^-7 of its magnitude at most), and an
    intermediate rounded the other way moves what is computed from it by at most one of its roundings (2^-8) of that
    output's largest element.  Almost all elements are identical."""
    o = _oracle(H, O, True)
    for k in NAMES:
        ref = G.from_bits(fix[f"{G.case_name(H, O, 'bf16')}_{k}"]).double()
        d = (o[k] - ref).abs()
        assert (d <= 2 ** -7 * ref.abs() + 2 ** -8 * ref.abs().max()).all(), k
        assert (d == 0).double().mean() >= 0.97, k


@pytest.mark.parametrize("H,O", [(H, O) for H in G.HS for O in G.OS])
def test_oracle_reproduces_fp32_fixture(fix, H, O):
    """Unrounded fp64 against the fp32 module: fp32 sums of at most 512 products, relative error below 1e-5 of the
    largest element."""
    o = _oracle(H, O, False)
    for k in NAMES:
        ref = torch.from_numpy(fix[f"{G.case_name(H, O, 'fp32')}_{k}"]).double()
        assert (o[k] - ref).abs().max() <= 1e-5 * ref.abs().max(), k


def _args(N=3, H=128, O=8, dtype=torch.bfloat16):
    return [torch.zeros(N, H, dtype=dtype), torch.zeros(512, H, dtype=dtype), torch.zeros(512, dtype=dtype),
            torch.zeros(128, 512, dtype=dtype), torch.zeros(128, dtype=dtype), torch.zeros(O, 128, dtype=dtype)]


def test_value_error_envelope():
    from rlinf_b200 import ops

    f = ops.vla_value_head
    with pytest.raises(ValueError, match="activation"):
        f(*_args(), activation="relu")
    with pytest.raises(ValueError, match="b2"):
        f(*_args(), b2=torch.zeros(8, dtype=torch.bfloat16))
    for i, name in enumerate(("hidden", "w0", "b0", "w1", "b1", "w2")):
        a = _args()
        a[i] = a[i].float()
        with pytest.raises(ValueError, match=f"{name} must be bfloat16"):
            f(*a)
    for i, name, bad in ((1, "w0", (256, 128)), (2, "b0", (256,)), (3, "w1", (64, 512)), (3, "w1", (128, 256)),
                         (4, "b1", (64,)), (5, "w2", (8, 64))):
        a = _args()
        a[i] = torch.zeros(bad, dtype=torch.bfloat16)
        with pytest.raises(ValueError, match=name):
            f(*a)
    for O in (33, 0):
        with pytest.raises(ValueError, match="w2"):
            f(*_args(O=O))
    for H in (96, 32, 8256):
        with pytest.raises(ValueError, match="hidden"):
            f(*_args(H=H))
    with pytest.raises(ValueError, match="hidden must be \\[N, H\\]"):
        a = _args()
        a[0] = torch.zeros(2, 3, 128, dtype=torch.bfloat16)
        f(*a)
    with pytest.raises(ValueError, match="hidden must be a CUDA tensor"):
        f(*_args())
    a = _args()
    a[1] = torch.zeros(512, 128, dtype=torch.bfloat16, device="meta")
    with pytest.raises(ValueError, match="w0 is on meta"):
        f(*a)


def _lib_loaded():
    if not os.path.exists(_lib.LIB_PATH):
        build.build()
    return _lib.load()


def test_c_envelope_returns_invalid_argument():
    lib = _lib_loaded()
    p = _lib.c_void_p(1 << 20)
    fwd, bwd, ws = lib.rb200_vla_value_head_fwd, lib.rb200_vla_value_head_bwd, lib.rb200_vla_value_head_workspace_bytes
    assert ws(40, 4096) == 40 * (512 + 128 + 512) * 2 and ws(0, 64) == 0
    assert ws(-1, 4096) == -1 and ws(40, 4100) == -1 and ws(40, 8256) == -1 and ws(40, 0) == -1

    def f(x=p, rs=4096, n=40, H=4096, O=8, z0=p, v=p, w1=p):
        return fwd(x, rs, n, H, p, p, w1, p, p, O, z0, None, v, None)

    assert f(x=None) == -1 and f(z0=None) == -1 and f(v=None) == -1
    assert f(n=-1) == -2 and f(H=4160 - 32) == -2 and f(O=0) == -2 and f(O=33) == -2 and f(rs=4032) == -2
    assert f(rs=4100) == -4 and f(x=_lib.c_void_p((1 << 20) + 8)) == -4 and f(w1=_lib.c_void_p((1 << 20) + 2)) == -4
    assert f(n=0) == 0  # nothing to do, nothing launched
    wsb = ws(40, 4096)

    def b(x=p, n=40, H=4096, O=8, dx=p, dw0=p, wsp=p, wsb=wsb, w0=p, gv=p):
        return bwd(x, 4096, n, H, w0, p, p, O, p, p, gv, dx, dw0, p, p, p, p, wsp, wsb, None)

    assert bwd(p, 4096, 40, 4096, p, p, p, 8, p, p, p, *([None] * 6), p, wsb, None) == -1  # no output at all
    assert b(gv=None) == -1 and b(wsp=None) == -1 and b(w0=None) == -1 and b(x=None) == -1
    assert b(n=-1) == -2 and b(O=33) == -2 and b(H=100) == -2
    assert b(wsb=wsb - 1) == -3
    assert b(dx=_lib.c_void_p((1 << 20) + 4)) == -4


@pytest.mark.parametrize("name", ["rb200_vla_value_head_workspace_bytes", "rb200_vla_value_head_fwd",
                                  "rb200_vla_value_head_bwd"])
def test_ctypes_signature_matches_header(name):
    src = open(os.path.join(ROOT, "include", "rlinf_b200.h")).read()
    m = re.search(rf"(int|int64_t) {name}\((.*?)\);", src, flags=re.S)
    ctype = {"int": _lib.c_int, "int64_t": _lib.c_int64}
    want = []
    for q in (q.strip() for q in m.group(2).split(",")):
        want.append(_lib.c_void_p if "*" in q or q.startswith("rb200_stream_t") else ctype[q.rsplit(" ", 1)[0]])
    res, args = _lib.SIGNATURES[name]
    assert res is ctype[m.group(1)] and args == want


def _nvcc():
    try:
        return build._nvcc()
    except RuntimeError:
        pytest.skip("nvcc not found")


def test_kernels_do_not_spill_and_use_no_serialised_wgmma(tmp_path):
    cmd = [_nvcc(), *build.NVCC_FLAGS, "-Xptxas", "-v", "-c", os.path.join(build.CSRC, "vla_value_head.cu"), "-o",
           str(tmp_path / "x.o")]
    out = subprocess.run(cmd, capture_output=True, text=True)
    log = out.stdout + out.stderr
    assert out.returncode == 0, log
    entries = re.findall(r"Compiling entry function '([^']+)'.*?(\d+) bytes spill stores, (\d+) bytes spill loads", log,
                         flags=re.S)
    # l0_fwd, tail_fwd, tail_bwd, small_grads and the two gemm_kernel instances
    assert len(entries) == 6 and all(e[1:] == ("0", "0") for e in entries), log
    assert "C7512" not in log and "C7514" not in log and "C7510" not in log and "serialized" not in log, log


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


def sass_digests(tmp_path, objs):
    out = {}
    for obj in objs:
        parts = re.split(r"^\s*Function : (\S+)\s*$", _sass(tmp_path, obj), flags=re.M)
        out[obj] = {parts[i]: hashlib.sha256(parts[i + 1].encode()).hexdigest() for i in range(1, len(parts), 2)}
    return out


def test_existing_objects_keep_their_sass(tmp_path):
    """The new file adds a source and a header section only: the objects built from common.cuh and the header
    (the reasoning critic's value head, the PPO and token losses, the logits, top-k and LM-head kernels) keep their
    SASS."""
    want = json.load(open(DIGESTS))
    assert sass_digests(tmp_path, sorted(want)) == want
