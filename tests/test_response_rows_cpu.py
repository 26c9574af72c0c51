"""Response-rows plans on the CPU: the oracle reproduces the reference's layout code (tests/golden/
golden_response_rows.npz, tests/golden/make_golden_response_rows.py) bit for bit on every response column, the
reference's masked columns hold what DESIGN.md §2 says, each constructor's a_b / R / errors match, the plan kernel's
ctypes signature matches the header, the kernel does not spill, and the four objects the op runs on compile to the
parent's SASS.  No GPU."""
from __future__ import annotations

import hashlib
import json
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

import response_rows_oracle as O
from rlinf_b200 import build
from rlinf_b200 import response_rows as RR

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "golden_response_rows.npz")
DIGESTS = os.path.join(HERE, "golden", "sass_digests_response_rows.json")


@pytest.fixture(scope="module")
def g():
    return {k: torch.from_numpy(v) for k, v in np.load(GOLDEN, allow_pickle=False).items()}


def _meta(g):
    V, H, P, L, S, PAD = (int(x) for x in g["meta"])
    return V, H, P, L, S, PAD


def _plan_of(g, case):
    _, _, MP, L, S, _ = _meta(g)
    r, p = g["response_lengths"], g["prompt_lengths"]
    if case == "fsdp_padded":
        return RR.padded(len(r), S, L, r), O.first_rows("padded", r, S=S, L=L), 0
    if case.startswith("fsdp_packed"):
        return (RR.fsdp_packed(p, r, MP, response_len=L), O.first_rows("fsdp_packed", r, prompt_lengths=p), 1)
    cu = g[f"{case}_train_cu"]
    return (RR.megatron_thd(cu, g["seq_lengths"], r, response_len=L),
            O.first_rows("megatron_thd", r, cu_seqlens_padded=cu, seq_lengths=g["seq_lengths"]), 0)


FSDP = ["fsdp_padded", "fsdp_packed_var", "fsdp_packed_fixed"]
MEGATRON = [f"megatron_tp{P}_{v}" for P in (1, 2) for v in ("var", "fixed")]


def _row_values(g, case):
    k = case if case in FSDP else f"{case}_train"
    h, tok = g[f"{k}_hidden"], g[f"{k}_tokens"]
    if case in FSDP:
        return O.fsdp_row_values(h, g["W"], tok, float(g["temperature"]))
    P = int(case.split("_")[1][2:])
    return O.megatron_row_values(h, g["W"], tok, float(g["temperature"]), P)


def _ref(g, case, what):
    if case in FSDP:
        return g[f"{case}_{what}"]
    return g[f"{case}_train_{what}"]


@pytest.mark.parametrize("case", FSDP + MEGATRON)
def test_oracle_reproduces_reference_response_columns(g, case):
    _, _, _, L, _, _ = _meta(g)
    r = g["response_lengths"]
    plan, a, shift = _plan_of(g, case)
    assert plan.first_rows.tolist() == a
    assert plan.num_rows == O.num_rows(r, shift)
    lp_rows, ent_rows = _row_values(g, case)
    lp, ent = O.to_cells(lp_rows, a, r, L), O.to_cells(ent_rows, a, r, L, shift)
    valid = torch.arange(L)[None] < r[:, None]
    ref_lp, ref_ent = _ref(g, case, "logprobs"), _ref(g, case, "entropy")
    assert torch.equal(lp[valid], ref_lp[valid])
    assert torch.equal(ent[valid], ref_ent[valid])
    assert not lp[~valid].any() and not ent[~valid].any()


def test_reference_masked_columns(g):
    """What the reference leaves at j >= r_b (this op writes zeros there; DESIGN.md §2)."""
    _, _, _, L, _, PAD = _meta(g)
    r = g["response_lengths"]
    masked = torch.arange(L)[None] >= r[:, None]
    # FSDP packed: zeros, both outputs
    for case in ("fsdp_packed_var", "fsdp_packed_fixed"):
        assert not g[f"{case}_logprobs"][masked].any() and not g[f"{case}_entropy"][masked].any()
    # FSDP without packing: every column holds the row's values, so padded columns hold log p(pad)
    _, a, _ = _plan_of(g, "fsdp_padded")
    lp_rows, ent_rows = _row_values(g, "fsdp_padded")
    full = torch.full_like(r, L)
    assert torch.equal(g["fsdp_padded_logprobs"], O.to_cells(lp_rows, a, full, L))
    assert torch.equal(g["fsdp_padded_entropy"], O.to_cells(ent_rows, a, full, L))
    tok = g["fsdp_padded_tokens"].view(len(r), -1)[:, -L:]
    assert (tok[masked] == PAD).all()
    for case in MEGATRON:
        # inference: multiplied by the response mask -> zeros
        assert not g[f"{case}_infer_logprobs"][masked].any()
        # training forward: column r_b (when r_b < L) holds log p(pad | last token) and its entropy, the rest 0
        _, a, _ = _plan_of(g, case)
        h, tok = g[f"{case}_train_hidden"], g[f"{case}_train_tokens"]
        lp_rows, ent_rows = O.megatron_row_values(h, g["W"], tok, float(g["temperature"]), int(case[11]),
                                                  torch.full_like(tok, PAD))
        lp, ent = g[f"{case}_train_logprobs"], g[f"{case}_train_entropy"]
        for b in range(len(r)):
            rb = int(r[b])
            if rb < L:
                assert lp[b, rb] == lp_rows[a[b] - 1 + rb] and ent[b, rb] == ent_rows[a[b] - 1 + rb]
                assert not lp[b, rb + 1:].any() and not ent[b, rb + 1:].any()


def test_fsdp_packed_entropy_is_one_row_later(g):
    """The packed branch's entropy at column j is the entropy of the row at token j, not of the row predicting it."""
    _, _, _, L, _, _ = _meta(g)
    r = g["response_lengths"]
    _, a, _ = _plan_of(g, "fsdp_packed_var")
    _, ent_rows = _row_values(g, "fsdp_packed_var")
    valid = torch.arange(L)[None] < r[:, None]
    aligned = O.to_cells(ent_rows, a, r, L, 0)
    assert not torch.equal(aligned[valid], g["fsdp_packed_var_entropy"][valid])
    assert torch.equal(O.to_cells(ent_rows, a, r, L, 1)[valid], g["fsdp_packed_var_entropy"][valid])


def test_constructors_first_rows_and_counts():
    p, r = [3, 6, 1], [5, 0, 8]
    plan = RR.padded(3, 14, 8, r)
    assert plan.first_rows.tolist() == [6, 20, 34] and plan.num_rows == 13 and plan.entropy_shift == 0
    plan = RR.fsdp_packed(p, r, 6, response_len=8)
    assert plan.first_rows.tolist() == [3, 14, 15] and plan.num_rows == 15 and plan.entropy_shift == 1
    plan = RR.megatron_thd([0, 8, 14, 24], [8, 6, 9], r, response_len=8)
    assert plan.first_rows.tolist() == [3, 14, 15] and plan.num_rows == 13
    assert plan.end_row == 23
    assert not plan.on_device


@pytest.mark.parametrize("make, msg", [
    (lambda: RR.megatron_thd([0, 4, 8], [6, 3], [2, 1], response_len=4), "overlap"),
    (lambda: RR.fsdp_packed([3, 0], [2, 2], 6, response_len=4), "no prompt token"),
    (lambda: RR.megatron_thd([0, 8, 16], [8, 4], [2, 4], response_len=4), "no prompt token"),
    (lambda: RR.padded(2, 8, 8, [1, 1]), "no prompt token"),
    (lambda: RR.padded(2, 12, 8, [9, 1]), r"outside \[0, response_len\]"),
    (lambda: RR.fsdp_packed([3, 2], [-1, 2], 6, response_len=4), r"outside \[0, response_len\]"),
    (lambda: RR.megatron_thd([-2, 8, 16], [8, 4], [2, 1], response_len=4), r"outside \[0, T\)"),
    (lambda: RR.megatron_thd([0, 8, 16], [8, 4], [2, 1], response_len=4, cp_size=2), "context parallelism"),
    (lambda: RR.fsdp_packed([7, 2], [1, 2], 6, response_len=4), "max_prompt_len"),
    (lambda: RR.megatron_thd([0, 8], [8, 4], [2, 1], response_len=4), "cu_seqlens_padded"),
])
def test_constructor_errors(make, msg):
    with pytest.raises(ValueError, match=msg):
        make()


def test_ranges_past_T_are_checked_against_the_hidden_rows():
    plan = RR.fsdp_packed([3, 2], [2, 2], 6, response_len=4)
    assert plan.end_row == 9
    with pytest.raises(ValueError, match=r"outside \[0, T\)"):
        plan.index(torch.zeros(8, dtype=torch.int64), 8)
    with pytest.raises(ValueError, match="needs T = 24"):
        RR.padded(2, 12, 8, [1, 1]).index(torch.zeros(20, dtype=torch.int64), 20)


def test_ctypes_signature_matches_header():
    from rlinf_b200 import _lib

    src = open(os.path.join(os.path.dirname(HERE), "include", "rlinf_b200.h")).read()
    decl = re.search(r"int rb200_response_rows_plan\((.*?)\);", src, flags=re.S).group(1)
    params = [p.strip() for p in decl.split(",")]
    ctype = {"int": _lib.c_int, "int64_t": _lib.c_int64}
    want = [_lib.c_void_p if ("*" in p or p.startswith("rb200_stream_t")) else ctype[p.rsplit(" ", 1)[0]]
            for p in params]
    res, args = _lib.SIGNATURES["rb200_response_rows_plan"]
    assert res is _lib.c_int and args == want


def _nvcc():
    try:
        return build._nvcc()
    except RuntimeError:
        pytest.skip("nvcc not found")


def test_plan_kernel_does_not_spill(tmp_path):
    cmd = [_nvcc(), *build.NVCC_FLAGS, "-Xptxas", "-v", "-c", os.path.join(build.CSRC, "response_rows.cu"), "-o",
           str(tmp_path / "response_rows.o")]
    out = subprocess.run(cmd, capture_output=True, text=True)
    log = out.stdout + out.stderr
    assert out.returncode == 0, log
    entries = re.findall(r"Compiling entry function '([^']+)'.*?(\d+) bytes spill stores, (\d+) bytes spill loads", log,
                         flags=re.S)
    assert len(entries) == 1 and entries[0][1:] == ("0", "0"), log


def normalised_sass(text: str) -> str:
    text = re.sub(r"_GLOBAL__N__[0-9a-f]+_\d+_\w+?_cu_[0-9a-f]+", "_GLOBAL__N_", text)
    return "\n".join(line for line in text.splitlines() if not line.strip().startswith("identifier"))


@pytest.mark.parametrize("obj", ["lmhead.o", "logits.o", "vocab_parallel.o", "gather.o"])
def test_existing_objects_keep_their_sass(tmp_path, obj):
    nvcc = _nvcc()
    cuobjdump = shutil.which("cuobjdump") or os.path.join(os.path.dirname(nvcc), "cuobjdump")
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not found")
    o = tmp_path / obj
    subprocess.run([nvcc, *build.NVCC_FLAGS, "-c", os.path.join(build.CSRC, obj[:-2] + ".cu"), "-o", str(o)],
                   check=True, capture_output=True)
    sass = subprocess.run([cuobjdump, "-sass", str(o)], check=True, capture_output=True, text=True).stdout
    assert hashlib.sha256(normalised_sass(sass).encode()).hexdigest() == json.load(open(DIGESTS))[obj]
