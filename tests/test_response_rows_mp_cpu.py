"""The Megatron SP / CP response-rows plan on the CPU: the oracle's ownership is the reference's preprocess_packed_seqs
chunking (tests/golden/golden_response_rows_mp.npz), the host plan's counts are the oracle's on every rank, at tp = cp
= 1 the plan reads the rows and targets megatron_thd reads, constructor errors, the ctypes signatures match the header,
the new kernels do not spill, and the objects the op runs on keep the parent's SASS.  No GPU."""
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

import response_rows_mp_oracle as O
import response_rows_oracle as O1
from rlinf_b200 import build
from rlinf_b200 import response_rows as RR

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "golden_response_rows_mp.npz")
DIGESTS = os.path.join(HERE, "golden", "sass_digests_response_rows_mp.json")


def _batch(tp, cp, fixed=None):
    p = torch.tensor([7, 30, 3, 12, 1, 20])
    r = torch.tensor([48, 0, 29, 17, 40, 5])
    n = p + r
    align = 2 * cp * tp if cp > 1 else tp
    N = n + (align - n % align) % align
    cu = torch.cat([torch.zeros(1, dtype=torch.int64), torch.cumsum(N, 0)])
    return cu, n, r, (int(cu[-1]) if fixed is None else fixed) // cp


@pytest.fixture(scope="module")
def g():
    return {k: torch.from_numpy(v) for k, v in np.load(GOLDEN, allow_pickle=False).items()}


def _cases(g):
    return sorted(k[:-len("_meta")] for k in g if k.endswith("_meta"))


def test_fixture_covers_the_grids(g):
    grids = {tuple(int(x) for x in g[f"{k}_meta"][:3]) for k in _cases(g)}
    assert grids == {(2, 1, 1), (1, 2, 0), (2, 2, 1)}


def test_fixture_has_ranks_without_prediction_rows(g):
    """The sparse batch leaves a whole CP rank (in both CP grids) and a TP shard (in every SP grid) without a
    prediction row: those ranks still take part in every collective."""
    empty_cp, empty_tp = set(), set()
    for key in _cases(g):
        tp, cp, sp, L, bsz, T_c, _ = (int(x) for x in g[f"{key}_meta"])
        per = O.prediction_rows(g[f"{key}_cu"], g[f"{key}_n"], g[f"{key}_r"], cp)
        Ts = T_c // tp
        if any(not rows for rows in per):
            empty_cp.add((tp, cp))
        if sp and any(not any(k * Ts <= t < (k + 1) * Ts for t, _, _ in rows) for rows in per for k in range(tp)):
            empty_tp.add((tp, cp))
    assert empty_cp == {(1, 2), (2, 2)} and empty_tp == {(2, 1), (2, 2)}


def test_reference_inference_output_is_the_training_columns_and_zeros(g):
    """The inference path (`log_probs[:, -L-1:-1] * response_mask`) holds the training output's response columns and
    zeros past r_b - exactly what the op returns, in both paths."""
    for key in _cases(g):
        L = int(g[f"{key}_meta"][3])
        valid = torch.arange(L)[None] < g[f"{key}_r"][:, None]
        infer, train = g[f"{key}_infer_logprobs"], g[f"{key}_logprobs"]
        assert torch.equal(infer[valid], train[valid]) and not infer[~valid].any(), key


def test_oracle_ownership_is_the_references(g):
    """preprocess_packed_seqs applied to position ids on each rank puts position p of sequence b exactly where the
    oracle says (under SP, at the rank's shard of its CP rank's stream)."""
    for key in _cases(g):
        tp, cp, sp, L, bsz, T_c, _ = (int(x) for x in g[f"{key}_meta"])
        cu, n = g[f"{key}_cu"], g[f"{key}_n"]
        own = O.owner(cu, n, cp)
        Ts = T_c // tp if sp else T_c
        for c in range(cp):
            for k in range(tp):
                pos = g[f"{key}_c{c}_k{k}_positions"]  # the shard of the stream of position ids (+1, 0 = padding)
                want = torch.zeros(Ts, dtype=torch.int64)
                for (b, p), (cc, t) in own.items():
                    if cc == c and (not sp or k * Ts <= t < (k + 1) * Ts):
                        want[t - (k * Ts if sp else 0)] = p + 1
                assert torch.equal(pos.long(), want), (key, c, k)


def test_oracle_reproduces_reference_forward(g):
    """Per-row values of the reference's vocabulary-parallel entropy / log-probs on each CP rank's stream, placed in
    cells by the oracle, are the reference's response columns bit for bit."""
    W = g["W"]
    for key in _cases(g):
        tp, cp, sp, L, bsz, T_c, _ = (int(x) for x in g[f"{key}_meta"])
        cu, n, r = g[f"{key}_cu"], g[f"{key}_n"], g[f"{key}_r"]
        resp = g[f"{key}_responses"]
        per = O.prediction_rows(cu, n, r, cp)
        lp = torch.zeros(bsz, L)
        for c in range(cp):
            parts = [g[f"{key}_c{c}_k{k}_hidden"] for k in range(tp)]
            h = torch.cat(parts) if sp else parts[0]
            tg = torch.zeros(T_c, dtype=torch.int64)
            for t, b, j in per[c]:
                tg[t] = resp[b, j]
            vals, _ = O1.megatron_row_values(h[None], W, tg, float(g["temperature"]), tp, tg)
            for t, b, j in per[c]:
                lp[b, j] = vals[t]
        valid = torch.arange(L)[None] < r[:, None]
        assert torch.equal(lp[valid], g[f"{key}_logprobs"][valid]), key


def test_reference_gradient_lies_on_owned_prediction_rows(g):
    """The reference's dX of Σ g·log_probs[:, -L-1:-1] is non-zero exactly on the prediction rows a rank holds: other
    CP ranks' cells arrive detached."""
    for key in _cases(g):
        tp, cp, sp, L, bsz, T_c, _ = (int(x) for x in g[f"{key}_meta"])
        per = O.prediction_rows(g[f"{key}_cu"], g[f"{key}_n"], g[f"{key}_r"], cp)
        Ts = T_c // tp if sp else T_c
        for c in range(cp):
            rows = {t for t, _, _ in per[c]}
            for k in range(tp):
                nz = g[f"{key}_c{c}_k{k}_grad"].reshape(Ts, -1).ne(0).any(-1)
                want = torch.tensor([(x + (k * Ts if sp else 0)) in rows for x in range(Ts)])
                assert torch.equal(nz, want), (key, c, k)


@pytest.mark.parametrize("tp, cp, sp", [(2, 1, True), (4, 1, True), (8, 1, True), (1, 2, False), (2, 2, True),
                                        (2, 4, True), (2, 4, False), (2, 2, False)])
@pytest.mark.parametrize("fixed", [None, 1024])
def test_host_counts_match_oracle(tp, cp, sp, fixed):
    cu, n, r, T_c = _batch(tp, cp, fixed)
    plan = RR.megatron_parallel(cu, n, r, response_len=48, tp_size=tp, cp_size=cp, sequence_parallel=sp)
    assert not plan.on_device
    m = O.rank_maps(cu, n, r, torch.zeros(6, 48, dtype=torch.int64).tolist(), 48, tp, cp, sp, T_c, 0, 0)
    assert plan.counts(T_c) == m["counts"]
    assert sum(sum(x) if sp else x[0] for x in m["counts"]) == int(r.sum())


def test_tp1_cp1_reads_what_megatron_thd_reads():
    cu, n, r, T = _batch(1, 1)
    thd = RR.megatron_thd(cu, n, r, response_len=48)
    m = O.rank_maps(cu, n, r, torch.zeros(6, 48, dtype=torch.int64).tolist(), 48, 1, 1, False, T, 0, 0)
    a = O1.first_rows("megatron_thd", r, cu_seqlens_padded=cu, seq_lengths=n)
    rows, _ = O1.rows_and_targets(a, r, torch.zeros(T + 1, dtype=torch.int64), 0)
    assert m["rows"] == rows and thd.num_rows == m["R"]
    assert m["cells"] == [b * 48 + j for b in range(6) for j in range(int(r[b]))]


@pytest.mark.parametrize("make, msg", [
    (lambda: RR.megatron_parallel([0, 6, 16], [6, 4], [2, 1], response_len=4, cp_size=2, tp_size=2), "multiple of 2"),
    (lambda: RR.megatron_parallel([4, 12, 20], [8, 4], [2, 1], response_len=4, cp_size=4), "multiple of 2"),
    (lambda: RR.megatron_parallel([0, 4, 8], [6, 3], [2, 1], response_len=4), "overlap"),
    (lambda: RR.megatron_parallel([0, 8, 16], [8, 4], [2, 4], response_len=4), "no prompt token"),
    (lambda: RR.megatron_parallel([0, 8, 16], [8, 4], [5, 1], response_len=4), r"outside \[0, response_len\]"),
    (lambda: RR.megatron_parallel([-2, 8, 16], [8, 4], [2, 1], response_len=4), r"outside \[0, T\)"),
    (lambda: RR.megatron_parallel([0, 8], [8, 4], [2, 1], response_len=4), "cu_seqlens_padded"),
    (lambda: RR.megatron_parallel([0, 8, 16], [8, 4], [2, 1], response_len=4, tp_size=8, cp_size=16), "<= 64"),
])
def test_constructor_errors(make, msg):
    with pytest.raises(ValueError, match=msg):
        make()


def test_shard_too_small_is_checked_before_any_launch():
    plan = RR.megatron_parallel([0, 8, 16], [8, 4], [2, 1], response_len=4, tp_size=2, cp_size=2,
                                sequence_parallel=True)
    with pytest.raises(ValueError, match="too few rows"):
        plan.index(torch.zeros(2, 4, dtype=torch.int64), 3, 0, 0)  # T_c = 6 < 16 / 2
    with pytest.raises(ValueError, match="outside the plan's"):
        plan.index(torch.zeros(2, 4, dtype=torch.int64), 4, 2, 0)


@pytest.mark.parametrize("name", ["rb200_response_rows_mp_plan", "rb200_response_rows_mp_pack_grad"])
def test_ctypes_signature_matches_header(name):
    from rlinf_b200 import _lib

    src = open(os.path.join(os.path.dirname(HERE), "include", "rlinf_b200.h")).read()
    decl = re.search(rf"int {name}\((.*?)\);", src, flags=re.S).group(1)
    params = [p.strip() for p in decl.split(",")]
    ctype = {"int": _lib.c_int, "int64_t": _lib.c_int64}
    want = [_lib.c_void_p if ("*" in p or p.startswith("rb200_stream_t")) else ctype[p.rsplit(" ", 1)[0]]
            for p in params]
    res, args = _lib.SIGNATURES[name]
    assert res is _lib.c_int and args == want


def _nvcc():
    try:
        return build._nvcc()
    except RuntimeError:
        pytest.skip("nvcc not found")


def test_new_kernels_do_not_spill(tmp_path):
    cmd = [_nvcc(), *build.NVCC_FLAGS, "-Xptxas", "-v", "-c", os.path.join(build.CSRC, "response_rows_mp.cu"), "-o",
           str(tmp_path / "response_rows_mp.o")]
    out = subprocess.run(cmd, capture_output=True, text=True)
    log = out.stdout + out.stderr
    assert out.returncode == 0, log
    entries = re.findall(r"Compiling entry function '([^']+)'.*?(\d+) bytes spill stores, (\d+) bytes spill loads", log,
                         flags=re.S)
    assert len(entries) == 2 and all(e[1:] == ("0", "0") for e in entries), log


def normalised_sass(text: str) -> str:
    text = re.sub(r"_GLOBAL__N__[0-9a-f]+_\d+_\w+?_cu_[0-9a-f]+", "_GLOBAL__N_", text)
    return "\n".join(line for line in text.splitlines() if not line.strip().startswith("identifier"))


@pytest.mark.parametrize("obj", ["gather.o", "lmhead.o", "logits.o", "vocab_parallel.o", "response_rows.o"])
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
