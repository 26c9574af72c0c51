"""Reasoning step bookkeeping without a GPU: the torch-on-CPU oracle (tests/reasoning_step_oracle.py) against the
reference fixture (tests/golden/golden_reasoning_step.npz: compute_rollout_metrics(_dynamic), the Megatron loss_func
tails and _process_fwd_bwd_outputs over gloo at data-parallel sizes 2 and 4); the ctypes mirrors against the C
compiler's layout of the header; the C envelope; no spills in the new kernels; and the SASS of token_loss.o,
token_critic_loss.o and ppo_loss.o as at the parent commit (tests/golden/sass_digests_reasoning_step.json)."""
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

import reasoning_step_oracle as O
from rlinf_b200 import _lib, build

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_golden_reasoning_step as G  # noqa: E402

FIX = os.path.join(HERE, "golden", "golden_reasoning_step.npz")
DIGESTS = os.path.join(HERE, "golden", "sass_digests_reasoning_step.json")
PS = (2, 4)


@pytest.fixture(scope="module")
def g():
    return dict(np.load(FIX))


def _same(a, b, P=2):
    """Bit for bit at 2 ranks; at 4, where gloo adds the ranks in an order of its own, within one fp32 rounding per
    added rank (2^-23 relative to the result or to 1, whichever is larger, for these O(1) metrics)."""
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    if a.shape != b.shape:
        return False
    tol = 0.0 if P == 2 else (P - 1) * 2.0 ** -23
    return bool(np.all((np.abs(a - b) <= tol * np.maximum(np.abs(b), 1.0)) | (np.isnan(a) & np.isnan(b))))


@pytest.mark.parametrize("P", PS)
@pytest.mark.parametrize("case", ["values", "novalues", "dynamic"])
def test_oracle_reproduces_reference_rollout_metrics(g, P, case):
    batches = [G.rollout_batch(case, r) for r in range(P)]
    want = O.rollout_metrics(batches, G.L, dynamic=case == "dynamic", reference=True)
    for r in range(P):
        keys = list(g[f"P{P}_r{r}_rollout_{case}_keys"])
        assert keys == list(want), (keys, list(want))
        assert _same(g[f"P{P}_r{r}_rollout_{case}_vals"], [want[k] for k in keys], P), (r, case)
    lens = np.concatenate([b["response_lengths"].numpy() for b in batches])
    assert np.array_equal(g[f"P{P}_r0_rollout_{case}_dlens"], lens)


@pytest.mark.parametrize("P", PS)
def test_all_masked_rank_is_the_reference_error(g, P):
    batches = [G.rollout_batch("empty", r) for r in range(P)]
    assert O.rollout_metrics(batches, G.L) == "RuntimeError"
    assert str(g[f"P{P}_r1_rollout_empty_error"]) == "RuntimeError"


def _actor_oracle(P, vts):
    rows = [[] for _ in range(P)]
    res = []
    gvt = None
    if vts:
        gvt = np.float32(sum(float(G.actor_inputs(r, mb, P)[2].sum()) for r in range(P) for mb in range(G.N_MB)))
        gvt = np.float32(torch.tensor(float(gvt), dtype=torch.float32) / G.N_MB)
    final = G.ACTOR_KEYS.index("actor/final_loss")
    for mb in range(G.N_MB):
        per = []
        for r in range(P):
            vals, loss, mask = G.actor_inputs(r, mb, P)
            per.append((vals.numpy(), np.float32(loss), int(mask.sum())))
        out = O.epilogue(per, final, G.ACTOR_KEYS.index("actor/ratio"), 0, G.EARLY_STOP, gvt, G.N_MB)
        res.append(out)
        for r in range(P):
            rows[r].append(out[r][2])
    return res, rows


@pytest.mark.parametrize("P", PS)
@pytest.mark.parametrize("case", list(G.ACTOR_CASES))
def test_oracle_reproduces_reference_actor_tail_and_step(g, P, case):
    res, rows = _actor_oracle(P, G.ACTOR_CASES[case])
    for r in range(P):
        for mb in range(G.N_MB):
            scale, scaled, red = res[mb][r]
            assert _same(g[f"P{P}_r{r}_actor_{case}_mb{mb}_loss"], scaled, P), (r, mb)
            assert _same(g[f"P{P}_r{r}_actor_{case}_mb{mb}_metrics"], red, P), (r, mb)
            assert (scale == 0) == (mb == 1)  # early stop on micro-batch 1 only
        assert list(g[f"P{P}_r{r}_actor_{case}_step_keys"]) == list(G.ACTOR_KEYS)
        assert _same(g[f"P{P}_r{r}_actor_{case}_step_vals"], O.step_finish(rows[r]), P)


@pytest.mark.parametrize("P", PS)
@pytest.mark.parametrize("case", G.CRITIC_CASES)
def test_oracle_reproduces_reference_critic_tail_and_step(g, P, case):
    order = [k for k in G.CRITIC_KEYS if k not in G.EV] + list(G.EV)  # averaged keys first, then the SUM keys
    perm = [G.CRITIC_KEYS.index(k) for k in order]
    final = order.index("critic/final_value_loss")
    rows = [[] for _ in range(P)]
    for mb in range(G.N_MB):
        per = []
        for r in range(P):
            vals, loss = G.critic_inputs(r, mb, case, P)
            per.append((vals.numpy()[perm], np.float32(loss), None))
        out = O.epilogue(per, final, None, len(G.EV))
        for r in range(P):
            scale, scaled, red = out[r]
            assert scale == 1 and _same(g[f"P{P}_r{r}_critic_{case}_mb{mb}_loss"], scaled)
            assert _same(g[f"P{P}_r{r}_critic_{case}_mb{mb}_metrics"][perm], red, P), (r, mb)
            rows[r].append(red)
    for r in range(P):
        keys = list(g[f"P{P}_r{r}_critic_{case}_step_keys"])
        assert keys == ["critic/value_loss", "critic/value_clip_ratio", "critic/final_value_loss",
                        "critic/explained_variance"]
        assert _same(g[f"P{P}_r{r}_critic_{case}_step_vals"], O.step_finish(rows[r], len(G.EV)), P)
    ev = g[f"P{P}_r0_critic_{case}_step_vals"][-1]
    assert np.isnan(ev) == (case != "regular")


STRUCTS = {"rb200_reasoning_record_args": _lib.ReasoningRecordArgs, "rb200_mb_epilogue_args": _lib.MbEpilogueArgs}


def test_struct_layouts_match_header(tmp_path):
    lines = []
    for cname, cls in STRUCTS.items():
        lines.append(f'  printf("{cname} sizeof %zu\\n", sizeof({cname}));')
        lines += [f'  printf("{cname} {f[0]} %zu %zu\\n", offsetof({cname}, {f[0]}), sizeof((({cname}*)0)->{f[0]}));'
                  for f in cls._fields_]
    lines.append('  printf("enums %d %d %d %d %d\\n", RB200_RR_NUM, RB200_RM_NUM, RB200_EPI_MAX_KEYS, '
                 'RB200_RR_VALUES_MEAN, RB200_RM_VERDICT);')
    src = tmp_path / "layout.c"
    src.write_text("#include <stddef.h>\n#include <stdio.h>\n#include \"rlinf_b200.h\"\nint main(void) {\n" +
                   "\n".join(lines) + "\n  return 0;\n}\n")
    cc = os.environ.get("CC") or shutil.which("gcc") or shutil.which("cc")
    assert cc, "no host C compiler (gcc) found"
    exe = tmp_path / "layout"
    subprocess.run([cc, "-std=c99", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    out = subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split("\n")
    got = {tuple(line.split()[:2]): tuple(int(v) for v in line.split()[2:]) for line in out if line}
    assert got[("enums", str(_lib.RR_NUM))] == (_lib.RM_NUM, _lib.EPI_MAX_KEYS, _lib.RR_VALUES_MEAN, _lib.RM_VERDICT)
    for cname, cls in STRUCTS.items():
        assert got[(cname, "sizeof")] == (C.sizeof(cls),)
        for f in cls._fields_:
            d = getattr(cls, f[0])
            assert got[(cname, f[0])] == (d.offset, d.size), (cname, f[0])


def test_metric_slots_match_header():
    src = open(os.path.join(ROOT, "include", "rlinf_b200.h")).read()
    body = re.search(r"enum \{\s*RB200_RM_NUM_SEQ = 0,(.*?)\};", src, flags=re.S).group(1)
    names = ["NUM_SEQ"] + re.findall(r"RB200_RM_(\w+)", body)
    assert names.index("VERDICT") == _lib.RM_VERDICT and names.index("NUM_LENGTHS_MAX") == _lib.RM_NUM_LENGTHS_MAX
    assert sorted(_lib.RM_SLOTS.values()) == list(range(len(_lib.RM_SLOTS)))


@pytest.mark.parametrize("name", ["rb200_reasoning_record_workspace_bytes", "rb200_reasoning_rollout_finish",
                                  "rb200_mask_count_f32", "rb200_step_metrics_finish"])
def test_ctypes_signature_matches_header(name):
    src = open(os.path.join(ROOT, "include", "rlinf_b200.h")).read()
    m = re.search(rf"(int|int64_t) {name}\((.*?)\);", src, flags=re.S)
    params = [q.strip() for q in m.group(2).split(",")]
    ctype = {"int": _lib.c_int, "int64_t": _lib.c_int64, "int32_t": C.c_int32}
    want = [_lib.c_void_p if ("*" in q or q.startswith("rb200_stream_t")) else ctype[q.rsplit(" ", 1)[0]]
            for q in params]
    res, args = _lib.SIGNATURES[name]
    assert res is ctype[m.group(1)] and args == want


def test_c_envelope_returns_invalid_argument():
    if not os.path.exists(_lib.LIB_PATH):
        build.build()
    lib = _lib.load()
    assert lib.rb200_reasoning_record_workspace_bytes(0, 8) == -1
    assert lib.rb200_reasoning_record_workspace_bytes(65536, 8) == -1
    assert lib.rb200_reasoning_record_workspace_bytes(2, 1025) == 2 * 2 * 8 * 8
    a = _lib.ReasoningRecordArgs()
    assert lib.rb200_reasoning_rollout_record(C.byref(a), None) == -1
    assert lib.rb200_reasoning_rollout_finish(None, 1, None, 0, None, None) == -1
    p = C.c_void_p(1 << 20)
    assert lib.rb200_reasoning_rollout_finish(p, 0, None, 0, p, None) == -2
    e = _lib.MbEpilogueArgs()
    assert lib.rb200_mb_epilogue_pack(C.byref(e), None) == -2  # no keys
    e.n_avg, e.final_slot, e.ratio_slot, e.dp, e.num_microbatches, e.n_mb = 2, 0, -1, 1, 1, 1
    assert lib.rb200_mb_epilogue_pack(C.byref(e), None) == -1  # no buffers
    e.mb = 1
    assert lib.rb200_mb_epilogue_apply(C.byref(e), None) == -3  # mb outside [0, n_mb)
    assert lib.rb200_step_metrics_finish(p, 0, 2, 0, p, None) == -2
    assert lib.rb200_mask_count_f32(None, 8, 1, 8, p, 1 << 20, p, None) == -1


def _nvcc():
    try:
        return build._nvcc()
    except RuntimeError:
        pytest.skip("nvcc not found")


def test_new_kernels_do_not_spill(tmp_path):
    cmd = [_nvcc(), *build.NVCC_FLAGS, "-Xptxas", "-v", "-c", os.path.join(build.CSRC, "reasoning_stats.cu"), "-o",
           str(tmp_path / "x.o")]
    out = subprocess.run(cmd, capture_output=True, text=True)
    log = out.stdout + out.stderr
    assert out.returncode == 0, log
    entries = re.findall(r"Compiling entry function '([^']+)'.*?(\d+) bytes spill stores, (\d+) bytes spill loads", log,
                         flags=re.S)
    assert len(entries) == 7 and all(e[1:] == ("0", "0") for e in entries), log


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
    for obj in ("token_loss.o", "token_critic_loss.o", "ppo_loss.o"):
        parts = re.split(r"^\s*Function : (\S+)\s*$", _sass(tmp_path, obj), flags=re.M)
        out[obj] = {parts[i]: hashlib.sha256(parts[i + 1].encode()).hexdigest() for i in range(1, len(parts), 2)}
    return out


def test_existing_objects_keep_their_sass(tmp_path):
    assert sass_digests(tmp_path) == json.load(open(DIGESTS))
