"""The reasoning critic on the CPU: the reference fixture (tests/golden/golden_critic.npz) replayed through the oracle
(tests/critic_oracle.py), the argument envelope of ops.megatron_response_values and reasoning_critic_loss (Python
ValueError, C invalid-argument status), the ctypes signatures and struct layout against the header, no spills in the
new kernels, and the SASS the new code must leave alone: ppo_loss.o, gather.o and response_rows_mp.o whole, and every
kernel of token_loss.o, as at the parent commit (tests/golden/sass_digests_critic.json).  No GPU."""
from __future__ import annotations

import ctypes as C
import hashlib
import json
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

import critic_oracle as CO
import response_rows_mp_oracle as O
from rlinf_b200 import _lib, build, ops
from rlinf_b200 import response_rows as RR
from rlinf_b200.algorithms import reasoning_critic_loss

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
GOLDEN = os.path.join(HERE, "golden", "golden_critic.npz")
DIGESTS = os.path.join(HERE, "golden", "sass_digests_critic.json")


@pytest.fixture(scope="module")
def g():
    return {k: torch.from_numpy(v) for k, v in np.load(GOLDEN, allow_pickle=False).items()}


def _cases(g):
    return sorted(k[:-len("_meta")] for k in g if k.endswith("_meta"))


def test_fixture_covers_the_grids_and_both_huber_branches(g):
    grids = {tuple(int(x) for x in g[f"{k}_meta"][:3]) for k in _cases(g)}
    assert grids == {(1, 1, 0), (2, 1, 1), (1, 2, 0), (2, 2, 1)}
    linear = False
    for key in _cases(g):
        delta = float(g[f"{key}_hyper"][1])
        m = g[f"{key}_mask"].bool()
        e = (g[f"{key}_returns"] - g[f"{key}_train_values"])[m].abs()
        linear |= bool((e >= delta).any())
    assert linear
    assert any(not g[f"{k}_mask"].any(-1).all() for k in _cases(g))  # a row without a valid token


def test_fixture_has_ranks_without_response_rows(g):
    empty = set()
    for key in _cases(g):
        tp, cp, sp, L, bsz, T_c = (int(x) for x in g[f"{key}_meta"][:6])
        per = O.prediction_rows(g[f"{key}_cu"], g[f"{key}_n"], g[f"{key}_r"], cp)
        if any(not rows for rows in per):
            empty.add((tp, cp))
    assert {(1, 2), (2, 2)} <= empty


def test_oracle_reproduces_reference_values(g):
    """The oracle's bf16 Linear on each CP rank's stream, placed in cells, is the reference's inference output bit for
    bit, and the training vpreds' response columns."""
    w = g["w"].to(torch.bfloat16)
    for key in _cases(g):
        tp, cp, sp, L, bsz, T_c = (int(x) for x in g[f"{key}_meta"][:6])
        streams = []
        for c in range(cp):
            parts = [g[f"{key}_c{c}_k{k}_hidden"] for k in range(tp)]
            streams.append((torch.cat(parts) if sp else parts[0]).to(torch.bfloat16))
        v = CO.head_values(streams, w, g[f"{key}_cu"], g[f"{key}_n"], g[f"{key}_r"], cp, L)
        assert torch.equal(v, g[f"{key}_infer_values"]), key
        valid = torch.arange(L)[None] < g[f"{key}_r"][:, None]
        assert torch.equal(v[valid], g[f"{key}_train_values"][valid]), key
        assert torch.equal(v, v.bfloat16().float())  # the reference rounds to bf16 before .float()


def test_oracle_reproduces_reference_loss_and_metrics(g):
    """compute_ppo_critic_loss on the reference's training vpreds, restated by the oracle with fp32 sums: the loss, every
    metric and d loss / d vpreds bit for bit; on the op's values (zeros past r_b) everything but the unmasked
    value_clip_ratio stays the same."""
    for key in _cases(g):
        value_clip, delta = (float(x) for x in g[f"{key}_hyper"])
        ret, prev, mask = g[f"{key}_returns"], g[f"{key}_prev_values"], g[f"{key}_mask"].bool()
        loss, m, grad = CO.critic_loss(g[f"{key}_train_values"], ret, prev, mask, value_clip, delta, sums="fp32")
        assert torch.equal(loss, g[f"{key}_loss"]), key
        assert torch.equal(torch.stack([m[k] for k in CO.KEYS]), g[f"{key}_metrics"]), key
        assert torch.equal(grad, g[f"{key}_vgrad"]), key
        loss2, m2, grad2 = CO.critic_loss(g[f"{key}_infer_values"], ret, prev, mask, value_clip, delta, sums="fp32")
        assert torch.equal(loss2, loss) and torch.equal(grad2, grad), key
        for k in CO.KEYS:
            if k != "critic/value_clip_ratio":
                assert torch.equal(m2[k], m[k]), (key, k)


def test_reference_gradients_lie_on_owned_rows_and_are_bf16_products(g):
    """The reference's dX of the loss is bf16(bf16(g) w) on the response rows a rank holds and zero elsewhere (other CP
    ranks' cells arrive detached; under SP each TP rank takes its own rows)."""
    w = g["w"]
    for key in _cases(g):
        tp, cp, sp, L, bsz, T_c = (int(x) for x in g[f"{key}_meta"][:6])
        per = O.prediction_rows(g[f"{key}_cu"], g[f"{key}_n"], g[f"{key}_r"], cp)
        gv = g[f"{key}_vgrad"].bfloat16().float()
        Ts = T_c // tp if sp else T_c
        for c in range(cp):
            for k in range(tp):
                want = torch.zeros(Ts, w.shape[1], dtype=torch.bfloat16)
                for t, b, j in per[c]:
                    if not sp or k * Ts <= t < (k + 1) * Ts:
                        want[t - (k * Ts if sp else 0)] = (gv[b, j] * w[0]).bfloat16()
                got = g[f"{key}_c{c}_k{k}_grad"].reshape(Ts, -1).bfloat16()
                assert torch.equal(got, want), (key, c, k)


def _host_plan(tp=1, cp=1, sp=False):
    return RR.megatron_parallel([0, 8, 16], [8, 6], [2, 1], response_len=4, tp_size=tp, cp_size=cp,
                                sequence_parallel=sp)


@pytest.mark.parametrize("make, msg", [
    (lambda: ops.megatron_response_values(torch.zeros(16, 64, dtype=torch.bfloat16),
                                          torch.zeros(1, 64, dtype=torch.bfloat16), object()), "megatron_parallel"),
    (lambda: ops.megatron_response_values(torch.zeros(16, 64), torch.zeros(1, 64, dtype=torch.bfloat16),
                                          _host_plan()), "bfloat16"),
    (lambda: ops.megatron_response_values(torch.zeros(16, 64, dtype=torch.bfloat16),
                                          torch.zeros(2, 64, dtype=torch.bfloat16), _host_plan()), r"\[1, H\]"),
    (lambda: ops.megatron_response_values(torch.zeros(16, 64, dtype=torch.bfloat16),
                                          torch.zeros(64, dtype=torch.bfloat16), _host_plan()), r"\[1, H\]"),
    (lambda: ops.megatron_response_values(torch.zeros(16, 96, dtype=torch.bfloat16),
                                          torch.zeros(1, 96, dtype=torch.bfloat16), _host_plan()), "H % 64"),
    (lambda: ops.megatron_response_values(torch.zeros(16, 8256, dtype=torch.bfloat16),
                                          torch.zeros(1, 8256, dtype=torch.bfloat16), _host_plan()), "H % 64"),
    (lambda: ops.megatron_response_values(torch.zeros(16, 64, dtype=torch.bfloat16),
                                          torch.zeros(1, 128, dtype=torch.bfloat16), _host_plan()), "hidden size"),
    (lambda: ops.megatron_response_values(torch.zeros(16, 2, 64, dtype=torch.bfloat16),
                                          torch.zeros(1, 64, dtype=torch.bfloat16), _host_plan()), r"\[rows, 1, H\]"),
    (lambda: ops.megatron_response_values(torch.zeros(8, 64, dtype=torch.bfloat16),
                                          torch.zeros(1, 64, dtype=torch.bfloat16), _host_plan(2, 1, True)),
     "the tp group has 1 ranks"),
    (lambda: ops.megatron_response_values(torch.zeros(8, 64, dtype=torch.bfloat16),
                                          torch.zeros(1, 64, dtype=torch.bfloat16), _host_plan(1, 2)),
     "the cp group has 1 ranks"),
])
def test_values_envelope(make, msg):
    with pytest.raises(ValueError, match=msg):
        make()


def test_values_take_cuda_tensors():
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(_lib.Rb200Error):
        ops.megatron_response_values(torch.zeros(16, 64, dtype=torch.bfloat16),
                                     torch.zeros(1, 64, dtype=torch.bfloat16), _host_plan())


def test_megatron_thd_still_rejects_cp():
    with pytest.raises(ValueError, match="context parallelism"):
        RR.megatron_thd([0, 8, 16], [8, 6], [2, 1], response_len=4, cp_size=2)


@pytest.mark.parametrize("kw, msg", [
    (dict(returns=torch.zeros(2, 3)), "returns has shape"),
    (dict(prev_values=torch.zeros(2, 4, dtype=torch.float64)), "prev_values must be torch.float32"),
    (dict(loss_mask=torch.ones(2, 4)), "loss_mask must be bool or uint8"),
    (dict(loss_mask=None), "loss_mask has shape None"),
    (dict(values=torch.zeros(8)), r"\[bsz, L\]"),
    (dict(values=torch.zeros(0, 4)), "empty values"),
    (dict(value_clip=None), "value_clip is required"),
])
def test_loss_envelope(kw, msg):
    args = dict(values=torch.zeros(2, 4), returns=torch.zeros(2, 4), prev_values=torch.zeros(2, 4),
                loss_mask=torch.ones(2, 4, dtype=torch.bool), value_clip=0.5)
    args.update(kw)
    with pytest.raises(ValueError, match=msg):
        reasoning_critic_loss(args.pop("values"), args.pop("returns"), args.pop("prev_values"), args.pop("loss_mask"),
                              **args)


def test_c_envelope_returns_invalid_argument():
    """The value-head entry points check the envelope before touching the device: any H outside it, a short row stride
    and unaligned pointers return invalid-argument statuses."""
    lib = _lib.load()
    p = C.c_void_p(1 << 20)
    for H in (0, 32, 96, 8256):
        assert lib.rb200_value_head_workspace_bytes(16, H) == -1
        assert lib.rb200_value_head_fwd(p, H, p, 16, H, p, p, None) == -2
        assert lib.rb200_value_head_bwd(p, H, p, 16, H, p, p, p, 16, p, p, p, 1 << 20, None) == -2
    assert lib.rb200_value_head_workspace_bytes(0, 64) == -1
    assert lib.rb200_value_head_workspace_bytes(65, 64) == 2 * 64 * 4
    assert lib.rb200_value_head_fwd(p, 32, p, 16, 64, p, p, None) == -2  # row stride < H
    assert lib.rb200_value_head_fwd(C.c_void_p((1 << 20) + 2), 64, p, 16, 64, p, p, None) == -4
    assert lib.rb200_value_head_fwd(p, 68, p, 16, 64, p, p, None) == -4  # row stride not a multiple of 8
    assert lib.rb200_value_head_fwd(None, 64, p, 16, 64, p, p, None) == -1
    assert lib.rb200_value_head_bwd(p, 64, p, 16, 64, p, p, p, 16, None, None, p, 0, None) == -1
    assert lib.rb200_value_head_bwd(p, 64, p, 16, 64, p, p, p, 16, None, p, p, 16, None) == -3  # workspace short
    a = _lib.TokenCriticLossArgs()
    assert lib.rb200_token_critic_loss(C.byref(a), None) == -1


@pytest.mark.parametrize("name", ["rb200_value_head_workspace_bytes", "rb200_value_head_fwd", "rb200_value_head_bwd"])
def test_ctypes_signature_matches_header(name):
    src = open(os.path.join(ROOT, "include", "rlinf_b200.h")).read()
    m = re.search(rf"(int|int64_t) {name}\((.*?)\);", src, flags=re.S)
    params = [q.strip() for q in m.group(2).split(",")]
    ctype = {"int": _lib.c_int, "int64_t": _lib.c_int64}
    want = [_lib.c_void_p if ("*" in q or q.startswith("rb200_stream_t")) else ctype[q.rsplit(" ", 1)[0]]
            for q in params]
    res, args = _lib.SIGNATURES[name]
    assert res is ctype[m.group(1)] and args == want


def test_critic_loss_struct_layout_matches_header(tmp_path):
    cls, cname = _lib.TokenCriticLossArgs, "rb200_token_critic_loss_args"
    lines = [f'  printf("sizeof %zu\\n", sizeof({cname}));']
    lines += [f'  printf("{f[0]} %zu %zu\\n", offsetof({cname}, {f[0]}), sizeof((({cname}*)0)->{f[0]}));'
              for f in cls._fields_]
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
    assert _lib.SIGNATURES["rb200_token_critic_loss"] == (_lib.c_int, [C.POINTER(cls), _lib.c_void_p])


def _nvcc():
    try:
        return build._nvcc()
    except RuntimeError:
        pytest.skip("nvcc not found")


@pytest.mark.parametrize("src, n", [("value_head.cu", 4), ("token_critic_loss.cu", 2)])
def test_new_kernels_do_not_spill(tmp_path, src, n):
    cmd = [_nvcc(), *build.NVCC_FLAGS, "-Xptxas", "-v", "-c", os.path.join(build.CSRC, src), "-o",
           str(tmp_path / "x.o")]
    out = subprocess.run(cmd, capture_output=True, text=True)
    log = out.stdout + out.stderr
    assert out.returncode == 0, log
    entries = re.findall(r"Compiling entry function '([^']+)'.*?(\d+) bytes spill stores, (\d+) bytes spill loads", log,
                         flags=re.S)
    assert len(entries) == n and all(e[1:] == ("0", "0") for e in entries), log


def _sass(tmp_path, obj):
    nvcc = _nvcc()
    cuobjdump = shutil.which("cuobjdump") or os.path.join(os.path.dirname(nvcc), "cuobjdump")
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not found")
    o = tmp_path / obj
    subprocess.run([nvcc, *build.NVCC_FLAGS, "-c", os.path.join(build.CSRC, obj[:-2] + ".cu"), "-o", str(o)],
                   check=True, capture_output=True)
    return subprocess.run([cuobjdump, "-sass", str(o)], check=True, capture_output=True, text=True).stdout


def _drop_identifiers(text):
    return "\n".join(line for line in text.splitlines() if not line.strip().startswith("identifier"))


@pytest.mark.parametrize("obj", ["ppo_loss.o", "gather.o", "response_rows_mp.o"])
def test_objects_keep_their_sass(tmp_path, obj):
    text = re.sub(r"_GLOBAL__N__[0-9a-f]+_\d+_\w+?_cu_[0-9a-f]+", "_GLOBAL__N_", _sass(tmp_path, obj))
    assert hashlib.sha256(_drop_identifiers(text).encode()).hexdigest() == json.load(open(DIGESTS))[obj]


def test_token_loss_kernels_keep_their_sass(tmp_path):
    """Each of the four kernels of token_loss.o, which the critic loss launches for its mask counts, disassembles to
    the parent's SASS."""
    text = re.sub(r"_GLOBAL__N__[0-9a-f]{8}_\d+_token_loss_cu_[0-9a-f]{8}", "_GLOBAL__N_", _sass(tmp_path, "token_loss.o"))
    parts = re.split(r"^\s*Function : (\S+)\s*$", _drop_identifiers(text), flags=re.M)
    got = {parts[i]: hashlib.sha256(parts[i + 1].encode()).hexdigest() for i in range(1, len(parts), 2)}
    assert got == json.load(open(DIGESTS))["token_loss.o"]
