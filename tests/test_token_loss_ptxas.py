"""Compiler checks of the token-level reasoning loss (csrc/token_loss.cu) with the library's own flags: none of its
kernels spills registers, and the objects whose per-unit arithmetic moved into the shared headers ppo_unit.cuh and
kl_unit.cuh (ppo_loss.o, misc.o, adv_extra.o) disassemble to exactly the SASS they had before the move.  The digests in
tests/golden/sass_digests_loss.json are of `cuobjdump -sass` with the anonymous-namespace hash and the source path
normalised away."""
from __future__ import annotations

import hashlib
import json
import os
import re
import shutil
import subprocess

import pytest

from rlinf_b200 import build

DIGESTS = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "sass_digests_loss.json")


def _nvcc():
    try:
        return build._nvcc()
    except RuntimeError:
        pytest.skip("nvcc not found")


def normalised_sass(text: str) -> str:
    text = re.sub(r"_GLOBAL__N__[0-9a-f]+_\d+_\w+?_cu_[0-9a-f]+", "_GLOBAL__N_", text)
    return "\n".join(line for line in text.splitlines() if not line.strip().startswith("identifier"))


def test_token_loss_kernels_do_not_spill(tmp_path):
    cmd = [_nvcc(), *build.NVCC_FLAGS, "-Xptxas", "-v", "-c", os.path.join(build.CSRC, "token_loss.cu"), "-o",
           str(tmp_path / "token_loss.o")]
    out = subprocess.run(cmd, capture_output=True, text=True)
    log = out.stdout + out.stderr
    assert out.returncode == 0, log
    entries = re.findall(r"Compiling entry function '([^']+)'.*?(\d+) bytes spill stores, (\d+) bytes spill loads", log,
                         flags=re.S)
    kernels = {name: (int(s), int(l)) for name, s, l in entries}
    assert len(kernels) == 4, log  # count, totals, main, finalize
    assert set(kernels.values()) == {(0, 0)}, kernels


@pytest.mark.parametrize("obj", ["ppo_loss.o", "misc.o", "adv_extra.o"])
def test_shared_arithmetic_leaves_existing_sass_unchanged(tmp_path, obj):
    nvcc = _nvcc()
    cuobjdump = shutil.which("cuobjdump") or os.path.join(os.path.dirname(nvcc), "cuobjdump")
    if not os.path.exists(cuobjdump):
        pytest.skip("cuobjdump not found")
    o = tmp_path / obj
    subprocess.run([nvcc, *build.NVCC_FLAGS, "-c", os.path.join(build.CSRC, obj[:-2] + ".cu"), "-o", str(o)],
                   check=True, capture_output=True)
    sass = subprocess.run([cuobjdump, "-sass", str(o)], check=True, capture_output=True, text=True).stdout
    want = json.load(open(DIGESTS))[obj]
    assert hashlib.sha256(normalised_sass(sass).encode()).hexdigest() == want
