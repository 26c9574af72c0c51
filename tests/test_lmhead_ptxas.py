"""ptxas report of the fused LM-head log-prob kernels (csrc/lmhead.cu), compiled with the library's own flags: no
kernel's wgmmas may be serialised (C7512 / C7514) and none may spill registers."""
from __future__ import annotations

import os
import re
import subprocess

import pytest

from rlinf_b200 import build

SRC = os.path.join(build.CSRC, "lmhead.cu")


def test_lmhead_kernels_not_serialised_and_no_spills(tmp_path):
    try:
        nvcc = build._nvcc()
    except RuntimeError:
        pytest.skip("nvcc not found")
    cmd = [nvcc, *build.NVCC_FLAGS, "-Xptxas", "-v", "-c", SRC, "-o", str(tmp_path / "lmhead.o")]
    out = subprocess.run(cmd, capture_output=True, text=True)
    log = out.stdout + out.stderr
    assert out.returncode == 0, log
    assert "wgmma.mma_async instructions are serialized" not in log, log
    assert "C7512" not in log and "C7514" not in log, log
    entries = re.findall(r"Compiling entry function '([^']+)'.*?(\d+) bytes spill stores, (\d+) bytes spill loads", log,
                         flags=re.S)
    kernels = {name: (int(s), int(l)) for name, s, l in entries if "lmhead" in name}
    # the four epilogues of lmhead_kernel and the combine kernel
    assert len(kernels) == 5, log
    assert set(kernels.values()) == {(0, 0)}, kernels
