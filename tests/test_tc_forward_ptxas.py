"""ptxas report of the forward GEMM kernel (csrc/tc_forward_h.cu), compiled with the library's own flags: its wgmmas
may not be serialised (C7512 / C7514) and it may not spill registers."""
from __future__ import annotations

import os
import re
import subprocess

import pytest

from rlinf_b200 import build

SRC = os.path.join(build.CSRC, "tc_forward_h.cu")


def test_tc_forward_kernel_not_serialised_and_no_spills(tmp_path):
    try:
        nvcc = build._nvcc()
    except RuntimeError:
        pytest.skip("nvcc not found")
    cmd = [nvcc, *build.NVCC_FLAGS, "-Xptxas", "-v", "-c", SRC, "-o", str(tmp_path / "tc_forward_h.o")]
    out = subprocess.run(cmd, capture_output=True, text=True)
    log = out.stdout + out.stderr
    assert out.returncode == 0, log
    assert "wgmma.mma_async instructions are serialized" not in log, log
    assert "C7512" not in log and "C7514" not in log, log
    entries = re.findall(r"Compiling entry function '([^']+)'.*?(\d+) bytes spill stores, (\d+) bytes spill loads", log,
                         flags=re.S)
    kernels = {name: (int(s), int(l)) for name, s, l in entries if "tc_h_fwd_kernel" in name}
    assert len(kernels) == 1, log
    assert list(kernels.values()) == [(0, 0)], kernels
