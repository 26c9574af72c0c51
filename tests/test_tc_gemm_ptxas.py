"""ptxas report of the wgmma GEMM kernels (csrc/tc_gemm_h.cu), compiled with the library's own flags: no tc_h_* kernel
may have its wgmmas serialised (C7512: each wgmma waits for the previous one) or spill registers."""
from __future__ import annotations

import os
import re
import subprocess

import pytest

from rlinf_b200 import build

SRC = os.path.join(build.CSRC, "tc_gemm_h.cu")


def _nvcc():
    try:
        return build._nvcc()
    except RuntimeError:
        pytest.skip("nvcc not found")


def test_tc_gemm_kernels_not_serialised_and_no_spills(tmp_path):
    cmd = [_nvcc(), *build.NVCC_FLAGS, "-Xptxas", "-v", "-c", SRC, "-o", str(tmp_path / "tc_gemm_h.o")]
    out = subprocess.run(cmd, capture_output=True, text=True)
    log = out.stdout + out.stderr
    assert out.returncode == 0, log

    serialised = [ln for ln in log.splitlines() if "wgmma.mma_async instructions are serialized" in ln and "tc_h_" in ln]
    assert not serialised, "\n".join(serialised)

    # "Compiling entry function 'NAME'" is followed by "N bytes stack frame, S bytes spill stores, L bytes spill loads"
    entries = re.findall(r"Compiling entry function '([^']+)'.*?(\d+) bytes spill stores, (\d+) bytes spill loads", log,
                         flags=re.S)
    kernels = {name: (int(s), int(l)) for name, s, l in entries if "tc_h_" in name}
    assert len(kernels) == 4, log  # tc_h_gemm_kernel<0>, <1>, tc_h_wgrad_kernel<128>, <256>
    spilling = {k: v for k, v in kernels.items() if v != (0, 0)}
    assert not spilling, spilling
