"""ptxas report of the vocabulary-parallel kernels (csrc/vocab_parallel.cu, the shard row passes of csrc/logits.cu),
compiled with the library's own flags: none may spill, and no wgmma of those files may be serialised (C7512 / C7514).
The fused shard forward and backward run the lmhead.cu kernels that test_lmhead_ptxas.py checks."""
from __future__ import annotations

import os
import re
import subprocess

import pytest

from rlinf_b200 import build


@pytest.mark.parametrize("src,names,count", [("vocab_parallel.cu", ("kernel",), 3), ("logits.cu", ("vp_",), 4)])
def test_vp_kernels_not_serialised_and_no_spills(tmp_path, src, names, count):
    try:
        nvcc = build._nvcc()
    except RuntimeError:
        pytest.skip("nvcc not found")
    cmd = [nvcc, *build.NVCC_FLAGS, "-Xptxas", "-v", "-c", os.path.join(build.CSRC, src), "-o", str(tmp_path / "x.o")]
    out = subprocess.run(cmd, capture_output=True, text=True)
    log = out.stdout + out.stderr
    assert out.returncode == 0, log
    assert "wgmma.mma_async instructions are serialized" not in log, log
    assert "C7512" not in log and "C7514" not in log, log
    entries = re.findall(r"Compiling entry function '([^']+)'.*?(\d+) bytes spill stores, (\d+) bytes spill loads", log,
                         flags=re.S)
    kernels = {name: (int(s), int(l)) for name, s, l in entries if any(n in name for n in names)}
    assert len(kernels) == count, log
    assert set(kernels.values()) == {(0, 0)}, kernels
