"""Build librlinf_b200.so in-tree with nvcc for sm_90a (H100; cross-compiles without a GPU).

    python -m rlinf_b200.build [--force] [--verbose]

The .so, the object files and the freshness stamp are build products (git-ignored).
"""
from __future__ import annotations

import glob
import hashlib
import os
import shutil
import subprocess
import sys

PKG_DIR = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(PKG_DIR, "csrc")
LIB_PATH = os.path.join(PKG_DIR, "librlinf_b200.so")
STAMP = os.path.join(PKG_DIR, ".librlinf_b200.stamp")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC,-O3",
    "--expt-relaxed-constexpr",
    "-Xptxas", "-warn-spills",
]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found; librlinf_b200.so cannot be built")


def sources() -> list[str]:
    return sorted(glob.glob(os.path.join(CSRC, "*.cu")))


def _digest() -> str:
    h = hashlib.sha256()
    files = sources() + sorted(glob.glob(os.path.join(CSRC, "*.cuh"))) + [
        os.path.join(os.path.dirname(PKG_DIR), "include", "rlinf_b200.h")]
    for f in files:
        h.update(os.path.basename(f).encode())
        with open(f, "rb") as fh:
            h.update(fh.read())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def is_fresh() -> bool:
    if not (os.path.exists(LIB_PATH) and os.path.exists(STAMP)):
        return False
    with open(STAMP) as fh:
        return fh.read().strip() == _digest()


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and is_fresh():
        return LIB_PATH
    objdir = os.path.join(PKG_DIR, "build")
    os.makedirs(objdir, exist_ok=True)
    nvcc = _nvcc()
    objs = []
    procs = []
    for src in sources():
        obj = os.path.join(objdir, os.path.basename(src)[:-3] + ".o")
        cmd = [nvcc, *NVCC_FLAGS, "-dc" if False else "-c", src, "-o", obj]
        if verbose:
            cmd.insert(1, "-Xptxas=-v")
            print(" ".join(cmd), flush=True)
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
        objs.append(obj)
    failed = False
    for src, p in procs:
        out, _ = p.communicate()
        if out.strip() and (verbose or p.returncode != 0 or "warning" in out.lower()):
            print(f"--- {os.path.basename(src)} ---\n{out}", flush=True)
        failed |= p.returncode != 0
    if failed:
        raise RuntimeError("nvcc failed")
    link = [nvcc, "-shared", "-gencode", "arch=compute_90a,code=sm_90a", "-Xcompiler", "-fPIC",
            "-o", LIB_PATH, *objs, "-lcudart_static" if False else "-lcudart"]
    subprocess.run(link, check=True)
    with open(STAMP, "w") as fh:
        fh.write(_digest())
    return LIB_PATH


if __name__ == "__main__":
    path = build(force="--force" in sys.argv, verbose="--verbose" in sys.argv)
    print(path)
