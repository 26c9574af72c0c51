"""CPU-side checks of the C-ABI library: it loads and exports every symbol the header declares, and the ctypes structs
match the header's layouts.  No compute calls (no GPU here)."""
import ctypes as C
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared_symbols():
    src = open(os.path.join(ROOT, "include", "rlinf_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(rb200_[a-z0-9_]+)\s*\(", src)))


def test_library_exports_every_declared_symbol_and_abi_version():
    from rlinf_b200 import _lib

    if not os.path.exists(_lib.LIB_PATH):
        from rlinf_b200 import build

        build.build()
    lib = _lib.load()
    declared = _declared_symbols()
    assert len(declared) >= 18
    for name in declared:
        assert hasattr(lib, name), f"{name} declared in include/rlinf_b200.h but not exported"
        assert name in _lib.SIGNATURES, f"{name} has no ctypes signature in rlinf_b200/_lib.py"
    assert lib.rb200_abi_version() == 2
    assert lib.rb200_strerror(-2).decode().startswith("non-positive")


def test_struct_layouts_match_ctypes(tmp_path):
    """sizeof / offsetof / field size of every field of the ABI structs, as the host C compiler lays them out, against
    the ctypes mirrors in rlinf_b200/_lib.py: a field out of order or of the wrong width would otherwise load fine and
    corrupt a launch."""
    import shutil
    import subprocess

    from rlinf_b200 import _lib

    structs = {"rb200_rollout_args": _lib.RolloutArgs, "rb200_mlp_layout": _lib.MlpLayout,
               "rb200_ppo_args": _lib.PpoArgs, "rb200_dppo_args": _lib.DppoArgs}
    lines = []
    for cname, cls in structs.items():
        lines.append(f'  printf("{cname} sizeof %zu\\n", sizeof({cname}));')
        for f in cls._fields_:
            lines.append(f'  printf("{cname} {f[0]} %zu %zu\\n", offsetof({cname}, {f[0]}), '
                         f'sizeof((({cname}*)0)->{f[0]}));')
    src = tmp_path / "layout.c"
    src.write_text("#include <stddef.h>\n#include <stdio.h>\n#include \"rlinf_b200.h\"\nint main(void) {\n" +
                   "\n".join(lines) + "\n  return 0;\n}\n")
    cc = os.environ.get("CC") or shutil.which("gcc") or shutil.which("cc")
    assert cc, "no host C compiler (gcc) found"
    exe = tmp_path / "layout"
    subprocess.run([cc, "-std=c99", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    out = subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split("\n")
    got = {tuple(line.split()[:2]): tuple(int(v) for v in line.split()[2:]) for line in out if line}
    for cname, cls in structs.items():
        assert got[(cname, "sizeof")] == (C.sizeof(cls),), cname
        for f in cls._fields_:
            d = getattr(cls, f[0])
            assert got[(cname, f[0])] == (d.offset, d.size), (cname, f[0])
    # rb200_rollout_args is ordered pointers, 64-bit, 32-bit, doubles: no padding anywhere
    assert C.sizeof(_lib.RolloutArgs) == sum(getattr(_lib.RolloutArgs, f[0]).size for f in _lib.RolloutArgs._fields_)


def test_missing_library_fails_loudly(monkeypatch, tmp_path):
    from rlinf_b200 import _lib

    monkeypatch.setattr(_lib, "_LIB", None)
    monkeypatch.setattr(_lib, "LIB_PATH", str(tmp_path / "nope.so"))
    with pytest.raises(_lib.Rb200Error, match="no CPU or PyTorch fallback"):
        _lib.load()


def test_no_cpu_fallback_for_cpu_tensors():
    import torch

    from rlinf_b200 import _lib

    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(_lib.Rb200Error):
        _lib.default_device()
    with pytest.raises(_lib.Rb200Error):
        _lib.ptr(torch.zeros(4))


def test_product_code_never_imports_oracle():
    pkg = os.path.join(ROOT, "rlinf_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh")):
                text = open(os.path.join(dirpath, f)).read()
                assert "import oracle" not in text and "from oracle" not in text, os.path.join(dirpath, f)


def test_registry_surface():
    import rlinf_b200.algorithms as A

    assert {"gae", "grpo"} <= set(A.ADV_REGISTRY)
    assert {"actor_critic", "actor"} <= set(A.LOSS_REGISTRY)
    with pytest.raises(ValueError, match="not registered"):
        A.get_adv_and_returns("nope")
    with pytest.raises(ValueError, match="not registered"):
        A.get_policy_loss("nope")
