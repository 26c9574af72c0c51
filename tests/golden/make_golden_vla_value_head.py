"""Reference fixture of the OpenVLA value head: golden_vla_value_head.npz.

    python tests/golden/make_golden_vla_value_head.py     (needs the reference checkout; CPU only)

Runs the unmodified reference module models/embodiment/modules/value_head.py, loaded by file path, on the CPU in bf16
and in fp32: ValueHead(H, output_dim=O) (hidden_sizes (512, 128), GELU, bias_last=False) for H in HS, O in OS, N rows,
forward and the backward of a seeded upstream gradient.  Inputs and parameters are not stored: make_inputs()
regenerates them from the case's seed.  Stored per case and dtype: the values, dX, db0, db1 and dW2 in full, and the
rows W0_ROWS of dW0 and W1_ROWS of dW1 (each row of a weight gradient is its own reduction over the N rows).  bf16
tensors are stored as their uint16 bit patterns.

The module's constructor calls nn.init.kaiming_normal_(nonlinearity="gelu"), which torch.nn.init.calculate_gain does
not know; in the reference it runs under transformers' from_pretrained, where the nn.init functions are no-ops.  It is
built the same way here, with kaiming_normal_ a no-op during construction, and its parameters are then set from the
seed.
"""
from __future__ import annotations

import importlib.util
import os

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "golden_vla_value_head.npz")
REFERENCE_ROOT = os.environ.get("RLINF_REFERENCE_ROOT", "/root/reference")

HS = (256, 512)
OS = (1, 8, 25)
N = 13
W0_ROWS = slice(None, None, 64)
W1_ROWS = slice(None, None, 32)
DTYPES = {"bf16": torch.bfloat16, "fp32": torch.float32}


def case_name(H: int, O: int, dt: str) -> str:
    return f"h{H}_o{O}_{dt}"


def make_inputs(H: int, O: int, seed: int = 0) -> dict:
    """fp32 tensors x [N, H], w0 [512, H], b0, w1 [128, 512], b1, w2 [O, 128], gv [N, O], every value exact in bf16
    (so the bf16 and fp32 modules see the same numbers)."""
    g = torch.Generator().manual_seed(1000 * H + O + 7919 * seed)

    def r(*shape, std=1.0):
        return (torch.randn(*shape, generator=g) * std).to(torch.bfloat16).float()

    return {"x": r(N, H), "w0": r(512, H, std=(2.0 / 512) ** 0.5), "b0": r(512, std=0.1),
            "w1": r(128, 512, std=(2.0 / 128) ** 0.5), "b1": r(128, std=0.1), "w2": r(O, 128, std=0.02),
            "gv": r(N, O)}


def bits(t: torch.Tensor) -> np.ndarray:
    return t.detach().contiguous().view(torch.int16).numpy().view(np.uint16)


def from_bits(a: np.ndarray) -> torch.Tensor:
    return torch.from_numpy(a.astype(np.uint16).view(np.int16)).view(torch.bfloat16)


def _load_value_head_class():
    path = os.path.join(REFERENCE_ROOT, "rlinf", "models", "embodiment", "modules", "value_head.py")
    spec = importlib.util.spec_from_file_location("reference_value_head", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod.ValueHead


def run_reference(ValueHead, H: int, O: int, dtype) -> dict:
    inp = make_inputs(H, O)
    init = torch.nn.init.kaiming_normal_
    torch.nn.init.kaiming_normal_ = lambda t, *a, **k: t  # from_pretrained's no-op init
    try:
        head = ValueHead(H, hidden_sizes=(512, 128), output_dim=O, activation="gelu", bias_last=False)
    finally:
        torch.nn.init.kaiming_normal_ = init
    with torch.no_grad():
        for name, key in (("mlp.0.weight", "w0"), ("mlp.0.bias", "b0"), ("mlp.2.weight", "w1"),
                          ("mlp.2.bias", "b1"), ("mlp.4.weight", "w2")):
            head.get_parameter(name).copy_(inp[key])
    head = head.to(dtype)
    x = inp["x"].to(dtype).requires_grad_(True)
    v = head(x)
    v.backward(inp["gv"].to(dtype))
    m = head.mlp
    return {"v": v, "dx": x.grad, "dw0": m[0].weight.grad[W0_ROWS], "db0": m[0].bias.grad,
            "dw1": m[2].weight.grad[W1_ROWS], "db1": m[2].bias.grad, "dw2": m[4].weight.grad}


def main():
    ValueHead = _load_value_head_class()
    out = {}
    for H in HS:
        for O in OS:
            for dt, dtype in DTYPES.items():
                res = run_reference(ValueHead, H, O, dtype)
                for k, t in res.items():
                    out[f"{case_name(H, O, dt)}_{k}"] = bits(t) if dt == "bf16" else t.detach().numpy()
    np.savez_compressed(OUT, **out)
    print(OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
