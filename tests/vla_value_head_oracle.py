"""fp64 restatement of the OpenVLA value head, ValueHead(H, (512, 128), O, "gelu", bias_last=False).mlp, and of
autograd's backward through it.  With bf16=True every tensor the bf16 module materialises is rounded to bf16 where
the module rounds it (each Linear's output, each GELU's output, each gradient autograd forms); the sums themselves are
fp64.  With bf16=False nothing is rounded: the exact result for the given (bf16-valued) inputs."""
from __future__ import annotations

import math

import torch

D0, D1 = 512, 128


def _round(t: torch.Tensor, bf16: bool) -> torch.Tensor:
    return t.to(torch.bfloat16).to(torch.float64) if bf16 else t


def gelu(z: torch.Tensor) -> torch.Tensor:
    return z * 0.5 * (1.0 + torch.erf(z / math.sqrt(2.0)))


def gelu_grad(z: torch.Tensor) -> torch.Tensor:
    return 0.5 * (1.0 + torch.erf(z / math.sqrt(2.0))) + z * torch.exp(-0.5 * z * z) / math.sqrt(2.0 * math.pi)


def _f64(*ts):
    return [t.detach().to(torch.float64) for t in ts]


def forward(x, w0, b0, w1, b1, w2, bf16: bool = True):
    """(values [N, O], saved = (z0, a0, z1, a1)), all fp64."""
    x, w0, b0, w1, b1, w2 = _f64(x, w0, b0, w1, b1, w2)
    z0 = _round(x @ w0.T + b0, bf16)
    a0 = _round(gelu(z0), bf16)
    z1 = _round(a0 @ w1.T + b1, bf16)
    a1 = _round(gelu(z1), bf16)
    return _round(a1 @ w2.T, bf16), (z0, a0, z1, a1)


def backward(x, w0, w1, w2, saved, gv, bf16: bool = True) -> dict:
    """Gradients of sum(values * gv) for the forward's saved tensors: dx, dw0, db0, dw1, db1, dw2 (fp64)."""
    x, w0, w1, w2, gv = _f64(x, w0, w1, w2, gv)
    z0, a0, z1, a1 = saved
    da1 = _round(gv @ w2, bf16)
    dz1 = _round(da1 * gelu_grad(z1), bf16)
    da0 = _round(dz1 @ w1, bf16)
    dz0 = _round(da0 * gelu_grad(z0), bf16)
    return {"dx": _round(dz0 @ w0, bf16), "dw0": _round(dz0.T @ x, bf16), "db0": _round(dz0.sum(0), bf16),
            "dw1": _round(dz1.T @ a0, bf16), "db1": _round(dz1.sum(0), bf16), "dw2": _round(gv.T @ a1, bf16)}
