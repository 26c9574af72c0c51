"""Envelope of ops.linear_logprobs_entropy: operands outside it raise ValueError naming the condition, before any
device work."""
from __future__ import annotations

import pytest
import torch

from rlinf_b200 import ops


def test_fp32_operands_rejected():
    x = torch.zeros(4, 64)
    w = torch.zeros(10, 64)
    with pytest.raises(ValueError, match="bfloat16"):
        ops.linear_logprobs_entropy(x, w, torch.zeros(4, dtype=torch.int64))


def test_fp16_weight_rejected():
    x = torch.zeros(4, 64, dtype=torch.bfloat16)
    w = torch.zeros(10, 64, dtype=torch.float16)
    with pytest.raises(ValueError, match="bfloat16"):
        ops.linear_logprobs_entropy(x, w, torch.zeros(4, dtype=torch.int64))


@pytest.mark.parametrize("H", [96, 32, 8256])
def test_hidden_size_outside_envelope_rejected(H):
    x = torch.zeros(4, H, dtype=torch.bfloat16)
    w = torch.zeros(10, H, dtype=torch.bfloat16)
    with pytest.raises(ValueError, match="H % 64 == 0"):
        ops.linear_logprobs_entropy(x, w, torch.zeros(4, dtype=torch.int64))


def test_mismatched_hidden_size_rejected():
    x = torch.zeros(4, 128, dtype=torch.bfloat16)
    w = torch.zeros(10, 64, dtype=torch.bfloat16)
    with pytest.raises(ValueError, match="hidden size"):
        ops.linear_logprobs_entropy(x, w, torch.zeros(4, dtype=torch.int64))
