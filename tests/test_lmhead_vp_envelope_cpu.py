"""Envelope of the vocabulary-parallel log-prob ops: unequal shards, windows outside [0, P * Vs), ranks outside
[0, P), wrong dtypes and label smoothing raise ValueError naming the condition, before any device work."""
from __future__ import annotations

import pytest
import torch

from rlinf_b200 import ops

X = torch.zeros(4, 64, dtype=torch.bfloat16)
W = torch.zeros(10, 64, dtype=torch.bfloat16)
T = torch.zeros(4, dtype=torch.int64)


def test_fp32_hidden_rejected():
    with pytest.raises(ValueError, match="bfloat16"):
        ops.vocab_parallel_linear_logprobs_entropy(X.float(), W, T)


def test_fp16_logits_rejected():
    with pytest.raises(ValueError, match="float32 or bfloat16"):
        ops.vocab_parallel_entropy_and_log_probs(torch.zeros(4, 10, dtype=torch.float16), T)
    with pytest.raises(ValueError, match="float32 or bfloat16"):
        ops.logits_vp_partials(torch.zeros(4, 10, dtype=torch.float16), T, 0, 2)


def test_unequal_shards_rejected():
    with pytest.raises(ValueError, match="shards must be equal"):
        ops.vocab_parallel_linear_logprobs_entropy(X, W, T, vocab_size=12)
    with pytest.raises(ValueError, match="shards must be equal"):
        ops.lmhead_vp_partials(X, W, T, 0, 2, vocab_size=21)
    with pytest.raises(ValueError, match="shards must be equal"):
        ops.logits_vp_partials(torch.zeros(4, 10), T, 1, 2, vocab_size=19)


@pytest.mark.parametrize("window", [(5, 21), (-1, 3), (7, 7), (12, 9)])
def test_window_outside_the_sharded_vocabulary_rejected(window):
    with pytest.raises(ValueError, match="window"):
        ops.lmhead_vp_partials(X, W, T, 1, 2, window=window)
    with pytest.raises(ValueError, match="window"):
        ops.vp_combine(torch.zeros(2, 4, 4), T, 10, window=window)


def test_window_outside_a_single_rank_rejected():
    with pytest.raises(ValueError, match="window"):
        ops.vocab_parallel_linear_logprobs_entropy(X, W, T, window=(0, 11))


def test_rank_outside_the_group_rejected():
    with pytest.raises(ValueError, match="rank"):
        ops.lmhead_vp_partials(X, W, T, 2, 2)


def test_label_smoothing_rejected():
    with pytest.raises(ValueError, match="label_smoothing"):
        ops.vocab_parallel_entropy_and_log_probs(torch.zeros(4, 10), T, label_smoothing=0.1)


def test_malformed_records_rejected():
    with pytest.raises(ValueError, match="records"):
        ops.vp_combine(torch.zeros(2, 4, 3), T, 10)
