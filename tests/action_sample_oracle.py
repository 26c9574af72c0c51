"""fp64 oracle of the OpenVLA-OFT rollout's action-token step (csrc/action_sample.cu, ops.sample_action_tokens) and
the reference's numpy de-tokeniser (predict_action_batch :390-404, _unnormalize_actions :167-203).  Kept apart from
oracle/, which stays as it is."""
from __future__ import annotations

import numpy as np
import torch


def window_logprobs(x, lo: int, hi: int, do_sample: bool, T: float = 1.0, k: int = 0) -> torch.Tensor:
    """[..., hi - lo] fp64 log-probabilities over the window of x [..., V]: greedy at T = 1 over the whole window;
    sampling with the window's values >= the k-th largest kept (0 < k < W, ties kept, selected before the temperature)
    and z = x / T.  Columns that are not kept are -inf."""
    w = torch.as_tensor(x)[..., lo:hi].double()
    W = hi - lo
    if do_sample and 0 < k < W:
        thr = torch.topk(w, k, dim=-1).values[..., -1:]
        w = w.masked_fill(w < thr, float("-inf"))
    z = w / T if do_sample else w
    return torch.log_softmax(z, dim=-1)


def greedy_tokens(x, lo: int, hi: int) -> torch.Tensor:
    """argmax over the window, lowest index on ties, as absolute vocabulary ids."""
    return torch.as_tensor(x)[..., lo:hi].argmax(-1) + lo


def detokenize(tokens, vocab_size: int, bin_centers, low, high, mask) -> np.ndarray:
    """The reference's numpy de-tokenisation and unnormalisation of tokens [bsz, L] (L a multiple of action_dim), in its
    order of operations: fp64, the same bits as the reference."""
    tokens = np.asarray(tokens)
    action_dim = len(low)
    d = vocab_size - tokens.reshape(-1, action_dim)
    d = np.clip(d - 1, a_min=0, a_max=len(bin_centers) - 1)
    n = np.asarray(bin_centers)[d]
    high, low = np.asarray(high, dtype=np.float64), np.asarray(low, dtype=np.float64)
    out = np.where(np.asarray(mask), 0.5 * (n + 1) * (high - low + 1e-8) + low, n)
    return out.reshape(tokens.shape)
