"""Two-stage fused hidden-layer backward (csrc/tc_backward_h.cu) at shapes where a CTA reuses its stages and ends on a
partial k-block, against the separate wgrad + dgrad kernels (GPU).

n = 3161: 99 k-blocks of 32 samples, the last one 25 rows; with two towers each CTA takes 3 k-blocks, so stage 0 is
reused for the zero-filled tail.  n = 20001: 626 k-blocks, the last one 1 row; with two towers a CTA takes 19 k-blocks
(each stage many times over, an odd count) and the last chunk 18."""
import pytest
import torch

pytestmark = pytest.mark.gpu

FLAG_UNFUSED = 4  # rb200_debug_set_flags bit: wgrad + dgrad as two kernels


def _run(lib, L, Z, W, H, amax_in, flags):
    ng, n = Z.shape[0], Z.shape[1]
    dZp = torch.full_like(Z, float("nan"))
    dW = torch.linspace(-1e-3, 1e-3, ng * 65536, device="cuda").reshape(ng, 256, 256)  # accumulates (+=)
    colsum = torch.linspace(-1e-4, 1e-4, ng * 256, device="cuda").reshape(ng, 256)  # accumulates (+=)
    amax_out = torch.zeros(ng, device="cuda")
    work = torch.empty(ng * (131072 + 256 * ((n + 15) // 16)), device="cuda")
    lib.rb200_debug_set_flags(flags)
    try:
        L.check(lib.rb200_tc_dgrad_wgrad_h(L.ptr(Z), L.ptr(W), L.ptr(H), L.ptr(dZp), L.ptr(dW), L.ptr(colsum),
                                           L.ptr(amax_in), L.ptr(amax_out), n, ng, L.ptr(work), L.stream_ptr()),
                "tc_dgrad_wgrad_h")
        torch.cuda.synchronize()
    finally:
        lib.rb200_debug_set_flags(0)
    return dZp, dW, colsum, amax_out


@pytest.mark.parametrize("n", [3161, 20001])
@pytest.mark.parametrize("ng", [1, 2])
def test_stage_reuse_bit_identical_to_two_kernels(n, ng):
    from rlinf_b200 import _lib as L

    lib = L.load()
    g = torch.Generator(device="cuda").manual_seed(7000 + 10 * ng + n)
    Z = torch.randn(ng, n, 256, device="cuda", generator=g) * 1e-7 * torch.exp(
        torch.randn(ng, n, 1, device="cuda", generator=g))
    H = torch.tanh(torch.randn(ng, n, 256, device="cuda", generator=g))
    W = torch.randn(ng, 256, 256, device="cuda", generator=g) / 16
    amax_in = Z.abs().flatten(1).max(dim=1).values.contiguous()
    ref = _run(lib, L, Z, W, H, amax_in, FLAG_UNFUSED)
    runs = [_run(lib, L, Z, W, H, amax_in, 0) for _ in range(2)]
    for a, b in zip(runs[0], runs[1]):  # deterministic: same bits every call
        assert torch.equal(a, b)
    dZp, dW, colsum, amax_out = runs[0]
    assert torch.equal(dZp, ref[0]), (dZp - ref[0]).abs().max().item()
    assert torch.equal(amax_out, ref[3]), (amax_out, ref[3])
    assert torch.equal(dW, ref[1]), (dW - ref[1]).abs().max().item()
    assert torch.equal(colsum, ref[2]), (colsum - ref[2]).abs().max().item()
