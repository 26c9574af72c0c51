"""Fused hidden-layer backward (csrc/tc_backward_h.cu) against the separate wgrad + dgrad kernels it replaces (GPU)."""
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


def _inputs(n, ng, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    # gradient-like dZ (~1e-7, rows spread over e^+-4) so that the amax scaling is active; H = tanh activations
    Z = torch.randn(ng, n, 256, device="cuda", generator=g) * 1e-7 * torch.exp(torch.randn(ng, n, 1, device="cuda", generator=g))
    H = torch.tanh(torch.randn(ng, n, 256, device="cuda", generator=g))
    W = torch.randn(ng, 256, 256, device="cuda", generator=g) / 16
    amax_in = Z.abs().flatten(1).max(dim=1).values.contiguous()
    return Z, W, H, amax_in


@pytest.mark.parametrize("n", [1, 127, 128, 129, 4097, 262144])
@pytest.mark.parametrize("ng", [1, 2])
def test_fused_backward_bit_identical_to_two_kernels(n, ng):
    from rlinf_b200 import _lib as L

    lib = L.load()
    Z, W, H, amax_in = _inputs(n, ng, 1000 * ng + n)
    ref = _run(lib, L, Z, W, H, amax_in, FLAG_UNFUSED)
    runs = [_run(lib, L, Z, W, H, amax_in, 0) for _ in range(3)]
    dZp, dW, colsum, amax_out = runs[0]
    for r in runs[1:]:  # deterministic: same bits every call
        for a, b in zip(runs[0], r):
            assert torch.equal(a, b)
    assert torch.equal(dZp, ref[0]), (dZp - ref[0]).abs().max().item()
    assert torch.equal(amax_out, ref[3]), (amax_out, ref[3])
    assert torch.equal(dW, ref[1]), (dW - ref[1]).abs().max().item()
    assert torch.equal(colsum, ref[2]), (colsum - ref[2]).abs().max().item()  # added in the dgrad kernel's order
    assert amax_out.tolist() == [dZp[g].abs().max().item() for g in range(ng)]


@pytest.mark.parametrize("n", [4097, 70000])
def test_fused_backward_matches_fp64(n):
    """dW and dZ_{L-1} of the fused kernel against an fp64 computation (the bound of test_tc_wgrad_h_matches_fp64)."""
    from rlinf_b200 import _lib as L

    lib = L.load()
    Z, W, H, amax_in = _inputs(n, 1, n)
    dZp, dW, colsum, _ = _run(lib, L, Z, W, H, amax_in, 0)
    Zd, Hd, Wd = Z[0].double(), H[0].double(), W[0].double()
    dW0 = torch.linspace(-1e-3, 1e-3, 65536, device="cuda").reshape(256, 256).double()
    ref_w = Zd.t() @ Hd
    err_w = ((dW[0].double() - dW0 - ref_w).abs() / (Zd.abs().t() @ Hd.abs()).clamp_min(1e-300)).max().item()
    assert err_w < 2e-6, err_w
    amax = Zd.abs().max()
    ref_d = (Zd @ Wd) * (1 - Hd * Hd)
    scale_d = (Zd.abs() @ Wd.abs()) * (1 - Hd * Hd) + amax * 2.0 ** -16 * Wd.abs().sum(dim=0, keepdim=True)
    err_d = ((dZp[0].double() - ref_d).abs() / scale_d.clamp_min(1e-300)).max().item()
    assert err_d < 2e-6, err_d
