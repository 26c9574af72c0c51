"""The forward GEMM of the MLP towers (tc_h_fwd_kernel, csrc/tc_forward_h.cu) against tc_h_gemm_kernel<0>, the kernel
it replaced for K <= 256: the same bits for every shape, operand scaling and group count (GPU)."""
import pytest
import torch

pytestmark = pytest.mark.gpu

MODE_FWD, MODE_REF = 0, 2  # rb200_tc_gemm_h: the shipped forward / tc_h_gemm_kernel<0>


def _gemm(lib, L, A, B, mode, amax):
    M, K = A.shape
    C = torch.full((M, 256), float("nan"), device="cuda")
    work = torch.empty(512 * K, device="cuda")
    L.check(lib.rb200_tc_gemm_h(L.ptr(A), L.ptr(B), L.ptr(C), M, K, mode, L.ptr(amax), L.ptr(work), L.stream_ptr()),
            "tc_gemm_h")
    torch.cuda.synchronize()
    return C


def _operand(n, K, scaling, g):
    A = torch.randn(n, K, device="cuda", generator=g)
    if scaling == "small":  # max|A| far below 2^-1: scaled up by its published max
        A = A * 1e-3 * torch.exp(torch.randn(n, 1, device="cuda", generator=g))
    elif scaling == "col17":  # one column at 2^17 (would overflow fp16 unscaled): scaled down
        A[:, K // 3] = 2.0 ** 17 * torch.tanh(A[:, K // 3])
        A[0, K // 3] = 2.0 ** 17
    return A


@pytest.mark.parametrize("n", [1, 63, 64, 65, 4096, 4097, 20001, 262144])
@pytest.mark.parametrize("K", [32, 96, 128, 256])
@pytest.mark.parametrize("scaling", [None, "small", "col17"])
def test_forward_bit_identical_to_reference_kernel(n, K, scaling):
    from rlinf_b200 import _lib as L

    lib = L.load()
    g = torch.Generator(device="cuda").manual_seed(7 * n + K)
    A = _operand(n, K, scaling, g)
    B = torch.randn(256, K, device="cuda", generator=g) / K ** 0.5
    amax = A.abs().max().reshape(1) if scaling else None
    ref = _gemm(lib, L, A, B, MODE_REF, amax)
    out = _gemm(lib, L, A, B, MODE_FWD, amax)
    assert torch.equal(out, ref), (out - ref).abs().max().item()
    assert torch.equal(_gemm(lib, L, A, B, MODE_FWD, amax), out)  # deterministic


def _tower_acts(pol, states, values):
    """H1, H2, H3 of the actor tower and, with values, G1, G2, G3 of the value tower, as the training forward keeps them."""
    n = states.shape[0]
    action = torch.zeros(n, pol.act_dim, device="cuda")
    pol.forward_train(states, action, compute_values=values)
    torch.cuda.synchronize()
    acts = pol._scratch["acts"]
    return [acts[i * n * 256:(i + 1) * n * 256].view(n, 256).clone() for i in range(6 if values else 3)]


@pytest.mark.parametrize("n", [1, 65, 4097, 20001])
@pytest.mark.parametrize("obs", [96, 128, 256])
@pytest.mark.parametrize("scaling", [None, "small", "col17"])
def test_two_tower_forward(n, obs, scaling):
    """Both towers in one launch per layer (layer 0: four CTAs per row tile on the same observations).  With the value
    tower given the actor's weights, every layer of both towers equals the one-tower launch bit for bit; layer 0
    equals tanh of the reference kernel's product plus the bias, to the tolerance of the epilogue's tanh."""
    from rlinf_b200 import _lib as L
    from rlinf_b200.policy import MLPPolicy

    lib = L.load()
    g = torch.Generator(device="cuda").manual_seed(n + obs)
    pol = MLPPolicy(obs_dim=obs, action_dim=8, seed=n)
    p = dict(pol.named_parameters())
    for i, v in ((0, 0), (2, 2), (4, 4)):
        p[f"backbone.{i}.bias"].copy_(0.1 * torch.randn(256, device="cuda", generator=g))
        p[f"value_head.mlp.{v}.weight"].copy_(p[f"backbone.{i}.weight"])
        p[f"value_head.mlp.{v}.bias"].copy_(p[f"backbone.{i}.bias"])
    pol.mark_params_changed()
    states = _operand(n, obs, scaling, g)

    both = _tower_acts(pol, states, True)
    one = _tower_acts(pol, states, False)
    for layer in range(3):
        assert torch.equal(both[layer], one[layer]), layer
        assert torch.equal(both[3 + layer], both[layer]), layer

    amax = states.abs().max().reshape(1) if scaling else None  # outside [2^-1, 2^15): the forward's own scale
    z = _gemm(lib, L, states, p["backbone.0.weight"].contiguous(), MODE_REF, amax)
    err = (one[0] - torch.tanh(z + p["backbone.0.bias"])).abs().max().item()
    assert err < 1e-6, err
