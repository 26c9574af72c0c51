import sys, torch
sys.path.insert(0, '.')
from rlinf_b200 import _lib as L
lib = L.load()
for n, IN in [(32, 32), (64, 32), (256, 256)]:
    Z = torch.zeros(n, 256, device='cuda'); H = torch.zeros(n, IN, device='cuda')
    # structured operands: Z[m, o] = (m+1) * 0.001 if o == m % 256 ... use simple patterns
    Z[:, :] = torch.arange(256, device='cuda').float().view(1, 256) * 0.01 + 1.0
    H[:, :] = torch.arange(IN, device='cuda').float().view(1, IN) * 0.1 + 1.0
    Z *= (torch.arange(n, device='cuda').float().view(n, 1) % 3 + 1)
    dW = torch.zeros(256, IN, device='cuda')
    work = torch.empty(2 * n * (256 + IN), device='cuda')
    L.check(lib.rb200_tc_wgrad_h(L.ptr(Z), L.ptr(H), L.ptr(dW), n, IN, None, L.stream_ptr()), "w")
    torch.cuda.synchronize()
    ref = Z.double().T @ H.double()
    print(f"n={n} IN={IN} dW absmax {dW.abs().max().item():.4f} ref absmax {ref.abs().max().item():.4f} nonzero {int((dW != 0).sum())}/{dW.numel()}")
    print(" dW[0,:4]", dW[0, :4].tolist(), "ref", ref[0, :4].tolist())
    print(" dW[1,:4]", dW[1, :4].tolist(), "ref", ref[1, :4].tolist())
    print(" dW[128,:4]", dW[128, :4].tolist(), "ref", ref[128, :4].tolist())
    r = (dW.double() / ref)
    print(" ratio stats", r.min().item(), r.max().item())
