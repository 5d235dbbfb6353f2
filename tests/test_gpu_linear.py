"""wgmma primitives end to end: weight packing + hg_linear vs a plain fp32 torch reference."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _ref(X, W, b):
    return (X.double() @ W.double().t() + (b.double() if b is not None else 0)).float()


@pytest.mark.parametrize("M,K,N,Nb,passes,tol", [
    (128, 64, 256, 256, 3, 2e-5),
    (128, 256, 256, 256, 3, 2e-5),
    (1000, 256, 768, 256, 3, 2e-5),     # ragged M, 3 N-blocks (style-projection shape family)
    (300, 192, 48, 48, 3, 2e-5),        # small N block, K not a multiple of 256
    (128 * 160, 256, 256, 256, 3, 2e-5),  # more tiles than SMs: persistent loop + barrier phases
    (512, 256, 256, 256, 1, 8e-3),      # plain bf16 mode
])
def test_linear_matches_fp32(pkg, M, K, N, Nb, passes, tol):
    from importlib import import_module
    abi = import_module("3dhumangan_b200.abi")
    abi.require_device()
    g = torch.Generator(device="cuda").manual_seed(M + K + N)
    X = torch.randn(M, K, device="cuda", generator=g)
    W = torch.randn(N, K, device="cuda", generator=g) / K ** 0.5
    b = torch.randn(N, device="cuda", generator=g)
    img, Nb_ = abi.pack_weight(W, Nb=Nb)
    Y = abi.linear(X, img, Nb_, N, bias=b, passes=passes)
    torch.cuda.synchronize()
    ref = _ref(X, W, b)
    err = (Y - ref).norm() / ref.norm()
    assert torch.isfinite(Y).all()
    assert err < tol, f"rel-L2 {err:.3e}"
    # element-wise bound too (catches a single mis-addressed tile)
    assert (Y - ref).abs().max() < tol * 50 * ref.abs().max()
