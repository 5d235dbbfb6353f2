"""Dense layers of the two mapping networks on the wgmma GEMM (`hg_linear`), differentiable.

    y = x @ (gain * W)^T + b          x [M,K], W [N,K], b [N]

(reference: `nn.Linear` inside MappingNetwork, lib/components/mapping_networks.py:13-41, and
`FullyConnectedLayer.forward` :107-121 with its equalised-learning-rate gains).  Forward, data gradient and weight
gradient are all the same kernel: dX = dY @ (gain W), dW = gain * dY^T @ X (a GEMM whose contraction runs over the batch).
`hg_linear` contracts over at most 256 columns per launch, so longer contractions (hidden_dim 384 / 420, or a batch of
10 000 latents in `generate_avg_latent`) are split and summed.  No cuBLAS / ATen matmul on this path.
"""
import torch

from .. import abi

_KMAX = 256


def _rows(t):
    """Row-major copy with canonical strides (a [K,1] transpose reports is_contiguous() with stride(1) == K)."""
    if t.stride(1) == 1 and t.stride(0) == t.shape[1] and (t.data_ptr() % 16) == 0:
        return t
    out = torch.empty(t.shape, dtype=torch.float32, device=t.device)
    out.copy_(t)
    return out


def _gemm_nt(a, b, scale=1.0, bias=None, passes=3):
    """a [M,K] @ (scale * b [N,K])^T (+ bias) -> [M,N] fp32, through hg_linear in contraction slices of <= 256."""
    a = a.float()
    b = b.float()
    M, K = a.shape
    N = b.shape[0]
    out = None
    for k0 in range(0, K, _KMAX):
        k1 = min(K, k0 + _KMAX)
        img, Nb = abi.pack_weight(_rows(b[:, k0:k1]), scale=float(scale))
        xa = a[:, k0:k1]
        if xa.stride(1) != 1 or (xa.data_ptr() % 16) != 0 or xa.shape[0] == 1:
            xa = _rows(xa)
        part = abi.linear(xa, img, Nb, N, bias=bias if k0 == 0 else None, passes=passes)
        out = part if out is None else out.add_(part)
    return out


class Dense(torch.autograd.Function):
    @staticmethod
    @torch.amp.custom_fwd(device_type="cuda", cast_inputs=torch.float32)
    def forward(ctx, x, w, bias, gain, passes):
        abi.require_device()
        ctx.save_for_backward(x, w)
        ctx.gain, ctx.passes, ctx.has_bias = float(gain), passes, bias is not None
        return _gemm_nt(x.detach(), w.detach(), gain, None if bias is None else bias.detach().float().contiguous(), passes)

    @staticmethod
    @torch.amp.custom_bwd(device_type="cuda")
    def backward(ctx, dy):
        x, w = ctx.saved_tensors
        dx = dw = db = None
        if ctx.needs_input_grad[0]:                       # dX = dY @ (gain W): "weight" of the GEMM is W^T
            dx = Dense.apply(dy, w.t(), None, ctx.gain, ctx.passes)
        if ctx.needs_input_grad[1]:                       # dW = gain * dY^T @ X: contraction over the batch
            dw = Dense.apply(dy.t(), x.t(), None, ctx.gain, ctx.passes)
        if ctx.has_bias and ctx.needs_input_grad[2]:
            db = dy.sum(0)
        return dx, dw, db, None, None


def dense(x, w, bias=None, gain=1.0, passes=3):
    """x [..., K] -> [..., N]."""
    lead = x.shape[:-1]
    y = Dense.apply(x.reshape(-1, x.shape[-1]), w, bias, gain, passes)
    return y.reshape(*lead, w.shape[0])
