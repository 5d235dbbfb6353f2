"""Training-mode U-Net discriminator: autograd graph over the sm_90a primitives.

The inference path (`discriminator_ops.discriminator_forward`) folds LeakyReLU / up-sample / concat / residual into
the convolution kernel.  For training the same network is an ordinary autograd graph whose nodes are this library's
ops, so that first-order gradients w.r.t. images (generator step) and parameters (discriminator step) come out of
`loss.backward()`:

    convolution      `Conv2dSame`  forward `hg_conv2d`, data gradient `hg_conv2d` with the rotated / transposed filter,
                                   weight gradient `ConvWgrad` = `hg_conv2d_wgrad_taps` (wgmma); both backward nodes
                                   are themselves differentiable (R1 double backward, phase_trainer.py:259-294)
    LeakyReLU        `ops.bias_act` (hg_bias_act / hg_bias_act_grad)
    avg-pool / nearest up-sample   `ops.upfirdn2d` with a 2x2 box filter (its backward is another upfirdn pass)
    spectral norm    `hg_spectral_norm` (one launch for all layers: power iteration, buffers in place) + a differentiable
                     W / sigma scale node (`synthesis_ops.SpectralScale`)
    residual add, channel concat, the full-extent `latent_layer`: torch (`+`, `cat`, one library GEMM)

Mirrors UNetDiscriminator.forward / ResBlock.forward (lib/discriminators/unet_discriminators.py:47-72, 125-160).
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

from .. import abi
from ..ops import bias_act as _ba
from ..ops import upfirdn2d as _uf


def _pack(w):
    """[Cout,Cin,k,k] -> packed operand image of hg_conv2d (tap-major K)."""
    Cout, Cin, kh, kw = w.shape
    wm = torch.empty(Cout, kh * kw * Cin, dtype=torch.float32, device=w.device)      # explicit strides (K, 1) even for K == 1
    wm.copy_(w.permute(0, 2, 3, 1).reshape(Cout, kh * kw * Cin))
    Nb = min(256, (Cout + 15) // 16 * 16)
    return abi.pack_weight(wm, Nb=Nb)


def _conv_raw(x, w, bias, passes):
    """Stride-1 'same' convolution through hg_conv2d; output channels in chunks of 512 (two N blocks per launch)."""
    B, Cin, H, W = x.shape
    Cout, k = w.shape[0], w.shape[2]
    outs = []
    for c0 in range(0, Cout, 512):
        wc = w[c0:c0 + 512]
        img, Nb = _pack(wc)
        outs.append(abi.conv2d(x, img, wc.shape[0], Nb, ksize=k, H=H, W=W, bias=None if bias is None else bias[c0:c0 + 512].contiguous(),
                               passes=passes))
    return outs[0] if len(outs) == 1 else torch.cat(outs, 1)


def _rot(w):
    """Filter of the data gradient: 180-degree rotation, input and output channels exchanged (differentiable in w)."""
    return w.flip(2, 3).transpose(0, 1)


class Conv2dSame(torch.autograd.Function):
    """Stride-1 'same' convolution y = w * x + b.  Differentiable to ANY order: its backward is composed of `Conv2dSame`
    (data gradient: the same kernel with the rotated filter) and `ConvWgrad` nodes, whose backwards are again those two --
    which is what the reference trainer's R1 term needs (`torch.autograd.grad(..., create_graph=True)` through the
    discriminator on the do_r1 phases, then `d_loss.backward()` through that graph: phase_trainer.py:259-294)."""

    @staticmethod
    @torch.amp.custom_fwd(device_type="cuda", cast_inputs=torch.float32)
    def forward(ctx, x, w, bias, passes):
        x = x.float().contiguous()
        ctx.save_for_backward(x, w)
        ctx.passes, ctx.has_bias = passes, bias is not None
        return _conv_raw(x, w.detach().float(), None if bias is None else bias.detach().float(), passes)

    @staticmethod
    @torch.amp.custom_bwd(device_type="cuda")
    def backward(ctx, dy):
        x, w = ctx.saved_tensors
        dx = dw = db = None
        if ctx.needs_input_grad[0]:
            dx = Conv2dSame.apply(dy, _rot(w), None, ctx.passes)
        if ctx.needs_input_grad[1] or (ctx.has_bias and ctx.needs_input_grad[2]):
            dw, db = ConvWgrad.apply(dy, x, w.shape[2], ctx.passes)
            if not ctx.has_bias:
                db = None
        return dx, dw, db, None


class ConvWgrad(torch.autograd.Function):
    """(dy [B,Co,H,W], x [B,Ci,H,W]) -> dw[co,ci,i,j] = sum_{b,p} dy[b,co,p] x[b,ci,p+(i,j)-k//2],  db[co] = sum dy.
    Bilinear in (dy, x); its two gradients are convolutions again."""

    @staticmethod
    @torch.amp.custom_fwd(device_type="cuda", cast_inputs=torch.float32)
    def forward(ctx, dy, x, ksize, passes):
        dy, x = dy.float().contiguous(), x.float().contiguous()
        ctx.save_for_backward(dy, x)
        ctx.passes = passes
        return abi.conv2d_wgrad(dy, x, ksize, passes=passes)

    @staticmethod
    @torch.amp.custom_bwd(device_type="cuda")
    def backward(ctx, ddw, ddb):
        dy, x = ctx.saved_tensors
        g_dy = g_x = None
        if ctx.needs_input_grad[0]:          # d/d dy[b,co,p] = sum_{ci,k} ddw[co,ci,k] x[b,ci,p+k] (+ ddb[co])
            g_dy = Conv2dSame.apply(x, ddw, ddb, ctx.passes)
        if ctx.needs_input_grad[1]:          # d/d x[b,ci,q] = sum_{co,k} ddw[co,ci,k] dy[b,co,q-k]
            g_x = Conv2dSame.apply(dy, _rot(ddw), None, ctx.passes)
        return g_dy, g_x, None, None


def _lrelu(x, rec=None):
    if rec is not None:
        rec.append(x.detach() > 0)
    return _ba.bias_act(x, None, act="lrelu", alpha=0.2, gain=1.0)


class _Resample2x(torch.autograd.Function):
    """avg_pool2d(x, 2) (up=False) / nearest 2x up-sample (up=True) on `hg_resample2x`; each is the other's adjoint up to
    a factor, so the backward is the other direction of the same kernel (and differentiable again)."""

    @staticmethod
    def forward(ctx, x, up, scale):
        ctx.up, ctx.scale = up, scale
        return abi.resample2x(x.float().contiguous(), up, scale)

    @staticmethod
    def backward(ctx, dy):
        # y = s * U x  =>  dx = s * U^T dy with U^T = block sum;   y = s * P x (block sum)  =>  dx = s * P^T dy = s * nearest(dy)
        return _Resample2x.apply(dy, not ctx.up, ctx.scale), None, None


def _pool(x):
    W = x.shape[3]
    if x.shape[2] % 2 or W % 4:          # odd sizes / tiny maps: the general resampler (a 2x2 box through upfirdn2d)
        return _uf.upfirdn2d(x, torch.full((2, 2), 0.25, device=x.device), down=2)
    return _Resample2x.apply(x, False, 0.25)


def _up(x):
    if x.shape[3] % 2:
        return _uf.upfirdn2d(x, torch.ones(2, 2, device=x.device), up=2, padding=[1, 0, 1, 0])
    return _Resample2x.apply(x, True, 1.0)


def discriminator_forward_train(module, images, passes=3, masks=None):
    """Differentiable forward.  `masks`: optional list that receives the LeakyReLU masks in application order (tests)."""
    abi.require_device()
    P = dict(list(module.named_parameters()) + list(module.named_buffers()))
    training = module.training
    sn = not module._cfg.get("disable_spectral_norm", False)
    nb = module.num_blocks
    B = images.shape[0]
    from .discriminator_ops import sn_layer_names
    from .synthesis_ops import sn_weights
    w_sn = sn_weights(P, [n + "." for n in sn_layer_names(P)], training) if sn else {}

    def conv(name, x, spectral=True):
        w = w_sn[name + "."] if (sn and spectral) else P[name + ".weight"]
        return Conv2dSame.apply(x, w, P[name + ".bias"], passes)

    x = images.float()
    skips = []
    for i in range(nb):
        blk = f"body_down.{i}"
        learned = (blk + ".conv_s.bias") in P
        if i == 0:                                   # first block: pool, then the 1x1 shortcut (:58-63)
            s = _pool(x)
            if learned:
                s = conv(blk + ".conv_s", s)
            dx = conv(blk + ".conv1", x)
        else:
            s = conv(blk + ".conv_s", x) if learned else x
            s = _pool(s)
            dx = conv(blk + ".conv1.1", _lrelu(x, masks))
        dx = conv(blk + ".conv2.1", _lrelu(dx, masks))
        x = s + _pool(dx)
        skips.append(x)
    if min(x.shape[2:4]) > 1:
        w = P["latent_layer.weight"]
        latents = F.linear(x.reshape(B, -1), w.reshape(w.shape[0], -1), P["latent_layer.bias"])
    else:
        latents = torch.zeros(B, module.latent_dim, dtype=x.dtype, device=x.device)
    for i in range(nb):
        blk = f"body_up.{i}"
        xin = x if i == 0 else torch.cat((skips[-i - 1], x), 1)
        learned = (blk + ".conv_s.bias") in P
        # shortcut: conv_s(up(x)) == up(conv_s(x)) exactly (1x1 convolution, nearest up-sampling): convolve at the low resolution
        s = _up(conv(blk + ".conv_s", xin)) if learned else _up(xin)
        dx = conv(blk + ".conv1.2", _up(_lrelu(xin, masks)))
        dx = conv(blk + ".conv2.1", _lrelu(dx, masks))
        x = s + dx
    pred = conv("layer_up_last", x, spectral=False)
    seg = conv("output_layer", x, spectral=False)
    sd = module.semantic_dim
    out = {"prediction": pred, "latents": latents, "segments": seg[:, sd:]}
    if sd > 0:
        out["semantics"] = seg[:, :sd]
    return out
