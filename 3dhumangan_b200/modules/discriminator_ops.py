"""Host-side schedule of the U-Net discriminator on the sm_90a convolution kernels (csrc/dconv.cu).

Mirrors `UNetDiscriminator.forward` / `ResBlock.forward` (lib/discriminators/unet_discriminators.py:47-72,
125-160).  Per ResBlock: two implicit-GEMM 3x3 convolutions with LeakyReLU / nearest up-sample / channel
concat folded into the operand producer and the residual add folded into the second conv's epilogue (up
path) or into the pooling kernel (down path); the two 1x1 heads run as ONE convolution with 27 outputs.
Spectral normalisation (one power iteration per training forward, buffers updated in place) is ONE launch of
`hg_spectral_norm` for all 30 convolutions; 1/sigma is applied while packing the bf16 operand image.
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

from .. import abi


def sn_layer_names(P):
    """State-dict prefixes (without the trailing dot) of the spectral-normed convolutions, in registration order."""
    return [k[:-len(".weight_orig")] for k in P if k.endswith(".weight_orig")]


def _sigma_inv_all(P, training):
    """{name: 1/sigma [1]} for every spectral-normed convolution: ONE `hg_spectral_norm` launch (power iteration with the
    u / v buffers updated in place when training), unet_discriminators.py:18."""
    names = sn_layer_names(P)
    inv = abi.spectral_norm([P[n + ".weight_orig"].detach() for n in names], [P[n + ".weight_u"] for n in names],
                            [P[n + ".weight_v"] for n in names], training)
    return {n: inv[i:i + 1] for i, n in enumerate(names)}


def _pack_conv(w, scale_dev=None):
    """[Cout,Cin,kh,kw] -> packed [Cout, tap*Cin] operand image (K padded to 64 for the 3-channel stem)."""
    Cout, Cin, kh, kw = w.shape
    wm = w.permute(0, 2, 3, 1).reshape(Cout, kh * kw * Cin).contiguous().float()
    Nb = min(256, (Cout + 15) // 16 * 16)
    img, Nb = abi.pack_weight(wm, Nb=Nb, scale_dev=scale_dev)
    return img, Nb


@torch.no_grad()
def discriminator_forward(module, images, passes=None):
    abi.require_device()
    from .generator import _precision_passes
    passes = _precision_passes() if passes is None else passes
    training = module.training
    P = dict(list(module.named_parameters()) + list(module.named_buffers()))
    x = images.float().contiguous()
    B = x.shape[0]
    nb = module.num_blocks
    sn = not module._cfg.get("disable_spectral_norm", False)
    inv_sigma = _sigma_inv_all(P, training) if sn else {}

    def conv(name, x1, *, ksize, H, W, x2=None, up2=False, pre_lrelu=False, residual=None, res_up2=False):
        if sn:
            img, Nb = _pack_conv(P[name + ".weight_orig"], inv_sigma[name])
        else:
            img, Nb = _pack_conv(P[name + ".weight"])
        Cout = P[name + ".bias"].shape[0]
        return abi.conv2d(x1, img, Cout, Nb, ksize=ksize, H=H, W=W, x2=x2, up2=up2, pre_lrelu=pre_lrelu,
                          bias=P[name + ".bias"], residual=residual, res_up2=res_up2, passes=passes)

    skips = []
    for i in range(nb):
        blk = f"body_down.{i}"
        H, W = x.shape[2], x.shape[3]
        learned = (blk + ".conv_s.bias") in P
        if i == 0:                                  # first block pools BEFORE the 1x1 shortcut (:58-63)
            s = abi.pool_add(x, True)
            if learned:
                s = conv(blk + ".conv_s", s, ksize=1, H=H // 2, W=W // 2)
            dx = conv(blk + ".conv1", x, ksize=3, H=H, W=W)
            dx = conv(blk + ".conv2.1", dx, ksize=3, H=H, W=W, pre_lrelu=True)
            x = abi.pool_add(dx, True, s, False)
        else:                                       # 1x1 shortcut, then pool (:65-70)
            s = conv(blk + ".conv_s", x, ksize=1, H=H, W=W) if learned else x
            dx = conv(blk + ".conv1.1", x, ksize=3, H=H, W=W, pre_lrelu=True)
            dx = conv(blk + ".conv2.1", dx, ksize=3, H=H, W=W, pre_lrelu=True)
            x = abi.pool_add(dx, True, s, True)
        skips.append(x)

    if min(x.shape[2:4]) > 1:
        w = P["latent_layer.weight"]
        latents = abi.dense(x.reshape(B, -1), w.reshape(w.shape[0], -1).contiguous(), P["latent_layer.bias"])
    else:
        latents = torch.zeros(B, module.latent_dim, dtype=x.dtype, device=x.device)

    for i in range(nb):
        blk = f"body_up.{i}"
        x1, x2 = (x, None) if i == 0 else (skips[-i - 1], x)
        H, W = x1.shape[2] * 2, x1.shape[3] * 2
        learned = (blk + ".conv_s.bias") in P
        if learned:
            # shortcut = conv_s(up(x)) (:65-67) == up(conv_s(x)): a 1x1 convolution commutes with nearest up-sampling exactly, so it
            # runs at the LOW resolution (a quarter of the pixels) and is up-sampled by the residual read of conv2's epilogue
            s = conv(blk + ".conv_s", x1, x2=x2, ksize=1, H=H // 2, W=W // 2)
            res_up2 = True
        else:
            if x2 is not None:
                raise RuntimeError("hg3d: identity shortcut over a concatenated input does not occur in this architecture")
            s, res_up2 = x1, True
        dx = conv(blk + ".conv1.2", x1, x2=x2, ksize=3, H=H, W=W, up2=True, pre_lrelu=True)
        x = conv(blk + ".conv2.1", dx, ksize=3, H=H, W=W, pre_lrelu=True, residual=s, res_up2=res_up2)

    # heads: prediction (1 ch) and segmentation logits (output_dim ch) as one 1x1 convolution
    H, W = x.shape[2], x.shape[3]
    wh = torch.cat([P["layer_up_last.weight"], P["output_layer.weight"]], 0)
    bh = torch.cat([P["layer_up_last.bias"], P["output_layer.bias"]], 0).contiguous()
    img, Nb = _pack_conv(wh)
    heads = abi.conv2d(x, img, wh.shape[0], Nb, ksize=1, H=H, W=W, bias=bh, passes=passes)
    sd = module.semantic_dim
    out = {"prediction": heads[:, :1], "latents": latents, "segments": heads[:, 1 + sd:]}
    if sd > 0:
        out["semantics"] = heads[:, 1:1 + sd]
    return out
