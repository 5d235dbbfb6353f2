"""`lib.discriminators` surface: UNetDiscriminator (reference: lib/discriminators/unet_discriminators.py:7-160).

Parameter tree, names and initialisation follow the reference (spectral-normed 3x3 / 1x1 convs in
`body_down` / `body_up` ResBlocks, plain heads `layer_up_last`, `output_layer`, `latent_layer`), so a
reference `state_dict` loads strictly.  The forward pass runs the implicit-GEMM convolution kernels
of csrc/dconv.cu when they are present in the library; there is no cuDNN / eager fallback.
"""
from __future__ import annotations

import math

import torch
import torch.nn as nn


def _conv(cin, cout, k, spectral):
    layer = nn.Conv2d(cin, cout, k, stride=1, padding=k // 2)
    return nn.utils.spectral_norm(layer) if spectral else layer


class ResBlock(nn.Module):
    """Parameter holder of one residual block (unet_discriminators.py:7-72).  The positions inside the Sequentials
    fix the state_dict keys: `conv1.1.*` (down), `conv1.2.*` (up), `conv1.*` (first block), `conv2.1.*`."""

    def __init__(self, fin, fout, up_or_down, first=False, **kwargs):
        super().__init__()
        spectral = not kwargs.get("disable_spectral_norm", False)
        self.up_or_down, self.first, self.learned_shortcut = up_or_down, first, fin != fout
        head = _conv(fin, fout, 3, spectral)
        if not first:
            pre = [nn.LeakyReLU(0.2, False)] + ([nn.Upsample(scale_factor=2)] if up_or_down > 0 else [])
            head = nn.Sequential(*pre, head)
        self.conv1 = head
        self.conv2 = nn.Sequential(nn.LeakyReLU(0.2, False), _conv(fout, fout, 3, spectral))
        if self.learned_shortcut:
            self.conv_s = _conv(fin, fout, 1, spectral)


def _channel_plan(cin, nb):
    """(down, up) lists of (in, out) channels: the up path consumes [skip | x] concatenations (:96-113)."""
    width = [cin, 128, 128, 256, 256, 512, 512, 512, 512]
    down = [(width[i], width[i + 1]) for i in range(nb)]
    up = [(width[nb], width[nb - 1])]
    up += [(2 * width[nb - i], width[nb - i - 1]) for i in range(1, nb - 1)]
    up += [(2 * width[1], 64)]
    return width, down, up


class UNetDiscriminator(nn.Module):
    def __init__(self, **kwargs):
        super().__init__()
        self.epoch, self.step = 0, 0
        self.semantic_dim, self.label_dim = kwargs.get("semantic_dim", 0), kwargs.get("label_dim", 0)
        self.output_dim = self.semantic_dim + self.label_dim
        self.latent_dim = kwargs["latent_dim"]
        Hg, Wg = kwargs["gen_height"], kwargs["gen_width"]
        self.num_blocks = nb = min(kwargs.get("discriminator_blocks", 6), int(math.log2(max(Hg, Wg))) - 1)
        self.channels, down, up = _channel_plan(6 if kwargs.get("dual_discrimination", False) else 3, nb)
        # registration order (up before down, then the heads) is the reference's state_dict order
        self.body_up = nn.ModuleList(ResBlock(i, o, 1, **kwargs) for i, o in up)
        self.body_down = nn.ModuleList(ResBlock(i, o, -1, first=(k == 0), **kwargs) for k, (i, o) in enumerate(down))
        self.layer_up_last = nn.Conv2d(64, 1, 1)
        self.output_layer = nn.Conv2d(64, self.output_dim, 1)
        self.latent_layer = nn.Conv2d(self.channels[nb], self.latent_dim, (Hg >> nb, Wg >> nb))
        # The reference calls `self.apply(kaiming_leaky_init)` (:121, :74-78).  On a spectral-normed conv `module.weight` is
        # `weight_orig.data` at that point (torch.nn.utils.spectral_norm registers the plain attribute from the same
        # storage), so the in-place kaiming draw re-initialises `weight_orig` of all 33 spectral-normed convolutions as
        # well as the three plain heads: std = sqrt(2 / (1 + 0.2^2)) / sqrt(fan_in).
        for m in self.modules():
            if isinstance(m, nn.Conv2d):
                w = m.weight_orig if hasattr(m, "weight_orig") else m.weight
                with torch.no_grad():
                    nn.init.kaiming_normal_(w, a=0.2, mode="fan_in", nonlinearity="leaky_relu")
        with torch.no_grad():
            self.output_layer.weight.mul_(0.25)
        self._cfg = {k: v for k, v in kwargs.items() if isinstance(k, str)}

    def forward(self, images, conditions, alpha, **kwargs):
        """-> {"prediction": [B,1,H,W], "latents": [B,L], "segments": [B,label_dim,H,W]} (:125-160).
        `conditions`, `alpha` and other kwargs are accepted and ignored, as in the reference."""
        from . import discriminator_ops
        from .generator import _precision_passes
        if torch.is_grad_enabled() and (images.requires_grad or any(p.requires_grad for p in self.parameters())):
            # discriminator / generator step of the trainer: the autograd graph over the sm_90a primitives
            from . import discriminator_train
            return discriminator_train.discriminator_forward_train(self, images, passes=_precision_passes(kwargs),
                                                                   masks=kwargs.get("hg_record_masks"))
        passes = _precision_passes(kwargs)
        return discriminator_ops.discriminator_forward(self, images, passes=passes)
