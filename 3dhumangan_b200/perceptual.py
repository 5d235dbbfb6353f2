"""VGG16 perceptual loss on sm_90a: the reference's `VGGPerceptualLoss` (lib/components/perceptual_loss.py), differentiable
w.r.t. its input.

Same constructor (plus `weights`), same `forward(input, target)` -> list of 4 scalar losses, same `get_features`, same
state_dict keys (`blocks.l.N.weight / .bias` with torchvision's layer indices, buffers `mean` / `std`).  The network is ONE
autograd node (`_PerceptualLoss`):

    forward    hg_vgg_input (1 -> 3 channels, (x - mean) / std, bilinear resize to 224x224) -> per block: hg_maxpool2x2 (blocks
               1-3), then every 3x3 convolution on hg_conv2d (fp32x3) with its bias in the epilogue and ReLU on hg_bias_act ->
               hg_smooth_l1 against the target's block output.  Every ReLU output is saved.
    backward   per block, last to first: hg_vgg_level_bwd (ReLU mask, un-pooling of the gradient from the block above and the
               smooth-L1 gradient in one pass), then each convolution's data gradient on hg_conv2d with the rotated filter and
               the ReLU masks inside the block on hg_bias_act_grad; finally hg_vgg_input_adjoint down to the input image.

The VGG weights are frozen, as in the reference (:16-18): no weight gradient is ever launched, and a VGG parameter that
requires grad under autograd raises.  The operand images of the convolutions (and of their rotated filters) are packed
once and again only when a weight changes (data pointer or version counter: `load_state_dict`, `.to()`, in-place edits of
the parameter; an edit through `.data` bypasses the version counter and is not seen).

Weights are never downloaded: `weights=None` reads torchvision's cached `vgg16-397923af.pth` under
`torch.hub.get_dir()/checkpoints` and raises, naming that path, when it is missing.
"""
from __future__ import annotations

import os
from collections import OrderedDict

import torch

from . import abi
from .modules.discriminator_train import _pack, _rot
from .ops import bias_act as _ba

LAYERS = ((0, 2), (5, 7), (10, 12, 14), (17, 19, 21))         # convolutions of VGG16 features[:4], [4:9], [9:16], [16:23]
CHANNELS = {0: (3, 64), 2: (64, 64), 5: (64, 128), 7: (128, 128), 10: (128, 256), 12: (256, 256), 14: (256, 256),
            17: (256, 512), 19: (512, 512), 21: (512, 512)}
WEIGHTS_FILE = "vgg16-397923af.pth"
_RELU = (2, 0.0, 1.0, -1.0)          # hg_bias_act: relu, gain 1, no clamp


def default_weights_path():
    """Where `torchvision.models.vgg16(pretrained=True)` caches its weights."""
    return os.path.join(torch.hub.get_dir(), "checkpoints", WEIGHTS_FILE)


class _Conv3x3(torch.nn.Module):
    """Parameter holder of one frozen VGG convolution (the kernels read the parameters; this module has no forward)."""

    def __init__(self, cin, cout):
        super().__init__()
        self.weight = torch.nn.Parameter(torch.zeros(cout, cin, 3, 3), requires_grad=False)
        self.bias = torch.nn.Parameter(torch.zeros(cout), requires_grad=False)


def _maxpool(x):
    B, C, H, W = x.shape
    y = torch.empty(B, C, H // 2, W // 2, dtype=torch.float32, device=x.device)
    abi.call("hg_maxpool2x2", abi.ptr(x), abi.ptr(y), B * C, H, W, abi.stream())
    return y


class _PerceptualLoss(torch.autograd.Function):
    """(input [B,C,H,W], module, 4 target block outputs) -> 4 smooth-L1 losses; the gradient reaches `input` only."""

    @staticmethod
    @torch.amp.custom_fwd(device_type="cuda", cast_inputs=torch.float32)
    def forward(ctx, x, net, t0, t1, t2, t3):
        keep = ctx.needs_input_grad[0]
        imgs = net._images()
        outs, acts = net._run(x, imgs, keep)
        ts = [t.contiguous() for t in (t0, t1, t2, t3)]
        for o, t in zip(outs, ts):
            if t.shape != o.shape:
                raise RuntimeError(f"hg3d: target features {tuple(t.shape)} do not match the input's {tuple(o.shape)}")
        ws = torch.empty(2 * torch.cuda.get_device_properties(x.device).multi_processor_count, dtype=torch.float64, device=x.device)
        losses = []
        with torch.cuda.device_of(x):
            for o, t in zip(outs, ts):
                loss = torch.empty(1, dtype=torch.float32, device=x.device)
                abi.call("hg_smooth_l1", abi.ptr(o), abi.ptr(t), o.numel(), abi.ptr(loss), abi.ptr(ws), abi.stream())
                losses.append(loss.reshape(()))
        if keep:
            ctx.net, ctx.imgs, ctx.in_shape = net, imgs, tuple(x.shape)
            ctx.save_for_backward(*acts, *ts)
        return tuple(losses)

    @staticmethod
    @torch.amp.custom_bwd(device_type="cuda")
    @torch.autograd.function.once_differentiable
    def backward(ctx, *gs):
        saved = ctx.saved_tensors
        dx = ctx.net._backward(ctx.imgs, saved[:10], saved[10:], [g.float().contiguous() for g in gs], ctx.in_shape)
        return dx, None, None, None, None, None


class VGGPerceptualLoss(torch.nn.Module):
    """Drop-in for lib/components/perceptual_loss.py's VGGPerceptualLoss.  Inputs are images in [0, 1], [B,1|3,H,W].
    weights: None (torchvision's cached file), a path to that file, or a state_dict in torchvision's `features.N.*` keys."""

    def __init__(self, resize=True, weights=None):
        super().__init__()
        blocks = []
        for idxs in LAYERS:
            blk = torch.nn.Module()
            for i in idxs:
                blk.add_module(str(i), _Conv3x3(*CHANNELS[i]))
            blocks.append(blk)
        self.blocks = torch.nn.ModuleList(blocks)
        self.resize = resize
        self.register_buffer("mean", torch.tensor([0.485, 0.456, 0.406]).view(1, 3, 1, 1))
        self.register_buffer("std", torch.tensor([0.229, 0.224, 0.225]).view(1, 3, 1, 1))
        self._packed = None
        if weights is None or isinstance(weights, (str, os.PathLike)):
            path = default_weights_path() if weights is None else os.fspath(weights)
            if not os.path.isfile(path):
                raise RuntimeError(f"hg3d: VGG16 weights not found at {path}: place torchvision's {WEIGHTS_FILE} there or pass "
                                   "`weights=` (a path or a state_dict); they are never downloaded")
            weights = torch.load(path, map_location="cpu", weights_only=True)
        self.load_torchvision(weights)

    @torch.no_grad()
    def load_torchvision(self, state):
        """Copy the convolutions of features[:23] from a torchvision VGG16 state_dict (`features.N.weight / .bias`)."""
        for l, idxs in enumerate(LAYERS):
            for i in idxs:
                conv = self.blocks[l]._modules[str(i)]
                for name in ("weight", "bias"):
                    key = f"features.{i}.{name}"
                    if key not in state:
                        raise RuntimeError(f"hg3d: VGG16 state_dict has no {key!r}")
                    getattr(conv, name).copy_(state[key])

    def _convs(self):
        return [self.blocks[l]._modules[str(i)] for l, idxs in enumerate(LAYERS) for i in idxs]

    def _images(self):
        """[((img, Nb), (rotated img, Nb))] per convolution, packed again only when a weight tensor changed."""
        convs = self._convs()
        key = tuple((c.weight.data_ptr(), c.weight._version, str(c.weight.device)) for c in convs)
        if self._packed is None or self._packed[0] != key:
            with torch.no_grad():
                imgs = [(_pack(c.weight.float()), _pack(_rot(c.weight.float()))) for c in convs]
            self._packed = (key, imgs)
        return self._packed[1]

    def _check(self, x):
        abi.require_device()
        if x.dim() != 4 or x.shape[1] not in (1, 3):
            raise RuntimeError(f"hg3d: VGGPerceptualLoss takes [B,1|3,H,W] images (got {tuple(x.shape)})")
        if torch.is_grad_enabled() and any(p.requires_grad for p in self.parameters()):
            raise RuntimeError("hg3d: gradients w.r.t. the VGG16 weights are not built (the reference freezes them)")

    def _run(self, x, imgs, keep):
        """x [B,C,H,W] -> (the four block outputs, the ten ReLU outputs when `keep`)."""
        x = x.float().contiguous()
        B, C, H, W = x.shape
        Ho, Wo = (224, 224) if self.resize else (H, W)
        mean = self.mean.float().reshape(3).contiguous()
        std = self.std.float().reshape(3).contiguous()
        h = torch.empty(B, 3, Ho, Wo, dtype=torch.float32, device=x.device)
        outs, acts = [], []
        k = 0
        with torch.cuda.device_of(x):
            abi.call("hg_vgg_input", abi.ptr(x), C, B, H, W, abi.ptr(mean), abi.ptr(std), abi.ptr(h), Ho, Wo, abi.stream())
            for l, idxs in enumerate(LAYERS):
                if l > 0:
                    h = _maxpool(h)
                for i in idxs:
                    conv = self.blocks[l]._modules[str(i)]
                    img, Nb = imgs[k][0]
                    h = abi.conv2d(h, img, CHANNELS[i][1], Nb, ksize=3, H=h.shape[2], W=h.shape[3],
                                   bias=conv.bias.float().contiguous(), passes=3)
                    h = _ba._launch_fwd(h, None, 1, _RELU)
                    if keep:
                        acts.append(h)
                    k += 1
                outs.append(h)
        return outs, acts

    def _backward(self, imgs, acts, ts, gs, in_shape):
        """Data-gradient chain from the four losses' incoming gradients `gs` (device scalars) down to the input image."""
        B, C, H, W = in_shape
        ends = [sum(len(b) for b in LAYERS[:l + 1]) - 1 for l in range(4)]
        dev = acts[0].device
        dpool = None
        with torch.cuda.device_of(acts[0]):
            for l in reversed(range(4)):
                y = acts[ends[l]]
                dpre = torch.empty_like(y)
                abi.call("hg_vgg_level_bwd", abi.ptr(y), abi.ptr(ts[l]), abi.ptr(dpool), abi.ptr(gs[l]), 1.0 / y.numel(),
                         abi.ptr(dpre), y.shape[0] * y.shape[1], y.shape[2], y.shape[3], abi.stream())
                idxs = LAYERS[l]
                for j in reversed(range(len(idxs))):
                    k = ends[l] - (len(idxs) - 1 - j)
                    img, Nb = imgs[k][1]
                    din = abi.conv2d(dpre, img, CHANNELS[idxs[j]][0], Nb, ksize=3, H=y.shape[2], W=y.shape[3], passes=3)
                    if j > 0:
                        dpre = _ba._launch_grad(din, None, None, acts[k - 1], None, 1, 1, _RELU)
                    else:
                        dpool = din
            std = self.std.float().reshape(3).contiguous()
            dx = torch.empty(B, C, H, W, dtype=torch.float32, device=dev)
            abi.call("hg_vgg_input_adjoint", abi.ptr(dpool), B, dpool.shape[2], dpool.shape[3], abi.ptr(std), abi.ptr(dx), C, H, W,
                     abi.stream())
        return dx

    def target_features(self, target):
        """The four block outputs of a fixed target (no gradient), for `loss`: an inversion computes them once."""
        self._check(target)
        if torch.is_grad_enabled() and target.requires_grad:
            raise RuntimeError("hg3d: gradients w.r.t. the perceptual loss's target are not built")
        with torch.no_grad():
            return self._run(target, self._images(), False)[0]

    def loss(self, input, target_features, lambdas=None):
        """-> the four smooth-L1 losses against `target_features(target)` (a list), or sum_i lambdas[i] * L_i when `lambdas`
        is given.  Differentiable w.r.t. `input`."""
        self._check(input)
        if len(target_features) != 4:
            raise RuntimeError("hg3d: expected the four block outputs of `target_features`")
        losses = list(_PerceptualLoss.apply(input, self, *target_features))
        if lambdas is None:
            return losses
        if len(lambdas) != 4:
            raise RuntimeError("hg3d: perceptual lambdas are one weight per block (4)")
        return sum(float(w) * v for w, v in zip(lambdas, losses))

    def forward(self, input, target):
        """The reference's forward (:26-49): the target's features are computed on every call."""
        return self.loss(input, self.target_features(target))

    def get_features(self, input):
        """The relu4_3 features of `input` (:51-63); not differentiable here."""
        self._check(input)
        if torch.is_grad_enabled() and input.requires_grad:
            raise RuntimeError("hg3d: gradients through VGGPerceptualLoss.get_features are not built (use `loss`)")
        with torch.no_grad():
            return self._run(input, self._images(), False)[0][-1]
