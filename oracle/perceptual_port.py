"""fp64 restatement of the reference's VGG16 perceptual loss (lib/components/perceptual_loss.py) in torch functional ops, and the
seeded VGG16 weights that stand in for the pretrained ones (which are never downloaded) in the fixture and the tests.

`VGGPerceptualLoss.forward(input, target)` (:26-49): a 1-channel input is repeated to 3 channels, normalised with the ImageNet
mean / std, optionally resized to 224x224 (bilinear, align_corners=False), and run through VGG16 `features[:23]` in four blocks
ending at relu1_2, relu2_2, relu3_3 and relu4_3 (a 2x2 max-pool opens blocks 1-3); each block contributes
`smooth_l1_loss(x, y)` (mean, beta = 1) between the input's and the target's features."""
from __future__ import annotations

import math
from collections import OrderedDict

import torch
import torch.nn.functional as F

CFG = [64, 64, "M", 128, 128, "M", 256, 256, 256, "M", 512, 512, 512, "M", 512, 512, 512, "M"]       # torchvision's vgg16
BLOCKS = ((0, 2), (5, 7), (10, 12, 14), (17, 19, 21))       # convolution indices of features[:4], [4:9], [9:16], [16:23]
MEAN = (0.485, 0.456, 0.406)
STD = (0.229, 0.224, 0.225)


def seeded_vgg16_state(seed=0):
    """torchvision's `features.N.weight / .bias` for the 13 convolutions of VGG16, drawn layer by layer from ONE
    torch.Generator(seed): weight = randn * sqrt(2 / (9 Cin)) (He-normal, fan-in), then bias = 0.01 * randn."""
    g = torch.Generator().manual_seed(seed)
    sd = OrderedDict()
    idx, cin = 0, 3
    for v in CFG:
        if v == "M":
            idx += 1
            continue
        sd[f"features.{idx}.weight"] = torch.randn(v, cin, 3, 3, generator=g) * math.sqrt(2.0 / (9 * cin))
        sd[f"features.{idx}.bias"] = 0.01 * torch.randn(v, generator=g)
        idx, cin = idx + 2, v
    return sd


def seeded_vgg16(seed=0, **_):
    """Stand-in for `torchvision.models.vgg16(pretrained=True)`: an object whose `.features` has torchvision's layers and
    indices (Conv2d 3x3 pad 1, ReLU(inplace=True), MaxPool2d(2, 2)) and the seeded weights."""
    layers, cin = [], 3
    for v in CFG:
        if v == "M":
            layers.append(torch.nn.MaxPool2d(kernel_size=2, stride=2))
        else:
            layers += [torch.nn.Conv2d(cin, v, kernel_size=3, padding=1), torch.nn.ReLU(inplace=True)]
            cin = v
    m = torch.nn.Module()
    m.features = torch.nn.Sequential(*layers)
    m.features.load_state_dict({k[len("features."):]: v for k, v in seeded_vgg16_state(seed).items()})
    return m


def module_params(torchvision_state):
    """torchvision `features.N.*` -> the reference module's `blocks.l.N.*` (the convolutions of features[:23] only)."""
    out = OrderedDict()
    for l, idxs in enumerate(BLOCKS):
        for i in idxs:
            for p in ("weight", "bias"):
                out[f"blocks.{l}.{i}.{p}"] = torchvision_state[f"features.{i}.{p}"]
    return out


def transform(x, resize):
    x = x.double()
    if x.shape[1] != 3:
        x = x.repeat(1, 3, 1, 1)
    mean = torch.tensor(MEAN, dtype=x.dtype, device=x.device).view(1, 3, 1, 1)
    x = (x - mean) / torch.tensor(STD, dtype=x.dtype, device=x.device).view(1, 3, 1, 1)
    if resize:
        x = F.interpolate(x, size=(224, 224), mode="bilinear", align_corners=False)
    return x


def features(params, x, resize, masks=None, pre=None, pool_index=None):
    """-> the four block outputs in fp64.  params: `blocks.l.N.weight / .bias`.  masks: 10 boolean tensors that replace the
    ReLUs' (pre-activation > 0) in layer order; pool_index: 3 tensors of flat argmax indices (max_pool2d's return_indices) that
    replace the max-pools' choices (same-mask evaluation of a device result); pre: a list that receives the 10
    pre-activations."""
    h = transform(x, resize)
    outs, k = [], 0
    for l, idxs in enumerate(BLOCKS):
        if l > 0:
            if pool_index is None:
                h = F.max_pool2d(h, kernel_size=2, stride=2)
            else:
                idx = pool_index[l - 1]
                h = h.flatten(2).gather(2, idx.flatten(2)).view(idx.shape)
        for i in idxs:
            h = F.conv2d(h, params[f"blocks.{l}.{i}.weight"].double(), params[f"blocks.{l}.{i}.bias"].double(), padding=1)
            if pre is not None:
                pre.append(h)
            h = F.relu(h) if masks is None else h * masks[k].to(h)
            k += 1
        outs.append(h)
    return outs


def losses(params, x, target, resize, masks=None, pre=None, pool_index=None):
    """The reference's `forward(input, target)`: four smooth-L1 losses, differentiable w.r.t. `x`."""
    fx = features(params, x, resize, masks, pre, pool_index)
    with torch.no_grad():
        ft = features(params, target, resize)
    return [F.smooth_l1_loss(a, b) for a, b in zip(fx, ft)]
