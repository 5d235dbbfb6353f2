"""fp64 restatement of the FID Inception-v3 graph in torch functional ops, with BatchNorm unfolded, and the seeded state that
stands in for pytorch-fid's pretrained weights (which are never downloaded) in the tests.

The architecture is torchvision's `Inception3` (torchvision/models/inception.py: BasicConv2d = conv without bias, BatchNorm
eps 1e-3, ReLU; blocks Mixed_5b .. Mixed_7c) as pytorch-fid's `fid_inception_v3` (pytorch_fid/inception.py) modifies it:
the pool branch of Mixed_5b-d (FIDInceptionA), Mixed_6b-e (FIDInceptionC) and Mixed_7b (FIDInceptionE_1) averages with
count_include_pad=False, Mixed_7c (FIDInceptionE_2) max-pools (3, 1, 1).  pytorch-fid's `InceptionV3` feeds it images in
[0, 1] resized to 299x299 (bilinear, align_corners=False) and mapped to 2x - 1, and returns the 2048-d global average of
Mixed_7c's output."""
from __future__ import annotations

import math
from collections import OrderedDict

import torch
import torch.nn.functional as F

EPS = 1e-3
BLOCKS = ("Mixed_5b", "Mixed_5c", "Mixed_5d", "Mixed_6a", "Mixed_6b", "Mixed_6c", "Mixed_6d", "Mixed_6e", "Mixed_7a",
          "Mixed_7b", "Mixed_7c")


def _pair(v):
    return (v, v) if isinstance(v, int) else tuple(v)


class _Graph:
    """conv(name, x, cout, k, stride, padding) = relu(bn(conv(x))) in fp64 from `sd` (torchvision names).  With `make` a
    missing layer is created first: make(name, x, cin, cout, kh, kw, stride, padding) fills `sd`."""

    def __init__(self, sd, make=None):
        self.sd, self.make = sd, make

    def conv(self, name, x, cout, k, stride=1, padding=0):
        kh, kw = _pair(k)
        if self.make is not None and f"{name}.conv.weight" not in self.sd:
            self.make(name, x, x.shape[1], cout, kh, kw, stride, _pair(padding))
        p = lambda s: self.sd[f"{name}.{s}"].to(x)
        w = p("conv.weight")
        assert tuple(w.shape) == (cout, x.shape[1], kh, kw), (name, tuple(w.shape))
        y = F.conv2d(x, w, stride=stride, padding=_pair(padding))
        y = F.batch_norm(y, p("bn.running_mean"), p("bn.running_var"), p("bn.weight"), p("bn.bias"), training=False, eps=EPS)
        return F.relu(y)


def stem(g, x):
    """Conv2d_1a_3x3 .. maxpool2: [B,3,299,299] -> [B,192,35,35]."""
    x = g.conv("Conv2d_1a_3x3", x, 32, 3, stride=2)
    x = g.conv("Conv2d_2a_3x3", x, 32, 3)
    x = g.conv("Conv2d_2b_3x3", x, 64, 3, padding=1)
    x = F.max_pool2d(x, 3, 2)
    x = g.conv("Conv2d_3b_1x1", x, 80, 1)
    x = g.conv("Conv2d_4a_3x3", x, 192, 3)
    return F.max_pool2d(x, 3, 2)


def _avg(x):
    return F.avg_pool2d(x, 3, 1, 1, count_include_pad=False)


def inception_a(g, n, x, pool_features):
    b1 = g.conv(f"{n}.branch1x1", x, 64, 1)
    b5 = g.conv(f"{n}.branch5x5_2", g.conv(f"{n}.branch5x5_1", x, 48, 1), 64, 5, padding=2)
    b3 = g.conv(f"{n}.branch3x3dbl_1", x, 64, 1)
    b3 = g.conv(f"{n}.branch3x3dbl_2", b3, 96, 3, padding=1)
    b3 = g.conv(f"{n}.branch3x3dbl_3", b3, 96, 3, padding=1)
    bp = g.conv(f"{n}.branch_pool", _avg(x), pool_features, 1)
    return torch.cat([b1, b5, b3, bp], 1)


def inception_b(g, n, x):
    b3 = g.conv(f"{n}.branch3x3", x, 384, 3, stride=2)
    bd = g.conv(f"{n}.branch3x3dbl_1", x, 64, 1)
    bd = g.conv(f"{n}.branch3x3dbl_2", bd, 96, 3, padding=1)
    bd = g.conv(f"{n}.branch3x3dbl_3", bd, 96, 3, stride=2)
    return torch.cat([b3, bd, F.max_pool2d(x, 3, 2)], 1)


def inception_c(g, n, x, c7):
    b1 = g.conv(f"{n}.branch1x1", x, 192, 1)
    b7 = g.conv(f"{n}.branch7x7_1", x, c7, 1)
    b7 = g.conv(f"{n}.branch7x7_2", b7, c7, (1, 7), padding=(0, 3))
    b7 = g.conv(f"{n}.branch7x7_3", b7, 192, (7, 1), padding=(3, 0))
    bd = g.conv(f"{n}.branch7x7dbl_1", x, c7, 1)
    bd = g.conv(f"{n}.branch7x7dbl_2", bd, c7, (7, 1), padding=(3, 0))
    bd = g.conv(f"{n}.branch7x7dbl_3", bd, c7, (1, 7), padding=(0, 3))
    bd = g.conv(f"{n}.branch7x7dbl_4", bd, c7, (7, 1), padding=(3, 0))
    bd = g.conv(f"{n}.branch7x7dbl_5", bd, 192, (1, 7), padding=(0, 3))
    bp = g.conv(f"{n}.branch_pool", _avg(x), 192, 1)
    return torch.cat([b1, b7, bd, bp], 1)


def inception_d(g, n, x):
    b3 = g.conv(f"{n}.branch3x3_2", g.conv(f"{n}.branch3x3_1", x, 192, 1), 320, 3, stride=2)
    b7 = g.conv(f"{n}.branch7x7x3_1", x, 192, 1)
    b7 = g.conv(f"{n}.branch7x7x3_2", b7, 192, (1, 7), padding=(0, 3))
    b7 = g.conv(f"{n}.branch7x7x3_3", b7, 192, (7, 1), padding=(3, 0))
    b7 = g.conv(f"{n}.branch7x7x3_4", b7, 192, 3, stride=2)
    return torch.cat([b3, b7, F.max_pool2d(x, 3, 2)], 1)


def inception_e(g, n, x, pool):
    """pool 'avg': FIDInceptionE_1 (Mixed_7b); 'max': FIDInceptionE_2 (Mixed_7c)."""
    b1 = g.conv(f"{n}.branch1x1", x, 320, 1)
    b3 = g.conv(f"{n}.branch3x3_1", x, 384, 1)
    b3 = torch.cat([g.conv(f"{n}.branch3x3_2a", b3, 384, (1, 3), padding=(0, 1)),
                    g.conv(f"{n}.branch3x3_2b", b3, 384, (3, 1), padding=(1, 0))], 1)
    bd = g.conv(f"{n}.branch3x3dbl_1", x, 448, 1)
    bd = g.conv(f"{n}.branch3x3dbl_2", bd, 384, 3, padding=1)
    bd = torch.cat([g.conv(f"{n}.branch3x3dbl_3a", bd, 384, (1, 3), padding=(0, 1)),
                    g.conv(f"{n}.branch3x3dbl_3b", bd, 384, (3, 1), padding=(1, 0))], 1)
    p = _avg(x) if pool == "avg" else F.max_pool2d(x, 3, 1, 1)
    bp = g.conv(f"{n}.branch_pool", p, 192, 1)
    return torch.cat([b1, b3, bd, bp], 1)


def block(g, name, x):
    """One of BLOCKS by name, with the FID pooling."""
    if name in ("Mixed_5b", "Mixed_5c", "Mixed_5d"):
        return inception_a(g, name, x, {"Mixed_5b": 32}.get(name, 64))
    if name == "Mixed_6a":
        return inception_b(g, name, x)
    if name in ("Mixed_6b", "Mixed_6c", "Mixed_6d", "Mixed_6e"):
        return inception_c(g, name, x, {"Mixed_6b": 128, "Mixed_6e": 192}.get(name, 160))
    if name == "Mixed_7a":
        return inception_d(g, name, x)
    return inception_e(g, name, x, "avg" if name == "Mixed_7b" else "max")


def transform(images):
    """pytorch-fid's input: [B,3,H,W] in [0, 1] -> 299x299 bilinear (align_corners=False) -> 2x - 1, in fp64."""
    x = images.double()
    if x.shape[2:] != (299, 299):
        x = F.interpolate(x, size=(299, 299), mode="bilinear", align_corners=False)
    return 2 * x - 1


def network(g, x, upto=None):
    """The transformed input x -> the 2048 pooled features [B,2048]; `upto` (a block name) stops after that block."""
    x = stem(g, x)
    for n in BLOCKS:
        x = block(g, n, x)
        if n == upto:
            return x
    return x.mean(dim=(2, 3))


def fid_features(sd, images):
    """images [B,3,H,W] in [0, 1] -> [B,2048] fp64 with the state `sd` (torchvision names)."""
    return network(_Graph(sd), transform(images))


def calibration_images(seed=0, n=2, size=299):
    """Seeded smooth-ish test images in [0, 1]: low-resolution noise up-sampled, so the stem sees image-like statistics."""
    g = torch.Generator().manual_seed(seed)
    low = torch.rand(n, 3, size // 8, size // 8, generator=g, dtype=torch.float64)
    return F.interpolate(low, size=(size, size), mode="bilinear", align_corners=False).clamp(0, 1)


def seeded_fid_inception_state(seed=0):
    """A state_dict in torchvision's names for the 94 BasicConv2d layers (`<layer>.conv.weight`, `<layer>.bn.weight / .bias /
    .running_mean / .running_var`): weights randn * sqrt(2 / fan_in) drawn in graph order from ONE torch.Generator(seed), BN
    gamma = 1 + 0.1 randn and beta = 0.1 randn, and running statistics set to the per-channel mean / variance of each layer's
    convolution output in one fp64 pass over `calibration_images(seed)`, so that every layer is roughly normalised and the 2048
    features stay spread out after 94 ReLU layers."""
    gen = torch.Generator().manual_seed(seed)
    sd = OrderedDict()

    def make(name, x, cin, cout, kh, kw, stride, padding):
        w = torch.randn(cout, cin, kh, kw, generator=gen, dtype=torch.float64) * math.sqrt(2.0 / (cin * kh * kw))
        y = F.conv2d(x, w, stride=stride, padding=padding)
        sd[f"{name}.conv.weight"] = w.float()
        sd[f"{name}.bn.weight"] = (1 + 0.1 * torch.randn(cout, generator=gen, dtype=torch.float64)).float()
        sd[f"{name}.bn.bias"] = (0.1 * torch.randn(cout, generator=gen, dtype=torch.float64)).float()
        sd[f"{name}.bn.running_mean"] = y.mean(dim=(0, 2, 3)).float()
        sd[f"{name}.bn.running_var"] = y.var(dim=(0, 2, 3), unbiased=False).float()

    with torch.no_grad():
        network(_Graph(sd, make), transform(calibration_images(seed)))
    return sd
