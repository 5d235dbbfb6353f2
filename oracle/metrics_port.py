"""fp64 test oracle of 3dhumangan_b200/metrics.py, written from the metrics' definitions (no implementation of them is at hand to
pin against): KID's unbiased MMD^2 with the cubic kernel, k-NN radii and ball coverage from direct differences sum (a - b)^2
(not from the norm expansion the kernels use), and torchvision's VGG16 through fc7 with a seeded state that stands in for the
pretrained weights (which are never downloaded)."""
from __future__ import annotations

import math

import numpy as np
import torch
import torch.nn.functional as F

from oracle import perceptual_port as pp


# ---------------------------------------------------------------------------------------------------------------- KID
def kid_indices(n_gen, n_real, num_subsets, max_subset_size, seed):
    """The subset draw: m = min(n_real, n_gen, max_subset_size); rng = default_rng(seed); per subset the gen rows, then the
    real rows, each rng.choice(n, m, replace=False)."""
    m = min(n_real, n_gen, max_subset_size)
    rng = np.random.default_rng(seed)
    ig, ir = [], []
    for _ in range(num_subsets):
        ig.append(rng.choice(n_gen, m, replace=False))
        ir.append(rng.choice(n_real, m, replace=False))
    return np.array(ig), np.array(ir)


def kid_terms(gen, real, ig, ir):
    """t [S] fp64: per subset (sum_{i != j} k(g_i, g_j) + sum_{i != j} k(r_i, r_j)) / (m (m - 1)) - 2 sum_{i,j} k(g_i, r_j) / m^2,
    k(a, b) = (a.b / D + 1)^3.  gen / real: fp64 torch tensors on any device."""
    D = gen.shape[1]
    out = []
    for s in range(ig.shape[0]):
        g = gen[torch.as_tensor(ig[s], device=gen.device)]
        r = real[torch.as_tensor(ir[s], device=real.device)]
        m = g.shape[0]
        kgg = (g @ g.T / D + 1) ** 3
        krr = (r @ r.T / D + 1) ** 3
        kgr = (g @ r.T / D + 1) ** 3
        a = (kgg.sum() - kgg.diagonal().sum() + krr.sum() - krr.diagonal().sum()) / (m * (m - 1))
        out.append(float(a - 2 * kgr.sum() / (m * m)))
    return np.array(out)


def kid_brute(gen, real, ig, ir):
    """kid_terms as explicit double loops over i != j (numpy fp64), for small m."""
    gen, real = np.asarray(gen, np.float64), np.asarray(real, np.float64)
    D = gen.shape[1]
    k = lambda a, b: (float(a @ b) / D + 1) ** 3
    out = []
    for s in range(ig.shape[0]):
        g, r = gen[ig[s]], real[ir[s]]
        m = len(g)
        sxx = sum(k(g[i], g[j]) for i in range(m) for j in range(m) if i != j)
        syy = sum(k(r[i], r[j]) for i in range(m) for j in range(m) if i != j)
        sxy = sum(k(g[i], r[j]) for i in range(m) for j in range(m))
        out.append((sxx + syy) / (m * (m - 1)) - 2 * sxy / (m * m))
    return np.array(out)


# ---------------------------------------------------------------------------------------------------------- k-NN metrics
def sq_dists(a, b):
    """[na, nb] squared distances sum_d (a_i - b_j)^2 in fp64 from direct differences, in row chunks of at most 2^25 differences
    (any device)."""
    a, b = a.double(), b.double()
    rows = []
    step = max(1, (1 << 25) // (b.shape[0] * a.shape[1]))
    for i in range(0, a.shape[0], step):
        rows.append(((a[i:i + step, None, :] - b[None, :, :]) ** 2).sum(-1))
    return torch.cat(rows)


def knn_radii(x, k):
    """rho_k^2 [n]: the k-th smallest squared distance from row i to rows j != i (excluded by index)."""
    d = sq_dists(x, x)
    d.fill_diagonal_(float("inf"))
    return d.kthvalue(k, dim=1).values


def coverage(gen, real, rho2_gen, rho2_real):
    """(gen flags [n_gen], real flags [n_real]): gen row i inside some real ball (d^2 <= rho2_real[j]), real row j inside some
    gen ball (d^2 <= rho2_gen[i])."""
    d = sq_dists(gen, real)
    return (d <= rho2_real[None, :]).any(1), (d <= rho2_gen[:, None]).any(0)


def precision_recall(real, gen, k):
    rr, rg = knn_radii(real, k), knn_radii(gen, k)
    fg, fr = coverage(gen, real, rg, rr)
    return float(fg.double().mean()), float(fr.double().mean())


# ---------------------------------------------------------------------------------------------------------- VGG16 fc7
def seeded_vgg16_state(seed=0):
    """torchvision VGG16 state_dict: the convolutions of `perceptual_port.seeded_vgg16_state(seed)` plus classifier.0 / .3 / .6
    drawn from torch.Generator(seed + 1): weight = randn * sqrt(2 / fan_in) (He-normal, so fc7 activations neither vanish nor
    explode), bias = 0.01 * randn."""
    sd = pp.seeded_vgg16_state(seed)
    g = torch.Generator().manual_seed(seed + 1)
    for idx, (cin, cout) in ((0, (512 * 7 * 7, 4096)), (3, (4096, 4096)), (6, (4096, 1000))):
        sd[f"classifier.{idx}.weight"] = torch.randn(cout, cin, generator=g) * math.sqrt(2.0 / cin)
        sd[f"classifier.{idx}.bias"] = 0.01 * torch.randn(cout, generator=g)
    return sd


def vgg16_fc7(state, x01):
    """fp64 features of images in [0, 1] [B,3,H,W]: ImageNet mean / std, bilinear to 224x224 (align_corners=False, no
    antialias), VGG16 `features`, adaptive average pool to 7x7, flatten, relu(fc6), relu(fc7) (dropout is the identity)."""
    h = pp.transform(x01, resize=True)
    idx = 0
    for v in pp.CFG:
        if v == "M":
            h = F.max_pool2d(h, 2, 2)
            idx += 1
            continue
        h = F.relu(F.conv2d(h, state[f"features.{idx}.weight"].double(), state[f"features.{idx}.bias"].double(), padding=1))
        idx += 2
    h = F.adaptive_avg_pool2d(h, (7, 7)).flatten(1)
    h = F.relu(F.linear(h, state["classifier.0.weight"].double(), state["classifier.0.bias"].double()))
    return F.relu(F.linear(h, state["classifier.3.weight"].double(), state["classifier.3.bias"].double()))
