"""fp64 test oracle of 3dhumangan_b200/ppl.py, written from the definitions in that module's docstring: LPIPS (VGG, v0.1) on
torchvision's VGG16 with a seeded state (`metrics_port.seeded_vgg16_state`) and seeded non-negative `lin` weights, the PPL
input stage, slerp, and the PPL composition on `oracle.port`'s generator evaluated in fp64 (mapping networks, SIREN,
integration and synthesis network; rays and geometry features stay fp32, as the reference computes them)."""
from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as F

from oracle import perceptual_port as pp
from oracle import port

SHIFT = (-0.030, -0.088, -0.188)
SCALE = (0.458, 0.448, 0.450)
LIN_CHANNELS = (64, 128, 256, 512, 512)


def seeded_lin_state(seed=0):
    """The lpips package's `lin{k}.model.1.weight` [1, C, 1, 1], drawn level by level from ONE torch.Generator(seed + 2) as
    U[0, 1) (non-negative, as the v0.1 weights are)."""
    g = torch.Generator().manual_seed(seed + 2)
    return {f"lin{k}.model.1.weight": torch.rand(1, C, 1, 1, generator=g) for k, C in enumerate(LIN_CHANNELS)}


def input_stage(x, factor=1):
    """fp64: the mean of every factor x factor window, then (x - shift) / scale."""
    x = x.double()
    B, C, H, W = x.shape
    f = factor
    x = x.reshape(B, C, H // f, f, W // f, f).mean(dim=(3, 5))
    shift = torch.tensor(SHIFT, dtype=x.dtype, device=x.device).view(1, 3, 1, 1)
    return (x - shift) / torch.tensor(SCALE, dtype=x.dtype, device=x.device).view(1, 3, 1, 1)


def lpips(vgg_state, lin_state, a, b, factor=1):
    """[B] fp64 LPIPS between images a and b [B,3,H,W] in [-1, 1] (any device)."""
    B = a.shape[0]
    h = input_stage(torch.cat([a, b]), factor)
    total = torch.zeros(B, dtype=torch.float64, device=h.device)
    idx = level = 0
    for v in pp.CFG:
        if v == "M":
            fa, fb = h[:B], h[B:]
            na = fa / (fa.pow(2).sum(1, keepdim=True).sqrt() + 1e-10)
            nb = fb / (fb.pow(2).sum(1, keepdim=True).sqrt() + 1e-10)
            w = lin_state[f"lin{level}.model.1.weight"].double().to(h.device).view(1, -1, 1, 1)
            total = total + ((na - nb) ** 2 * w).sum(1).mean(dim=(1, 2))
            level += 1
            if level < len(LIN_CHANNELS):
                h = F.max_pool2d(h, 2, 2)
            idx += 1
            continue
        h = F.relu(F.conv2d(h, vgg_state[f"features.{idx}.weight"].double().to(h.device),
                            vgg_state[f"features.{idx}.bias"].double().to(h.device), padding=1))
        idx += 2
    return total


def slerp(a, b, t):
    a = a / a.norm(dim=-1, keepdim=True)
    b = b / b.norm(dim=-1, keepdim=True)
    d = (a * b).sum(dim=-1, keepdim=True)
    p = t * torch.acos(d)
    c = b - d * a
    c = c / c.norm(dim=-1, keepdim=True)
    r = a * torch.cos(p) + c * torch.sin(p)
    return r / r.norm(dim=-1, keepdim=True)


def filtered_mean(dist):
    d = np.sort(np.asarray(dist, dtype=np.float64))
    n = d.size
    lo = d[int(np.floor(0.01 * (n - 1)))]
    hi = d[int(np.ceil(0.99 * (n - 1)))]
    return lo, hi, float(d[(d >= lo) & (d <= hi)].mean())


# ------------------------------------------------------------------------------------------------------- the generator
def _params64(params):
    return {k: (v.double() if v.is_floating_point() else v) for k, v in params.items()}


def codes(params, z, cfg):
    """(freq, phase, styles) of latents z [n, L] in fp64: port.mapping_network / port.synthesis_mapping without their fp32
    input cast."""
    p = _params64(params)
    zz = z if cfg.get("neural_field_latent_input", True) else torch.zeros_like(z)
    x = port.normalize_2nd_moment(zz.double())
    for i in (0, 2, 4):
        x = F.leaky_relu(F.linear(x, p[f"neural_field_mapping_network.network.{i}.weight"],
                                  p[f"neural_field_mapping_network.network.{i}.bias"]), port.LRELU)
    fp = F.linear(x, p["neural_field_mapping_network.network.6.weight"], p["neural_field_mapping_network.network.6.bias"])
    half = fp.shape[-1] // 2
    x = port.normalize_2nd_moment(z.double())
    for i in range(7):
        x = port._fc(p, f"synthesis_mapping_network.trunk{i}", x, "lrelu")
    styles = port._fc(p, "synthesis_mapping_network.superres0", x, "lrelu")[:, None, :]
    return fp[..., :half], fp[..., half:], styles


def truncate(c, psi, averages):
    return c if psi >= 1.0 else tuple(a + psi * (x - a) for x, a in zip(c, averages))


def synthesize(params, freq, phase, styles, cond, cfg, u, noise):
    """Eval-mode images [n,3,Hg,Wg] fp64 from the codes: port.render in fp64, the bilinear style map and
    port.synthesis_network with running statistics."""
    p = _params64(params)
    _, fmap, _, _, _ = port.render(p, freq, phase, cond, cfg, u, noise, dtype=torch.float64)
    Hg, Wg = cfg["gen_height"], cfg["gen_width"]
    style = F.interpolate(fmap, (Hg, Wg), mode="bilinear")
    x0 = port.synthesis_input(p, freq.shape[0], Hg, Wg)
    return port.synthesis_network(p, x0, style, styles.double(), cfg, training=False)


def pair_distances(params, vgg_state, lin_state, z0, z1, t, cond, cfg, u, noise, space, epsilon, psi=1.0, averages=None):
    """dist [n] fp64 of the pairs (z0, z1, t) [n, L], [n, L], [n, 1] under one jitter (u, noise) for both endpoints:
    LPIPS(img(t), img(t + eps)) / eps^2 at StyleGAN2-ADA's downsampling factor.  cfg: nerf_noise 0 and the eval last_back."""
    z0, z1, t = z0.double(), z1.double(), t.double()
    if space == "w":
        c0, c1 = truncate(codes(params, z0, cfg), psi, averages), truncate(codes(params, z1, cfg), psi, averages)
        ends = [tuple(a + tt.view(-1, *[1] * (a.dim() - 1)) * (b - a) for a, b in zip(c0, c1)) for tt in (t, t + epsilon)]
    else:
        ends = [truncate(codes(params, slerp(z0, z1, tt), cfg), psi, averages) for tt in (t, t + epsilon)]
    imgs = [synthesize(params, *c, cond, cfg, u, noise) for c in ends]
    H = imgs[0].shape[2]
    return lpips(vgg_state, lin_state, imgs[0], imgs[1], H // 256 if H > 256 else 1) / (epsilon * epsilon)
