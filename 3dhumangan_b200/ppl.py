"""Perceptual path length (PPL) on sm_90a: LPIPS (VGG, v0.1) on the library's VGG16, and the path length of a generator with
both images of a pair rendered under one ray jitter.

LPIPS is the distance of the `lpips` package's `LPIPS(net='vgg', version='0.1')` between images a, b [B,3,H,W] in [-1, 1]:

    scaling    x -> (x - shift) / scale per channel, shift = (-0.030, -0.088, -0.188), scale = (0.458, 0.448, 0.450): ImageNet's
               mean / std applied to (x + 1) / 2.
    taps       torchvision VGG16 `features` after relu1_2, relu2_2, relu3_3, relu4_3 and relu5_3 (the ends of the slices [0:4],
               [4:9], [9:16], [16:23] and [23:30]), at the input's resolution: there is no resize to 224.
    per level  each pixel's channel vector f -> f / (||f||_2 + 1e-10); the squared difference of the two images' normalised
               features, weighted by the non-negative 1x1 `lin` weights (one per channel, no bias), summed over the channels
               and averaged over the H x W pixels.
    distance   the sum of the five levels.

The `lin` weights are the package's `weights/v0.1/vgg.pth`: `lin{0..4}.model.1.weight` of shapes [1, C, 1, 1] with C = 64,
128, 256, 512, 512.  They are never downloaded: `lin=None` reads `default_lin_path()` and raises, naming it, when it is
missing.  The VGG16 weights come from a `metrics.VGG16Features` (default: torchvision's cached `vgg16-397923af.pth`); its
packed convolution images are shared, and fc6 / fc7 are never packed for LPIPS.

    LPIPS.distance  the 13 convolutions on hg_conv2d (fp32x3) with ReLU on hg_bias_act and hg_maxpool2x2 between the slices,
                    both images of every pair in one batch; each level's head is one hg_lpips_level launch (fp64 norms,
                    differences and sums into a per-pair fp64 accumulator).
    input_stage     StyleGAN2-ADA's PPL box-downsampling by an integer factor f, then the scaling: hg_vgg_input for f <= 2
                    (a bilinear resize by 1/2 with align_corners=False is exactly the 2x2 box mean), hg_lpips_input otherwise.
                    Nothing is quantised or clamped: rounding to uint8 would erase an epsilon-sized difference.

PPL follows StyleGAN2-ADA's `ppl_zfull` / `ppl_wfull` / `ppl_zend` / `ppl_wend` (Karras et al. 2019): per pair i, latents z0,
z1 and t (0 for sampling "end", U[0, 1) for "full") drawn from (seed, i) alone; the images at t and t + epsilon (lerp of the
mapped codes in space "w", slerp of z in space "z"); dist_i = LPIPS / epsilon^2 after the factor-H // 256 box-downsampling of
images taller than 256; PPL = the mean of dist over [1st percentile (lower), 99th percentile (higher)].

The renderer jitters its samples on every call (`rng.draw`).  Both images of a pair see the same draws: before each of the two
renders the device RNG is seeded from (seed, batch index), inside `torch.random.fork_rng`, so the caller's RNG state is left as
it was.  With neural_field_latent_input False (every shipped curriculum) the render then is the same for both endpoints, and
PPL measures the synthesis network's path in style space."""
from __future__ import annotations

import os

import numpy as np
import torch

from . import abi, fid, metrics
from .modules.generator import _precision_passes
from .ops import bias_act as _ba
from .perceptual import _RELU, _maxpool

SHIFT = (-0.030, -0.088, -0.188)
SCALE = (0.458, 0.448, 0.450)
LIN_CHANNELS = (64, 128, 256, 512, 512)
LIN_FILE = "lpips_vgg_v0.1.pth"
SPACES = ("w", "z")
SAMPLINGS = ("end", "full")
AVERAGE_DRAWS = 10000


def default_lin_path():
    """Where LPIPS's lin weights are read from when `lin=None`: the `lpips` package's weights/v0.1/vgg.pth, copied to
    torch.hub.get_dir()/checkpoints/lpips_vgg_v0.1.pth."""
    return os.path.join(torch.hub.get_dir(), "checkpoints", LIN_FILE)


def load_lin(lin=None):
    """lin: None (`default_lin_path()`), a path, or a state_dict in the `lpips` package's names -> {name: [1,C,1,1] fp32}."""
    if lin is None or isinstance(lin, (str, os.PathLike)):
        path = default_lin_path() if lin is None else os.fspath(lin)
        if not os.path.isfile(path):
            raise RuntimeError(f"hg3d: LPIPS lin weights not found at {path}: place the lpips package's weights/v0.1/vgg.pth there "
                               "or pass `lin=` (a path or a state_dict); they are never downloaded")
        lin = torch.load(path, map_location="cpu", weights_only=True)
    out = {}
    for k, C in enumerate(LIN_CHANNELS):
        name = f"lin{k}.model.1.weight"
        if name not in lin:
            raise RuntimeError(f"hg3d: LPIPS lin state_dict has no {name!r}")
        w = lin[name]
        if tuple(w.shape) != (1, C, 1, 1):
            raise RuntimeError(f"hg3d: LPIPS {name!r} has shape {tuple(w.shape)}, expected (1, {C}, 1, 1)")
        if bool((w < 0).any()):
            raise RuntimeError(f"hg3d: LPIPS {name!r} has negative weights; the v0.1 lin layers are non-negative")
        out[name] = w.detach().float().cpu()
    return out


class _Lin(torch.nn.Module):
    def __init__(self, C):
        super().__init__()
        self.weight = torch.nn.Parameter(torch.zeros(1, C, 1, 1), requires_grad=False)


def _check_images(x, what):
    abi.require_device()
    if not torch.is_tensor(x) or x.dim() != 4 or x.shape[1] != 3 or not x.is_cuda or not x.is_floating_point():
        raise RuntimeError(f"hg3d: {what} takes float CUDA images [B,3,H,W] (got "
                           f"{tuple(x.shape) if torch.is_tensor(x) else type(x).__name__})")
    if torch.is_grad_enabled() and x.requires_grad:
        raise RuntimeError(f"hg3d: gradients through {what} are not built")


class LPIPS(torch.nn.Module):
    """LPIPS (VGG, v0.1) on this library's kernels; no gradients.  vgg: a `metrics.VGG16Features` (default: torchvision's
    cached weights); lin: see `load_lin`.  The state_dict holds `vgg.*` and the lpips package's `lin{k}.model.1.weight`."""

    def __init__(self, vgg=None, lin=None):
        super().__init__()
        self.vgg = metrics.VGG16Features() if vgg is None else vgg
        for k, C in enumerate(LIN_CHANNELS):
            m = torch.nn.Module()
            m.model = torch.nn.Module()
            m.model.add_module("1", _Lin(C))
            self.add_module(f"lin{k}", m)
        self.register_buffer("shift", torch.tensor(SHIFT), persistent=False)
        self.register_buffer("scale", torch.tensor(SCALE), persistent=False)
        self.load_lin(lin)

    @torch.no_grad()
    def load_lin(self, lin):
        for name, w in load_lin(lin).items():
            self.get_parameter(name).copy_(w)

    def _lin(self, k):
        return self.get_parameter(f"lin{k}.model.1.weight").reshape(-1).float().contiguous()

    def input_stage(self, x, factor=1):
        """x [B,3,H,W] float -> [B,3,H/f,W/f] fp32: the mean of every f x f window, then (x - shift) / scale.  H and W must be
        divisible by f."""
        _check_images(x, "LPIPS.input_stage")
        f = int(factor)
        B, _, H, W = x.shape
        if f != factor or f < 1:
            raise ValueError(f"LPIPS.input_stage: the factor must be a positive integer (got {factor!r})")
        if H % f or W % f:
            raise ValueError(f"LPIPS.input_stage: {H} x {W} images are not divisible by the factor {f}")
        x = x.float().contiguous()
        shift, scale = self.shift.float().contiguous(), self.scale.float().contiguous()
        out = torch.empty(B, 3, H // f, W // f, dtype=torch.float32, device=x.device)
        with torch.cuda.device_of(x):
            if f <= 2:
                abi.call("hg_vgg_input", abi.ptr(x), 3, B, H, W, abi.ptr(shift), abi.ptr(scale), abi.ptr(out), H // f, W // f,
                         abi.stream())
            else:
                abi.call("hg_lpips_input", abi.ptr(x), B, H, W, f, abi.ptr(shift), abi.ptr(scale), abi.ptr(out), abi.stream())
        return out

    def distance(self, a, b, factor=1):
        """-> [B] fp64: LPIPS between a[i] and b[i], images [B,3,H,W] in [-1, 1], after `input_stage(·, factor)`."""
        _check_images(a, "LPIPS.distance")
        _check_images(b, "LPIPS.distance")
        if a.shape != b.shape or a.device != b.device:
            raise RuntimeError(f"hg3d: LPIPS.distance takes two batches of one shape on one device (got {tuple(a.shape)} on "
                               f"{a.device}, {tuple(b.shape)} on {b.device})")
        if any(p.requires_grad for p in self.parameters()) and torch.is_grad_enabled():
            raise RuntimeError("hg3d: gradients w.r.t. the LPIPS weights are not built")
        B = a.shape[0]
        with torch.no_grad(), torch.cuda.device_of(a):
            h = self.input_stage(torch.cat([a, b]), factor)
            dev = h.device
            acc = torch.zeros(B, dtype=torch.float64, device=dev)
            nbytes = int(abi.lib().hg_lpips_workspace_bytes(B))
            ws = torch.empty(nbytes // 8, dtype=torch.float64, device=dev)
            convs = iter(zip(self.vgg._convs(), self.vgg.conv_images()))
            level = 0
            for v in metrics.CFG:
                if v == "M":
                    # the end of a slice: relu1_2, relu2_2, relu3_3, relu4_3, relu5_3
                    _, C, Hh, Ww = h.shape
                    abi.call("hg_lpips_level", abi.ptr(h[:B]), abi.ptr(h[B:]), abi.ptr(self._lin(level)), B, C, Hh * Ww,
                             abi.ptr(acc), abi.ptr(ws), nbytes, abi.stream())
                    level += 1
                    if level < len(LIN_CHANNELS):
                        h = _maxpool(h)
                    continue
                conv, (img, Nb) = next(convs)
                h = abi.conv2d(h, img, v, Nb, ksize=3, H=h.shape[2], W=h.shape[3], bias=conv.bias.float().contiguous(), passes=3)
                h = _ba._launch_fwd(h, None, 1, _RELU)
        return acc


# ------------------------------------------------------------------------------------------------------------ sampling
def downsample_factor(H):
    """StyleGAN2-ADA's PPL factor: images taller than 256 are box-downsampled by H // 256."""
    return H // 256 if H > 256 else 1


def _rng(seed, index, tag):
    # numpy's SeedSequence keeps every bit of (seed, index, tag); torch's CPU generator would keep 32 bits of one seed
    return np.random.default_rng([int(seed), int(index), int(tag)])


def pair_draws(seed, index, dim, sampling):
    """(z0 [dim], z1 [dim], t) of pair `index`: z0, z1 and t each from their own generator seeded from (seed, index, tag
    0 / 1 / 2), so they depend on neither the batching nor the rank; t = 0 for sampling "end", U[0, 1) for "full"."""
    z0 = torch.from_numpy(_rng(seed, index, 0).standard_normal(dim)).float()
    z1 = torch.from_numpy(_rng(seed, index, 1).standard_normal(dim)).float()
    t = float(_rng(seed, index, 2).random()) if sampling == "full" else 0.0
    return z0, z1, t


def jitter_seed(seed, batch):
    """The device-RNG seed of both renders of batch `batch`."""
    return (int(seed) << 32) + int(batch)


def batches(num_samples, batch_size, rank=0, world=1):
    """[(k, indices)] of this rank: pairs cut into batches of `batch_size` in index order, batch k on rank k % world."""
    nb = -(-num_samples // batch_size)
    return [(k, list(range(k * batch_size, min((k + 1) * batch_size, num_samples)))) for k in range(rank, nb, world)]


def slerp(a, b, t):
    """StyleGAN2-ADA's slerp of the rows of a, b [n, D] at t [n, 1]: normalise a and b; d = a.b; p = t acos(d);
    c = normalise(b - d a); normalise(a cos p + c sin p)."""
    a = a / a.norm(dim=-1, keepdim=True)
    b = b / b.norm(dim=-1, keepdim=True)
    d = (a * b).sum(dim=-1, keepdim=True)
    p = t * torch.acos(d)
    c = b - d * a
    c = c / c.norm(dim=-1, keepdim=True)
    r = a * torch.cos(p) + c * torch.sin(p)
    return r / r.norm(dim=-1, keepdim=True)


def filtered_mean(dist):
    """-> (lo, hi, ppl): lo = 1st percentile (method "lower"), hi = 99th (method "higher"), ppl = mean of dist in [lo, hi]."""
    d = np.asarray(dist, dtype=np.float64)
    lo = np.percentile(d, 1, method="lower")
    hi = np.percentile(d, 99, method="higher")
    return float(lo), float(hi), float(d[(d >= lo) & (d <= hi)].mean())


def _check_args(cfg, space, sampling, epsilon):
    if space not in SPACES:
        raise ValueError(f"ppl: space must be one of {SPACES} (got {space!r})")
    if sampling not in SAMPLINGS:
        raise ValueError(f"ppl: sampling must be one of {SAMPLINGS} (got {sampling!r})")
    if not epsilon >= 0:
        raise ValueError(f"ppl: epsilon must not be negative (got {epsilon!r})")
    if _precision_passes(cfg) == 1:
        raise RuntimeError("hg3d: PPL needs hg_precision='fp32x3': the single-pass bf16 generator's error is far above an "
                           "epsilon step")


def _run_cfg(cfg):
    run = dict(cfg)
    run.update(nerf_noise=0, last_back=cfg.get("eval_last_back", False))
    return run


@torch.no_grad()
def truncation_averages(G, cfg, seed=0, n=AVERAGE_DRAWS):
    """(freq, phase, styles) averaged over the codes of n latents drawn from (seed, tag 3): the one set of averages both
    endpoints of every pair are truncated towards."""
    dev = next(G.parameters()).device
    z = torch.from_numpy(_rng(seed, 0, 3).standard_normal((n, cfg["latent_dim"]))).float().to(dev)
    return tuple(c.mean(dim=0, keepdim=True) for c in G.truncated_codes(z, 1.0, cfg))


@torch.no_grad()
def pair_codes(G, cfg, indices, seed=0, space="w", sampling="end", epsilon=1e-4, truncation_psi=1.0, averages=None):
    """The generator codes (freq, phase, styles) of both endpoints of pairs `indices`: [(codes at t), (codes at t + eps)].
    Interpolation in fp64 (codes in "w", unit latents in "z"), then fp32."""
    dev = next(G.parameters()).device
    draws = [pair_draws(seed, i, cfg["latent_dim"], sampling) for i in indices]
    z0 = torch.stack([d[0] for d in draws]).to(dev)
    z1 = torch.stack([d[1] for d in draws]).to(dev)
    t = torch.tensor([[d[2]] for d in draws], dtype=torch.float64, device=dev)
    if space == "w":
        c0 = G.truncated_codes(z0, truncation_psi, cfg, averages)
        c1 = G.truncated_codes(z1, truncation_psi, cfg, averages)
        return [tuple(a.double().lerp(b.double(), tt.view(-1, *[1] * (a.dim() - 1))).float() for a, b in zip(c0, c1))
                for tt in (t, t + epsilon)]
    return [G.truncated_codes(slerp(z0.double(), z1.double(), tt).float(), truncation_psi, cfg, averages) for tt in (t, t + epsilon)]


@torch.no_grad()
def pair_images(G, cfg, indices, seed=0, batch=0, space="w", sampling="end", epsilon=1e-4, truncation_psi=1.0, conditions=None,
                averages=None):
    """-> (img0, img1) [n,3,H,W] fp32: the images at t and t + epsilon of pairs `indices`, as `path_length` renders batch
    `batch`: G.eval(), nerf_noise 0, last_back = eval_last_back, one body and camera per pair (`conditions(indices)`,
    default `fid.synthetic_conditions(seed)`), and the device RNG seeded from (seed, batch) before each of the two renders,
    inside torch.random.fork_rng.  epsilon = 0 gives two renders of the same codes."""
    _check_args(cfg, space, sampling, epsilon)
    dev = next(G.parameters()).device
    if conditions is None:
        conditions = fid.synthetic_conditions(seed)
    if truncation_psi < 1.0 and averages is None:
        averages = truncation_averages(G, cfg, seed)
    run = _run_cfg(cfg)
    G.eval()
    ends = pair_codes(G, cfg, indices, seed, space, sampling, epsilon, truncation_psi, averages)
    cond = {k: v.to(dev) for k, v in conditions(list(indices)).items()}
    imgs = []
    with torch.random.fork_rng(devices=[dev]):
        for freq, phase, styles in ends:
            torch.cuda.default_generators[dev.index].manual_seed(jitter_seed(seed, batch))
            imgs.append(G.synthesize(freq, phase, styles, cond, **run)["rgbs"])
    return imgs[0], imgs[1]


def path_length(G, cfg, num_samples, batch_size, seed=0, space="w", sampling="end", epsilon=1e-4, truncation_psi=1.0,
                conditions=None, lpips=None):
    """Perceptual path length of generator G -> {"ppl": float, "dist": [num_samples] fp64 numpy, "lo": float, "hi": float}.

    Pairs are rendered by `pair_images` batch by batch (`batches`), each distance is LPIPS(img_t, img_t+eps) / eps^2 at
    `downsample_factor(H)`, and PPL is `filtered_mean(dist)` on the host.  Under torch.distributed batch k runs on rank k %
    world and the distances are all-gathered into index order, so every rank returns the same result, and the distances
    depend on (seed, batch_size) and not on the world size.  conditions: (indices) -> conditions dict (default
    `fid.synthetic_conditions(seed)`); lpips: an `LPIPS` (default: the cached weight files)."""
    import torch.distributed as dist
    _check_args(cfg, space, sampling, epsilon)
    if not epsilon > 0:
        raise ValueError(f"ppl: epsilon must be positive (got {epsilon!r})")
    if num_samples < 2:
        raise ValueError(f"ppl: num_samples must be at least 2 (got {num_samples})")
    if batch_size < 1:
        raise ValueError(f"ppl: batch_size must be at least 1 (got {batch_size})")
    dev = next(G.parameters()).device
    if lpips is None:
        lpips = LPIPS().to(dev)
    if conditions is None:
        conditions = fid.synthetic_conditions(seed)
    rank, world = 0, 1
    if dist.is_available() and dist.is_initialized():
        rank, world = dist.get_rank(), dist.get_world_size()
    averages = truncation_averages(G, cfg, seed) if truncation_psi < 1.0 else None
    nb = -(-num_samples // batch_size)
    per = -(-nb // world)
    local = torch.zeros(per * batch_size, dtype=torch.float64, device=dev)
    for j, (k, idx) in enumerate(batches(num_samples, batch_size, rank, world)):
        a, b = pair_images(G, cfg, idx, seed, k, space, sampling, epsilon, truncation_psi, conditions, averages)
        local[j * batch_size:j * batch_size + len(idx)] = lpips.distance(a, b, downsample_factor(a.shape[2])) / (epsilon * epsilon)
    if world > 1:
        parts = [torch.empty_like(local) for _ in range(world)]
        dist.all_gather(parts, local)
    else:
        parts = [local]
    out = torch.empty(num_samples, dtype=torch.float64, device=dev)
    for k in range(nb):
        n_k = min(batch_size, num_samples - k * batch_size)
        j = (k // world) * batch_size
        out[k * batch_size:k * batch_size + n_k] = parts[k % world][j:j + n_k]
    d = out.cpu().numpy()
    lo, hi, ppl = filtered_mean(d)
    return {"ppl": ppl, "dist": d, "lo": lo, "hi": hi}
