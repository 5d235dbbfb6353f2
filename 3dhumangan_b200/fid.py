"""FID on sm_90a: pytorch-fid's Inception-v3, fp64 feature statistics and the Frechet distance, for generators and image sets.

    FIDInceptionV3        pytorch-fid's `fid_inception_v3`: torchvision's `Inception3(num_classes=1008, aux_logits=False)`
                          with the FID pooling (average pooling without the padding in Mixed_5b-d, 6b-e and 7b, max pooling
                          (3, 1, 1) in Mixed_7c), same parameter / buffer names.  `features(images)` -> [B,2048]: hg_vgg_input
                          (bilinear to 299x299, 2x - 1), the 94 convolutions on hg_conv2d_general (BatchNorm folded in fp64,
                          bias + ReLU in the epilogue, each branch written into its block's concatenation), the pools on
                          hg_pool3x3 and the 8x8 average on hg_global_avgpool.
    FeatureStats          n, sum x and sum x x^T in fp64 on the device (hg_feature_moments), all-reduced across ranks.
    frechet_distance      host fp64 numpy, without scipy.
    generator_statistics  the statistics of a generator's images, sampled as the sample app samples them.

The Inception weights are never downloaded: `weights=None` reads pytorch-fid's cached `pt_inception-2015-12-05-6726825d.pth`
under `torch.hub.get_dir()/checkpoints` and raises, naming that path, when it is missing."""
from __future__ import annotations

import os

import numpy as np
import torch

from . import abi

WEIGHTS_FILE = "pt_inception-2015-12-05-6726825d.pth"
DIM = 2048
BN_EPS = 1e-3


def default_weights_path():
    """Where pytorch-fid caches its Inception weights."""
    return os.path.join(torch.hub.get_dir(), "checkpoints", WEIGHTS_FILE)


def _pair(v):
    return (v, v) if isinstance(v, int) else tuple(v)


class BasicConv2d(torch.nn.Module):
    """Parameter holder of torchvision's BasicConv2d (conv without bias, BatchNorm eps 1e-3, ReLU); the kernels read it."""

    def __init__(self, cin, cout, kernel_size, stride=1, padding=0):
        super().__init__()
        kh, kw = _pair(kernel_size)
        self.cin, self.cout, self.stride = cin, cout, stride
        self.kh, self.kw = kh, kw
        self.ph, self.pw = _pair(padding)
        self.conv = torch.nn.Module()
        self.conv.weight = torch.nn.Parameter(torch.zeros(cout, cin, kh, kw), requires_grad=False)
        self.bn = torch.nn.Module()
        self.bn.weight = torch.nn.Parameter(torch.ones(cout), requires_grad=False)
        self.bn.bias = torch.nn.Parameter(torch.zeros(cout), requires_grad=False)
        self.bn.register_buffer("running_mean", torch.zeros(cout))
        self.bn.register_buffer("running_var", torch.ones(cout))

    def tensors(self):
        return (self.conv.weight, self.bn.weight, self.bn.bias, self.bn.running_mean, self.bn.running_var)

    def folded(self):
        """-> (W [Cout, kh*kw*Cin] fp32 in the packed order [Cout, kh, kw, Cin], bias [Cout] fp32), BatchNorm folded in fp64 on
        the host: W' = W * gamma / sqrt(var + eps), b' = beta - mean * gamma / sqrt(var + eps)."""
        w, gamma, beta, mean, var = (t.detach().to("cpu", torch.float64) for t in self.tensors())
        s = gamma / torch.sqrt(var + BN_EPS)
        wf = (w * s.view(-1, 1, 1, 1)).permute(0, 2, 3, 1).reshape(self.cout, -1)
        return wf.float().contiguous(), (beta - mean * s).float()


class InceptionA(torch.nn.Module):
    def __init__(self, cin, pool_features):
        super().__init__()
        self.branch1x1 = BasicConv2d(cin, 64, 1)
        self.branch5x5_1 = BasicConv2d(cin, 48, 1)
        self.branch5x5_2 = BasicConv2d(48, 64, 5, padding=2)
        self.branch3x3dbl_1 = BasicConv2d(cin, 64, 1)
        self.branch3x3dbl_2 = BasicConv2d(64, 96, 3, padding=1)
        self.branch3x3dbl_3 = BasicConv2d(96, 96, 3, padding=1)
        self.branch_pool = BasicConv2d(cin, pool_features, 1)

    def run(self, net, x):
        out = net.buffer(x, 224 + self.branch_pool.cout, x.shape[2], x.shape[3])
        net.conv(self.branch1x1, x, out, 0)
        net.conv(self.branch5x5_2, net.conv(self.branch5x5_1, x), out, 64)
        net.conv(self.branch3x3dbl_3, net.conv(self.branch3x3dbl_2, net.conv(self.branch3x3dbl_1, x)), out, 128)
        net.conv(self.branch_pool, net.pool(x, 1, 1, True), out, 224)
        return out


class InceptionB(torch.nn.Module):
    def __init__(self, cin):
        super().__init__()
        self.branch3x3 = BasicConv2d(cin, 384, 3, stride=2)
        self.branch3x3dbl_1 = BasicConv2d(cin, 64, 1)
        self.branch3x3dbl_2 = BasicConv2d(64, 96, 3, padding=1)
        self.branch3x3dbl_3 = BasicConv2d(96, 96, 3, stride=2)

    def run(self, net, x):
        Ho, Wo = (x.shape[2] - 3) // 2 + 1, (x.shape[3] - 3) // 2 + 1
        out = net.buffer(x, 480 + x.shape[1], Ho, Wo)
        net.conv(self.branch3x3, x, out, 0)
        net.conv(self.branch3x3dbl_3, net.conv(self.branch3x3dbl_2, net.conv(self.branch3x3dbl_1, x)), out, 384)
        net.pool(x, 2, 0, False, out, 480)
        return out


class InceptionC(torch.nn.Module):
    def __init__(self, cin, c7):
        super().__init__()
        self.branch1x1 = BasicConv2d(cin, 192, 1)
        self.branch7x7_1 = BasicConv2d(cin, c7, 1)
        self.branch7x7_2 = BasicConv2d(c7, c7, (1, 7), padding=(0, 3))
        self.branch7x7_3 = BasicConv2d(c7, 192, (7, 1), padding=(3, 0))
        self.branch7x7dbl_1 = BasicConv2d(cin, c7, 1)
        self.branch7x7dbl_2 = BasicConv2d(c7, c7, (7, 1), padding=(3, 0))
        self.branch7x7dbl_3 = BasicConv2d(c7, c7, (1, 7), padding=(0, 3))
        self.branch7x7dbl_4 = BasicConv2d(c7, c7, (7, 1), padding=(3, 0))
        self.branch7x7dbl_5 = BasicConv2d(c7, 192, (1, 7), padding=(0, 3))
        self.branch_pool = BasicConv2d(cin, 192, 1)

    def run(self, net, x):
        out = net.buffer(x, 768, x.shape[2], x.shape[3])
        net.conv(self.branch1x1, x, out, 0)
        b = net.conv(self.branch7x7_2, net.conv(self.branch7x7_1, x))
        net.conv(self.branch7x7_3, b, out, 192)
        b = net.conv(self.branch7x7dbl_1, x)
        for layer in (self.branch7x7dbl_2, self.branch7x7dbl_3, self.branch7x7dbl_4):
            b = net.conv(layer, b)
        net.conv(self.branch7x7dbl_5, b, out, 384)
        net.conv(self.branch_pool, net.pool(x, 1, 1, True), out, 576)
        return out


class InceptionD(torch.nn.Module):
    def __init__(self, cin):
        super().__init__()
        self.branch3x3_1 = BasicConv2d(cin, 192, 1)
        self.branch3x3_2 = BasicConv2d(192, 320, 3, stride=2)
        self.branch7x7x3_1 = BasicConv2d(cin, 192, 1)
        self.branch7x7x3_2 = BasicConv2d(192, 192, (1, 7), padding=(0, 3))
        self.branch7x7x3_3 = BasicConv2d(192, 192, (7, 1), padding=(3, 0))
        self.branch7x7x3_4 = BasicConv2d(192, 192, 3, stride=2)

    def run(self, net, x):
        Ho, Wo = (x.shape[2] - 3) // 2 + 1, (x.shape[3] - 3) // 2 + 1
        out = net.buffer(x, 512 + x.shape[1], Ho, Wo)
        net.conv(self.branch3x3_2, net.conv(self.branch3x3_1, x), out, 0)
        b = net.conv(self.branch7x7x3_1, x)
        for layer in (self.branch7x7x3_2, self.branch7x7x3_3):
            b = net.conv(layer, b)
        net.conv(self.branch7x7x3_4, b, out, 320)
        net.pool(x, 2, 0, False, out, 512)
        return out


class InceptionE(torch.nn.Module):
    """avg_pool: FIDInceptionE_1 (Mixed_7b) averages without the padding; else FIDInceptionE_2 (Mixed_7c) max-pools."""

    def __init__(self, cin, avg_pool):
        super().__init__()
        self.avg_pool = avg_pool
        self.branch1x1 = BasicConv2d(cin, 320, 1)
        self.branch3x3_1 = BasicConv2d(cin, 384, 1)
        self.branch3x3_2a = BasicConv2d(384, 384, (1, 3), padding=(0, 1))
        self.branch3x3_2b = BasicConv2d(384, 384, (3, 1), padding=(1, 0))
        self.branch3x3dbl_1 = BasicConv2d(cin, 448, 1)
        self.branch3x3dbl_2 = BasicConv2d(448, 384, 3, padding=1)
        self.branch3x3dbl_3a = BasicConv2d(384, 384, (1, 3), padding=(0, 1))
        self.branch3x3dbl_3b = BasicConv2d(384, 384, (3, 1), padding=(1, 0))
        self.branch_pool = BasicConv2d(cin, 192, 1)

    def run(self, net, x):
        out = net.buffer(x, 2048, x.shape[2], x.shape[3])
        net.conv(self.branch1x1, x, out, 0)
        b = net.conv(self.branch3x3_1, x)
        net.conv(self.branch3x3_2a, b, out, 320)
        net.conv(self.branch3x3_2b, b, out, 704)
        b = net.conv(self.branch3x3dbl_2, net.conv(self.branch3x3dbl_1, x))
        net.conv(self.branch3x3dbl_3a, b, out, 1088)
        net.conv(self.branch3x3dbl_3b, b, out, 1472)
        net.conv(self.branch_pool, net.pool(x, 1, 1, self.avg_pool), out, 1856)
        return out


class FIDInceptionV3(torch.nn.Module):
    """pytorch-fid's Inception-v3 for FID on this library's kernels; no gradients.
    weights: None (pytorch-fid's cached file), a path to such a file, or a state_dict in torchvision's names (`fc.*` is ignored,
    `num_batches_tracked` may be present or absent)."""

    def __init__(self, weights=None):
        super().__init__()
        self.Conv2d_1a_3x3 = BasicConv2d(3, 32, 3, stride=2)
        self.Conv2d_2a_3x3 = BasicConv2d(32, 32, 3)
        self.Conv2d_2b_3x3 = BasicConv2d(32, 64, 3, padding=1)
        self.Conv2d_3b_1x1 = BasicConv2d(64, 80, 1)
        self.Conv2d_4a_3x3 = BasicConv2d(80, 192, 3)
        self.Mixed_5b = InceptionA(192, 32)
        self.Mixed_5c = InceptionA(256, 64)
        self.Mixed_5d = InceptionA(288, 64)
        self.Mixed_6a = InceptionB(288)
        self.Mixed_6b = InceptionC(768, 128)
        self.Mixed_6c = InceptionC(768, 160)
        self.Mixed_6d = InceptionC(768, 160)
        self.Mixed_6e = InceptionC(768, 192)
        self.Mixed_7a = InceptionD(768)
        self.Mixed_7b = InceptionE(1280, True)
        self.Mixed_7c = InceptionE(2048, False)
        self._packed = None
        if weights is None or isinstance(weights, (str, os.PathLike)):
            path = default_weights_path() if weights is None else os.fspath(weights)
            if not os.path.isfile(path):
                raise RuntimeError(f"hg3d: FID Inception weights not found at {path}: place pytorch-fid's {WEIGHTS_FILE} there or "
                                   "pass `weights=` (a path or a state_dict); they are never downloaded")
            weights = torch.load(path, map_location="cpu", weights_only=True)
        self.load_torchvision(weights)

    @torch.no_grad()
    def load_torchvision(self, state):
        """Copy every parameter and running statistic from a torchvision-named Inception3 state_dict."""
        for name, t in list(self.named_parameters()) + list(self.named_buffers()):
            if name not in state:
                raise RuntimeError(f"hg3d: FID Inception state_dict has no {name!r}")
            src = state[name]
            if tuple(src.shape) != tuple(t.shape):
                raise RuntimeError(f"hg3d: FID Inception {name!r} has shape {tuple(src.shape)}, expected {tuple(t.shape)}")
            t.copy_(src)

    def layers(self):
        return [m for m in self.modules() if isinstance(m, BasicConv2d)]

    def _images(self):
        """{layer: (packed weight image, Nb, folded bias)}, packed again only when a tensor of a layer changed."""
        layers = self.layers()
        key = tuple((t.data_ptr(), t._version, str(t.device)) for m in layers for t in m.tensors())
        if self._packed is None or self._packed[0] != key:
            dev = self.Conv2d_1a_3x3.conv.weight.device
            imgs = {}
            with torch.no_grad():
                for m in layers:
                    w, b = m.folded()
                    nblocks = -(-m.cout // 128)
                    Nb = -(-m.cout // (16 * nblocks)) * 16
                    img, Nb = abi.pack_weight(w.to(dev), Nb=Nb)
                    imgs[m] = (img, Nb, b.to(dev))
            self._packed = (key, imgs)
        return self._packed[1]

    # ---- launch helpers used by the blocks' `run`
    @staticmethod
    def buffer(x, C, H, W):
        return torch.empty(x.shape[0], C, H, W, dtype=torch.float32, device=x.device)

    def conv(self, layer, x, out=None, c0=0):
        """relu(bn(conv(x))) of `layer` into channels [c0, c0 + Cout) of `out` (a new tensor when None)."""
        img, Nb, bias = self._imgs[layer]
        B, C, H, W = x.shape
        Ho = (H + 2 * layer.ph - layer.kh) // layer.stride + 1
        Wo = (W + 2 * layer.pw - layer.kw) // layer.stride + 1
        if out is None:
            out = self.buffer(x, layer.cout, Ho, Wo)
        abi.call("hg_conv2d_general", abi.ptr(x), B, C, H, W, layer.kh, layer.kw, layer.stride, layer.ph, layer.pw, abi.ptr(img),
                 layer.cout, Nb, abi.ptr(bias), abi.ptr(out), out.shape[1], c0, 3, abi.stream())
        return out

    def pool(self, x, stride, pad, avg, out=None, c0=0):
        B, C, H, W = x.shape
        if out is None:
            out = self.buffer(x, C, (H + 2 * pad - 3) // stride + 1, (W + 2 * pad - 3) // stride + 1)
        abi.call("hg_pool3x3", abi.ptr(x), B, C, H, W, stride, pad, int(bool(avg)), abi.ptr(out), out.shape[1], c0, abi.stream())
        return out

    def _check(self, images):
        abi.require_device()
        if images.dim() != 4 or images.shape[1] != 3 or not images.is_cuda:
            raise RuntimeError(f"hg3d: FIDInceptionV3.features takes CUDA images [B,3,H,W] (got {tuple(images.shape)} on "
                               f"{images.device})")
        if images.dtype != torch.uint8 and not images.is_floating_point():
            raise RuntimeError(f"hg3d: FIDInceptionV3.features takes uint8 or float images (got {images.dtype})")
        if torch.is_grad_enabled() and (images.requires_grad or any(p.requires_grad for p in self.parameters())):
            raise RuntimeError("hg3d: gradients through FIDInceptionV3 are not built")

    def features(self, images):
        """images uint8 [B,3,H,W] (k -> k / 255) or float in [0, 1] -> the 2048 pooled features [B,2048] fp32."""
        self._check(images)
        with torch.no_grad(), torch.cuda.device_of(images):
            x = images.float() / 255 if images.dtype == torch.uint8 else images.float()
            x = x.contiguous()
            B, _, H, W = x.shape
            half = torch.full((3,), 0.5, dtype=torch.float32, device=x.device)
            h = self.buffer(x, 3, 299, 299)
            abi.call("hg_vgg_input", abi.ptr(x), 3, B, H, W, abi.ptr(half), abi.ptr(half), abi.ptr(h), 299, 299, abi.stream())
            self._imgs = self._images()
            try:
                h = self.conv(self.Conv2d_1a_3x3, h)
                h = self.conv(self.Conv2d_2a_3x3, h)
                h = self.conv(self.Conv2d_2b_3x3, h)
                h = self.pool(h, 2, 0, False)
                h = self.conv(self.Conv2d_3b_1x1, h)
                h = self.conv(self.Conv2d_4a_3x3, h)
                h = self.pool(h, 2, 0, False)
                for blk in (self.Mixed_5b, self.Mixed_5c, self.Mixed_5d, self.Mixed_6a, self.Mixed_6b, self.Mixed_6c, self.Mixed_6d,
                            self.Mixed_6e, self.Mixed_7a, self.Mixed_7b, self.Mixed_7c):
                    h = blk.run(self, h)
            finally:
                self._imgs = None
            out = torch.empty(B, DIM, dtype=torch.float32, device=x.device)
            abi.call("hg_global_avgpool", abi.ptr(h), B * DIM, h.shape[2] * h.shape[3], abi.ptr(out), abi.stream())
        return out


def to_uint8(rgbs):
    """Generator output in [-1, 1] -> uint8 images exactly as the sample app writes them (apps/sample_from_generator.py:59-62):
    clamp to [-1, 1], * 0.5 + 0.5, then clamp(* 255, 0, 255) truncated to uint8."""
    x = torch.clamp(rgbs, -1, 1) * 0.5 + 0.5
    return torch.clamp(x * 255, 0, 255).to(torch.uint8)


class FeatureStats:
    """Running n, sum x and sum x x^T of feature vectors in fp64.  CUDA features accumulate on the device with
    hg_feature_moments; features on the CPU (precomputed ones, say) accumulate on the host in fp64."""

    def __init__(self, dim=DIM, device="cuda"):
        self.dim = dim
        self.n = 0
        self.sum = torch.zeros(dim, dtype=torch.float64, device=device)
        self.gram = torch.zeros(dim, dim, dtype=torch.float64, device=device)

    def update(self, features):
        if features.dim() != 2 or features.shape[1] != self.dim:
            raise RuntimeError(f"hg3d: FeatureStats takes [n, {self.dim}] features (got {tuple(features.shape)})")
        if features.shape[0] == 0:
            return
        if features.device != self.sum.device:
            raise RuntimeError(f"hg3d: features on {features.device}, statistics on {self.sum.device}")
        if features.is_cuda:
            f = features.float().contiguous()
            with torch.cuda.device_of(f):
                abi.call("hg_feature_moments", abi.ptr(f), f.shape[0], self.dim, abi.ptr(self.sum), abi.ptr(self.gram), abi.stream())
        else:
            f = features.double()
            self.sum += f.sum(0)
            self.gram += f.T @ f
        self.n += int(features.shape[0])

    def all_reduce(self, group=None):
        """Sum the moments of every rank in ONE collective (a no-op without an initialised process group)."""
        import torch.distributed as dist
        if not (dist.is_available() and dist.is_initialized()):
            return self
        buf = torch.cat([torch.tensor([float(self.n)], dtype=torch.float64, device=self.sum.device), self.sum, self.gram.reshape(-1)])
        dist.all_reduce(buf, group=group)
        self.n = int(buf[0].item())
        self.sum.copy_(buf[1:1 + self.dim])
        self.gram.copy_(buf[1 + self.dim:].reshape(self.dim, self.dim))
        return self

    def mean_cov(self):
        """-> (mu [D], sigma [D,D]) fp64 numpy with np.cov semantics: sigma = (sum x x^T - n mu mu^T) / (n - 1)."""
        if self.n < 2:
            raise RuntimeError(f"hg3d: a covariance needs at least 2 feature vectors (have {self.n})")
        s = self.sum.cpu().numpy()
        g = self.gram.cpu().numpy()
        mu = s / self.n
        sigma = (g - self.n * np.outer(mu, mu)) / (self.n - 1)
        return mu, sigma

    def save(self, path):
        """pytorch-fid's statistics file: an .npz with `mu` and `sigma`."""
        mu, sigma = self.mean_cov()
        save_stats(path, mu, sigma)


def save_stats(path, mu, sigma):
    with open(path, "wb") as f:
        np.savez(f, mu=mu, sigma=sigma)


def load_stats(path):
    """-> (mu, sigma) fp64 from an .npz with keys `mu` and `sigma` (pytorch-fid's format; other keys are ignored)."""
    with np.load(path) as z:
        return z["mu"].astype(np.float64), z["sigma"].astype(np.float64)


def frechet_distance(mu1, sigma1, mu2, sigma2):
    """||mu1 - mu2||^2 + tr S1 + tr S2 - 2 tr sqrt(S1 S2) in fp64 numpy.  tr sqrt(S1 S2) = sum sqrt(max(lambda(R S2 R), 0))
    with R = S1^(1/2) from `eigh` (eigenvalues clamped at 0): R S2 R is symmetric and similar to S1 S2, so for PSD inputs
    this equals tr sqrtm(S1 S2) without sqrtm's complex round-off or an epsilon offset."""
    mu1, mu2 = np.asarray(mu1, np.float64), np.asarray(mu2, np.float64)
    s1, s2 = np.asarray(sigma1, np.float64), np.asarray(sigma2, np.float64)
    if mu1.shape != mu2.shape or s1.shape != s2.shape or s1.shape != (mu1.size, mu1.size):
        raise ValueError(f"frechet_distance: shapes {mu1.shape} {s1.shape} vs {mu2.shape} {s2.shape}")
    w, v = np.linalg.eigh((s1 + s1.T) / 2)
    r = (v * np.sqrt(np.clip(w, 0, None))) @ v.T
    m = r @ s2 @ r
    lam = np.linalg.eigvalsh((m + m.T) / 2)
    # eigenvalues under the solver's rounding level are zeros of a rank-deficient product (fewer samples than dimensions);
    # their square roots would add ~sqrt(eps * |lambda|_max) each
    lam[lam < lam.size * np.finfo(np.float64).eps * max(float(np.abs(lam).max()), 0.0)] = 0
    tr_sqrt = float(np.sqrt(lam).sum())
    d = mu1 - mu2
    return float(d @ d + np.trace(s1) + np.trace(s2) - 2 * tr_sqrt)


def latent(seed, index, dim):
    """z of image `index` under `seed`: its own torch.Generator, so it depends on neither the batching nor the rank."""
    return torch.randn(dim, generator=torch.Generator().manual_seed((int(seed) << 32) + int(index)))


def synthetic_conditions(seed=0):
    """(indices) -> the conditions of those images from `synthetic.make_conditions`, one seeded body per index."""
    from . import synthetic

    def conditions(indices):
        per = [synthetic.make_conditions(1, seed=(int(seed) << 32) + int(i)) for i in indices]
        return {k: torch.cat([c[k] for c in per]) for k in per[0]}
    return conditions


def generator_statistics(G, cfg, num_images, batch_size, seed=0, truncation_psi=1.0, conditions=None, inception=None):
    """FeatureStats of `num_images` images of generator G, sampled as apps/sample_from_generator.py samples them: G.eval(),
    `staged_forward` with nerf_noise = 0 and last_back = eval_last_back, z_i from (seed, i), images through `to_uint8`,
    `inception.features` and `FeatureStats.update` without leaving the device.

    conditions: (indices) -> conditions dict for those images; default `synthetic_conditions(seed)`, synthetic bodies from
    `synthetic.make_conditions`.  FID on synthetic poses is NOT comparable with the paper's, which conditions on SHHQ poses:
    pass the dataset's conditions to compare with it.  Under torch.distributed each rank renders indices rank::world and the
    moments are all-reduced, so every rank returns the statistics of all `num_images`.  The renderer's ray jitter draws from
    torch's global RNG, as in the sample app: seed it (torch.manual_seed) for a repeatable run."""
    import torch.distributed as dist
    dev = next(G.parameters()).device
    if inception is None:
        inception = FIDInceptionV3().to(dev)
    if conditions is None:
        conditions = synthetic_conditions(seed)
    rank, world = 0, 1
    if dist.is_available() and dist.is_initialized():
        rank, world = dist.get_rank(), dist.get_world_size()
    run = dict(cfg)
    run.update(nerf_noise=0, last_back=cfg.get("eval_last_back", False), truncation_psi=truncation_psi)
    G.eval()
    stats = FeatureStats(device=dev)
    mine = list(range(rank, num_images, world))
    for s in range(0, len(mine), batch_size):
        idx = mine[s:s + batch_size]
        z = torch.stack([latent(seed, i, run["latent_dim"]) for i in idx]).to(dev)
        cond = {k: v.to(dev) for k, v in conditions(idx).items()}
        with torch.no_grad():
            out = G.staged_forward(z, cond, **run)
            stats.update(inception.features(to_uint8(out["rgbs"])))
    return stats.all_reduce()
