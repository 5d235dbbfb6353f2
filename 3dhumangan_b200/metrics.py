"""KID and k-NN precision / recall on sm_90a, with the VGG16 fc7 features that precision / recall are defined on.

    VGG16Features       torchvision's VGG16 up to fc7 (`classifier.3`) after its ReLU, the 4096-d features of Kynkaanniemi et
                        al. 2019, with torchvision's parameter names.  `features(images)` -> [B,4096]: hg_vgg_input (ImageNet
                        mean / std, bilinear to 224x224), the 13 3x3 convolutions on hg_conv2d (fp32x3, bias in the epilogue,
                        ReLU on hg_bias_act), hg_maxpool2x2 after each block, and fc6 / fc7 as a 7x7 and a 1x1 convolution on
                        hg_conv2d_general in windows of 448 output channels.
    generator_features  the Inception pool features and the VGG16 fc7 features of a generator's images, from ONE generation pass
                        sampled exactly as `fid.generator_statistics` samples.
    kid                 KID (Binkowski et al. 2018): the unbiased MMD^2 with the kernel (a.b / D + 1)^3, averaged over subsets.
    precision_recall    Kynkaanniemi et al. 2019 with k-NN balls.
    save_features / load_features   one .npz with `inception` and `vgg16`.

FID from a feature bank is `fid.FeatureStats().update(feats["inception"])` and `fid.frechet_distance`.  KID and precision /
recall run on csrc/metrics.cu's fp64 pairwise engine: every product, sum and comparison is fp64, so the values depend on no
rounding of the distances.  StyleGAN2-ADA computes the k-NN distances in fp16 and drops the row itself with `kthvalue(k+1)`, so
its decisions can differ from these on near ties (and on duplicate rows, which count here at distance 0).

The VGG16 weights are never downloaded: `weights=None` reads torchvision's cached `vgg16-397923af.pth` (the file the
perceptual loss reads) and raises, naming that path, when it is missing."""
from __future__ import annotations

import os

import numpy as np
import torch

from . import abi, fid
from .modules.discriminator_train import _pack
from .ops import bias_act as _ba
from .perceptual import _RELU, WEIGHTS_FILE, _Conv3x3, _maxpool, default_weights_path

CFG = [64, 64, "M", 128, 128, "M", 256, 256, 256, "M", 512, 512, 512, "M", 512, 512, 512, "M"]    # torchvision's vgg16
DIM = 4096
FC_WINDOW = 448          # output channels per hg_conv2d_general launch of fc6 / fc7
MEAN = (0.485, 0.456, 0.406)
STD = (0.229, 0.224, 0.225)
MAX_K = 8


class _Linear(torch.nn.Module):
    """Parameter holder of one frozen fully connected layer (the kernels read it)."""

    def __init__(self, cin, cout):
        super().__init__()
        self.weight = torch.nn.Parameter(torch.zeros(cout, cin), requires_grad=False)
        self.bias = torch.nn.Parameter(torch.zeros(cout), requires_grad=False)


class VGG16Features(torch.nn.Module):
    """torchvision's VGG16 through fc7 and its ReLU on this library's kernels; no gradients.
    weights: None (torchvision's cached file), a path to that file, or a state_dict in torchvision's names (`features.N.*`,
    `classifier.0.*`, `classifier.3.*`; other keys such as `classifier.6.*` are ignored)."""

    def __init__(self, weights=None):
        super().__init__()
        feats = torch.nn.Module()
        idx, cin = 0, 3
        for v in CFG:
            if v == "M":
                idx += 1
                continue
            feats.add_module(str(idx), _Conv3x3(cin, v))
            idx, cin = idx + 2, v
        cls = torch.nn.Module()
        cls.add_module("0", _Linear(512 * 7 * 7, DIM))
        cls.add_module("3", _Linear(DIM, DIM))
        # registered directly: the state_dict keys are torchvision's `features.N.*`, while `self.features` is the method
        self._modules["features"] = feats
        self.classifier = cls
        self.register_buffer("mean", torch.tensor(MEAN), persistent=False)
        self.register_buffer("std", torch.tensor(STD), persistent=False)
        self._packed = None
        self._packed_convs = None
        if weights is None or isinstance(weights, (str, os.PathLike)):
            path = default_weights_path() if weights is None else os.fspath(weights)
            if not os.path.isfile(path):
                raise RuntimeError(f"hg3d: VGG16 weights not found at {path}: place torchvision's {WEIGHTS_FILE} there or pass "
                                   "`weights=` (a path or a state_dict); they are never downloaded")
            weights = torch.load(path, map_location="cpu", weights_only=True)
        self.load_torchvision(weights)

    @torch.no_grad()
    def load_torchvision(self, state):
        """Copy the 13 convolutions and fc6 / fc7 from a torchvision VGG16 state_dict."""
        for name, t in self.named_parameters():
            if name not in state:
                raise RuntimeError(f"hg3d: VGG16 state_dict has no {name!r}")
            src = state[name]
            if tuple(src.shape) != tuple(t.shape):
                raise RuntimeError(f"hg3d: VGG16 {name!r} has shape {tuple(src.shape)}, expected {tuple(t.shape)}")
            t.copy_(src)

    def _convs(self):
        return list(self._modules["features"].children())

    def conv_images(self):
        """Per convolution (img, Nb), packed again only when a convolution weight changed.  `ppl.LPIPS` reads these too, so
        an LPIPS on this network never packs fc6 / fc7."""
        convs = self._convs()
        key = tuple((c.weight.data_ptr(), c.weight._version, str(c.weight.device)) for c in convs)
        if self._packed_convs is None or self._packed_convs[0] != key:
            with torch.no_grad():
                self._packed_convs = (key, [_pack(c.weight.float()) for c in convs])
        return self._packed_convs[1]

    def _images(self):
        """(per convolution (img, Nb), per fc layer [(c0, Cout, img, Nb, bias)]), packed again only when a weight changed."""
        fcs = [self.classifier._modules["0"], self.classifier._modules["3"]]
        conv_imgs = self.conv_images()
        key = tuple((p.data_ptr(), p._version, str(p.device)) for layer in fcs for p in layer.parameters())
        if self._packed is None or self._packed[0] != key:
            with torch.no_grad():
                fc6 = fcs[0].weight.float().view(DIM, 512, 7, 7).permute(0, 2, 3, 1).reshape(DIM, -1)
                fc_imgs = []
                for w, layer in ((fc6, fcs[0]), (fcs[1].weight.float(), fcs[1])):
                    wins = []
                    for c0 in range(0, DIM, FC_WINDOW):
                        cout = min(FC_WINDOW, DIM - c0)
                        nblocks = -(-cout // 128)
                        img, Nb = abi.pack_weight(w[c0:c0 + cout].contiguous(), Nb=-(-cout // (16 * nblocks)) * 16)
                        wins.append((c0, cout, img, Nb, layer.bias[c0:c0 + cout].float().contiguous()))
                    fc_imgs.append(wins)
            self._packed = (key, fc_imgs)
        return conv_imgs, self._packed[1]

    def _check(self, images):
        abi.require_device()
        if images.dim() != 4 or images.shape[1] != 3 or not images.is_cuda:
            raise RuntimeError(f"hg3d: VGG16Features.features takes CUDA images [B,3,H,W] (got {tuple(images.shape)} on "
                               f"{images.device})")
        if images.dtype != torch.uint8 and not images.is_floating_point():
            raise RuntimeError(f"hg3d: VGG16Features.features takes uint8 or float images (got {images.dtype})")
        if torch.is_grad_enabled() and (images.requires_grad or any(p.requires_grad for p in self.parameters())):
            raise RuntimeError("hg3d: gradients through VGG16Features are not built")

    def features(self, images):
        """images uint8 [B,3,H,W] (k -> k / 255) or float in [0, 1] -> the fc7 activations after ReLU [B,4096] fp32."""
        self._check(images)
        with torch.no_grad(), torch.cuda.device_of(images):
            x = images.float() / 255 if images.dtype == torch.uint8 else images.float()
            x = x.contiguous()
            B, _, H, W = x.shape
            conv_imgs, fc_imgs = self._images()
            mean = self.mean.float().contiguous()
            std = self.std.float().contiguous()
            h = torch.empty(B, 3, 224, 224, dtype=torch.float32, device=x.device)
            abi.call("hg_vgg_input", abi.ptr(x), 3, B, H, W, abi.ptr(mean), abi.ptr(std), abi.ptr(h), 224, 224, abi.stream())
            convs = iter(zip(self._convs(), conv_imgs))
            for v in CFG:
                if v == "M":
                    h = _maxpool(h)
                    continue
                conv, (img, Nb) = next(convs)
                h = abi.conv2d(h, img, v, Nb, ksize=3, H=h.shape[2], W=h.shape[3], bias=conv.bias.float().contiguous(), passes=3)
                h = _ba._launch_fwd(h, None, 1, _RELU)
            # at 224 x 224 the map is 7 x 7, so torchvision's AdaptiveAvgPool2d((7, 7)) is the identity; classifier.2 / .5 are
            # dropout, the identity in eval
            for wins in fc_imgs:
                _, C, Hh, Ww = h.shape
                out = torch.empty(B, DIM, 1, 1, dtype=torch.float32, device=x.device)
                for c0, cout, img, Nb, bias in wins:
                    abi.call("hg_conv2d_general", abi.ptr(h), B, C, Hh, Ww, Hh, Ww, 1, 0, 0, abi.ptr(img), cout, Nb, abi.ptr(bias),
                             abi.ptr(out), DIM, c0, 3, abi.stream())
                h = out
        return h.reshape(B, DIM)


def generator_features(G, cfg, num_images, batch_size, seed=0, truncation_psi=1.0, conditions=None, inception=None, vgg=None):
    """{"inception": [N,2048], "vgg16": [N,4096]} fp32 on G's device: the features of `num_images` images of generator G,
    sampled exactly as `fid.generator_statistics` samples them (z_i = fid.latent(seed, i), `conditions` or
    `fid.synthetic_conditions(seed)`, `staged_forward` with nerf_noise = 0 and last_back = eval_last_back, `fid.to_uint8`); both
    detectors see the same uint8 batch.  Under torch.distributed each rank renders indices rank::world and the features are
    all-gathered into index order on every rank.  The renderer's ray jitter draws from torch's global RNG, as in the sample app:
    seed it (torch.manual_seed) for a repeatable run; it is drawn per batch, so the images depend on the world size unless the
    jitter is fixed."""
    import torch.distributed as dist
    dev = next(G.parameters()).device
    if inception is None:
        inception = fid.FIDInceptionV3().to(dev)
    if vgg is None:
        vgg = VGG16Features().to(dev)
    if conditions is None:
        conditions = fid.synthetic_conditions(seed)
    rank, world = 0, 1
    if dist.is_available() and dist.is_initialized():
        rank, world = dist.get_rank(), dist.get_world_size()
    run = dict(cfg)
    run.update(nerf_noise=0, last_back=cfg.get("eval_last_back", False), truncation_psi=truncation_psi)
    G.eval()
    mine = list(range(rank, num_images, world))
    per = max(-(-num_images // world), 1)
    local = torch.zeros(per, fid.DIM + DIM, dtype=torch.float32, device=dev)
    for s in range(0, len(mine), batch_size):
        idx = mine[s:s + batch_size]
        z = torch.stack([fid.latent(seed, i, run["latent_dim"]) for i in idx]).to(dev)
        cond = {k: v.to(dev) for k, v in conditions(idx).items()}
        with torch.no_grad():
            imgs = fid.to_uint8(G.staged_forward(z, cond, **run)["rgbs"])
            local[s:s + len(idx), :fid.DIM] = inception.features(imgs)
            local[s:s + len(idx), fid.DIM:] = vgg.features(imgs)
    if world > 1:
        parts = [torch.empty_like(local) for _ in range(world)]
        dist.all_gather(parts, local)
    else:
        parts = [local]
    out = torch.empty(num_images, fid.DIM + DIM, dtype=torch.float32, device=dev)
    for r, p in enumerate(parts):
        n_r = len(range(r, num_images, world))
        out[r::world] = p[:n_r]
    return {"inception": out[:, :fid.DIM].contiguous(), "vgg16": out[:, fid.DIM:].contiguous()}


def save_features(path, feats):
    """One .npz with `inception` [N,2048] and `vgg16` [N,4096] fp32."""
    with open(path, "wb") as f:
        np.savez(f, inception=_host(feats["inception"], fid.DIM), vgg16=_host(feats["vgg16"], DIM))


def load_features(path):
    """-> {"inception": [N,2048], "vgg16": [N,4096]} as fp32 CPU tensors."""
    with np.load(path) as z:
        out = {k: torch.from_numpy(np.ascontiguousarray(z[k], dtype=np.float32)) for k in ("inception", "vgg16")}
    if out["inception"].shape[0] != out["vgg16"].shape[0]:
        raise RuntimeError(f"hg3d: {path} holds {out['inception'].shape[0]} Inception and {out['vgg16'].shape[0]} VGG16 rows")
    _host(out["inception"], fid.DIM)
    _host(out["vgg16"], DIM)
    return out


def _host(t, dim):
    a = t.detach().cpu().numpy() if torch.is_tensor(t) else np.asarray(t)
    if a.ndim != 2 or a.shape[1] != dim:
        raise RuntimeError(f"hg3d: expected features [n, {dim}] (got {a.shape})")
    return a.astype(np.float32, copy=False)


def _pair(real, gen, what):
    """Shape checks first (they need no device), then the device; -> fp32 contiguous (real, gen)."""
    for name, t in (("real", real), ("gen", gen)):
        if not torch.is_tensor(t) or t.dim() != 2 or not t.is_floating_point():
            raise RuntimeError(f"hg3d: {what} takes float feature tensors [n, D] ({name}: "
                               f"{tuple(t.shape) if torch.is_tensor(t) else type(t).__name__})")
    if real.shape[1] != gen.shape[1] or real.shape[1] < 1:
        raise RuntimeError(f"hg3d: {what}: real and gen features differ in D ({real.shape[1]} vs {gen.shape[1]})")
    return real, gen


def _device(real, gen, what):
    if not (real.is_cuda and gen.is_cuda) or real.device != gen.device:
        raise RuntimeError(f"hg3d: {what} takes features on one CUDA device (real on {real.device}, gen on {gen.device})")
    abi.require_device()
    return real.float().contiguous(), gen.float().contiguous()


def kid_subsets(n_gen, n_real, num_subsets=100, max_subset_size=1000, seed=0):
    """-> (idx_gen, idx_real), each [num_subsets, m] int64, m = min(n_real, n_gen, max_subset_size): with
    rng = np.random.default_rng(seed), subset s draws rng.choice(n_gen, m, replace=False) and then rng.choice(n_real, m,
    replace=False)."""
    if isinstance(num_subsets, bool) or not isinstance(num_subsets, (int, np.integer)) or num_subsets < 1:
        raise ValueError(f"kid: num_subsets must be a positive integer (got {num_subsets!r})")
    m = min(int(n_real), int(n_gen), int(max_subset_size))
    if m < 2:
        raise ValueError(f"kid: subset size m = min(n_real={n_real}, n_gen={n_gen}, max_subset_size={max_subset_size}) = {m} "
                         "is below 2")
    rng = np.random.default_rng(seed)
    ig = np.empty((num_subsets, m), dtype=np.int64)
    ir = np.empty((num_subsets, m), dtype=np.int64)
    for s in range(num_subsets):
        ig[s] = rng.choice(n_gen, m, replace=False)
        ir[s] = rng.choice(n_real, m, replace=False)
    return ig, ir


def kid(real, gen, num_subsets=100, max_subset_size=1000, seed=0):
    """-> (mean_s t_s, std_s t_s (ddof 0), t [num_subsets] fp64 numpy): per subset the unbiased MMD^2 between m gen and m real
    features with k(a, b) = (a.b / D + 1)^3 (`kid_subsets` draws the rows), in fp64 on hg_kid."""
    real, gen = _pair(real, gen, "kid")
    ig, ir = kid_subsets(gen.shape[0], real.shape[0], num_subsets, max_subset_size, seed)
    real, gen = _device(real, gen, "kid")
    S, m = ig.shape
    dev = real.device
    with torch.cuda.device_of(real):
        idx_g = torch.from_numpy(ig).to(dev)
        idx_r = torch.from_numpy(ir).to(dev)
        nbytes = int(abi.lib().hg_kid_workspace_bytes(S, m))
        ws = torch.empty(nbytes // 8, dtype=torch.float64, device=dev)
        t = torch.empty(S, dtype=torch.float64, device=dev)
        abi.call("hg_kid", abi.ptr(gen), gen.shape[0], abi.ptr(real), real.shape[0], real.shape[1], abi.ptr(idx_g), abi.ptr(idx_r),
                 S, m, abi.ptr(t), abi.ptr(ws), nbytes, abi.stream())
    t = t.cpu().numpy()
    return float(t.mean()), float(t.std()), t


def _sqnorms(x):
    out = torch.empty(x.shape[0], dtype=torch.float64, device=x.device)
    abi.call("hg_row_sqnorms", abi.ptr(x), x.shape[0], x.shape[1], abi.ptr(out), abi.stream())
    return out


def _radii(x, sqn, k):
    rho2 = torch.empty(x.shape[0], dtype=torch.float64, device=x.device)
    abi.call("hg_knn_radii", abi.ptr(x), abi.ptr(sqn), x.shape[0], x.shape[1], k, abi.ptr(rho2), abi.stream())
    return rho2


def _check_k(k, n_real, n_gen):
    if isinstance(k, bool) or not isinstance(k, (int, np.integer)) or not 1 <= k <= MAX_K:
        raise ValueError(f"precision_recall: k must be an integer in [1, {MAX_K}] (got {k!r})")
    if k >= n_real or k >= n_gen:
        raise ValueError(f"precision_recall: k={k} needs more than k features in each set (n_real={n_real}, n_gen={n_gen})")


def precision_recall(real, gen, k=3):
    """-> (precision, recall): the fraction of gen rows inside some real row's k-NN ball, and of real rows inside some gen
    row's; a ball's radius is the distance to its centre's k-th nearest other row of its own set.  All in fp64 on
    hg_row_sqnorms / hg_knn_radii / hg_ball_coverage."""
    real, gen = _pair(real, gen, "precision_recall")
    _check_k(k, real.shape[0], gen.shape[0])
    real, gen = _device(real, gen, "precision_recall")
    dev = real.device
    ng, nr, D = gen.shape[0], real.shape[0], real.shape[1]
    with torch.cuda.device_of(real):
        sq_r, sq_g = _sqnorms(real), _sqnorms(gen)
        rho_r, rho_g = _radii(real, sq_r, k), _radii(gen, sq_g, k)
        row_flag = torch.empty(ng, dtype=torch.uint8, device=dev)
        col_flag = torch.empty(nr, dtype=torch.uint8, device=dev)
        counts = torch.empty(2, dtype=torch.int64, device=dev)
        abi.call("hg_ball_coverage", abi.ptr(gen), abi.ptr(sq_g), abi.ptr(rho_g), ng, abi.ptr(real), abi.ptr(sq_r), abi.ptr(rho_r), nr,
                 D, abi.ptr(row_flag), abi.ptr(col_flag), abi.ptr(counts), abi.stream())
    c = counts.cpu().tolist()
    return c[0] / ng, c[1] / nr
