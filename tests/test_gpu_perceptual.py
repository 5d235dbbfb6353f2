"""The VGG16 perceptual loss on sm_90a (3dhumangan_b200/perceptual.py, csrc/perceptual.cu): each new kernel against fp64,
the whole module against the fp64 oracle (oracle/perceptual_port.py, pinned to the reference by test_oracle_pin_perceptual.py)
on the GPU's ReLU masks, determinism, frozen weights, no torch op on the path, and latent inversion with the term."""
import importlib
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import perceptual_port as pp
from test_gpu_inversion import SPREAD, _released_like

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "perceptual.npz")
FIXTURE = {"rgb64x32": True, "rgb60x44_noresize": False, "gray48": True}


def _abi():
    return importlib.import_module("3dhumangan_b200.abi")


def _net(resize=True, seed=0):
    mod = importlib.import_module("3dhumangan_b200.perceptual")
    return mod.VGGPerceptualLoss(resize=resize, weights=pp.seeded_vgg16_state(seed)).cuda()


def _bilinear64(x, Ho, Wo):
    """fp64 bilinear resize (align_corners=False) at the source coordinates torch's fp32 kernel computes: the scale in / out
    and scale * (o + 0.5) - 0.5 rounded to fp32 (at 512 rows that rounding alone moves a sample by ~6e-5 pixels)."""
    def taps(n_in, n_out):
        s = np.float32(n_in) / np.float32(n_out)
        src = np.maximum(s * (np.arange(n_out, dtype=np.float32) + np.float32(0.5)) - np.float32(0.5), np.float32(0))
        i0 = np.minimum(src.astype(np.int64), n_in - 1)
        i1 = np.where(i0 < n_in - 1, i0 + 1, i0)
        return torch.from_numpy(i0), torch.from_numpy(i1), torch.from_numpy(src.astype(np.float64) - i0)
    y0, y1, ly = taps(x.shape[2], Ho)
    x0, x1, lx = taps(x.shape[3], Wo)
    ly, lx = ly[:, None], lx[None, :]
    r0, r1 = x[:, :, y0], x[:, :, y1]
    return (1 - ly) * ((1 - lx) * r0[..., x0] + lx * r0[..., x1]) + ly * ((1 - lx) * r1[..., x0] + lx * r1[..., x1])


def _transform(x, Ho, Wo, mean, std):
    abi = _abi()
    B, C, H, W = x.shape
    out = torch.empty(B, 3, Ho, Wo, device="cuda")
    abi.call("hg_vgg_input", abi.ptr(x), C, B, H, W, abi.ptr(mean), abi.ptr(std), abi.ptr(out), Ho, Wo, abi.stream())
    return out


def _adjoint(d, C, H, W, std):
    abi = _abi()
    B, _, Ho, Wo = d.shape
    dx = torch.empty(B, C, H, W, device="cuda")
    abi.call("hg_vgg_input_adjoint", abi.ptr(d), B, Ho, Wo, abi.ptr(std), abi.ptr(dx), C, H, W, abi.stream())
    return dx


@pytest.mark.parametrize("B,C,H,W,resize", [(1, 3, 512, 256, True), (1, 3, 512, 512, True), (2, 3, 224, 224, True),
                                            (1, 1, 48, 48, True), (3, 3, 60, 44, True), (3, 1, 64, 32, False)])
def test_input_transform_and_its_adjoint(B, C, H, W, resize):
    g = torch.Generator().manual_seed(H * W + B)
    x = torch.rand(B, C, H, W, generator=g)
    Ho, Wo = (224, 224) if resize else (H, W)
    mean, std = torch.tensor(pp.MEAN).cuda(), torch.tensor(pp.STD).cuda()
    got = _transform(x.cuda(), Ho, Wo, mean, std).cpu().double()
    ref = pp.transform(x, resize)                 # torch's fp64 interpolate: source coordinates in fp64
    assert (got - ref).abs().max() <= 2e-4 * ref.abs().max()
    if resize:
        ref = _bilinear64(pp.transform(x, False), Ho, Wo)
    # what is left is the rounding of the source coordinate (one fp32 ulp of ~50 on the up-sampling cases, times a pixel step)
    assert (got - ref).abs().max() <= 1e-5 * ref.abs().max()
    # the adjoint of the linear part (zero mean): <T x, y> = <x, T^T y>, and T^T y against fp64 autograd
    y = torch.rand(B, 3, Ho, Wo, generator=g)
    zero = torch.zeros(3, device="cuda")
    tx = _transform(x.cuda(), Ho, Wo, zero, std).cpu().double()
    tty = _adjoint(y.cuda(), C, H, W, std)
    lhs, rhs = float((tx * y.double()).sum()), float((x.double() * tty.cpu().double()).sum())
    print(f"{B}x{C}x{H}x{W}: <Tx,y> {lhs:.10e}  <x,T'y> {rhs:.10e}  rel {abs(lhs - rhs) / abs(lhs):.2e}")
    assert abs(lhs - rhs) <= 1e-6 * abs(lhs)
    xd = x.double().requires_grad_(True)
    lin = (xd.repeat(1, 3 // C, 1, 1)) / torch.tensor(pp.STD, dtype=torch.float64).view(1, 3, 1, 1)
    if resize:
        lin = _bilinear64(lin, 224, 224)
    (lin * y.double()).sum().backward()
    assert (tty.cpu().double() - xd.grad).abs().max() <= 1e-5 * xd.grad.abs().max()
    assert torch.equal(tty, _adjoint(y.cuda(), C, H, W, std))          # a gather: bit for bit


@pytest.mark.parametrize("shape", [(2, 5, 7, 9), (1, 64, 224, 224), (2, 8, 15, 11), (1, 3, 2, 3)])
def test_maxpool_equals_torch(shape):
    abi = _abi()
    x = torch.randn(*shape, generator=torch.Generator().manual_seed(1))
    P, H, W = shape[0] * shape[1], shape[2], shape[3]
    y = torch.empty(shape[0], shape[1], H // 2, W // 2, device="cuda")
    abi.call("hg_maxpool2x2", abi.ptr(x.cuda()), abi.ptr(y), P, H, W, abi.stream())
    assert torch.equal(y.cpu(), F.max_pool2d(x, 2, 2))


@pytest.mark.parametrize("planes,H,W,pooled,with_loss", [(16, 15, 11, True, True), (12, 28, 28, True, True),
                                                         (8, 28, 28, False, True), (6, 13, 10, True, False)])
def test_level_boundary_backward_matches_fp64(planes, H, W, pooled, with_loss):
    abi = _abi()
    g = torch.Generator().manual_seed(planes + H)
    y = torch.relu(torch.randn(planes, H, W, generator=g))        # a ReLU output: about half zeros, all-zero windows included
    t = torch.relu(torch.randn(planes, H, W, generator=g)) * 1.5
    dp = torch.randn(planes, H // 2, W // 2, generator=g)
    gs = torch.tensor(0.7)
    inv_n = 1.0 / y.numel()
    yd = y.double().requires_grad_(True)
    if pooled:
        (F.max_pool2d(yd[None], 2, 2)[0] * dp.double()).sum().backward()
    ref = yd.grad if pooled else torch.zeros_like(yd)
    if with_loss:
        ref = ref + 0.7 * inv_n * (y.double() - t.double()).clamp(-1, 1)
    ref = ref * (y > 0)
    out = torch.empty(planes, H, W, device="cuda")
    yc, tc, dpc, gc = y.cuda(), t.cuda(), dp.cuda(), gs.cuda()
    abi.call("hg_vgg_level_bwd", abi.ptr(yc), abi.ptr(tc) if with_loss else None, abi.ptr(dpc) if pooled else None,
             abi.ptr(gc) if with_loss else None, inv_n, abi.ptr(out), planes, H, W, abi.stream())
    assert (out.cpu().double() - ref).abs().max() <= 1e-6 * ref.abs().max()


def _case(name):
    if name in FIXTURE:
        gold = np.load(GOLD)
        return torch.from_numpy(gold[f"{name}_input"]), torch.from_numpy(gold[f"{name}_target"]), FIXTURE[name], gold
    g = torch.Generator().manual_seed(9)
    return torch.rand(2, 3, 512, 256, generator=g), torch.rand(2, 3, 512, 256, generator=g), True, None


@pytest.mark.parametrize("name", list(FIXTURE) + ["rgb512x256"])
def test_module_matches_fp64_oracle_on_the_gpu_masks(name):
    x, t, resize, gold = _case(name)
    net = _net(resize)
    xc = x.cuda().requires_grad_(True)
    losses = net(xc, t.cuda())
    sum(losses).backward()
    with torch.no_grad():
        acts = net._run(x.cuda(), net._images(), True)[1]
    masks = [a > 0 for a in acts]
    # the max-pools' choices too: at 224x224 a few dozen windows hold two entries within fp32x3 rounding of each other
    pool_index = [F.max_pool2d(acts[e], 2, 2, return_indices=True)[1] for e in (1, 3, 6)]
    params = {k: v.cuda() for k, v in pp.module_params(pp.seeded_vgg16_state(0)).items()}
    xd = x.cuda().double().requires_grad_(True)
    pre = []
    ref = pp.losses(params, xd, t.cuda(), resize, masks=masks, pre=pre, pool_index=pool_index)
    sum(ref).backward()
    near = sum(int((p.abs() <= 1e-6 * p.abs().max()).sum()) for p in pre)
    errs = [abs(float(a.detach()) - float(b.detach())) / abs(float(b.detach())) for a, b in zip(losses, ref)]
    gerr = float((xc.grad.double() - xd.grad).norm() / xd.grad.norm())
    print(f"{name}: block losses rel {['%.1e' % e for e in errs]}, input gradient rel-L2 {gerr:.2e}, "
          f"{near} pre-activations within 1e-6 of zero")
    assert max(errs) <= 1e-4 and gerr <= 1e-3
    if gold is not None:        # and against the reference's own fp32 numbers
        want = gold[f"{name}_losses"]
        assert all(abs(float(a.detach()) - w) <= 2e-4 * abs(w) for a, w in zip(losses, want))


def test_cached_target_features_and_repeated_backward_are_bit_identical():
    net = _net()
    g = torch.Generator().manual_seed(3)
    x, t = torch.rand(1, 3, 512, 256, generator=g).cuda(), torch.rand(1, 3, 512, 256, generator=g).cuda()
    grads, values = [], []
    for use_cache in (False, True, True):
        xc = x.clone().requires_grad_(True)
        losses = net.loss(xc, net.target_features(t)) if use_cache else net(xc, t)
        sum(losses).backward()
        values.append(torch.stack([v.detach() for v in losses]))
        grads.append(xc.grad)
    assert torch.equal(values[0], values[1]) and torch.equal(values[1], values[2])
    assert torch.equal(grads[0], grads[1]) and torch.equal(grads[1], grads[2])
    weighted = net.loss(x, net.target_features(t), (1.0, 0.5, 0.25, 2.0))
    assert abs(float(weighted) - float((values[0] * torch.tensor([1.0, 0.5, 0.25, 2.0], device="cuda")).sum())) <= 1e-6 * float(weighted)
    with torch.autocast("cuda", dtype=torch.bfloat16):
        auto = net(x, t)
    assert all(v.dtype == torch.float32 for v in auto) and torch.equal(torch.stack(auto), values[0])
    assert torch.equal(net.get_features(x), net.target_features(x)[3])


def test_frozen_weights_launch_no_weight_gradient_and_repack_on_change(monkeypatch):
    abi = _abi()
    net = _net()
    names = []
    call = abi.call

    def recorder(name, *a, **k):
        names.append(name)
        return call(name, *a, **k)
    monkeypatch.setattr(abi, "call", recorder)
    monkeypatch.setattr(abi, "conv2d_wgrad", lambda *a, **k: pytest.fail("a weight gradient was launched"))
    g = torch.Generator().manual_seed(4)
    x = torch.rand(2, 3, 96, 64, generator=g).cuda().requires_grad_(True)
    t = torch.rand(2, 3, 96, 64, generator=g).cuda()
    sum(net(x, t)).backward()
    torch.cuda.synchronize()
    assert not any("wgrad" in n for n in names)
    assert names.count("hg_conv2d") == 30 and names.count("hg_vgg_level_bwd") == 4 and names.count("hg_vgg_input_adjoint") == 1
    assert all(p.grad is None for p in net.parameters())
    # operand images: packed once, packed again after an in-place edit, `load_state_dict` or `.to()`
    imgs = net._images()
    assert net._images() is imgs
    w = net.blocks[2]._modules["12"].weight
    with torch.no_grad():
        w.mul_(2.0)
    imgs2 = net._images()
    assert imgs2 is not imgs
    net.load_state_dict(_net(seed=1).state_dict())
    assert net._images() is not imgs2
    w.requires_grad_(True)
    with pytest.raises(RuntimeError, match="not built"):
        net(x, t)
    with torch.no_grad():
        net(x, t)                      # no autograd: the flag does not matter


def test_no_torch_convolution_pooling_interpolation_or_loss_on_the_path():
    net = _net()
    g = torch.Generator().manual_seed(5)
    x = torch.rand(1, 3, 512, 256, generator=g).cuda().requires_grad_(True)
    t = torch.rand(1, 3, 512, 256, generator=g).cuda()
    sum(net(x, t)).backward()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA]) as prof:
        sum(net(x, t)).backward()
        torch.cuda.synchronize()
    names = {e.name for e in prof.events()}
    for bad in ("aten::convolution", "aten::cudnn_convolution", "max_pool2d", "upsample_bilinear2d", "smooth_l1_loss"):
        assert not any(bad in n for n in names), (bad, sorted(n for n in names if bad in n))


@pytest.mark.parametrize("which", ["tiny", "420"])
def test_inversion_with_the_perceptual_term(pkg, which):
    inv = importlib.import_module("3dhumangan_b200.inversion")
    G, cfg, cond = _released_like(pkg, which)
    state = {k: v.clone() for k, v in G.state_dict().items()}
    flags = [p.requires_grad for p in G.parameters()]
    net = _net()
    vgg = {k: v.clone() for k, v in net.state_dict().items()}
    torch.manual_seed(11)
    with torch.no_grad():
        target = G(torch.randn(1, cfg["latent_dim"], device="cuda"), cond, **cfg)["rgbs"]
    kw = dict(cfg, perceptual_lambda=(1, 1, 1, 1))       # the merged config's own perceptual_lambda is [0, 0, 0, 0]
    runs = [inv.invert(G, target, cond, space="film", steps=60, lr=0.02, seed=5, perceptual=net, **kw) for _ in range(2)]
    torch.cuda.synchronize()
    losses = runs[0]["losses"]
    print(f"{which} + perceptual: objective {losses[0]:.4e} -> {losses[-1]:.4e} ({losses[0] / losses[-1]:.1f}x) in 60 steps")
    assert len(losses) == 60 and all(v == v for v in losses)
    assert losses[-1] * 10 <= losses[0]
    spread = max(abs(a - b) / b for a, b in zip(runs[1]["losses"], losses))
    image_spread = float((runs[1]["image"] - runs[0]["image"]).norm() / runs[0]["image"].norm())
    print(f"{which} + perceptual: second run differs by {spread:.2e} (objective), {image_spread:.2e} (final image)")
    # The perceptual path repeats bit for bit for identical inputs (test above), but the generator's run-to-run differences
    # (its atomic sums) grow more over 60 steps of this objective than of the pixel loss alone.  Measured in two invocations:
    # 420 4.0e-5 / 2.2e-4 on the objective, 4.3e-6 / 4.4e-6 on the final image; tiny (32x32 up-sampled 7x to 224x224)
    # 3.9e-2 / 3.8e-2 and 1.3e-3 / 7.4e-4.  The objective is held to 10x the larger value, the 420 image to SPREAD.
    bound = (2.2e-3, SPREAD) if which == "420" else (0.4, 1.3e-2)
    assert spread < bound[0] and image_spread < bound[1]
    assert all(torch.equal(v, state[k]) for k, v in G.state_dict().items())
    assert not G.training and [p.requires_grad for p in G.parameters()] == flags
    assert all(p.grad is None for p in G.parameters())
    assert all(torch.equal(v, vgg[k]) for k, v in net.state_dict().items())
    if which == "tiny":           # the perceptual term alone
        res = inv.invert(G, target, cond, space="film", steps=20, lr=0.02, seed=5, loss=None, perceptual=net,
                         **dict(cfg, perceptual_lambda=(1, 1, 0.5, 0.5)))
        assert res["losses"][-1] < res["losses"][0]
        with pytest.raises(RuntimeError, match="pixel loss, a perceptual loss"):
            inv.invert(G, target, cond, steps=1, loss=None, **cfg)
        with pytest.raises(RuntimeError, match="switches the perceptual term off"):
            inv.invert(G, target, cond, steps=1, perceptual=net, **cfg)
