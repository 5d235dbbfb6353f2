"""Conditional (reconstruction) phases on the GPU: the latent-pool lookup and its dense gradient, the latent regression and the
smooth-L1 photometric mode of hg_image_loss against fp64, then `Trainer(fused=True)`'s conditional discriminator and generator
steps against the same steps composed from the oracle (oracle/port.py, oracle/perceptual_port.py) under torch autograd, and one
conditional iteration under fp16 autocast + GradScaler with FusedAdam."""
import importlib

import pytest
import torch
import torch.nn.functional as F

from oracle import perceptual_port as pp

pytestmark = pytest.mark.gpu


def _ops():
    return importlib.import_module("3dhumangan_b200.ops.trainer_ops")


# ----------------------------------------------------------------------------------------------------------------------
# kernels
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("P,L", [(1000, 256), (37, 420), (219047, 420)])
def test_latent_pool_gather_and_dense_gradient_match_torch(P, L):
    ops = _ops()
    g = torch.Generator().manual_seed(P + L)
    pool = torch.randn(P, L, generator=g).cuda().requires_grad_(True)
    idx = torch.tensor([17, 3, P - 1, 17, 0, 3, 17, 12], dtype=torch.int64)          # unsorted, repeated
    dz = torch.randn(idx.numel(), L, generator=g)
    out = ops.latent_pool_gather(pool, idx.cuda())
    assert torch.equal(out.detach(), pool.detach()[idx.cuda()])
    grads = []
    for _ in range(2):
        pool.grad = None
        ops.latent_pool_gather(pool, idx.cuda()).backward(dz.cuda())
        grads.append(pool.grad.clone())
    torch.cuda.synchronize()
    ref = torch.zeros(P, L, dtype=torch.float64).index_add_(0, idx, dz.double()).float()
    assert torch.equal(grads[0].cpu(), ref)                 # fp64 sums in batch order, rounded once
    assert torch.equal(grads[0], grads[1])                  # no atomics: repeats bit for bit
    untouched = torch.ones(P, dtype=torch.bool)
    untouched[idx] = False
    assert not grads[0][untouched.cuda()].any()


def test_latent_pool_indices_out_of_range_stay_in_bounds():
    ops = _ops()
    P, L = 8, 64
    pool = torch.randn(P, L, device="cuda", requires_grad=True)
    idx = torch.tensor([2, P, -1, 2], dtype=torch.int64, device="cuda")
    out = ops.latent_pool_gather(pool, idx)
    assert torch.equal(out[0], pool.detach()[2]) and torch.equal(out[3], pool.detach()[2])
    assert torch.isnan(out[1]).all() and torch.isnan(out[2]).all()
    dz = torch.randn(4, L, device="cuda")
    out.backward(dz)
    torch.cuda.synchronize()
    expect = torch.zeros(P, L, device="cuda")
    expect[2] = (dz[0].double() + dz[3].double()).float()
    assert torch.equal(pool.grad, expect)


def _normalize64(x):
    return x * (x.square().mean(dim=1, keepdim=True) + 1e-8).rsqrt()


@pytest.mark.parametrize("B", [1, 4, 32])
@pytest.mark.parametrize("L", [64, 256, 420])
def test_latent_loss_matches_fp64(B, L):
    ops = _ops()
    g = torch.Generator().manual_seed(B * 1000 + L)
    pred = torch.randn(B, L, generator=g) * 1.5
    target = torch.randn(B, L, generator=g)
    target[:, : L // 4] = pred[:, : L // 4] * 0.97           # |d| < beta on part of every row: both smooth-L1 branches
    if B > 1:
        pred[1] = 0                                           # a row of zeros: n(0) = 0, the eps branch of the Jacobian
        target[0] = 0
    p64 = pred.double().requires_grad_(True)
    ref = F.smooth_l1_loss(_normalize64(p64), _normalize64(target.double()), beta=0.1)
    ref.backward(torch.tensor(2.5, dtype=torch.float64))
    p = pred.cuda().requires_grad_(True)
    loss = ops.latent_loss(p, target.cuda(), beta=0.1)
    (loss * 2.5).backward()
    again = ops.latent_loss(pred.cuda(), target.cuda(), beta=0.1)
    torch.cuda.synchronize()
    assert float(loss.detach()) == pytest.approx(float(ref), rel=2e-6, abs=1e-9)
    assert torch.equal(loss.detach(), again)
    scale = float(p64.grad.abs().max())
    err = float((p.grad.cpu().double() - p64.grad).abs().max())
    assert err <= 1e-5 * scale, (err, scale)


@pytest.mark.parametrize("masked", [False, True])
def test_image_loss_smooth_l1_mode_matches_fp64_and_the_other_modes_hold(masked):
    ops = _ops()
    g = torch.Generator().manual_seed(5 + masked)
    B, H, W = 3, 17, 23
    pred = torch.rand(B, 3, H, W, generator=g) * 2 - 1
    target = pred + (torch.rand(B, 3, H, W, generator=g) * 2 - 1) * 0.3          # |d| on both sides of beta = 0.1
    mask = (torch.rand(B, 1, H, W, generator=g) > 0.3).float() if masked else None
    m64 = mask.double() if masked else torch.ones(B, 1, H, W, dtype=torch.float64)
    for kind, rho in (("smooth_l1", lambda d: torch.where(d.abs() < 0.1, 0.5 * d * d / 0.1, d.abs() - 0.05)),
                      ("l2", lambda d: d * d), ("charbonnier", lambda d: torch.sqrt(d * d + 1e-6))):
        p64 = pred.double().requires_grad_(True)
        ref = (m64 * rho(p64 - target.double())).mean()
        ref.backward()
        p = pred.cuda().requires_grad_(True)
        loss = ops.image_loss(p, target.cuda(), None if mask is None else mask.cuda(), kind=kind, eps=1e-3, beta=0.1)
        loss.backward()
        again = ops.image_loss(pred.cuda(), target.cuda(), None if mask is None else mask.cuda(), kind=kind, eps=1e-3, beta=0.1)
        torch.cuda.synchronize()
        assert float(loss) == pytest.approx(float(ref), rel=1e-6), kind
        assert torch.equal(loss.detach(), again), kind
        err = float((p.grad.cpu().double() - p64.grad).abs().max())
        assert err <= 1e-6 * float(p64.grad.abs().max()), (kind, err)


# ----------------------------------------------------------------------------------------------------------------------
# whole steps
# ----------------------------------------------------------------------------------------------------------------------
def _setup(pkg, port, monkeypatch, B=2, seed=7):
    gen = importlib.import_module("3dhumangan_b200.modules.generator")
    disc = importlib.import_module("3dhumangan_b200.modules.discriminator")
    rng = importlib.import_module("3dhumangan_b200.rng")
    cfg = pkg.configs.baseline_config("tiny")
    cfg.update(gen_height=64, gen_width=64, render_height=8, render_width=8, num_steps=32, nerf_noise=0.5, grad_clip=1e9,
               batch_split=1, latent_lambda=1.0, photometric_lambda=1.0, perceptual_lambda=[1.0, 1.0, 1.0, 1.0])
    cfg["phases"] = [{"name": "cond", "uncond": False, "rotate": False, "gen_modal": "rgbs", "do_r1": False}]
    pg = {k: v.cuda() for k, v in port.init_generator_params(cfg, seed=5, sigma_gain=200.0, sigma_bias=1.0).items()}
    pd = {k: v.cuda() for k, v in port.init_discriminator_params(cfg, seed=6).items()}
    codes, app = pkg.synthetic.make_appearance(B, cfg["dataset_length"], cfg["latent_dim"], seed=seed)
    pg["latent_pool.latents"] = codes.cuda()
    G = gen.Map3DGenerator(**cfg).cuda().train()
    G.load_state_dict(pg, strict=True)
    G.set_device(torch.device("cuda:0"))
    D = disc.UNetDiscriminator(**cfg).cuda().train()
    D.load_state_dict(pd, strict=True)
    # the full-extent latent head sees a 2x2 bottleneck at 64x64: it is live (a 1x1 bottleneck would make it constant zero)
    assert min(D.latent_layer.weight.shape[2:]) > 1
    g = torch.Generator().manual_seed(seed)
    cond = {k: v.cuda() for k, v in pkg.synthetic.make_conditions(B, seed=8).items()}
    cond.update({k: v.cuda() for k, v in app.items()})
    batch = dict(z_d=torch.randn(B, cfg["latent_dim"], generator=g).cuda(), z_g=torch.randn(B, cfg["latent_dim"], generator=g).cuda(),
                 cond=cond, images=torch.randn(B, 3, 64, 64, generator=g).clamp_(-1, 1).cuda(),
                 labels=torch.randint(0, cfg["label_dim"], (B, 64, 64), generator=g).cuda())
    u, noise = rng.draw_render_noise(B, 64, 32, "cuda", cfg["sample_dist"])
    monkeypatch.setattr(rng, "draw_render_noise", lambda *a, **k: (u, noise))
    vgg = importlib.import_module("3dhumangan_b200.perceptual").VGGPerceptualLoss(weights=pp.seeded_vgg16_state(0)).cuda()
    return cfg, pg, pd, G, D, batch, (u, noise), vgg


def _rel_errs(named, ref, min_count):
    scale = max(float(v.norm()) for v in ref.values() if v is not None)
    errs = {}
    for n, p in named:
        r = ref.get(n)
        if r is None or float(r.norm()) < 1e-6 * scale:
            continue
        assert p.grad is not None, n
        errs[n] = float((p.grad.double() - r.double()).norm() / r.double().norm())
    assert len(errs) >= min_count, len(errs)
    vals = sorted(errs.values())
    assert vals[len(vals) // 2] < 2e-2, (vals[len(vals) // 2], sorted(errs.items(), key=lambda kv: -kv[1])[:5])
    assert vals[-1] < 0.3, sorted(errs.items(), key=lambda kv: -kv[1])[:5]
    return errs


def _no_tf32():
    old = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    return old


def test_conditional_discriminator_step_matches_oracle_composition(pkg, port, monkeypatch):
    ts = importlib.import_module("3dhumangan_b200.train_step")
    old = _no_tf32()
    try:
        cfg, pg, pd, G, D, batch, (u, noise), vgg = _setup(pkg, port, monkeypatch)
        idx, cond = batch["cond"]["indices"], batch["cond"]
        with torch.no_grad():
            zc = pg["latent_pool.latents"][idx]
            fake = port.generator_forward(pg, zc, cond, cfg, u, noise, training=True)["rgbs"]
        P = {k: (v.clone().requires_grad_(True) if v.is_floating_point() and "weight_u" not in k and "weight_v" not in k else v.clone())
             for k, v in pd.items()}
        st = {}
        out_real = port.discriminator_forward(P, batch["images"], cfg, training=True, stats_out=st)
        P2 = dict(P)
        P2.update({k: v.detach() for k, v in st.items()})
        out_gen = port.discriminator_forward(P2, fake, cfg, training=True)
        Ld = cfg["label_dim"]
        seg = ts.segmentation_loss(out_real["segments"], batch["labels"], Ld) + \
            ts.segmentation_loss(out_gen["segments"], torch.zeros_like(batch["labels"]), Ld)
        lat = ts.latent_regression_loss(out_gen["latents"], zc) + ts.latent_regression_loss(out_real["latents"], cond["latents"])
        ref_loss = seg * cfg["segmentation_lambda"] + lat * cfg["latent_lambda"]
        ref_loss.backward()
        ref_grads = {k: v.grad for k, v in P.items() if v.requires_grad}
        t = ts.Trainer(G, D, cfg, amp=False, ddp=False, perceptual=vgg)
        loss = t.train_discriminator(batch)
        torch.cuda.synchronize()
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old
    assert float(lat) > 1e-3 * float(ref_loss)
    assert abs(float(loss) - float(ref_loss)) < 2e-3 * abs(float(ref_loss)), (float(loss), float(ref_loss))
    errs = _rel_errs(D.named_parameters(), ref_grads, 25)
    assert "latent_layer.weight" in errs


def test_conditional_generator_step_matches_oracle_composition(pkg, port, monkeypatch):
    ts = importlib.import_module("3dhumangan_b200.train_step")
    old = _no_tf32()
    try:
        cfg, pg, pd, G, D, batch, (u, noise), vgg = _setup(pkg, port, monkeypatch)
        idx, cond = batch["cond"]["indices"], batch["cond"]
        P = {k: (v.clone().requires_grad_(True) if v.is_floating_point() else v.clone()) for k, v in pg.items()}
        z = P["latent_pool.latents"][idx]
        fake = port.generator_forward(P, z, cond, cfg, u, noise, training=True)["rgbs"]
        out = port.discriminator_forward(pd, fake, cfg, training=True)
        lat = ts.latent_regression_loss(out["latents"], z.detach()) + F.smooth_l1_loss(batch["z_g"], cond["latents"], beta=0.1)
        vparams = pp.module_params(pp.seeded_vgg16_state(0))
        vparams = {k: v.cuda() for k, v in vparams.items()}
        perc = sum(pp.losses(vparams, 0.5 * fake + 0.5, 0.5 * batch["images"] + 0.5, True)).float()
        photo = F.smooth_l1_loss(fake, batch["images"], beta=0.1)
        seg = ts.segmentation_loss(out["segments"], batch["labels"], cfg["label_dim"])
        ref_loss = lat * cfg["latent_lambda"] + perc + photo * cfg["photometric_lambda"] + seg * cfg["segmentation_lambda"]
        ref_loss.backward()
        ref_grads = {k: v.grad for k, v in P.items() if isinstance(v, torch.Tensor) and v.requires_grad}
        t = ts.Trainer(G, D, cfg, amp=False, ddp=False, perceptual=vgg)
        d_before = [p.detach().clone() for p in D.parameters()]
        loss = t.train_generator(batch)
        torch.cuda.synchronize()
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old
    for n in ("perc", "photo", "lat"):
        assert float(locals()[n]) > 1e-3 * float(ref_loss), n
    assert abs(float(loss) - float(ref_loss)) < 2e-3 * abs(float(ref_loss)), (float(loss), float(ref_loss))
    errs = _rel_errs(G.named_parameters(), ref_grads, 100)
    pool, ref_pool = G.latent_pool.latents.grad, ref_grads["latent_pool.latents"]
    touched = torch.zeros(pool.shape[0], dtype=torch.bool, device="cuda")
    touched[idx] = True
    assert not pool[~touched].any()                           # rows not indexed: exactly zero
    assert float((pool[touched] - ref_pool[touched]).norm() / ref_pool[touched].norm()) < 2e-2, errs.get("latent_pool.latents")
    for p, q in zip(D.parameters(), d_before):                 # the frozen discriminator passes the gradient, keeps its weights
        assert torch.equal(p.detach(), q)


def test_conditional_iteration_under_amp_with_fused_adam(pkg, port, monkeypatch):
    ts = importlib.import_module("3dhumangan_b200.train_step")
    B = 4
    cfg, pg, pd, G, D, batch, _, vgg = _setup(pkg, port, monkeypatch, B=B, seed=9)
    t = ts.Trainer(G, D, cfg, amp=True, ddp=False, perceptual=vgg)
    assert isinstance(t.optimizer_G, _ops().FusedAdam)
    idx = batch["cond"]["indices"]
    touched = torch.zeros(G.latent_pool.latents.shape[0], dtype=torch.bool, device="cuda")
    touched[idx] = True
    pool0 = G.latent_pool.latents.detach().clone()
    k = [i for i, p in enumerate(p for p in G.parameters() if p.requires_grad) if p is G.latent_pool.latents][0]
    for _ in range(2):                  # the first step may be skipped while GradScaler finds its scale
        d, g = t.iteration(batch)
        assert torch.isfinite(d) and torch.isfinite(g)
    torch.cuda.synchronize()
    pool = G.latent_pool.latents.detach()
    shadow = t.ema.shadow_params[k]
    assert bool((pool[touched] != pool0[touched]).any(dim=1).all())         # every indexed row moved
    assert torch.equal(pool[~touched], pool0[~touched])                     # the rest of the pool is outside the graph
    assert bool((shadow[touched] != pool0[touched]).any(dim=1).all())
    assert torch.equal(shadow[~touched], pool0[~touched])
    for p in list(G.parameters()) + list(D.parameters()):
        assert torch.isfinite(p).all()
