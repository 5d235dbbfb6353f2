"""hierarchical_sample=True on the device: hg_sample_fine against the oracle's sample_pdf, hg_merge_samples against
torch.sort + gather, the renderer at 256 (fused) and 384 / 420 (zero-padded) against the oracle with the device's fine
depths injected, the training renderer's gradients over the merged samples against fp64 autograd, CUDA-graph replay and
one trainer iteration."""
import importlib

import pytest
import torch

from golden_util import rel_l2
import hierarchical_oracle
from test_oracle_pin_hierarchical import hierarchical_case

pytestmark = pytest.mark.gpu


def _mod(name):
    return importlib.import_module("3dhumangan_b200." + name)


# ------------------------------------------------------------------------------------------------ hg_sample_fine
def _sampling_case(kind, B=2, Rw=8, Rh=4, S=32, seed=0):
    g = torch.Generator().manual_seed(seed)
    R = Rw * Rh
    zs = torch.linspace(0.88, 1.12, S)
    z = (zs + (torch.rand(B, R, S, generator=g) - 0.5) * (zs[1] - zs[0]) + 10.0)
    if kind == "miss":            # every density zero: uniform pdf
        sigma = -torch.rand(B, R, S, generator=g) - 1.0
    elif kind == "dominant":      # one opaque sample per ray
        sigma = torch.full((B, R, S), -5.0)
        hit = torch.randint(2, S - 2, (B, R), generator=g)
        sigma.scatter_(2, hit[..., None], 1e4)
    else:                         # a dense shell: transmittance 0 behind it, so most cdf bins are narrower than eps
        sigma = torch.randn(B, R, S, generator=g) * 50 + 200
    noise = torch.randn(B, R, S, 1, generator=g)
    u_pdf = torch.rand(B * R, S, generator=g)
    return z, sigma, noise, u_pdf


def _oracle_pdf(port, z, sigma, noise, u_pdf, noise_std, clamp):
    B, R, S = z.shape
    out = torch.cat([torch.zeros(B, R, S, 3), sigma[..., None]], -1).double()
    _, _, w = port.ray_integration(out, z.double()[..., None], noise.double(), noise_std, False, False, clamp)
    w = w.reshape(B * R, S) + 1e-5
    zf = z.double().reshape(B * R, S)
    mid = 0.5 * (zf[:, :-1] + zf[:, 1:])
    wt = w[:, 1:-1] + 1e-5
    cdf = torch.cat([torch.zeros(B * R, 1, dtype=torch.float64), torch.cumsum(wt / wt.sum(-1, keepdim=True), -1)], -1)
    return hierarchical_oracle.sample_pdf(mid, w[:, 1:-1], u_pdf.double()), cdf, mid


@pytest.mark.parametrize("kind", ["miss", "dominant", "shell"])
@pytest.mark.parametrize("clamp, noise_std", [("relu", 0.0), ("softplus", 0.5)])
def test_sample_fine_matches_sample_pdf(port, kind, clamp, noise_std):
    abi = _mod("abi")
    z, sigma, noise, u_pdf = _sampling_case(kind)
    B, R, S = z.shape
    Rw, Rh = 8, 4
    c2w = torch.eye(4).repeat(B, 1, 1)
    c2w[:, :3, 3] = torch.tensor([0.1, -0.2, 0.3])
    c2w[1, :3, :3] = torch.tensor([[0.0, 0.0, 1.0], [0.0, 1.0, 0.0], [-1.0, 0.0, 0.0]])
    focals = torch.tensor([9.0, 11.0])
    xs, ys = torch.linspace(-Rw / Rh, Rw / Rh, Rw), torch.linspace(-1, 1, Rh)
    fz, pts = abi.sample_fine(sigma.reshape(B, R * S).cuda(), 1, z.reshape(B, R * S).cuda(), noise.reshape(B, R * S).cuda(),
                              u_pdf.cuda(), noise_std=noise_std, clamp_mode=clamp, xs=xs.cuda(), ys=ys.cuda(), focals=focals.cuda(),
                              cam2world=c2w.cuda(), B=B, Rw=Rw, Rh=Rh, S=S)
    ref, cdf, mid = _oracle_pdf(port, z, sigma, noise, u_pdf, noise_std, clamp)
    width = (mid[:, 1:] - mid[:, :-1]).mean(-1, keepdim=True)
    # the chosen bin is the same wherever u is not within 1e-6 of a cdf knot
    far = ((u_pdf.double()[:, :, None] - cdf[:, None, :]).abs() > 1e-6).all(-1)
    err = ((fz.cpu().double().reshape(B * R, S) - ref).abs() / width)[far]
    assert far.float().mean() > 0.9
    assert err.max() <= 1e-2, float(err.max())
    assert err.median() <= 1e-4, float(err.median())
    # fine points: cam2world . (0,0,0,1) + cam2world[:3,:3] . normalize(x, y, focal) * z
    x = xs[None, :].expand(Rh, Rw).reshape(-1)
    y = ys[:, None].expand(Rh, Rw).reshape(-1)
    d = torch.stack([x[None].expand(B, -1), y[None].expand(B, -1), focals[:, None].expand(B, R)], -1)
    d = d / (d.norm(dim=-1, keepdim=True) + 1e-12)
    dw = torch.einsum("bij,brj->bri", c2w[:, :3, :3], d)
    want = c2w[:, None, None, :3, 3] + dw[:, :, None] * fz.cpu().reshape(B, R, S, 1)
    assert (pts.cpu().reshape(B, R, S, 3) - want).abs().max() < 1e-5


def test_merge_samples_equals_sort_and_gather():
    abi = _mod("abi")
    B, R, S = 2, 96, 32
    g = torch.Generator().manual_seed(3)
    cz = (torch.rand(B, R, S, generator=g) * 0.01 + 0.005).cumsum(-1)
    fz = torch.rand(B, R, S, generator=g) * cz[..., -1:]
    fz[:, :, :4] = cz[:, :, 3:7]                 # exact ties: the fine sample comes first
    crec, frec = torch.randn(B, R * S, 36, generator=g), torch.randn(B, R * S, 36, generator=g)
    rec, z, perm = abi.merge_samples(frec.cuda(), fz.reshape(B, -1).cuda(), crec.cuda(), cz.reshape(B, -1).cuda(), B=B, R=R, S=S,
                                     want_perm=True)
    all_z = torch.cat([fz, cz], -1)
    _, order = torch.sort(all_z, dim=-1, stable=True)
    assert torch.equal(perm.cpu().reshape(B, R, 2 * S).long(), order)
    assert torch.equal(z.cpu().reshape(B, R, 2 * S), torch.gather(all_z, -1, order))
    all_rec = torch.cat([frec.reshape(B, R, S, 36), crec.reshape(B, R, S, 36)], 2)
    want = torch.gather(all_rec, 2, order[..., None].expand(-1, -1, -1, 36))
    assert torch.equal(rec.cpu().reshape(B, R, 2 * S, 36), want)


# ------------------------------------------------------------------------------------------------ renderer forward
def _device_fine(P, freq, phase, cond, cfg, u, noise):
    h = _mod("modules.hierarchical").merged_records(P, freq, phase, cond, cfg, u, noise, want_nearest=True, want_fine=True)
    return h["fine_z"].cpu(), h["nearest"].cpu().long()


def _cuda_noise(pkg, noise):
    return pkg.rng.HierarchicalNoise(noise.coarse.cuda(), noise.u_pdf.cuda(), noise.final.cuda())


@pytest.mark.parametrize("name", ["relu_n0", "relu_n5", "softplus_n0", "softplus_n5"])
def test_render_256_matches_oracle(pkg, port, name):
    ren = _mod("modules.render_ops")
    cfg, params, cond, z, (u, noise), gold = hierarchical_case(name)
    with torch.no_grad():
        freq, phase = port.mapping_network(params, z)
    gp = {k: v.cuda() for k, v in params.items()}
    cg = {k: v.cuda() for k, v in cond.items()}
    nd = _cuda_noise(pkg, noise)
    fz, near = _device_fine(gp, freq.cuda(), phase.cuda(), cg, cfg, u.cuda(), nd)
    out = ren.render_forward(gp, freq.cuda(), phase.cuda(), cg, cfg, u.cuda(), nd, want_weights=True, want_nearest=True)
    torch.cuda.synchronize()
    with torch.no_grad():
        rgb_r, fmap, depth, w, idx, _ = hierarchical_oracle.render(params, freq, phase, cond, cfg, u, noise, fine_z=fz)
        *_, idx_self, fz_self = hierarchical_oracle.render(params, freq, phase, cond, cfg, u, noise)
    B, R = z.shape[0], cfg["render_width"] * cfg["render_height"]
    ro = out["ray_out"].cpu()
    assert torch.equal(out["nearest"].cpu().long(), near)
    assert (near != idx).float().mean() < 2e-3
    assert rel_l2(out["weights"].cpu().reshape(w.shape), w) < 1e-3
    assert rel_l2(ro[..., :256], fmap.permute(0, 2, 3, 1).reshape(B, R, -1)) < 1e-3, "feature maps"
    assert rel_l2(ro[..., 256:259], ((rgb_r + 1) / 2).permute(0, 2, 3, 1).reshape(B, R, 3)) < 1e-3, "rgb"
    assert rel_l2(ro[..., 259:260], depth) < 1e-4, "depth"
    # the device's own samples against the oracle's own: coarse sigmas that differ in fp32 rounding move a sample whose u
    # lies near a cdf knot into the neighbouring bin; reported, with the nearest-vertex decisions that change
    fine_differs = (fz.reshape(-1, cfg["num_steps"]) - fz_self).abs().max()
    print(f"{name}: max |fine z device - oracle| {float(fine_differs):.2e}, "
          f"nearest-vertex differences with the oracle's own samples {(near != idx_self).float().mean().item():.2e}")


@pytest.mark.parametrize("C", [384, 420])
def test_render_wide_matches_oracle(pkg, port, C):
    wo = _mod("modules.wide_ops")
    cfg, _, cond, z, (u, noise), _ = hierarchical_case("softplus_n5")
    cfg.update(hidden_dim=C, feature_dim=C, latent_dim=C, legacy_mode=C == 420, last_back=C == 420)
    params = port.init_generator_params(cfg, seed=9, sigma_gain=200.0, sigma_bias=1.0)
    zz = torch.randn(z.shape[0], C, generator=torch.Generator().manual_seed(1))
    with torch.no_grad():
        freq, phase = port.mapping_network(params, zz)
    gp = {k: v.cuda() for k, v in params.items()}
    cg = {k: v.cuda() for k, v in cond.items()}
    nd = _cuda_noise(pkg, noise)
    fz, near = _device_fine(gp, freq.cuda(), phase.cuda(), cg, cfg, u.cuda(), nd)
    feats, rgb01, depth_k = wo.render_forward_wide(gp, freq.cuda(), phase.cuda(), cg, cfg, u.cuda(), nd)
    torch.cuda.synchronize()
    with torch.no_grad():
        rgb_r, fmap, depth, w, idx, _ = hierarchical_oracle.render(params, freq, phase, cond, cfg, u, noise, fine_z=fz)
    B, R = z.shape[0], cfg["render_width"] * cfg["render_height"]
    assert (near != idx).float().mean() < 2e-3
    assert rel_l2(feats.cpu(), fmap.permute(0, 2, 3, 1).reshape(B, R, -1)) < 1e-3
    assert rel_l2(rgb01.cpu(), ((rgb_r + 1) / 2).permute(0, 2, 3, 1).reshape(B, R, 3)) < 1e-3
    assert rel_l2(depth_k.cpu(), depth) < 1e-4


# ------------------------------------------------------------------------------------------------ gradients
@pytest.mark.parametrize("C", [256, 384])
def test_training_renderer_gradients_over_merged_samples(pkg, port, C):
    """The training renderer on the merged 2S records: neural-field parameter and freq / phase gradients against fp64
    autograd of the oracle's MLP + integration over the same records (the fine depths carry no gradient)."""
    rt = _mod("modules.render_train")
    wo = _mod("modules.wide_ops")
    hier = _mod("modules.hierarchical")
    cfg, _, cond, z, (u, noise), _ = hierarchical_case("relu_n5")
    cfg.update(hidden_dim=C, feature_dim=C, latent_dim=C, white_back=True)
    params = port.init_generator_params(cfg, seed=13, sigma_gain=60.0, sigma_bias=2.0)
    names = [n for n in params if n.startswith("neural_field.")]
    g = torch.Generator().manual_seed(2)
    freq, phase = torch.randn(z.shape[0], 4 * C, generator=g), torch.randn(z.shape[0], 4 * C, generator=g)
    gp = {n: v.cuda().requires_grad_(n in names) for n, v in params.items()}
    cg = {k: v.cuda() for k, v in cond.items()}
    h = hier.merged_records(gp, freq.cuda(), phase.cuda(), cg, cfg, u.cuda(), _cuda_noise(pkg, noise))
    rec, zv, rcfg, nz = h["rec"], h["z_vals"], h["cfg"], h["noise"]
    B, N = zv.shape
    S2 = rcfg["num_steps"]
    R = N // S2
    wgt = torch.randn(B, R, 3 + C, generator=g)
    if C == 256:
        ray, tape = rt.mlp_forward_train(gp, freq.cuda(), phase.cuda(), rec, zv, nz, rcfg)
    else:
        tape = {}
        wo.render_forward_wide(gp, freq.cuda(), phase.cuda(), None, rcfg, None, nz, tape=tape, records=(rec, zv))
    dfq, dph = rt.mlp_backward(tape, wgt[..., 3:].cuda(), wgt[..., :3].cuda())
    torch.cuda.synchronize()
    # fp64 oracle over the same records, with the device's ReLU mask on sigma (the gradient is discontinuous there)
    mask = ((tape["sig"].cpu().double() + nz.cpu().double() * cfg["nerf_noise"]) > 0).double().reshape(B, R, S2, 1)
    pc = {n: params[n].clone().double().requires_grad_(True) for n in names}
    fq, ph = freq.double().requires_grad_(True), phase.double().requires_grad_(True)
    r = rec.cpu().double()
    dirs = torch.zeros(B, N, 3, dtype=torch.float64)
    dirs[..., -1] = -1
    raw = port.siren(pc, r[..., :3], fq, ph, r[..., 3:34], dirs, 1.0, C, 4)
    relu = port.F.relu
    try:
        port.F.relu = lambda v: v * mask
        rgbf, _, _ = port.ray_integration(raw.reshape(B, R, S2, -1), zv.cpu().double().reshape(B, R, S2, 1),
                                          nz.cpu().double().reshape(B, R, S2, 1), cfg["nerf_noise"], True, False, "relu")
    finally:
        port.F.relu = relu
    (rgbf * wgt.double()).sum().backward()
    assert 0.05 < mask.mean().item() < 0.95
    rel = lambda a, b: ((a - b).norm() / b.norm()).item()
    bad = {n: e for n in names if (e := rel(gp[n].grad.cpu().double(), pc[n].grad)) > 1e-3}
    assert not bad, sorted(bad.items(), key=lambda t: -t[1])
    assert rel(dfq.cpu().double(), fq.grad) < 1e-3
    assert rel(dph.cpu().double(), ph.grad) < 1e-3


# ------------------------------------------------------------------------------------------------ generator surface
def _tiny_generator(pkg, port, C=256, **over):
    gen = _mod("modules.generator")
    cfg = pkg.configs.baseline_config("tiny")
    cfg.update(gen_height=64, gen_width=64, render_height=8, render_width=8, num_steps=32, nerf_noise=0.5,
               hierarchical_sample=True, hidden_dim=C, feature_dim=C, latent_dim=C, **over)
    G = gen.Map3DGenerator(**cfg).cuda()
    G.load_state_dict({k: v.cuda() for k, v in port.init_generator_params(cfg, seed=5, sigma_gain=200.0, sigma_bias=1.0).items()})
    G.set_device(torch.device("cuda:0"))
    return G, cfg


def test_cuda_graph_replay_equals_eager(pkg, port, monkeypatch):
    rng = _mod("rng")
    G, cfg = _tiny_generator(pkg, port)
    G.eval()
    B = 2
    z = torch.randn(B, cfg["latent_dim"], generator=torch.Generator().manual_seed(4)).cuda()
    cond = {k: v.cuda() for k, v in pkg.synthetic.make_conditions(B, seed=3).items()}
    torch.manual_seed(8)
    u, noise = rng.draw_hierarchical_noise(B, 64, 32, "cuda", cfg["sample_dist"])
    monkeypatch.setattr(rng, "draw", lambda *a, **k: (u, noise))          # the same draws on both sides
    with torch.no_grad():
        oe = G(z, cond, **cfg)
        og = G(z, cond, hg_cuda_graph=True, **cfg)
        og2 = G(z, cond, hg_cuda_graph=True, **cfg)                       # a replay of the captured graph
    torch.cuda.synchronize()
    for o in (og, og2):
        assert rel_l2(o["rgbs_render"].cpu(), oe["rgbs_render"].cpu()) < 1e-6
        assert rel_l2(o["rgbs"].cpu(), oe["rgbs"].cpu()) < 1e-4      # fp32 atomics in the BN statistics are order-dependent


@pytest.mark.parametrize("C", [256, 420])
def test_staged_forward_sample_app_settings(pkg, port, C):
    G, cfg = _tiny_generator(pkg, port, C=C, legacy_mode=C == 420)
    G.eval()
    B = 1
    z = torch.randn(B, cfg["latent_dim"], generator=torch.Generator().manual_seed(4)).cuda()
    cond = {k: v.cuda() for k, v in pkg.synthetic.make_conditions(B, seed=3).items()}
    kw = {k: v for k, v in cfg.items() if k not in ("render_height", "render_width")}
    kw.update(nerf_noise=0.0, last_back=True)
    out = G.staged_forward(z, cond, cfg["render_height"], cfg["render_width"], truncation_psi=0.7, **kw)
    assert out["rgbs"].shape == (B, 3, 64, 64) and torch.isfinite(out["rgbs"]).all()
    assert out["depths"].shape == (B, 1, 8, 8) and torch.isfinite(out["depths"]).all()


def test_refusals_keep_their_messages(pkg, port):
    G, cfg = _tiny_generator(pkg, port)
    B = 1
    z = torch.randn(B, cfg["latent_dim"]).cuda()
    cond = {k: v.cuda() for k, v in pkg.synthetic.make_conditions(B, seed=3).items()}
    G.train()
    with pytest.raises(RuntimeError, match="lock_view_dependence=False"):
        with torch.no_grad():
            G(z, cond, **dict(cfg, lock_view_dependence=False))
    with pytest.raises(RuntimeError, match="last_back=True is an inference-only setting"):
        G(z, cond, **dict(cfg, last_back=True))
    with pytest.raises(RuntimeError, match="power of two"):
        with torch.no_grad():
            G(z, cond, **dict(cfg, num_steps=24))


def test_trainer_iteration(pkg, port):
    disc = _mod("modules.discriminator")
    ts = _mod("train_step")
    G, cfg = _tiny_generator(pkg, port)
    G.train()
    D = disc.UNetDiscriminator(**cfg).cuda().train()
    t = ts.Trainer(G, D, cfg, amp=False, ddp=False)
    B = 2
    batch = dict(cond={k: v.cuda() for k, v in pkg.synthetic.make_conditions(B, seed=1).items()},
                 images=torch.randn(B, 3, 64, 64, device="cuda").clamp_(-1, 1),
                 labels=torch.randint(1, cfg["label_dim"], (B, 64, 64), device="cuda"))
    p0 = [p.detach().clone() for p in G.parameters() if p.requires_grad]
    d, g_ = t.iteration(batch)
    assert torch.isfinite(d) and torch.isfinite(g_)
    ps = [p for p in G.parameters() if p.requires_grad]
    assert all(torch.isfinite(p).all() for p in ps)
    assert sum(int(not torch.equal(a, b.detach())) for a, b in zip(p0, ps)) > 100
