"""Parity at the BENCHMARKED sizes (BASELINE.json configs C2 / C3 / C5), not only on the tiny fixtures.

At C2 every persistent CTA of the synthesis kernels walks ~28 tiles per image and the render kernel ~16 per image (ring-phase
wraps, accumulator drains, many tiles per CTA) -- code paths the 32x32 fixtures never reach.  The checker is the
oracle (`oracle/port.py`, pinned to the unmodified reference by tests/test_oracle_pin.py) executed ON THE GPU in plain
fp32 torch with TF32 disabled; B = 2 keeps it to a few seconds.  Tolerance: 1e-3 relative L2 (the north_star's
"within 1e-3 relative fp32"); nearest-vertex indices bit-exact.
"""
import importlib

import pytest
import torch

from golden_util import rel_l2

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _exact_fp32_checker():
    """The oracle's convolutions / matmuls must be true fp32 on the device (cuDNN defaults to TF32)."""
    old = (torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32)
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old


def _to(d, dev):
    return {k: (v.to(dev) if isinstance(v, torch.Tensor) else v) for k, v in d.items()}


def _generator(cfg, params):
    gen = importlib.import_module("3dhumangan_b200.modules.generator")
    G = gen.Map3DGenerator(**cfg).cuda()
    G.load_state_dict(params, strict=True)
    G.set_device(torch.device("cuda", 0))
    G.train()
    return G


def _case(pkg, port, name, B, seed, **over):
    cfg = pkg.configs.baseline_config(name)
    cfg.update(over)
    params = port.init_generator_params(cfg, seed=seed, sigma_gain=200.0, sigma_bias=1.0)     # densities that actually occlude
    cond = pkg.synthetic.make_conditions(B, seed=seed + 1)
    z = torch.randn(B, cfg["latent_dim"], generator=torch.Generator().manual_seed(seed + 2))
    g = torch.Generator(device="cuda").manual_seed(seed + 3)
    R, S = cfg["render_height"] * cfg["render_width"], cfg["num_steps"]
    u = torch.rand(B, R, S, 1, device="cuda", generator=g)
    noise = torch.randn(B, R, S, 1, device="cuda", generator=g)
    return cfg, params, cond, z, u, noise


@pytest.mark.parametrize("mode,graph", [("mixed", False), ("mixed", True), ("isolated", False)])
def test_generator_forward_at_c2_size(pkg, port, monkeypatch, mode, graph):
    """Map3DGenerator.forward at gen 512x512 / render 96x96x32 / hidden 256 (config C2), B = 2: 8 192 synthesis tiles and
    4 608 render tiles over 148 persistent CTAs.  Final pixels, rendered pixels, feature maps, every block's activation,
    BatchNorm running statistics and the spectral-norm vector against the oracle."""
    B = 2
    cfg, params, cond, z, u, noise = _case(pkg, port, "C2", B, 40, nerf_noise=0.5, map3d_mode=mode,
                                           legacy_mode=(mode == "isolated"))
    rng = importlib.import_module("3dhumangan_b200.rng")
    monkeypatch.setattr(rng, "draw_render_noise", lambda *a, **k: (u, noise))
    G = _generator(cfg, params)
    cg, zg = _to(cond, "cuda"), z.cuda()
    with torch.no_grad():
        # graph=True: the returned pixels come from the REPLAY of the captured forward (the warm-up run's effects on the
        # buffers are rolled back before the capture), i.e. exactly one forward from the initial state, like the oracle's
        out = G(zg, cg, **dict(cfg, hg_cuda_graph=graph))
    torch.cuda.synchronize()
    pg = _to(params, "cuda")
    stats = {}
    with torch.no_grad():
        ref = port.generator_forward(pg, zg, cg, cfg, u, noise, training=True, stats_out=stats)
    assert torch.isfinite(out["rgbs"]).all()
    assert rel_l2(out["rgbs_render"], ref["rgbs_render"]) < 1e-3
    assert rel_l2(out["rgbs"], ref["rgbs"]) < 1e-3, rel_l2(out["rgbs"], ref["rgbs"])
    assert float((out["rgbs"] - ref["rgbs"]).abs().max() / ref["rgbs"].abs().max()) < 5e-3
    if not graph:
        sd = G.state_dict()
        for k in (0, 4, 8):
            blk = f"synthesis_network.network.m3d_{k}."
            assert rel_l2(sd[blk + "spade_1.first_norm.running_var"], stats[blk + "spade_1.first_norm.running_var"]) < 1e-3
            assert rel_l2(sd[blk + "conv_1.weight_u"], stats[blk + "conv_1.weight_u"]) < 1e-4


def test_render_and_synthesis_blocks_at_c2_size(pkg, port):
    """The two halves separately at C2 size: ray records [B,R,260] (features, rgb, depth), bit-exact nearest-vertex indices
    on the kernel's own sample points, and the activation after EVERY SPADE block."""
    render_ops = importlib.import_module("3dhumangan_b200.modules.render_ops")
    synthesis_ops = importlib.import_module("3dhumangan_b200.modules.synthesis_ops")
    B = 2
    cfg, params, cond, z, u, noise = _case(pkg, port, "C2", B, 50, nerf_noise=0.5)
    pg, cg, zg = _to(params, "cuda"), _to(cond, "cuda"), z.cuda()
    Rh, Rw, S = cfg["render_height"], cfg["render_width"], cfg["num_steps"]
    with torch.no_grad():
        freq, phase = port.mapping_network(pg, torch.zeros_like(zg))          # neural_field_latent_input=False
        styles = port.synthesis_mapping(pg, zg)
        r = render_ops.render_forward(pg, freq, phase, cg, cfg, u, noise, want_weights=True, want_nearest=True)
        rgb_r, fmap, depth, w, idx = port.render(pg, freq, phase, cg, cfg, u, noise)
    torch.cuda.synchronize()
    ray = r["ray_out"]
    feat = ray[..., :256].reshape(B, Rh, Rw, 256).permute(0, 3, 1, 2)
    assert rel_l2(feat, fmap) < 1e-3, rel_l2(feat, fmap)
    assert rel_l2(ray[..., 256:259].reshape(B, Rh, Rw, 3).permute(0, 3, 1, 2) * 2 - 1, rgb_r) < 1e-3
    assert rel_l2(ray[..., 259:260], depth) < 1e-4
    assert rel_l2(r["weights"].reshape(B, Rh * Rw, S), w.reshape(B, Rh * Rw, S)) < 1e-3
    # nearest vertex: kernel vs the oracle's search.  Both sides compute the sample points themselves (the kernel with
    # fused multiply-adds), so a point within an ulp of a bisector plane may legitimately differ; everything else is equal.
    near = r["nearest"].reshape(B, -1).long()
    differ = int((near != idx).sum())
    assert differ <= 1e-5 * idx.numel(), (differ, idx.numel())
    # (bit-exactness on identical points: test_nearest_vertex_bit_exact_at_c2_size below)
    with torch.no_grad():
        ref_rgb, ref_int = port.synthesis_network(pg, port.synthesis_input(pg, B, cfg["gen_height"], cfg["gen_width"]),
                                                  torch.nn.functional.interpolate(fmap, (cfg["gen_height"], cfg["gen_width"]),
                                                                                  mode="bilinear"),
                                                  styles, cfg, training=True, return_internal=True)
        P2 = {k: v.clone() for k, v in pg.items()}
        got_rgb, got_int = synthesis_ops.synthesis_forward(P2, ray, styles.reshape(B, -1), cfg, training=True, return_internal=True)
    torch.cuda.synchronize()
    for k in range(cfg["synthesis_blocks"]):
        e = rel_l2(got_int[f"m3d_{k}"], ref_int[f"m3d_{k}"])
        assert e < 1e-3, (k, e)
    assert rel_l2(got_rgb, ref_rgb) < 1e-3


def test_nearest_vertex_bit_exact_at_c2_size(pkg, port):
    """K=1 nearest posed vertex for all 2 x 294 912 sample points of a C2 batch (rays + jitter + camera transform inside the
    kernel): indices and squared distances bit-exact against the oracle's search over the SAME points."""
    abi = importlib.import_module("3dhumangan_b200.abi")
    B = 2
    cfg, params, cond, z, u, noise = _case(pkg, port, "C2", B, 60)
    cg = _to(cond, "cuda")
    Rw, Rh, S = cfg["render_width"], cfg["render_height"], cfg["num_steps"]
    f32 = dict(dtype=torch.float32, device="cuda")
    geo = abi.geo_features(cg["vertices"], cg["tpose_vertices"], cg["skeletons_xyz"], abi.vertex_ik(cg["fk_matrices"], cg["lbs_weights"]),
                           input_scaler=2.0 / cfg["side_length"], legacy_mode=False, xs=torch.linspace(-Rw / Rh, Rw / Rh, Rw, **f32),
                           ys=torch.linspace(-1, 1, Rh, **f32), zs=torch.linspace(cfg["ray_start"], cfg["ray_end"], S, **f32),
                           focals=cg["intrinsics"][:, 0, 0], scales=cg["scales"], cam2world=cg["cam2world_matrices"],
                           jitter=u.reshape(B, -1), want_points=True, want_nearest=True)
    torch.cuda.synchronize()
    d2, idx = port.knn1(geo["points"], cg["vertices"])
    assert torch.equal(geo["nearest"].reshape(B, -1).long(), idx), int((geo["nearest"].reshape(B, -1).long() != idx).sum())
    assert torch.equal(geo["nearest_d2"].reshape(B, -1), d2)


def test_render_at_c5_size(pkg, port):
    """Config C5's renderer shape: 192x192 rays x 128 samples (a tile of 128 points is ONE ray; 36 864 tiles for one image)."""
    render_ops = importlib.import_module("3dhumangan_b200.modules.render_ops")
    B = 1
    cfg, params, cond, z, u, noise = _case(pkg, port, "C5", B, 70, nerf_noise=0.5)
    pg, cg, zg = _to(params, "cuda"), _to(cond, "cuda"), z.cuda()
    Rh, Rw, S = cfg["render_height"], cfg["render_width"], cfg["num_steps"]
    with torch.no_grad():
        freq, phase = port.mapping_network(pg, zg)
        r = render_ops.render_forward(pg, freq, phase, cg, cfg, u, noise)
        rgb_r, fmap, depth, w, idx = port.render(pg, freq, phase, cg, cfg, u, noise)
    torch.cuda.synchronize()
    ray = r["ray_out"]
    feat = ray[..., :256].reshape(B, Rh, Rw, 256).permute(0, 3, 1, 2)
    assert rel_l2(feat, fmap) < 1e-3, rel_l2(feat, fmap)
    assert rel_l2(ray[..., 256:259].reshape(B, Rh, Rw, 3).permute(0, 3, 1, 2) * 2 - 1, rgb_r) < 1e-3
    assert rel_l2(ray[..., 259:260], depth) < 1e-4


@pytest.mark.parametrize("path", ["inference", "training"])
def test_discriminator_at_512(pkg, port, path):
    """UNetDiscriminator.forward at 512x512, B = 2 (the shape of a C3 discriminator pass), both implementations:
    the fused inference kernels and the autograd graph of the training path."""
    disc = importlib.import_module("3dhumangan_b200.modules.discriminator")
    cfg = pkg.configs.baseline_config("C2")
    params = port.init_discriminator_params(cfg, seed=81)
    B = 2
    img = torch.randn(B, 3, 512, 512, generator=torch.Generator().manual_seed(82)).clamp(-1, 1).cuda()
    pg = _to(params, "cuda")
    with torch.no_grad():
        ref = port.discriminator_forward(pg, img, cfg, training=True)
    D = disc.UNetDiscriminator(**cfg).cuda()
    D.load_state_dict(params, strict=True)
    D.train()
    if path == "inference":
        with torch.no_grad():
            out = D(img, None, alpha=1.0, **cfg)
    else:
        out = D(img.requires_grad_(True), None, alpha=1.0, **cfg)
        assert out["segments"].requires_grad
    torch.cuda.synchronize()
    for k in ("prediction", "latents", "segments"):
        e = rel_l2(out[k].detach(), ref[k])
        assert e < 1e-3, (k, e)


@pytest.mark.parametrize("name,over", [("C1", {}), ("C2native", dict(hidden_dim=420, latent_dim=420, feature_dim=420, map3d_mode="isolated",
                                                                  legacy_mode=True))])
def test_other_widths_at_config_size(pkg, port, monkeypatch, name, over):
    """BASELINE config C1 (MAP3DBN: hidden 384, gen 256x256, render 64x64) and the released checkpoint's shape (MAP3DBN512L:
    hidden 420, 512x256, render 96x48, isolated + legacy) through the module call, on the zero-padded blocked-GEMM path
    (modules/wide_ops.py), against the oracle on the device."""
    B = 1
    cfg, params, cond, z, u, noise = _case(pkg, port, name, B, 90, nerf_noise=0.5, **over)
    rng = importlib.import_module("3dhumangan_b200.rng")
    monkeypatch.setattr(rng, "draw_render_noise", lambda *a, **k: (u, noise))
    G = _generator(cfg, params)
    cg, zg = _to(cond, "cuda"), z.cuda()
    with torch.no_grad():
        out = G(zg, cg, **cfg)
    torch.cuda.synchronize()
    pg = _to(params, "cuda")
    stats = {}
    with torch.no_grad():
        ref = port.generator_forward(pg, zg, cg, cfg, u, noise, training=True, stats_out=stats)
    assert out["rgbs"].shape == ref["rgbs"].shape
    assert rel_l2(out["rgbs_render"], ref["rgbs_render"]) < 1e-3, rel_l2(out["rgbs_render"], ref["rgbs_render"])
    assert rel_l2(out["rgbs"], ref["rgbs"]) < 1e-3, rel_l2(out["rgbs"], ref["rgbs"])
    blk = "synthesis_network.network.m3d_8."
    assert rel_l2(G.state_dict()[blk + "spade_1.first_norm.running_var"], stats[blk + "spade_1.first_norm.running_var"]) < 1e-3
    # the sample app's entry point on this width: truncated, eval-mode statistics after a few train-mode forwards
    with torch.no_grad():
        for _ in range(2):
            G(zg, cg, **cfg)
        G.eval()
        o2 = G.staged_forward(zg, cg, truncation_psi=0.7, **dict(cfg, nerf_noise=0, last_back=True))
    assert o2["rgbs"].shape == ref["rgbs"].shape and torch.isfinite(o2["rgbs"]).all()
    assert o2["depths"].shape == (B, 1, cfg["render_height"], cfg["render_width"])
