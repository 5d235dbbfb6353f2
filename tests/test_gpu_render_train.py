"""Training-mode renderer (layer-by-layer FiLM-SIREN over tile-blocked points + compositing) and its backward against
the restated reference (oracle.port.siren + ray_integration) in fp64 with autograd, at hidden_dim 256 (render_train's
forward) and at the zero-padded widths 384 / 420 (wide_ops' forward); one backward serves all three."""
import importlib

import pytest
import torch

pytestmark = pytest.mark.gpu


def _setup(port, C, B=2, R=8, S=32, seed=11, noise_std=0.0):
    pkg = importlib.import_module("3dhumangan_b200")
    cfg = pkg.configs.baseline_config("tiny")
    cfg.update(hidden_dim=C, feature_dim=C, num_steps=S, nerf_noise=noise_std, white_back=True, last_back=False, clamp_mode="relu")
    params = port.init_generator_params(cfg, seed=seed, sigma_gain=60.0, sigma_bias=2.0)
    names = [n for n in params if n.startswith("neural_field.")]
    g = torch.Generator().manual_seed(seed + 1)
    N = R * S
    pts = torch.rand(B, N, 3, generator=g) * 2 - 1
    geo = torch.rand(B, N, 31, generator=g)
    z = (torch.rand(B, R, S, generator=g) * 0.02 + 0.03).cumsum(-1) + 8.0
    freq = torch.randn(B, 4 * C, generator=g)
    phase = torch.randn(B, 4 * C, generator=g)
    noise = torch.randn(B, R, S, 1, generator=g)
    wgt = torch.randn(B, R, 3 + C, generator=g)
    return cfg, params, names, pts, geo, z, freq, phase, noise, wgt


def _oracle(port, monkeypatch, cfg, params, names, pts, geo, z, freq, phase, noise, wgt, mask):
    import torch.nn.functional as TF
    B, R, S = z.shape
    pc = {n: params[n].clone().double().requires_grad_(True) for n in names}
    fq, ph = freq.clone().double().requires_grad_(True), phase.clone().double().requires_grad_(True)
    dirs = torch.zeros(B, R * S, 3, dtype=torch.float64)
    dirs[..., -1] = -1
    raw = port.siren(pc, pts.double(), fq, ph, geo.double(), dirs, 1.0, cfg["hidden_dim"], 4)
    with monkeypatch.context() as mp:
        if mask is not None:      # same ReLU mask on sigma as our pass (the gradient is discontinuous in it)
            mp.setattr(port.F, "relu", lambda v: v * mask)
        rgbf, depth, w = port.ray_integration(raw.reshape(B, R, S, -1), z.double()[..., None], noise.double(), cfg["nerf_noise"],
                                              True, False, "relu")
    return rgbf, depth, pc, fq, ph, raw


@pytest.mark.parametrize("C", [256, 384, 420])
@pytest.mark.parametrize("noise_std", [0.0, 0.5])
def test_render_train_forward_and_backward(port, monkeypatch, noise_std, C):
    rt = importlib.import_module("3dhumangan_b200.modules.render_train")
    wo = importlib.import_module("3dhumangan_b200.modules.wide_ops")
    cfg, params, names, pts, geo, z, freq, phase, noise, wgt = _setup(port, C, noise_std=noise_std)
    B, R, S = z.shape
    N = R * S
    pg = {n: params[n].clone().cuda().requires_grad_(True) for n in names}
    rec = torch.cat([pts, geo], -1).cuda()
    z_vals = z.reshape(B, N).cuda().contiguous()
    nz = noise.cuda() if noise_std > 0 else None
    if C == 256:        # the fused-width training forward
        ray_out, tape = rt.mlp_forward_train(pg, freq.cuda(), phase.cuda(), rec, z_vals, nz, cfg)
        feats, rgb01, depth_k = ray_out[..., :256], ray_out[..., 256:259], ray_out[..., 259:260]
    else:               # the zero-padded forward with a tape
        monkeypatch.setattr(rt, "geo_records", lambda *a, **k: (rec, z_vals))
        tape = {}
        feats, rgb01, depth_k = wo.render_forward_wide(pg, freq.cuda(), phase.cuda(), None, cfg, None, nz, tape=tape)
    dfq, dph = rt.mlp_backward(tape, wgt[..., 3:].cuda(), wgt[..., :3].cuda())
    torch.cuda.synchronize()

    # ---- forward against the plain fp64 oracle
    with torch.no_grad():
        rgbf, depth, *_ = _oracle(port, monkeypatch, cfg, params, names, pts, geo, z, freq, phase, noise, wgt, None)
    assert (feats.cpu().double() - rgbf[..., 3:]).abs().max() / rgbf[..., 3:].abs().max() < 1e-3
    assert (rgb01.cpu().double() - rgbf[..., :3]).abs().max() < 1e-3
    assert (depth_k.cpu().double()[..., 0] - depth[..., 0]).abs().max() / depth.abs().max() < 1e-4

    # ---- gradients against the fp64 oracle with our sigma mask
    pre = tape["sig"].cpu().double().reshape(B, R, S, 1) + (noise.double() * noise_std if noise_std > 0 else 0.0)
    mask = (pre > 0).double()
    rgbf, depth, pc, fq, ph, raw = _oracle(port, monkeypatch, cfg, params, names, pts, geo, z, freq, phase, noise, wgt, mask)
    (rgbf * wgt.double()).sum().backward()
    frac_pos = mask.mean().item()
    assert 0.05 < frac_pos < 0.95, frac_pos          # the test must exercise both sides of the clamp

    def rel(a, b):
        return ((a - b).norm() / b.norm()).item()

    bad = {}
    for n in names:
        assert pg[n].grad is not None and pg[n].grad.shape == pg[n].shape, n
        e = rel(pg[n].grad.cpu().double(), pc[n].grad)
        if e > 1e-3:
            bad[n] = e
    assert not bad, sorted(bad.items(), key=lambda t: -t[1])
    assert rel(dfq.cpu().double(), fq.grad) < 1e-3
    assert rel(dph.cpu().double(), ph.grad) < 1e-3
