"""CPU oracle of `Map3DGenerator.render(..., hierarchical_sample=True)`: the coarse-to-fine importance sampling on top of
the one-pass oracle in `oracle/port.py`.  TEST INFRASTRUCTURE ONLY.

Random draws are inputs (`rng.HierarchicalNoise`), as in `port.render`.  `fine_z` (tests only) replaces the sampled fine
depths, so that the device's own samples can be evaluated here: nearest-vertex decisions are then made on identical
depths, and the fine depths carry no gradient in the reference either.
"""
from __future__ import annotations

import torch

from oracle import port


def sample_pdf(bins, weights, u, eps=1e-5):
    """lib/generators/volume_rendering.py:261-303 with det=False; `u` [N_rays, N_importance] is the torch.rand draw."""
    n_rays, n_samples = weights.shape
    weights = weights + eps
    pdf = weights / torch.sum(weights, -1, keepdim=True)
    cdf = torch.cumsum(pdf, -1)
    cdf = torch.cat([torch.zeros_like(cdf[:, :1]), cdf], -1)
    u = u.contiguous()
    inds = torch.searchsorted(cdf, u)
    below = torch.clamp_min(inds - 1, 0)
    above = torch.clamp_max(inds, n_samples)
    n_imp = u.shape[1]
    inds_sampled = torch.stack([below, above], -1).view(n_rays, 2 * n_imp)
    cdf_g = torch.gather(cdf, 1, inds_sampled).view(n_rays, n_imp, 2)
    bins_g = torch.gather(bins, 1, inds_sampled).view(n_rays, n_imp, 2)
    denom = cdf_g[..., 1] - cdf_g[..., 0]
    denom[denom < eps] = 1
    return bins_g[..., 0] + (u - cdf_g[..., 0]) / denom * (bins_g[..., 1] - bins_g[..., 0])


def render(params, freq, phase, cond, cfg, u, noise, fine_z=None, dtype=None):
    """lib/generators/map3d_generator.py:381-523 with hierarchical_sample=True, coarse_steps = fine_steps = num_steps,
    lock_view_dependence=True, staged=False.  `noise` is an rng.HierarchicalNoise.
    Returns rgb_render, feature_maps, depth, weights [B,R,2S,1], nearest idx of the merged samples [B,R*2S], fine_z [B*R,S].
    `dtype`: as in `port.render` (the MLP and integrations in that dtype; rays, sampling and geometry features in fp32)."""
    Rw, Rh, S = cfg["render_width"], cfg["render_height"], cfg["num_steps"]
    Fd, H = cfg["feature_dim"], cfg["hidden_dim"]
    if not cfg.get("lock_view_dependence", False):
        raise ValueError("the oracle restates the locked view direction only")
    focals = cond["intrinsics"][:, 0, 0]
    scales = cond["scales"].float()
    c2w = cond["cam2world_matrices"]
    B = freq.shape[0]
    R = Rw * Rh
    cast = (lambda t: t) if dtype is None else (lambda t: t.to(dtype))
    pts, z, d = port.initial_rays(focals, scales, S, Rw, Rh, cfg["ray_start"], cfg["ray_end"])
    pw, z = port.jitter_and_transform(pts, z, d, c2w, u)
    geo_args = (cond["skeletons_xyz"], cond["vertices"], cond["tpose_vertices"], cond["fk_matrices"], cond["lbs_weights"],
                cfg.get("legacy_mode", False))

    def field(points):
        geo, idx = port.geo_features(points, *geo_args)
        dirs = torch.zeros_like(points)
        dirs[..., -1] = -1
        out = port.siren(params, cast(points), cast(freq), cast(phase), cast(geo), cast(dirs), 2.0 / cfg["side_length"], H,
                         cfg["neural_field_blocks"])
        return out.reshape(B, R, S, Fd + 4), idx.reshape(B, R, S)

    coarse, idx_c = field(pw.reshape(B, R * S, 3))
    with torch.no_grad():                                                                     # :450-472
        _, _, w = port.ray_integration(coarse, cast(z), cast(noise.coarse), cfg["nerf_noise"], False, False, cfg["clamp_mode"])
        w = w.reshape(B * R, S).float() + 1e-5
        zf = z.reshape(B * R, S)
        mid = 0.5 * (zf[:, :-1] + zf[:, 1:])
        fz = sample_pdf(mid, w[:, 1:-1], noise.u_pdf) if fine_z is None else fine_z.reshape(B * R, S).float()
        fz = fz.detach()
        dw = torch.bmm(c2w[:, :3, :3], d.permute(0, 2, 1)).permute(0, 2, 1)                  # volume_rendering.py:159-161
        hom = torch.zeros(B, 4, R, dtype=c2w.dtype)
        hom[:, 3] = 1
        org = torch.bmm(c2w, hom).permute(0, 2, 1)[..., :3]                                   # :163-167
        fine_pts = (org.unsqueeze(2) + dw.unsqueeze(2) * fz.reshape(B, R, S, 1)).reshape(B, R * S, 3)
    fine, idx_f = field(fine_pts)
    all_out = torch.cat([fine, coarse], -2)                                                   # :500-505
    all_z = torch.cat([fz.reshape(B, R, S, 1), z], -2)
    _, order = torch.sort(all_z, dim=-2, stable=True)
    all_z = torch.gather(all_z, -2, order)
    all_out = torch.gather(all_out, -2, order.expand(-1, -1, -1, Fd + 4))
    idx = torch.gather(torch.cat([idx_f, idx_c], -1), -1, order[..., 0]).reshape(B, R * 2 * S)
    rgbf, depth, w = port.ray_integration(all_out, cast(all_z), cast(noise.final), cfg["nerf_noise"], cfg.get("white_back", False),
                                          cfg.get("last_back", False), cfg["clamp_mode"])
    img = rgbf.reshape(B, Rh, Rw, Fd + 3).permute(0, 3, 1, 2)
    return img[:, :3] * 2 - 1, img[:, 3:], depth, w, idx, fz
