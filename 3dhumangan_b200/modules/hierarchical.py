"""hierarchical_sample=True: the NeRF / pi-GAN coarse-to-fine importance sampling of `Map3DGenerator.render`
(lib/generators/map3d_generator.py:450-511, lib/generators/volume_rendering.py:261-303).

Gradients never flow through the fine depths or the sampling weights (the reference computes them under no_grad and
detaches them), so a hierarchical render IS an ordinary render over 2S samples per ray whose point records come from the
depth-sorted merge of the S coarse and S fine samples.  `merged_records` builds those records:

    hg_geo_features    coarse rays, jitter, camera transform, nearest vertex, features   (as the one-pass render)
    pass 1             coarse sigma only: hg_render_mlp's per-point mode at 256, the layered trunk up to the sigma
                       head at the zero-padded widths; no tape
    hg_sample_fine     coarse weights, pdf, cdf, inverse cdf, fine points
    hg_geo_features    nearest vertex and features of the fine points (points_in mode)
    hg_merge_samples   stable depth sort of cat([fine, coarse]) + gather of records and depths

and every existing renderer (fused inference, layered training, zero-padded widths) then runs unchanged at
num_steps = 2S on them with the final noise draw.  The coarse points are evaluated twice (pass 1 and inside the 2S pass);
reusing the pass-1 outputs would need a scatter compositing forward and backward.
"""
from __future__ import annotations

import torch

from .. import abi


def check_steps(cfg):
    """The merged render runs the compositing kernels at 2S samples per ray: a power of two <= 128."""
    S = cfg["num_steps"]
    if not cfg.get("lock_view_dependence", False):
        raise RuntimeError("hg3d: lock_view_dependence=False is not used by any shipped curriculum and is not built")
    if S < 4 or S > 64 or S & (S - 1):
        raise RuntimeError(f"hg3d: hierarchical_sample=True renders 2 * num_steps samples per ray, which must be a power of "
                           f"two <= 128 (num_steps = {S})")
    return S


def ray_tables(cfg, dev):
    Rw, Rh, S = cfg["render_width"], cfg["render_height"], cfg["num_steps"]
    f32 = dict(dtype=torch.float32, device=dev)
    return (torch.linspace(-Rw / Rh, Rw / Rh, Rw, **f32), torch.linspace(-1, 1, Rh, **f32),
            torch.linspace(cfg["ray_start"], cfg["ray_end"], S, **f32))


def coarse_sigma(P, freq, phase, rec, cfg, passes, wblob=None):
    """Pass 1: raw sigma of every coarse point -> (tensor, element stride of consecutive points)."""
    B = freq.shape[0]
    S = cfg["num_steps"]
    if cfg["hidden_dim"] == 256:
        from . import render_ops
        g = lambda n: P["neural_field." + n].detach()
        if wblob is None:
            wblob = render_ops.pack_render_weights(P, geo_dim=cfg["geo_feature_dim"])
        heads_b = torch.cat([g("sigma_layer.bias").reshape(1), g("color_layer_linear.bias").reshape(3)]).float().contiguous()
        raw, _ = abi.render_mlp(rec, None, render_ops.film_table(P, freq.detach(), phase.detach()), wblob,
                                g("sigma_layer.weight").reshape(-1).float().contiguous(), g("color_layer_linear.weight").float().contiguous(),
                                g("feature_layer_linear.bias").float().contiguous(), heads_b, B=B, R=rec.shape[1] // S, S=S,
                                passes=passes, raw=True)
        return raw[..., 259], 260                 # per point (rgb 3, feat 256, sigma)
    from . import wide_ops
    return wide_ops.render_forward_wide(P, freq.detach(), phase.detach(), None, cfg, None, None, passes=passes,
                                        records=(rec, None), sigma_only=True), 1


@torch.no_grad()
def merged_records(P, freq, phase, cond, cfg, u, noise, *, passes=3, wblob=None, want_nearest=False, want_fine=False):
    """Records of the merged 2S-sample render.  `noise` is the rng.HierarchicalNoise of this render.
    Returns dict(rec [B,R*2S,36], z_vals [B,R*2S], cfg (num_steps = 2S), noise [B,R*2S] final draws,
    nearest [B,R*2S] when want_nearest, fine_z [B,R*S] / perm [B,R*2S] when want_fine)."""
    abi.require_device()
    S = check_steps(cfg)
    dev = freq.device
    B = freq.shape[0]
    Rw, Rh = cfg["render_width"], cfg["render_height"]
    R = Rw * Rh
    xs, ys, zs = ray_tables(cfg, dev)
    vik = abi.vertex_ik(cond["fk_matrices"], cond["lbs_weights"])
    geo_kw = dict(input_scaler=2.0 / cfg["side_length"], legacy_mode=cfg.get("legacy_mode", False), want_nearest=want_nearest)
    geo_c = abi.geo_features(cond["vertices"], cond["tpose_vertices"], cond["skeletons_xyz"], vik, xs=xs, ys=ys, zs=zs,
                             focals=cond["intrinsics"][:, 0, 0], scales=cond["scales"], cam2world=cond["cam2world_matrices"],
                             jitter=u.reshape(B, R * S) if u is not None else None, **geo_kw)
    sigma, stride = coarse_sigma(P, freq, phase, geo_c["rec"], cfg, passes, wblob=wblob)
    fine_z, pts = abi.sample_fine(sigma, stride, geo_c["z_vals"], noise.coarse.reshape(B, R * S), noise.u_pdf,
                                  noise_std=cfg["nerf_noise"], clamp_mode=cfg["clamp_mode"], xs=xs, ys=ys,
                                  focals=cond["intrinsics"][:, 0, 0], cam2world=cond["cam2world_matrices"], B=B, Rw=Rw, Rh=Rh, S=S)
    geo_f = abi.geo_features(cond["vertices"], cond["tpose_vertices"], cond["skeletons_xyz"], vik, points_in=pts, **geo_kw)
    rec, z_vals, perm = abi.merge_samples(geo_f["rec"], fine_z, geo_c["rec"], geo_c["z_vals"], B=B, R=R, S=S,
                                          want_perm=want_nearest or want_fine)
    out = {"rec": rec, "z_vals": z_vals, "cfg": dict(cfg, num_steps=2 * S),
           "noise": noise.final.reshape(B, R * 2 * S).float().contiguous(), "nearest": None}
    if want_nearest:
        both = torch.cat([geo_f["nearest"].reshape(B, R, S), geo_c["nearest"].reshape(B, R, S)], -1)
        out["nearest"] = torch.gather(both, 2, perm.reshape(B, R, 2 * S).long()).reshape(B, R * 2 * S)
    if want_fine:
        out.update(fine_z=fine_z, perm=perm)
    return out
