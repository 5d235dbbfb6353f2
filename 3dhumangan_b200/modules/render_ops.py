"""Host-side schedule of the pose-mapping renderer on top of the C ABI (csrc/geo.cu, csrc/render.cu).

Mirrors `Map3DGenerator.render` (lib/generators/map3d_generator.py:381-523) with lock_view_dependence=True.  Three
launches per one-pass call (hierarchical_sample=True first builds 2S merged samples per ray, modules/hierarchical.py):
`hg_vertex_ik` (inverse-LBS matrices per posed vertex), `hg_geo_features` (rays, jitter, camera
transform, exact K=1 nearest vertex, 31-d feature) and `hg_render_mlp` (FiLM-SIREN + compositing).
"""
from __future__ import annotations

import torch

from .. import abi


def pack_render_weights(P, prefix="neural_field.", geo_dim=31):
    """Concatenate the packed bf16 hi/lo operand images of the MLP in the kernel's schedule order
    (render.cu): W01 = [coord | geo] block matrix, network.0 (K=512: the geometry half first), network.1-3, color[:, 3:],
    feature."""
    g = lambda n: P[prefix + n]
    dev = g("network.0.layer.weight").device
    H = g("network.0.layer.weight").shape[0]
    if H != 256 or geo_dim + 3 > 36:
        raise RuntimeError("hg3d: the fused render kernel is built for hidden_dim == 256, geo_feature_dim <= 33")
    W01 = torch.zeros(2 * H, 3 + geo_dim, dtype=torch.float32, device=dev)
    W01[:H, :3] = g("first_layer_coord.layer.weight")
    W01[H:, 3:] = g("first_layer_mod.layer.weight")
    mats = [W01, g("network.0.layer.weight"), g("network.1.layer.weight"), g("network.2.layer.weight"),
            g("network.3.layer.weight"), g("color_layer_sine.layer.weight")[:, 3:], g("feature_layer_linear.weight")]
    imgs = [abi.pack_weight(m.float().contiguous() if m.stride(1) == 1 else m.float().contiguous(), Nb=256)[0] for m in mats]
    # network.0 runs its geometry half (K chunks 4-7) first: the kernel computes g before a (render.cu, layer schedule)
    half = imgs[1].numel() // 2
    imgs[1] = torch.cat([imgs[1][half:], imgs[1][:half]])
    blob = torch.cat(imgs)
    assert blob.numel() == abi.lib().hg_render_weight_blob_bytes(), blob.numel()
    return blob


def film_table(P, freq, phase, locked_dir=(0.0, 0.0, -1.0), prefix="neural_field."):
    """[B,7,2,256] (F, P) per layer so that the layer output is sin(F*acc + P) with acc = W x (no bias):
    sine layers: sin(30*(acc+b)); FiLM layers: sin(f*(acc+b)+phi), f = 15*freq+30 (modulated.py:43);
    the colour layer re-uses the LAST slice (modulated.py:68) and absorbs W[:, :3] . dir (view direction)."""
    g = lambda n: P[prefix + n]
    B = freq.shape[0]
    H = 256
    f = freq.float() * 15 + 30
    ph = phase.float()
    rows = []
    one = torch.full((B, H), 30.0, device=freq.device)
    rows.append((one, 30.0 * g("first_layer_coord.layer.bias")[None].expand(B, H)))
    rows.append((one, 30.0 * g("first_layer_mod.layer.bias")[None].expand(B, H)))
    for i in range(4):
        fi, pi = f[:, i * H:(i + 1) * H], ph[:, i * H:(i + 1) * H]
        rows.append((fi, fi * g(f"network.{i}.layer.bias")[None] + pi))
    fi, pi = f[:, -H:], ph[:, -H:]
    wd = g("color_layer_sine.layer.weight")[:, :3]
    # python-float arithmetic only: no host->device tensor creation, so the forward stays CUDA-graph capturable
    dterm = wd[:, 0] * float(locked_dir[0]) + wd[:, 1] * float(locked_dir[1]) + wd[:, 2] * float(locked_dir[2])
    rows.append((fi, fi * (g("color_layer_sine.layer.bias") + dterm)[None] + pi))
    return torch.stack([torch.stack([F_, P_], 1) for F_, P_ in rows], 1).contiguous()


@torch.no_grad()
def render_forward(P, freq, phase, cond, cfg, u, noise, *, passes=3, wblob=None, want_weights=False, want_nearest=False):
    """u [B,R,S,1] jitter draws, noise [B,R,S,1] sigma-noise draws (rng.draw_render_noise); with hierarchical_sample
    `noise` is the rng.HierarchicalNoise of the render and the integration runs over the 2S merged samples
    (modules/hierarchical.py).  Returns dict(ray_out [B,R,260], z_vals, weights, nearest)."""
    abi.require_device()
    if not cfg.get("lock_view_dependence", False):
        raise RuntimeError("hg3d: lock_view_dependence=False is not used by any shipped curriculum and is not built")
    dev = freq.device
    B = freq.shape[0]
    Rw, Rh, S = cfg["render_width"], cfg["render_height"], cfg["num_steps"]
    R = Rw * Rh
    if wblob is None:
        wblob = pack_render_weights(P, geo_dim=cfg["geo_feature_dim"])
    if cfg.get("hierarchical_sample", False):
        from . import hierarchical
        geo = hierarchical.merged_records(P, freq, phase, cond, cfg, u, noise, passes=passes, wblob=wblob,
                                          want_nearest=want_nearest)
        S, noise = 2 * S, geo["noise"]
    else:
        f32 = dict(dtype=torch.float32, device=dev)
        xs = torch.linspace(-Rw / Rh, Rw / Rh, Rw, **f32)
        ys = torch.linspace(-1, 1, Rh, **f32)
        zs = torch.linspace(cfg["ray_start"], cfg["ray_end"], S, **f32)
        vik = abi.vertex_ik(cond["fk_matrices"], cond["lbs_weights"])
        geo = abi.geo_features(cond["vertices"], cond["tpose_vertices"], cond["skeletons_xyz"], vik,
                               input_scaler=2.0 / cfg["side_length"], legacy_mode=cfg.get("legacy_mode", False),
                               xs=xs, ys=ys, zs=zs, focals=cond["intrinsics"][:, 0, 0], scales=cond["scales"],
                               cam2world=cond["cam2world_matrices"], jitter=u.reshape(B, R * S) if u is not None else None,
                               want_nearest=want_nearest)
    film = film_table(P, freq, phase)
    g = lambda n: P["neural_field." + n]
    heads_b = torch.cat([g("sigma_layer.bias").reshape(1), g("color_layer_linear.bias").reshape(3)]).float().contiguous()
    ray_out, weights = abi.render_mlp(
        geo["rec"], geo["z_vals"], film, wblob, g("sigma_layer.weight").reshape(-1).float().contiguous(),
        g("color_layer_linear.weight").float().contiguous(), g("feature_layer_linear.bias").float().contiguous(), heads_b,
        B=B, R=R, S=S, noise=noise.reshape(B, R * S).float().contiguous() if noise is not None else None,
        noise_std=cfg["nerf_noise"], white_back=cfg.get("white_back", False), last_back=cfg.get("last_back", False),
        clamp_mode=cfg["clamp_mode"], passes=passes, want_weights=want_weights)
    return {"ray_out": ray_out, "z_vals": geo["z_vals"], "weights": weights, "nearest": geo["nearest"]}


@torch.no_grad()
def siren_points(module, pts, freq, phase, geo, dirs, input_scaler=1.0, geo_scaler=1.0, passes=3):
    """Stand-alone COORDCONCATSIREN.forward: [B,N,3], [B,4H], [B,4H], [B,N,G], [B,N,3] -> [B,N,3+F+1].
    The view direction must be constant over all points (it is folded into the colour layer's offset)."""
    abi.require_device()
    squeeze = pts.dim() < 3
    if squeeze:
        pts, geo, dirs = pts.unsqueeze(1), geo.unsqueeze(1), dirs.unsqueeze(1)
    B, N, _ = pts.shape
    G = geo.shape[-1]
    d0 = dirs.reshape(-1, 3)[0]
    if not bool((dirs.reshape(-1, 3) == d0).all()):
        raise RuntimeError("hg3d: COORDCONCATSIREN.forward needs one view direction for all points "
                           "(lock_view_dependence=True in every shipped curriculum)")
    P = {"neural_field." + k: v for k, v in list(module.named_parameters()) + list(module.named_buffers())}
    rec = torch.zeros(B, N, 36, dtype=torch.float32, device=pts.device)
    rec[..., :3] = pts.float() * input_scaler
    rec[..., 3:3 + G] = geo.float() * geo_scaler
    wblob = pack_render_weights(P, geo_dim=G)
    film = film_table(P, freq, phase, locked_dir=tuple(float(v) for v in d0))
    g = lambda n: P["neural_field." + n]
    heads_b = torch.cat([g("sigma_layer.bias").reshape(1), g("color_layer_linear.bias").reshape(3)]).float().contiguous()
    S = 32
    Np = (N + S - 1) // S * S
    if Np != N:
        rec = torch.cat([rec, torch.zeros(B, Np - N, 36, dtype=torch.float32, device=pts.device)], 1)
    raw, _ = abi.render_mlp(rec.contiguous(), None, film, wblob, g("sigma_layer.weight").reshape(-1).float().contiguous(),
                            g("color_layer_linear.weight").float().contiguous(),
                            g("feature_layer_linear.bias").float().contiguous(), heads_b, B=B, R=Np // S, S=S,
                            passes=passes, raw=True)
    out = raw[:, :N]
    return out.squeeze(1) if squeeze else out
