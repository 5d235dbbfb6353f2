"""Geometry of the generator: the renderer's density on a lattice and its iso-surface as a triangle mesh.

`density_lattice` evaluates the density the volume renderer integrates -- the raw `sigma_layer` output of the FiLM-SIREN,
clamped by `clamp_mode`, without noise (`vr.ray_integration`'s sigma at nerf_noise 0) -- on a regular lattice in world
coordinates (the frame of `conditions["vertices"]`), in chunks of at most `chunk_points` points:

    lattice coordinates   torch
    hg_geo_features       nearest posed vertex + 31-d geometry feature of every point (points_in mode)
    sigma                 the sigma column of hg_render_mlp's per-point mode at hidden_dim 256; the zero-padded trunk up to
                          the sigma head (wide_ops.render_forward_wide, sigma_only) at 384 / 420 -- hierarchical.coarse_sigma

`extract_mesh` turns each lattice into a closed, consistently oriented mesh by marching tetrahedra (`abi.iso_surface`,
csrc/surface.cu) and colours its vertices with the NeRF colour head at the locked view direction (0, 0, -1): the per-point
rgb that the renderer composites.  `write_ply` stores a mesh as binary little-endian PLY.

What the surface depends on: with neural_field_latent_input False (all three shipped curricula) freq / phase come from
`neural_field_mapping_network(0)`, so the density does not depend on the latent and the mesh is the clothed-body geometry
the renderer learned for a POSE.  It follows the subject when freq / phase are given directly (e.g. `inversion.invert(
space="film")`'s result) or when a config sets neural_field_latent_input True.
"""
from __future__ import annotations

import math

import numpy as np
import torch

from . import abi
from .modules.generator import _precision_passes

CHUNK_POINTS = 1 << 17
# Device memory of one chunk on top of the lattice, per chunk point: the zero-padded trunk keeps at most four [2 x 256]-channel
# fp32 activations alive at once (8 KiB) next to the 128-channel point blocks and the point records; plus the packed weights
# and the FiLM tables.  tests/test_gpu_surface.py holds density_lattice to it at hidden_dim 420.
CHUNK_BYTES_PER_POINT = 10 << 10
CHUNK_BYTES_FIXED = 64 << 20


def _cfg(G, kwargs):
    cfg = G._cfg_for(kwargs, kwargs.get("render_height", 1), kwargs.get("render_width", 1))
    if cfg["hidden_dim"] > 512:
        raise RuntimeError("hg3d: the zero-padded path serves hidden_dim <= 512")
    if cfg["clamp_mode"] not in ("relu", "softplus"):
        raise RuntimeError("Need to choose clamp mode")          # volume_rendering.py:31
    return cfg


def default_level(cfg):
    """ln 2 / delta, delta = (ray_end - ray_start) / (num_steps - 1): the density at which one of the renderer's own sample
    intervals is half opaque (1 - exp(-delta * sigma) = 1/2).  cam2world is rigid (smpl.cam2world_fix_body: the inverse of a
    rotation, a translation and the body rotation), so delta is a world length too."""
    delta = (float(cfg["ray_end"]) - float(cfg["ray_start"])) / (int(cfg["num_steps"]) - 1)
    return math.log(2.0) / delta


def lattice_box(vertices, resolution, margin=0.1, bbox=None):
    """Lattice of one sample -> (origin (3 floats), spacing h, (nz, ny, nx)).  Default box: the AABB of the posed vertices
    [V,3], padded on every side by margin x its largest extent; `bbox` = ((x0, y0, z0), (x1, y1, z1)) overrides it.
    h = longest extent / (resolution - 1); points per axis = ceil(extent / h) + 1."""
    if not isinstance(resolution, int) or resolution < 2:
        raise RuntimeError(f"hg3d: surface resolution must be an integer >= 2 (got {resolution!r})")
    if bbox is not None:
        if len(bbox) != 2:
            raise RuntimeError(f"hg3d: bbox must be ((x0, y0, z0), (x1, y1, z1)) (got {bbox!r})")
        lo, hi = (np.asarray(c, dtype=np.float64).reshape(-1) for c in bbox)
        if lo.size != 3 or hi.size != 3 or not (np.isfinite(lo).all() and np.isfinite(hi).all()) or not (hi > lo).all():
            raise RuntimeError(f"hg3d: bbox must be ((x0, y0, z0), (x1, y1, z1)) with x1 > x0, y1 > y0, z1 > z0 (got {bbox!r})")
    else:
        if not margin >= 0:
            raise RuntimeError(f"hg3d: margin must be >= 0 (got {margin!r})")
        v = vertices.detach().double().cpu().numpy().reshape(-1, 3)
        lo, hi = v.min(0), v.max(0)
        pad = float(margin) * float((hi - lo).max())
        lo, hi = lo - pad, hi + pad
    ext = hi - lo
    h = float(ext.max()) / (resolution - 1)
    if not h > 0:
        raise RuntimeError("hg3d: the surface box has zero extent")
    counts = [int(math.ceil(e / h - 1e-9)) + 1 for e in ext]
    counts = [max(2, c) for c in counts]
    if counts[0] * counts[1] * counts[2] > 1 << 30:
        raise RuntimeError(f"hg3d: a {counts[2]} x {counts[1]} x {counts[0]} lattice exceeds 2^30 points")
    return tuple(float(c) for c in lo), h, (counts[2], counts[1], counts[0])


def _film(G, cfg, latent, freq, phase, truncation_psi):
    if (latent is None) == (freq is None or phase is None):
        raise RuntimeError("hg3d: pass either `latent` or both `freq` and `phase`")
    if latent is not None:
        freq, phase, _ = G.truncated_codes(latent, truncation_psi, cfg)
    return freq.float(), phase.float()


def _point_records(cond, b, pts, cfg):
    vik = abi.vertex_ik(cond["fk_matrices"][b:b + 1], cond["lbs_weights"][b:b + 1])
    return abi.geo_features(cond["vertices"][b:b + 1], cond["tpose_vertices"][b:b + 1], cond["skeletons_xyz"][b:b + 1], vik,
                            points_in=pts[None], input_scaler=2.0 / cfg["side_length"],
                            legacy_mode=cfg.get("legacy_mode", False))["rec"]


def _pad128(pts):
    n = pts.shape[0]
    m = (n + 127) // 128 * 128
    if m == n:
        return pts
    return torch.cat([pts, pts[-1:].expand(m - n, 3)])


class _Evaluator:
    """Per-point heads of one sample's FiLM-SIREN over given world points, in chunks of 128-point multiples."""

    def __init__(self, G, cfg, freq, phase, passes):
        from .modules import render_ops
        self.cfg, self.freq, self.phase, self.passes = dict(cfg, num_steps=128), freq, phase, passes
        self.P = G._params()
        self.wide = cfg["hidden_dim"] != 256
        self.wblob = None if self.wide else render_ops.pack_render_weights(self.P, geo_dim=cfg["geo_feature_dim"])

    def sigma(self, cond, b, pts):
        from .modules import hierarchical
        n = pts.shape[0]
        rec = _point_records(cond, b, _pad128(pts), self.cfg)
        sig, stride = hierarchical.coarse_sigma(self.P, self.freq[b:b + 1], self.phase[b:b + 1], rec, self.cfg, self.passes,
                                                wblob=self.wblob)
        sig = sig.reshape(-1)[:n]
        return torch.relu(sig) if self.cfg["clamp_mode"] == "relu" else torch.nn.functional.softplus(sig)

    def rgb(self, cond, b, pts):
        from .modules import render_ops, wide_ops
        n = pts.shape[0]
        rec = _point_records(cond, b, _pad128(pts), self.cfg)
        fq, ph = self.freq[b:b + 1], self.phase[b:b + 1]
        if self.wide:
            out = wide_ops.render_forward_wide(self.P, fq, ph, None, self.cfg, None, None, passes=self.passes, records=(rec, None),
                                               point_rgb=True)
            return out[0, :n]
        g = lambda k: self.P["neural_field." + k].detach()
        heads_b = torch.cat([g("sigma_layer.bias").reshape(1), g("color_layer_linear.bias").reshape(3)]).float().contiguous()
        raw, _ = abi.render_mlp(rec, None, render_ops.film_table(self.P, fq, ph), self.wblob,
                                g("sigma_layer.weight").reshape(-1).float().contiguous(), g("color_layer_linear.weight").float().contiguous(),
                                g("feature_layer_linear.bias").float().contiguous(), heads_b, B=1, R=rec.shape[1] // 128, S=128,
                                passes=self.passes, raw=True)
        return raw[0, :n, 0:3]


def _chunk(chunk_points):
    c = int(chunk_points)
    if c < 128:
        raise RuntimeError(f"hg3d: chunk_points must be >= 128 (got {chunk_points!r})")
    return c // 128 * 128


@torch.no_grad()
def density_lattice(G, conditions, *, latent=None, freq=None, phase=None, truncation_psi=1.0, resolution=256, bbox=None,
                    margin=0.1, chunk_points=CHUNK_POINTS, **cfg):
    """The renderer's density on a lattice per sample -> [dict(density [nz,ny,nx] fp32, origin (x, y, z), spacing h)].

    FiLM codes from `latent` ([B, latent_dim], honouring neural_field_latent_input, truncated towards `generate_avg_latent`
    as `staged_forward` does) or from `freq` / `phase` ([B, 4 * hidden_dim], the mapped space of `synthesize`).  `bbox`
    (one box for every sample) overrides the default box (`lattice_box`).  Peak device memory: the lattices plus about
    CHUNK_BYTES_PER_POINT x chunk_points + CHUNK_BYTES_FIXED bytes."""
    abi.require_device()
    cfg = _cfg(G, cfg)
    chunk = _chunk(chunk_points)
    freq, phase = _film(G, cfg, latent, freq, phase, truncation_psi)
    ev = _Evaluator(G, cfg, freq, phase, _precision_passes(cfg))
    dev = freq.device
    out = []
    for b in range(freq.shape[0]):
        origin, h, (nz, ny, nx) = lattice_box(conditions["vertices"][b], resolution, margin, bbox)
        lat = torch.empty(nz * ny * nx, dtype=torch.float32, device=dev)
        o = torch.tensor(origin, dtype=torch.float32, device=dev)
        for s in range(0, lat.numel(), chunk):
            i = torch.arange(s, min(s + chunk, lat.numel()), device=dev)
            idx = torch.stack([i % nx, i // nx % ny, i // (nx * ny)], 1).float()
            lat[s:s + i.numel()] = ev.sigma(conditions, b, o + h * idx)
        out.append({"density": lat.reshape(nz, ny, nx), "origin": origin, "spacing": h})
    return out


@torch.no_grad()
def extract_mesh(G, conditions, *, level=None, colors=True, latent=None, freq=None, phase=None, truncation_psi=1.0,
                 resolution=256, bbox=None, margin=0.1, chunk_points=CHUNK_POINTS, **cfg):
    """Iso-surface of `density_lattice` at `level` (default `default_level`) per sample -> [dict(vertices [V,3], faces [F,3]
    int32, normals [V,3], colors [V,3] in [0,1] or None, origin, spacing, level)], device tensors.  Faces wind
    counter-clockwise seen from outside (low density)."""
    abi.require_device()
    c = _cfg(G, cfg)
    if level is None:
        level = default_level(c)
    level = float(level)
    if not math.isfinite(level):
        raise RuntimeError(f"hg3d: iso level must be finite (got {level})")
    chunk = _chunk(chunk_points)
    freq, phase = _film(G, c, latent, freq, phase, truncation_psi)
    lats = density_lattice(G, conditions, freq=freq, phase=phase, resolution=resolution, bbox=bbox, margin=margin,
                           chunk_points=chunk, **cfg)
    ev = _Evaluator(G, c, freq, phase, _precision_passes(c)) if colors else None
    meshes = []
    for b, lat in enumerate(lats):
        verts, normals, faces = abi.iso_surface(lat["density"], level, lat["origin"], lat["spacing"])
        rgb = None
        if colors:
            rgb = torch.empty_like(verts)
            for s in range(0, verts.shape[0], chunk):
                rgb[s:s + chunk] = ev.rgb(conditions, b, verts[s:s + chunk])
        meshes.append({"vertices": verts, "faces": faces, "normals": normals, "colors": rgb, "origin": lat["origin"],
                       "spacing": lat["spacing"], "level": level})
    return meshes


def write_ply(path, mesh):
    """Binary little-endian PLY: vertex x y z nx ny nz (float) [+ red green blue (uchar)], faces as a uchar count + int list."""
    v = mesh["vertices"].detach().float().cpu().numpy()
    n = mesh["normals"].detach().float().cpu().numpy()
    f = mesh["faces"].detach().cpu().numpy().astype("<i4")
    rgb = mesh.get("colors")
    props = [("x", "<f4"), ("y", "<f4"), ("z", "<f4"), ("nx", "<f4"), ("ny", "<f4"), ("nz", "<f4")]
    if rgb is not None:
        props += [("red", "u1"), ("green", "u1"), ("blue", "u1")]
    rows = np.empty(v.shape[0], dtype=props)
    for k, name in enumerate(("x", "y", "z")):
        rows[name] = v[:, k]
    for k, name in enumerate(("nx", "ny", "nz")):
        rows[name] = n[:, k]
    if rgb is not None:
        c = np.clip(np.rint(rgb.detach().float().cpu().numpy() * 255.0), 0, 255).astype(np.uint8)
        for k, name in enumerate(("red", "green", "blue")):
            rows[name] = c[:, k]
    frows = np.empty(f.shape[0], dtype=[("n", "u1"), ("i", "<i4", (3,))])
    frows["n"] = 3
    frows["i"] = f
    kind = {"<f4": "float", "u1": "uchar"}
    head = ["ply", "format binary_little_endian 1.0", f"element vertex {v.shape[0]}"]
    head += [f"property {kind[t]} {name}" for name, t in props]
    head += [f"element face {f.shape[0]}", "property list uchar int vertex_indices", "end_header"]
    with open(path, "wb") as fh:
        fh.write(("\n".join(head) + "\n").encode("ascii"))
        fh.write(rows.tobytes())
        fh.write(frows.tobytes())
    return path
