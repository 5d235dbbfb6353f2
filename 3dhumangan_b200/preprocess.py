"""The segmentation targets of a training step on the device (SURVEY.md 8f-2): `SHHQPreprocessor` (lib/data/preprocessor.py)
with pytorch3d's MeshRasterizer replaced by csrc/raster.cu.

    pre = Preprocessor(**meta)                                        # gen_height, gen_width, coordinate_mode="fix_body"
    pre.init_smpl(faces [13776,3], faces_to_labels_from_densepose("densepose_data.json"))
    cond = pre(cond, rotate, **meta)                                  # draws the view like the reference, or
    cond = pre.forward_with_rotation(cond, h, v, r)                   # -> + cam2world_matrices, rasterized_segments [B,H,W] int64,
                                                                      #      rasterized_semantics [B,3,H,W]

`cond` is the dict of smpl.conditions_fix_body (scales, vertices, tpose_vertices, full_pose, R, T, ...).  The view rotation is
smpl.cam2world_fix_body; the rasterising camera (field of view 1 degree, negative focal length, T_raster) is built as
preprocessor.py:142-150 builds it, and the three kernels do the rest: projection, z-buffer, label resolve.  No gradients."""
from __future__ import annotations

import json
import math

import numpy as np
import torch
import torch.nn as nn

from . import abi, smpl

SMPL_VERTS, SMPL_FACES = 6890, 13776
FOCAL_RASTER = 1.0 / math.tan(math.pi * 1 / 180 / 2)


def faces_to_labels_from_densepose(path, n_faces=SMPL_FACES):
    """`get_preprocessor` (preprocessor.py:187-192): SMPL face -> DensePose face -> part label, int64 [n_faces]."""
    with open(path) as f:
        d = json.load(f)
    dp = torch.tensor(d["smpl_faces_to_densepose_faces"], dtype=torch.long)[list(range(n_faces))]
    return torch.tensor(d["densepose_faces_to_labels"], dtype=torch.long)[dp]


@torch.no_grad()
def rasterize_projected(proj, faces, faces_to_labels, tpose0, H, W, debug=False):
    """proj [B,V,3] (NDC x, y, view z; hg_raster_project's output), faces [F,3] int64, faces_to_labels [F] int64, tpose0 [V,3]
    -> dict(rasterized_segments [B,H,W] int64, rasterized_semantics [B,3,H,W]; with debug also pix_to_face [B,H,W] int64
    (b*F + face, -1), zbuf [B,H,W], bary [B,H,W,3])."""
    abi.require_device()
    B, V = proj.shape[0], proj.shape[1]
    F = faces.shape[0]
    dev = proj.device
    proj = proj.float().contiguous()
    faces = faces.to(dev, torch.int64).contiguous()
    labels = faces_to_labels.to(dev, torch.int64).contiguous()
    tpose0 = tpose0.to(dev, torch.float32).contiguous()
    if faces_to_labels.shape[0] != F or tpose0.shape[0] != V:
        raise RuntimeError("hg3d: faces_to_labels must have one entry per face and tpose0 one row per vertex")
    zkey = torch.empty(B, H, W, dtype=torch.int64, device=dev)
    out = {"rasterized_segments": torch.empty(B, H, W, dtype=torch.int64, device=dev),
           "rasterized_semantics": torch.empty(B, 3, H, W, dtype=torch.float32, device=dev)}
    if debug:
        out.update(pix_to_face=torch.empty(B, H, W, dtype=torch.int64, device=dev), zbuf=torch.empty(B, H, W, dtype=torch.float32, device=dev),
                   bary=torch.empty(B, H, W, 3, dtype=torch.float32, device=dev))
    with torch.cuda.device_of(proj):
        abi.call("hg_raster_faces", abi.ptr(proj), abi.ptr(faces), B, V, F, H, W, abi.ptr(zkey), abi.stream())
        abi.call("hg_raster_resolve", abi.ptr(proj), abi.ptr(faces), abi.ptr(labels), abi.ptr(tpose0), abi.ptr(zkey), B, V, F, H, W,
                 abi.ptr(out["rasterized_segments"]), abi.ptr(out["rasterized_semantics"]), abi.ptr(out.get("pix_to_face")),
                 abi.ptr(out.get("zbuf")), abi.ptr(out.get("bary")), abi.stream())
    return out


@torch.no_grad()
def project(verts, R, T, focal):
    """verts [B,V,3], R [B,3,3], T [B,3] -> [B,V,3] = (f X/Z, f Y/Z, Z) of X_view = X @ R + T (pytorch3d's row-vector
    world-to-view and in-NDC perspective projection, principal point 0)."""
    abi.require_device()
    B, V = verts.shape[0], verts.shape[1]
    verts = verts.float().contiguous()
    R = R.to(verts.device, torch.float32).contiguous()
    T = T.to(verts.device, torch.float32).contiguous()
    proj = torch.empty(B, V, 3, dtype=torch.float32, device=verts.device)
    with torch.cuda.device_of(verts):
        abi.call("hg_raster_project", abi.ptr(verts), abi.ptr(R), abi.ptr(T), float(np.float32(focal)), abi.ptr(proj), B, V, abi.stream())
    return proj


class Preprocessor(nn.Module):
    """`SHHQPreprocessor` (preprocessor.py:14-176) for coordinate_mode "fix_body", the mode of every shipped curriculum."""

    def __init__(self, gen_height, gen_width, **kwargs):
        super().__init__()
        self.height, self.width = int(gen_height), int(gen_width)
        self.mode = kwargs.get("coordinate_mode", "fix_body")
        if self.mode != "fix_body":
            raise NotImplementedError("hg3d: coordinate_mode %r is not used by any shipped curriculum and is not built" % self.mode)
        self.register_buffer("vertex_approximation", torch.zeros([SMPL_VERTS], dtype=torch.long))
        self.register_buffer("smpl_faces", torch.zeros([SMPL_FACES, 3], dtype=torch.long))
        self.register_buffer("smpl_faces_to_labels", torch.zeros([SMPL_FACES], dtype=torch.long))

    @torch.no_grad()
    def init_smpl(self, smpl_faces, smpl_faces_to_labels):
        smpl_faces = torch.as_tensor(smpl_faces)
        if smpl_faces.numel() and (int(smpl_faces.min()) < 0 or int(smpl_faces.max()) >= SMPL_VERTS):
            raise ValueError("hg3d: SMPL face indices must lie in [0, %d)" % SMPL_VERTS)
        self.smpl_faces.copy_(smpl_faces)
        self.smpl_faces_to_labels.copy_(torch.as_tensor(smpl_faces_to_labels))

    @torch.no_grad()
    def forward(self, data, rotate=False, **kwargs):
        """preprocessor.py:44-53: h / v drawn with torch.randn on the CPU generator (h first), r = 0."""
        B = data["scales"].shape[0]
        h = torch.randn(B) * (kwargs["h_stddev"] if rotate else 0) + kwargs["h_mean"]
        v = torch.randn(B) * (kwargs["v_stddev"] if rotate else 0) + kwargs["v_mean"]
        return self.forward_with_rotation(data, h, v, torch.zeros_like(h), **kwargs)

    @torch.no_grad()
    def forward_with_rotation(self, data, h_rotation, v_rotation, r_rotation, **kwargs):
        """preprocessor.py:56-68 / 72-98 / 138-176: sets cam2world_matrices, rasterized_segments, rasterized_semantics in `data`
        (and returns it)."""
        Rb = smpl.body_rotation(data, h_rotation, v_rotation, r_rotation)
        data["cam2world_matrices"] = smpl.cam2world_fix_body(data, h_rotation, v_rotation, r_rotation)
        R_raster = torch.inverse(Rb)
        T_raster = data["T"][:, :3, -1].clone()
        T_raster[:, -1] = FOCAL_RASTER / data["scales"] * 0.5
        proj = project(data["vertices"], R_raster, T_raster, -FOCAL_RASTER)
        out = rasterize_projected(proj, self.smpl_faces.to(proj.device), self.smpl_faces_to_labels.to(proj.device),
                                  data["tpose_vertices"][0], self.height, self.width)
        data.update(out)
        return data
