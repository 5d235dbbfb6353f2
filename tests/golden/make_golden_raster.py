"""Fixture for the SMPL label-map rasteriser (SURVEY.md 8f-2) from the reference's OWN code (build container only).

Runs the unmodified `SHHQPreprocessor.forward_with_rotation` (-> `_forward_fix_body`, `_forward_rasterize`,
lib/data/preprocessor.py:56-176) on seeded conditions of the 6 890-vertex synthetic surface
(`SMPLModel.synthetic_surface`; SMPL_NEUTRAL.pkl is licence-gated and absent), skinned and canonicalised by
oracle/smpl_port.py, with the DensePose face labels of tests/golden/densepose_data.json.  pytorch3d is not installed: its
`Meshes`, `PerspectiveCameras`, `euler_angles_to_matrix` and the preprocessor's `self.rasterizer` are the restatements of
oracle/raster_port.py and oracle/smpl_port.py, injected as make_golden_smpl.py injects `euler_angles_to_matrix`.  Everything
the reference builds around them -- the camera (field of view 1 degree, negative focal length, T_raster), the `% F` of packed
face ids, the barycentric argmax, the labels + 2 / background 1, the semantics of sample 0 -- runs as the reference wrote it.
Writes tests/golden/raster_conditions.npz with a 256x128 (MAP3DBN) and a 64x64 case."""
import importlib
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle", "shims"))
sys.path.insert(0, "/root/reference")

SHAPES = {"h256w128": (256, 128, 2, 0), "h64w64": (64, 64, 2, 1)}


def conditions(B, seed):
    """Seeded fix-body conditions of the synthetic surface, on the CPU oracle -> (cond dict, faces, (h, v, r))."""
    from oracle import smpl_port as sp
    smpl = importlib.import_module("3dhumangan_b200.smpl")
    model, faces = smpl.SMPLModel.synthetic_surface("cpu", seed=seed)
    g = torch.Generator().manual_seed(100 + seed)
    betas = torch.randn(B, 10, generator=g)
    pose = torch.randn(B, 24, 3, generator=g) * 0.15
    A, v_shaped, verts, J, Jt = sp.lbs(betas, pose.reshape(B, -1), model.v_template, model.shapedirs, model.posedirs, model.J_regressor,
                                       model.parents.long(), model.lbs_weights)
    rot = sp.batch_rodrigues(pose.reshape(-1, 3)).reshape(B, 24, 3, 3)
    orig_cam = torch.stack([1.2 + 0.2 * torch.rand(B, generator=g), torch.ones(B), 0.1 * torch.randn(B, generator=g),
                            0.1 * torch.randn(B, generator=g)], 1)
    cond = sp.conditions_fix_body(orig_cam, Jt, rot, v_shaped, A, model.lbs_weights, model.v_template)
    angles = torch.randn(3, B, generator=g) * torch.tensor([[0.4], [0.1], [0.0]])
    return cond, faces, angles


def main():
    from oracle import raster_port as rp
    from oracle import smpl_port as sp
    import lib.data.preprocessor as pp
    pp.euler_angles_to_matrix = lambda e, convention: sp.euler_xyz_to_matrix(e)
    pp.Meshes = rp.Meshes
    pp.PerspectiveCameras = rp.PerspectiveCameras
    labels = rp.faces_to_labels(os.path.join(HERE, "densepose_data.json"))
    out = {}
    for name, (H, W, B, seed) in SHAPES.items():
        cond, faces, ang = conditions(B, seed)
        pre = pp.SHHQPreprocessor(gen_height=H, gen_width=W)
        pre.rasterizer = rp.MeshRasterizer(H, W)
        pre.init_smpl(faces, labels)
        keep = {k: cond[k].clone() for k in ("vertices", "tpose_vertices", "full_pose", "R", "T", "scales")}
        data = pre.forward_with_rotation(dict(cond), ang[0], ang[1], ang[2])
        out.update({f"{name}_{k}": v.numpy() for k, v in keep.items()})
        out.update({f"{name}_angles": ang.numpy(), f"{name}_cam2world": data["cam2world_matrices"].numpy(),
                    f"{name}_segments": data["rasterized_segments"].numpy().astype(np.int8),
                    f"{name}_semantics": data["rasterized_semantics"].numpy()})
        fg = float((data["rasterized_segments"] > 1).float().mean())
        print(name, "foreground fraction %.3f" % fg, "labels", sorted(set(data["rasterized_segments"].unique().tolist()))[:6], "...")
    np.savez_compressed(os.path.join(HERE, "raster_conditions.npz"), **out)


if __name__ == "__main__":
    main()
