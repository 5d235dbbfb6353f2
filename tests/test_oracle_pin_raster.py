"""The rasteriser oracle (oracle/raster_port.py, SURVEY.md 8f-2) on hand-computed cases, against the reference's own
`SHHQPreprocessor.forward_with_rotation` (tests/golden/raster_conditions.npz, made by tests/golden/make_golden_raster.py), and
the DensePose label loader against the reference's indexing.  CPU only."""
import importlib
import json
import os

import numpy as np
import pytest
import torch

from oracle import raster_port as rp

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _tri(verts, faces, H, W):
    return rp.rasterize(np.asarray(verts, np.float32)[None], np.asarray(faces, np.int64), H, W)


def test_pixel_centres_and_one_triangle():
    assert np.array_equal(rp.pix_ndc(np.arange(4), 4, 4), np.float32([-0.75, -0.25, 0.25, 0.75]))
    # (x, y) = (1, 1), (-0.5, 1), (1, -0.5): NDC +x is left, +y up -> the image's top-left corner.  Centres on the hypotenuse
    # x + y = 0.5 have a barycentric of exactly 0 and stay outside (strict test).
    p2f, zbuf, bary = _tri([[1.0, 1.0, 2.0], [-0.5, 1.0, 2.0], [1.0, -0.5, 2.0]], [[0, 1, 2]], 4, 4)
    want = np.full((4, 4), -1)
    want[0, 0] = want[1, 0] = want[0, 1] = 0
    assert np.array_equal(p2f[0], want)
    assert np.all(zbuf[0][want == 0] == 2.0) and np.all(zbuf[0][want < 0] == -1)
    # (x, y) = (0.75, 0.25) at pixel (1, 0): affine barycentrics (b0, b1, b2) = (1/3, 1/6, 1/2)
    assert np.allclose(bary[0, 1, 0], [1 / 3, 1 / 6, 1 / 2], atol=1e-6)
    assert np.allclose(bary[0][want == 0].sum(-1), 1.0, atol=1e-6)


def test_non_square_image():
    # H=4, W=2: the width spans [-1, 1] (centres +-0.5), the height +-2 (centres -1.5 .. 1.5)
    assert np.array_equal(rp.pix_ndc(np.arange(2), 2, 4), np.float32([-0.5, 0.5]))
    assert np.array_equal(rp.pix_ndc(np.arange(4), 4, 2), np.float32([-1.5, -0.5, 0.5, 1.5]))
    p2f, _, _ = _tri([[-3.0, 1.0, 1.0], [3.0, 1.0, 1.0], [0.0, 4.0, 1.0]], [[0, 1, 2]], 4, 2)   # only y = 1.5: the top row
    assert np.array_equal(p2f[0] >= 0, np.array([[1, 1], [0, 0], [0, 0], [0, 0]], bool))
    p2f, _, _ = _tri([[0.0, -5.0, 1.0], [0.0, 5.0, 1.0], [3.0, 0.0, 1.0]], [[0, 1, 2]], 4, 2)    # only x = +0.5: the left column
    assert np.array_equal(p2f[0] >= 0, np.array([[1, 0]] * 4, bool))


def test_nearest_face_wins():
    v = [[2, 2, 3.0], [-2, 2, 3.0], [0, -2, 3.0], [1, 1, 1.0], [-1, 1, 1.0], [0, -1, 1.0]]
    p2f, zbuf, _ = _tri(v, [[0, 1, 2], [3, 4, 5]], 8, 8)
    near = p2f[0] == 1
    assert near.sum() > 4 and np.all(zbuf[0][near] == 1.0)
    assert np.all(zbuf[0][p2f[0] == 0] == 3.0) and (p2f[0] == 0).sum() > 0


def test_equal_depth_goes_to_the_lowest_face():
    v = [[2, 2, 1.5], [-2, 2, 1.5], [0, -2, 1.5], [2, 2, 1.5], [-2, 2, 1.5], [0, -2, 1.5]]
    p2f, _, _ = _tri(v, [[3, 4, 5], [0, 1, 2], [0, 1, 2]], 8, 8)        # three coplanar copies
    assert (p2f[0] >= 0).sum() > 10 and set(np.unique(p2f[0])) == {-1, 0}


def test_face_behind_the_camera_and_zero_area_are_skipped():
    p2f, _, _ = _tri([[1, 1, -1.0], [-1, 1, -1.0], [0, -1, -1.0]], [[0, 1, 2]], 8, 8)
    assert np.all(p2f == -1)
    p2f, _, _ = _tri([[1, 1, 1.0], [0, 0, 1.0], [-1, -1, 1.0], [0.5, 0.5, 1.0]], [[0, 1, 2], [3, 3, 3]], 8, 8)
    assert np.all(p2f == -1)


@pytest.mark.parametrize("name", ["h256w128", "h64w64"])
def test_oracle_matches_reference_preprocessor(name):
    smpl = importlib.import_module("3dhumangan_b200.smpl")
    g = np.load(os.path.join(GOLD, "raster_conditions.npz"))
    H, W = (256, 128) if name == "h256w128" else (64, 64)
    seed = 0 if name == "h256w128" else 1
    _, faces = smpl.SMPLModel.synthetic_surface("cpu", seed=seed)
    cond = {k: torch.from_numpy(g[f"{name}_{k}"]) for k in ("vertices", "tpose_vertices", "full_pose", "R", "T", "scales")}
    ang = torch.from_numpy(g[f"{name}_angles"])
    labels = rp.faces_to_labels(os.path.join(GOLD, "densepose_data.json"))
    out = rp.preprocess(cond, faces.numpy(), labels, H, W, ang[0], ang[1], ang[2])
    seg = g[f"{name}_segments"].astype(np.int64)
    assert (seg > 1).mean() > 0.1
    assert np.array_equal(out["rasterized_segments"].numpy(), seg)
    assert np.abs(out["rasterized_semantics"].numpy() - g[f"{name}_semantics"]).max() <= 1e-6


def test_densepose_labels_follow_the_reference_indexing():
    pre = importlib.import_module("3dhumangan_b200.preprocess")
    path = os.path.join(GOLD, "densepose_data.json")
    d = json.load(open(path))
    want = [d["densepose_faces_to_labels"][d["smpl_faces_to_densepose_faces"][i]] for i in range(13776)]
    got = pre.faces_to_labels_from_densepose(path)
    assert got.dtype == torch.int64 and got.shape == (13776,) and got.tolist() == want
    assert torch.equal(got, rp.faces_to_labels(path))
    assert 0 <= min(want) and max(want) + 2 < 26          # + 2 stays below label_dim


def test_synthetic_surface_is_a_closed_smpl_sized_mesh():
    smpl = importlib.import_module("3dhumangan_b200.smpl")
    model, faces = smpl.SMPLModel.synthetic_surface("cpu")
    V, F = model.v_template.shape[0], faces.shape[0]
    assert (V, F) == (6890, 13776) and F == 2 * V - 4
    e = torch.cat([faces[:, [0, 1]], faces[:, [1, 2]], faces[:, [2, 0]]])
    und = torch.sort(e, 1).values
    uniq, cnt = torch.unique(und, dim=0, return_counts=True)
    assert bool((cnt == 2).all()) and V - uniq.shape[0] + F == 2           # every edge in two faces, Euler characteristic 2
    assert torch.unique(torch.cat([e, e.flip(1)]), dim=0).shape[0] == e.shape[0]   # consistently oriented
    assert torch.allclose(model.lbs_weights.sum(1), torch.ones(V))


def test_preprocessor_refuses_unbuilt_modes_and_bad_faces():
    pre = importlib.import_module("3dhumangan_b200.preprocess")
    with pytest.raises(NotImplementedError):
        pre.Preprocessor(256, 128, coordinate_mode="fix_camera")
    p = pre.Preprocessor(256, 128)
    assert p.smpl_faces.dtype == torch.int64 and p.smpl_faces.shape == (13776, 3) and p.vertex_approximation.shape == (6890,)
    with pytest.raises(ValueError):
        p.init_smpl(torch.full((13776, 3), 6890), torch.zeros(13776, dtype=torch.long))
