"""The iso-surface rule (tests/surface_oracle.py, the restatement the kernel is tested against) on analytic fields, and the
host-side pieces of `3dhumangan_b200.surface`: lattice box, default level, PLY writer."""
import importlib
import math
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import surface_oracle as so  # noqa: E402


def grid(n, lo, hi):
    h = (hi - lo) / (n - 1)
    c = lo + h * np.arange(n)
    Z, Y, X = np.meshgrid(c, c, c, indexing="ij")
    return X, Y, Z, h


def closed(faces):
    assert faces.shape[0] > 0
    assert so.closed_and_oriented(faces), "an edge is not shared by exactly two oppositely wound faces"


def test_sphere_64():
    X, Y, Z, h = grid(64, -1.1, 1.1)
    r = 0.8
    v, n, f = so.iso_surface(r - np.sqrt(X ** 2 + Y ** 2 + Z ** 2), 0.0, (-1.1,) * 3, h)
    closed(f)
    assert so.euler_characteristic(f) == 2
    assert abs(so.signed_volume(v, f) / (4 / 3 * math.pi * r ** 3) - 1) < 0.01
    assert np.abs(np.linalg.norm(v.astype(np.float64), axis=1) - r).max() < h
    fn = so.face_normals(v, f)
    big = np.linalg.norm(fn, axis=1) > 1e-12
    assert (np.einsum("ij,ij->i", fn, v[f].mean(1))[big] > 0).all(), "face normals point inwards"
    assert (np.einsum("ij,ij->i", n, v) > 0).all(), "vertex normals point inwards"
    assert np.allclose(np.linalg.norm(n, axis=1), 1, atol=1e-6)


def test_torus_genus_one():
    X, Y, Z, h = grid(48, -1.0, 1.0)
    R, r = 0.6, 0.25
    v, _, f = so.iso_surface(r - np.sqrt((np.sqrt(X ** 2 + Y ** 2) - R) ** 2 + Z ** 2), 0.0, (-1.0,) * 3, h)
    closed(f)
    assert so.euler_characteristic(f) == 0
    assert so.components(f) == 1
    assert so.signed_volume(v, f) > 0


def test_two_spheres():
    X, Y, Z, h = grid(40, -1.0, 1.0)
    d = np.maximum(0.35 - np.sqrt((X - 0.45) ** 2 + Y ** 2 + Z ** 2), 0.3 - np.sqrt((X + 0.45) ** 2 + Y ** 2 + Z ** 2))
    v, _, f = so.iso_surface(d, 0.0, (-1.0,) * 3, h)
    closed(f)
    assert so.euler_characteristic(f) == 4
    assert so.components(f) == 2


def test_level_hit_at_lattice_points():
    """Integer field with the level taken at many lattice points: t is 0 there, vertices coincide, triangles degenerate,
    and the mesh is still closed and oriented by the combinatorial rule."""
    c = np.arange(21) - 10
    Z, Y, X = np.meshgrid(c, c, c, indexing="ij")
    field = (49 - (X ** 2 + Y ** 2 + Z ** 2)).astype(np.float32)
    assert (field == 0).sum() > 50
    v, _, f = so.iso_surface(field, 0.0)
    closed(f)
    assert so.euler_characteristic(f) == 2
    assert so.signed_volume(v, f) > 0
    assert (np.linalg.norm(so.face_normals(v, f), axis=1) == 0).any(), "expected degenerate triangles"


def test_random_noise_bordered_below_level():
    rng = np.random.default_rng(0)
    field = rng.standard_normal((13, 17, 11)).astype(np.float32)
    for ax in range(3):
        idx = [slice(None)] * 3
        idx[ax] = 0
        field[tuple(idx)] = -5
        idx[ax] = -1
        field[tuple(idx)] = -5
    v, n, f = so.iso_surface(field, 0.25)
    closed(f)
    assert so.signed_volume(v, f) > 0


def test_plane_cut_by_the_box_is_an_open_sheet():
    X, Y, Z, h = grid(24, 0.0, 1.0)
    for field, cos in ((0.43 - Z, 1.0), (0.5 - Z + 0.1 * X - 0.05 * Y, 1 / math.sqrt(1 + 0.01 + 0.0025))):
        v, n, f = so.iso_surface(field, 0.0, (0.0,) * 3, h)
        assert f.shape[0] > 0 and not so.closed_and_oriented(f)
        assert abs(so.area(v, f) - 1.0 / cos) < 1e-5
        fn = so.face_normals(v, f)
        big = np.linalg.norm(fn, axis=1) > 1e-9                 # collinear triangles: the normal is rounding noise
        assert (fn[big, 2] > 0).all() and big.sum() > f.shape[0] // 2, "the sheet faces the low side (z above the plane)"


def test_no_crossing_gives_an_empty_mesh():
    for field in (np.zeros((3, 4, 5), np.float32), np.ones((2, 2, 2), np.float32)):
        v, n, f = so.iso_surface(field, 0.5 if field.max() == 0 else 0.0)
        assert v.shape == (0, 3) and n.shape == (0, 3) and f.shape == (0, 3)


# ------------------------------------------------------------------------------------------------------------- host pieces
@pytest.fixture(scope="module")
def surface():
    return importlib.import_module("3dhumangan_b200.surface")


def test_lattice_box(surface):
    v = torch.tensor([[0.0, -1.0, 0.5], [0.4, 1.0, 0.73], [0.2, 0.0, 0.6]], dtype=torch.float64)
    origin, h, (nz, ny, nx) = surface.lattice_box(v, 101, margin=0.1)
    pad = 0.1 * 2.0
    assert np.allclose(origin, (0.0 - pad, -1.0 - pad, 0.5 - pad))
    assert math.isclose(h, (2.0 + 2 * pad) / 100)
    assert ny == 101
    assert nx == math.ceil((0.4 + 2 * pad) / h) + 1 and nz == math.ceil((0.23 + 2 * pad) / h) + 1
    for k, n in zip(range(3), (nx, ny, nz)):           # the lattice covers the padded box
        assert origin[k] + (n - 1) * h >= v[:, k].max().item() + pad - 1e-9
    origin, h, shape = surface.lattice_box(v, 11, bbox=((0, 0, 0), (1, 2, 0.5)))
    assert origin == (0.0, 0.0, 0.0) and math.isclose(h, 0.2) and shape == (4, 11, 6)
    for bad in (dict(resolution=1), dict(resolution=2.5), dict(bbox=((0, 0, 0), (1, 0, 1))), dict(bbox=((0, 0), (1, 1))),
                dict(margin=-0.1)):
        kw = dict(resolution=16)
        kw.update(bad)
        with pytest.raises(RuntimeError, match="hg3d:"):
            surface.lattice_box(v, **kw)
    with pytest.raises(RuntimeError, match="hg3d:.*2\\^30"):
        surface.lattice_box(torch.tensor([[0.0, 0, 0], [1, 1, 1]]), 1100, margin=0.0)


def test_default_level(pkg, surface):
    cfg = pkg.configs.baseline_config("C2")
    delta = (cfg["ray_end"] - cfg["ray_start"]) / (cfg["num_steps"] - 1)
    assert math.isclose(surface.default_level(cfg), math.log(2) / delta)
    assert math.isclose(1 - math.exp(-delta * surface.default_level(cfg)), 0.5)
    assert math.isclose(surface.default_level(dict(ray_start=-0.5, ray_end=0.55, num_steps=32)), math.log(2) * 31 / 1.05)


def read_ply(path):
    """Minimal binary little-endian PLY reader for the layout `write_ply` produces."""
    with open(path, "rb") as fh:
        data = fh.read()
    end = data.index(b"end_header\n") + len(b"end_header\n")
    head = data[:end].decode("ascii").splitlines()
    assert head[0] == "ply" and head[1] == "format binary_little_endian 1.0"
    nv = nf = 0
    props = []
    for line in head:
        w = line.split()
        if w[:2] == ["element", "vertex"]:
            nv = int(w[2])
        elif w[:2] == ["element", "face"]:
            nf = int(w[2])
        elif w[0] == "property" and w[1] != "list":
            props.append((w[2], {"float": "<f4", "uchar": "u1"}[w[1]]))
    verts = np.frombuffer(data, dtype=props, count=nv, offset=end)
    faces = np.frombuffer(data, dtype=[("n", "u1"), ("i", "<i4", (3,))], count=nf, offset=end + verts.nbytes)
    assert end + verts.nbytes + faces.nbytes == len(data)
    assert (faces["n"] == 3).all()
    return verts, faces["i"]


@pytest.mark.parametrize("with_colors", [True, False])
def test_ply_round_trip(surface, tmp_path, with_colors):
    X, Y, Z, h = grid(12, -1.0, 1.0)
    v, n, f = so.iso_surface(0.7 - np.sqrt(X ** 2 + Y ** 2 + Z ** 2), 0.0, (-1.0,) * 3, h)
    rgb = torch.rand(v.shape[0], 3, generator=torch.Generator().manual_seed(0)) if with_colors else None
    mesh = {"vertices": torch.from_numpy(v), "normals": torch.from_numpy(n), "faces": torch.from_numpy(f.astype(np.int32)),
            "colors": rgb}
    path = surface.write_ply(str(tmp_path / "m.ply"), mesh)
    rv, rf = read_ply(path)
    assert np.array_equal(np.stack([rv["x"], rv["y"], rv["z"]], 1), v)
    assert np.array_equal(np.stack([rv["nx"], rv["ny"], rv["nz"]], 1), n)
    assert np.array_equal(rf, f)
    if with_colors:
        got = np.stack([rv["red"], rv["green"], rv["blue"]], 1)
        assert np.array_equal(got, np.rint(rgb.numpy() * 255).astype(np.uint8))
    else:
        assert "red" not in rv.dtype.names
