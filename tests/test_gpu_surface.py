"""Surface extraction on the device: `hg_iso_count` / `hg_iso_emit` against the numpy restatement of the rule
(tests/surface_oracle.py), `surface.density_lattice` against the reference (tests/golden/surface_density.npz) and the fp64
oracle, and `surface.extract_mesh` end to end."""
import importlib
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import surface_oracle as so  # noqa: E402

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "surface_density.npz")
TOL = 1e-3            # relative L2 of the render tests' sigma (test_gpu_generator.py::test_siren_points_matches_oracle)


def _mod(name):
    return importlib.import_module("3dhumangan_b200." + name)


def rel_l2(a, b):
    a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double().cpu()
    return float((a - b).norm() / b.norm())


# ------------------------------------------------------------------------------------------------------------ the kernel
def _grid(n, lo, hi):
    h = (hi - lo) / (n - 1)
    c = lo + h * np.arange(n)
    Z, Y, X = np.meshgrid(c, c, c, indexing="ij")
    return X, Y, Z, h


def _fields():
    out = {}
    X, Y, Z, h = _grid(64, -1.1, 1.1)
    out["sphere64"] = (0.8 - np.sqrt(X ** 2 + Y ** 2 + Z ** 2), 0.0, (-1.1, -1.1, -1.1), h)
    X, Y, Z, h = _grid(48, -1.0, 1.0)
    out["torus"] = (0.25 - np.sqrt((np.sqrt(X ** 2 + Y ** 2) - 0.6) ** 2 + Z ** 2), 0.0, (-1.0,) * 3, h)
    X, Y, Z, h = _grid(40, -1.0, 1.0)
    out["two_spheres"] = (np.maximum(0.35 - np.sqrt((X - 0.45) ** 2 + Y ** 2 + Z ** 2), 0.3 - np.sqrt((X + 0.45) ** 2 + Y ** 2 + Z ** 2)),
                          0.0, (-1.0,) * 3, h)
    c = np.arange(21) - 10
    Zi, Yi, Xi = np.meshgrid(c, c, c, indexing="ij")
    out["level_at_points"] = (49.0 - (Xi ** 2 + Yi ** 2 + Zi ** 2), 0.0, (0.5, -2.0, 3.0), 0.25)
    rng = np.random.default_rng(0)
    bordered = rng.standard_normal((13, 17, 11))
    bordered[[0, -1]] = bordered[:, [0, -1]] = bordered[:, :, [0, -1]] = -5
    out["bordered_noise"] = (bordered, 0.25, (0.0, 0.0, 0.0), 1.0)
    X, Y, Z, h = _grid(24, 0.0, 1.0)
    out["plane"] = (0.5 - Z + 0.1 * X - 0.05 * Y, 0.0, (0.0,) * 3, h)
    out["empty"] = (np.zeros((3, 4, 5)), 0.5, (0.0,) * 3, 1.0)
    for shape in ((2, 2, 2), (3, 5, 7), (67, 33, 129)):
        out["noise_" + "x".join(map(str, shape))] = (rng.standard_normal(shape), 0.1, (-0.3, 0.2, 1.5), 0.01)
    return out


FIELDS = _fields()


def _check_against_oracle(field, level, origin, h):
    abi = _mod("abi")
    lat = torch.from_numpy(np.ascontiguousarray(field, dtype=np.float32)).cuda()
    v, n, f = abi.iso_surface(lat, level, origin, h)
    torch.cuda.synchronize()
    rv, rn, rf = so.iso_surface(lat.cpu().numpy(), level, origin, h)
    assert f.dtype == torch.int32 and v.dtype == n.dtype == torch.float32
    assert tuple(f.shape) == rf.shape and tuple(v.shape) == rv.shape
    assert np.array_equal(f.cpu().numpy(), rf), "faces differ from the oracle"
    ext = h * (max(field.shape) - 1)
    if rv.size:
        assert np.abs(v.cpu().numpy() - rv).max() <= 1e-6 * max(ext, 1.0)
        assert np.abs(n.cpu().numpy() - rn).max() <= 1e-6
    return v, n, f


@pytest.mark.parametrize("name", list(FIELDS))
def test_kernel_equals_oracle(name):
    field, level, origin, h = FIELDS[name]
    v, n, f = _check_against_oracle(field, level, origin, h)
    if name == "empty":
        assert v.shape == (0, 3) and n.shape == (0, 3) and f.shape == (0, 3)
    elif name in ("sphere64", "torus", "two_spheres", "level_at_points", "bordered_noise"):
        assert so.closed_and_oriented(f.cpu().numpy())


def test_kernel_equals_oracle_on_a_large_lattice():
    """2^24 points: the scans span 4096 blocks."""
    n = 256
    c = np.arange(n, dtype=np.float32) * np.float32(2 * np.pi / 64)
    Z, Y, X = np.meshgrid(c, c, c, indexing="ij")
    field = np.sin(X) * np.cos(Y) + np.sin(Y) * np.cos(Z) + np.sin(Z) * np.cos(X)        # gyroid, period 64 points
    v, _, f = _check_against_oracle(field, 0.3, (-1.0, -1.0, -1.0), 2.0 / (n - 1))
    assert f.shape[0] > 1_000_000


def test_repeatable_and_runs_the_library_kernels():
    abi = _mod("abi")
    field, level, origin, h = FIELDS["noise_67x33x129"]
    lat = torch.from_numpy(field.astype(np.float32)).cuda()
    a = abi.iso_surface(lat, level, origin, h)
    b = abi.iso_surface(lat, level, origin, h)
    for x, y in zip(a, b):
        assert torch.equal(x, y)
    # the kernel trace in a fresh process: a second profiler session in one process may record no device activity
    code = "\n".join([
        "import importlib, sys, torch",
        f"sys.path.insert(0, {ROOT!r})",
        "abi = importlib.import_module('3dhumangan_b200.abi')",
        "lat = torch.randn(33, 17, 65, device='cuda')",
        "abi.iso_surface(lat, 0.1)",
        "with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:",
        "    abi.iso_surface(lat, 0.1)",
        "    torch.cuda.synchronize()",
        "print(' '.join(e.key for e in prof.key_averages()))"])
    out = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stderr[-2000:]
    names = out.stdout
    for k in ("iso_count_kernel", "iso_scan_reduce_kernel", "iso_scan_blocks_kernel", "iso_scan_apply_kernel", "iso_emit_kernel"):
        assert k in names, (k, names)


def test_kernel_refusals():
    abi = _mod("abi")
    for shape in ((1, 4, 4), (4, 1, 4), (4, 4, 1)):
        with pytest.raises(RuntimeError, match="hg3d:"):
            abi.iso_surface(torch.zeros(shape, device="cuda"), 0.0)
    with pytest.raises(RuntimeError, match="hg3d:"):
        abi.iso_surface(torch.zeros(4, 4, 4, device="cuda"), float("nan"))
    with pytest.raises(RuntimeError, match="hg3d:"):
        abi.iso_surface(torch.zeros(4, 4, 4, device="cuda"), 0.0, spacing=0.0)
    with pytest.raises(RuntimeError, match="hg3d:"):
        abi.iso_surface(torch.zeros(4, 4, 4, device="cuda", dtype=torch.float64), 0.0)
    with pytest.raises(RuntimeError, match="2\\^30"):
        abi.iso_surface(torch.empty(1025, 1024, 1024, device="meta"), 0.0)


# ------------------------------------------------------------------------------------------------- density and meshes
def _generator(pkg, port, C=256, seed=31, **over):
    gen = _mod("modules.generator")
    cfg = pkg.configs.baseline_config("tiny")
    if C != 256:
        cfg.update(hidden_dim=C, feature_dim=C, latent_dim=C)
    cfg.update(over)
    G = gen.Map3DGenerator(**cfg).cuda()
    params = port.init_generator_params(cfg, seed=seed, sigma_gain=200.0, sigma_bias=1.0)
    G.load_state_dict({k: v.cuda() for k, v in params.items()})
    G.set_device(torch.device("cuda:0"))
    G.eval()
    return G, cfg, params


def _cond(pkg, seed=42, B=1):
    return {k: v.cuda() for k, v in pkg.synthetic.make_conditions(B, seed=seed).items()}


def _lattice_points(lat):
    nz, ny, nx = lat["density"].shape
    i = torch.arange(nz * ny * nx)
    idx = torch.stack([i % nx, i // nx % ny, i // (nx * ny)], 1).float()
    return torch.tensor(lat["origin"], dtype=torch.float32) + lat["spacing"] * idx


def _oracle_point_outputs(port, params, cfg, cond, b, pts, freq, phase):
    """port.geo_features + fp64 port.siren at world points [N,3] -> [N, 3+F+1] (rgb, feat, sigma)."""
    P = {k: v.double() for k, v in params.items() if v.is_floating_point()}
    c = {k: v[b:b + 1].cpu().float() for k, v in cond.items()}
    geo, _ = port.geo_features(pts.float()[None], c["skeletons_xyz"], c["vertices"], c["tpose_vertices"], c["fk_matrices"],
                               c["lbs_weights"], legacy_mode=cfg.get("legacy_mode", False))      # fp32, as the reference runs it
    geo = geo.double()
    p = pts.double()[None]
    dirs = torch.zeros_like(p)
    dirs[..., -1] = -1
    return port.siren(P, p, freq[b:b + 1].cpu().double(), phase[b:b + 1].cpu().double(), geo, dirs, 2.0 / cfg["side_length"],
                      cfg["hidden_dim"], 4)[0]


def test_density_matches_reference_golden(pkg, port):
    gold = np.load(GOLD)
    recipe = json.loads(str(gold["recipe"]))
    surface = _mod("surface")
    G, cfg, _ = _generator(pkg, port, seed=recipe["param_seed"])
    cond = _cond(pkg, recipe["cond_seed"])
    freq, phase = torch.from_numpy(gold["freq"]).cuda(), torch.from_numpy(gold["phase"]).cuda()
    lat = surface.density_lattice(G, cond, freq=freq, phase=phase, resolution=recipe["resolution"], margin=recipe["margin"],
                                  chunk_points=256)[0]
    assert tuple(lat["density"].shape) == tuple(gold["shape"])
    assert np.allclose(lat["origin"], gold["origin"], atol=1e-6) and abs(lat["spacing"] - float(gold["spacing"])) < 1e-9
    assert float((gold["density"] > 0).mean()) > 0.02
    assert rel_l2(lat["density"], torch.from_numpy(gold["density"])) < TOL
    # the latent path maps the golden's latent to the same codes (neural_field_latent_input False: a zero latent)
    z = torch.from_numpy(gold["z"]).cuda()
    lz = surface.density_lattice(G, cond, latent=z, resolution=recipe["resolution"], margin=recipe["margin"])[0]
    assert rel_l2(lz["density"], torch.from_numpy(gold["density"])) < TOL
    # a perturbed freq is caught by the tolerance
    bad = surface.density_lattice(G, cond, freq=freq + 0.5, phase=phase, resolution=recipe["resolution"], margin=recipe["margin"])[0]
    assert rel_l2(bad["density"], torch.from_numpy(gold["density"])) > 10 * TOL


@pytest.mark.parametrize("C,legacy", [(384, False), (420, True)])
def test_density_wide_matches_oracle(pkg, port, C, legacy):
    surface = _mod("surface")
    G, cfg, params = _generator(pkg, port, C=C, seed=33, legacy_mode=legacy)
    cond = _cond(pkg, 43)
    g = torch.Generator().manual_seed(5)
    freq, phase = torch.randn(1, 4 * C, generator=g).cuda(), torch.randn(1, 4 * C, generator=g).cuda()
    lat = surface.density_lattice(G, cond, freq=freq, phase=phase, resolution=14, chunk_points=384)[0]
    ref = torch.relu(_oracle_point_outputs(port, params, cfg, cond, 0, _lattice_points(lat), freq, phase)[:, -1])
    assert float((ref > 0).double().mean()) > 0.02
    assert rel_l2(lat["density"].reshape(-1), ref) < TOL
    bad = surface.density_lattice(G, cond, freq=freq + 0.5, phase=phase, resolution=14)[0]
    assert rel_l2(bad["density"].reshape(-1), ref) > 10 * TOL


@pytest.mark.parametrize("C", [256, 420])
def test_extract_mesh_end_to_end(pkg, port, C):
    surface = _mod("surface")
    G, cfg, params = _generator(pkg, port, C=C, seed=34, legacy_mode=C == 420)
    cond = _cond(pkg, 44, B=2)
    g = torch.Generator().manual_seed(6)
    freq, phase = torch.randn(2, 4 * C, generator=g).cuda(), torch.randn(2, 4 * C, generator=g).cuda()
    lats = surface.density_lattice(G, cond, freq=freq, phase=phase, resolution=40)
    for b, lat in enumerate(lats):
        level = float(lat["density"].median())
        mesh = surface.extract_mesh(G, {k: v[b:b + 1] for k, v in cond.items()}, freq=freq[b:b + 1], phase=phase[b:b + 1],
                                    resolution=40, level=level)[0]
        rv, rn, rf = so.iso_surface(lat["density"].cpu().numpy(), level, lat["origin"], lat["spacing"])
        assert rf.shape[0] > 100
        assert np.array_equal(mesh["faces"].cpu().numpy(), rf)
        assert np.abs(mesh["vertices"].cpu().numpy() - rv).max() <= 1e-6 * lat["spacing"] * max(lat["density"].shape)
        assert mesh["level"] == level and mesh["origin"] == lat["origin"] and mesh["spacing"] == lat["spacing"]
        pick = torch.linspace(0, rv.shape[0] - 1, min(rv.shape[0], 2000)).long()
        ref = _oracle_point_outputs(port, params, cfg, cond, b, mesh["vertices"].cpu()[pick], freq, phase)[:, :3]
        assert rel_l2(mesh["colors"].cpu()[pick], ref) < TOL
        nz, ny, nx = lat["density"].shape
        hi = torch.tensor(lat["origin"]) + lat["spacing"] * torch.tensor([nx - 1, ny - 1, nz - 1], dtype=torch.float64)
        v = cond["vertices"][b].cpu().double()
        assert (v >= torch.tensor(lat["origin"])).all() and (v <= hi).all()


def test_film_sources(pkg, port):
    surface = _mod("surface")
    G, cfg, _ = _generator(pkg, port, seed=35)
    cond = _cond(pkg, 45)
    z = torch.randn(1, cfg["latent_dim"], generator=torch.Generator().manual_seed(7)).cuda()
    kw = dict(resolution=16, neural_field_latent_input=True)
    torch.manual_seed(123)
    a = surface.density_lattice(G, cond, latent=z, truncation_psi=0.7, **kw)[0]["density"]
    torch.manual_seed(123)
    with torch.no_grad():
        _, afreq, aphase, _ = G.generate_avg_latent()
        freq, phase = G.neural_field_mapping_network(z)
    b = surface.density_lattice(G, cond, freq=afreq + 0.7 * (freq - afreq), phase=aphase + 0.7 * (phase - aphase), **kw)[0]["density"]
    assert torch.equal(a, b)
    c = surface.density_lattice(G, cond, latent=z, **kw)[0]["density"]
    d = surface.density_lattice(G, cond, freq=freq, phase=phase, **kw)[0]["density"]
    assert torch.equal(c, d)
    assert not torch.equal(a, c)


def test_peak_memory_is_bounded(pkg, port):
    surface = _mod("surface")
    G, cfg, _ = _generator(pkg, port, C=420, seed=36, legacy_mode=True)
    cond = _cond(pkg, 46)
    g = torch.Generator().manual_seed(8)
    freq, phase = torch.randn(1, 4 * 420, generator=g).cuda(), torch.randn(1, 4 * 420, generator=g).cuda()
    surface.density_lattice(G, cond, freq=freq, phase=phase, resolution=32)         # warm-up: packed weights, allocator
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    lat = surface.density_lattice(G, cond, freq=freq, phase=phase, resolution=256)[0]
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    lat_bytes = lat["density"].numel() * 4
    bound = surface.CHUNK_BYTES_PER_POINT * surface.CHUNK_POINTS + surface.CHUNK_BYTES_FIXED
    print(f"peak {peak / 2**20:.1f} MiB, lattice {lat_bytes / 2**20:.1f} MiB, bound {bound / 2**20:.1f} MiB")
    assert peak <= lat_bytes + bound


def test_refusals(pkg, port):
    surface = _mod("surface")
    gen = _mod("modules.generator")
    G, cfg, _ = _generator(pkg, port)
    cond = _cond(pkg)
    f = torch.zeros(1, 4 * 256, device="cuda")
    for kw in (dict(resolution=1), dict(resolution=3.5), dict(bbox=((0, 0, 0), (1, -1, 1))), dict(bbox=((0, 0, 0),))):
        with pytest.raises(RuntimeError, match="hg3d:"):
            surface.density_lattice(G, cond, freq=f, phase=f, **kw)
    with pytest.raises(RuntimeError, match="hg3d:"):
        surface.extract_mesh(G, cond, freq=f, phase=f, resolution=8, level=float("nan"))
    with pytest.raises(RuntimeError, match="hg3d:"):
        surface.density_lattice(G, cond, resolution=8)
    wide = pkg.configs.baseline_config("tiny")
    wide.update(hidden_dim=576, feature_dim=576, latent_dim=576)
    Gw = gen.Map3DGenerator(**wide)
    with pytest.raises(RuntimeError, match="hg3d: the zero-padded path serves hidden_dim <= 512"):
        surface.density_lattice(Gw, cond, freq=torch.zeros(1, 4 * 576, device="cuda"), phase=torch.zeros(1, 4 * 576, device="cuda"),
                                resolution=8)


def test_extract_mesh_tool(tmp_path):
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    from test_cpu_surface import read_ply
    out = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "extract_mesh.py"), "--config", "tiny", "--resolution", "48", "--level", "0",
                          "--out", str(tmp_path)], capture_output=True, text=True, timeout=900, cwd=ROOT)
    assert out.returncode == 0, out.stderr[-3000:]
    res = json.loads(out.stdout.strip().splitlines()[-1])
    verts, faces = read_ply(res["ply"][0])
    assert verts.shape[0] == res["V"][0] and faces.shape[0] == res["F"][0]
    assert res["F"][0] > 0 and faces.max() < verts.shape[0]
