"""Golden fixture of the renderer's density on a lattice, run by the UNMODIFIED reference on the CPU (build container only;
needs the reference checkout plus the test-only shims in oracle/shims).

    python tests/golden/make_golden_surface.py      # writes tests/golden/surface_density.npz

A 256-wide generator with seeded parameters (sigma_gain 200, sigma_bias 1, as the hierarchical fixture) and synthetic
conditions.  The lattice is `surface.lattice_box` of the posed vertices at a small resolution; at its points the reference's
`Map3DGenerator.get_geo_features` (map3d_generator.py:196-205) and `COORDCONCATSIREN.forward` (modulated.py:41-75) give the
raw sigma, with the renderer's input scaler 2 / side_length and the locked view direction (0, 0, -1).  The fixture holds the
lattice geometry, freq / phase, the raw sigma and the density clamped by clamp_mode, and the recipe as JSON.
"""
import copy
import importlib
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
RECIPE = {"config": "tiny", "param_seed": 31, "sigma_gain": 200.0, "sigma_bias": 1.0, "cond_seed": 42, "latent_seed": 131,
          "resolution": 14, "margin": 0.1}


def build_case(pkg, port):
    cfg = pkg.configs.baseline_config(RECIPE["config"])
    params = port.init_generator_params(cfg, seed=RECIPE["param_seed"], sigma_gain=RECIPE["sigma_gain"],
                                        sigma_bias=RECIPE["sigma_bias"])
    cond = pkg.synthetic.make_conditions(1, seed=RECIPE["cond_seed"])
    z = torch.randn(1, cfg["latent_dim"], generator=torch.Generator().manual_seed(RECIPE["latent_seed"]))
    return cfg, params, cond, z


def lattice_points(origin, h, shape):
    nz, ny, nx = shape
    i = torch.arange(nz * ny * nx)
    idx = torch.stack([i % nx, i // nx % ny, i // (nx * ny)], 1).float()
    return torch.tensor(origin, dtype=torch.float32) + h * idx


def main():
    sys.path.insert(0, ROOT)
    sys.path.insert(0, HERE)
    pkg = importlib.import_module("3dhumangan_b200")
    surface = importlib.import_module("3dhumangan_b200.surface")
    from oracle import port
    from make_golden import reference_modules
    gens, _, impl = reference_modules()
    cfg, params, cond, z = build_case(pkg, port)
    meta = dict(cfg)
    meta["neural_field_cls"] = getattr(impl, meta["neural_field_cls"])
    G = gens.Map3DGenerator(**meta)
    G.load_state_dict(copy.deepcopy(params), strict=True)
    G.set_device("cpu")
    G.eval()
    origin, h, shape = surface.lattice_box(cond["vertices"][0], RECIPE["resolution"], RECIPE["margin"])
    pts = lattice_points(origin, h, shape)[None]
    with torch.no_grad():
        freq, phase = G.neural_field_mapping_network(z if meta["neural_field_latent_input"] else torch.zeros_like(z))
        geo = G.get_geo_features(pts, cond["skeletons_xyz"], cond["vertices"], cond["tpose_vertices"], cond["fk_matrices"],
                                 cond["lbs_weights"])
        dirs = torch.zeros_like(pts)
        dirs[..., -1] = -1
        out = G.neural_field.forward(pts, freq, phase, geo, ray_directions=dirs, input_scaler=2. / G.side_length)
    sigma = out[0, :, -1]
    dens = torch.relu(sigma) if cfg["clamp_mode"] == "relu" else torch.nn.functional.softplus(sigma)
    print(shape, float(h), float(dens.mean()), float((dens > 0).float().mean()))
    np.savez_compressed(os.path.join(HERE, "surface_density.npz"), recipe=np.array(json.dumps(RECIPE)),
                        origin=np.array(origin), spacing=np.array(h), shape=np.array(shape), freq=freq.numpy(), phase=phase.numpy(),
                        z=z.numpy(), sigma=sigma.reshape(shape).numpy(), density=dens.reshape(shape).numpy(),
                        clamp_mode=np.array(cfg["clamp_mode"]))


if __name__ == "__main__":
    main()
