"""Golden fixture of `Map3DGenerator.render(..., hierarchical_sample=True)`, run by the UNMODIFIED reference on the CPU
(build container only; needs the reference checkout plus the test-only shims in oracle/shims).

    python tests/golden/make_golden_hierarchical.py      # writes tests/golden/g_hierarchical.npz

A tiny 256-wide generator (8x8 rays, 32 samples per ray, B = 2) under both clamp modes and nerf_noise 0 / 0.5.  The
reference draws its own randoms from the global torch RNG seeded with the stored seed; `rng.draw_hierarchical_noise`
replays the same sequence.  The fixture holds the outputs and, as JSON, the recipe.
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
OVER = dict(gen_height=32, gen_width=32, render_height=8, render_width=8, num_steps=32, hierarchical_sample=True)
# name: (clamp_mode, nerf_noise, param seed, sigma_gain, sigma_bias, batch)
CASES = {f"{clamp}_n{int(noise * 10)}": (clamp, noise, 20 + i, 200.0, 1.0, 2)
         for i, (clamp, noise) in enumerate((c, n) for c in ("relu", "softplus") for n in (0.0, 0.5))}
SEED = 4321


def build_case(pkg, port, name):
    clamp, noise, pseed, sg, sb, B = CASES[name]
    cfg = pkg.configs.baseline_config("C2")
    cfg.update(OVER)
    cfg.update(clamp_mode=clamp, nerf_noise=noise)
    params = port.init_generator_params(cfg, seed=pseed, sigma_gain=sg, sigma_bias=sb)
    cond = pkg.synthetic.make_conditions(B, seed=11 + pseed)
    z = torch.randn(B, cfg["latent_dim"], generator=torch.Generator().manual_seed(100 + pseed))
    return cfg, params, cond, z


def main():
    sys.path.insert(0, ROOT)
    sys.path.insert(0, HERE)
    pkg = importlib.import_module("3dhumangan_b200")
    from oracle import port
    from make_golden import reference_modules
    gens, _, impl = reference_modules()
    out = {"recipe": np.array(json.dumps({"over": OVER, "cases": CASES, "seed": SEED}))}
    for name in CASES:
        cfg, params, cond, z = build_case(pkg, port, name)
        meta = dict(cfg)
        meta["neural_field_cls"] = getattr(impl, meta["neural_field_cls"])
        G = gens.Map3DGenerator(**meta)
        G.load_state_dict(copy.deepcopy(params), strict=True)
        G.set_device("cpu")
        G.train()
        torch.manual_seed(SEED)
        with torch.no_grad():
            rr, fmap, depth, w, _ = G.render(*G.neural_field_mapping_network(z), cond, coarse_steps=meta["num_steps"],
                                             fine_steps=meta["num_steps"], **meta)
        for k, v in (("rgb_render", rr), ("feature_maps", fmap), ("depth", depth), ("weights", w)):
            out[f"{name}.{k}"] = v.numpy()
        print(name, tuple(rr.shape), float(depth.mean()), float(w.sum(2).mean()))
    np.savez_compressed(os.path.join(HERE, "g_hierarchical.npz"), **out)


if __name__ == "__main__":
    main()
