"""Extract the generator's surface as PLY meshes, on synthetic conditions: `3dhumangan_b200.surface.extract_mesh` with an
eval-mode generator set up as tools/invert.py sets it up.
    python tools/extract_mesh.py [--config 420|tiny] [--checkpoint generator.pth] [--resolution 256] [--level L]
                                 [--truncation 1.0] [--seed 0] [--out DIR]
Writes one PLY per sample to --out (a new temporary directory by default) and prints one JSON line: vertex and face counts,
the seconds of the density lattice alone and of the whole extraction (lattice, iso-surface, colours), the PLY paths.
Without --checkpoint the generator is randomly initialised, so the mesh shows the untrained density."""
import argparse
import importlib
import json
import os
import sys
import tempfile
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from invert import released_like  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", choices=["420", "tiny"], default="420")
    ap.add_argument("--checkpoint")
    ap.add_argument("--resolution", type=int, default=256)
    ap.add_argument("--level", type=float, help="iso level (default: ln 2 / the renderer's sample spacing)")
    ap.add_argument("--truncation", type=float, default=1.0)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--out")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("extract_mesh: needs a CUDA device")
    pkg = importlib.import_module("3dhumangan_b200")
    surface = importlib.import_module("3dhumangan_b200.surface")
    G, cfg, cond = released_like(pkg, args.config, args.checkpoint)
    out_dir = args.out or tempfile.mkdtemp(prefix="hg3d_mesh_")
    os.makedirs(out_dir, exist_ok=True)
    z = torch.randn(1, cfg["latent_dim"], generator=torch.Generator(device="cuda").manual_seed(args.seed), device="cuda")
    kw = dict(cfg, latent=z, truncation_psi=args.truncation, resolution=args.resolution)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    surface.density_lattice(G, cond, **kw)
    torch.cuda.synchronize()
    t1 = time.perf_counter()
    meshes = surface.extract_mesh(G, cond, level=args.level, **kw)
    torch.cuda.synchronize()
    t2 = time.perf_counter()
    paths = [surface.write_ply(os.path.join(out_dir, f"mesh_{b}.ply"), m) for b, m in enumerate(meshes)]
    print(json.dumps({"config": args.config, "resolution": args.resolution, "level": meshes[0]["level"],
                      "V": [int(m["vertices"].shape[0]) for m in meshes], "F": [int(m["faces"].shape[0]) for m in meshes],
                      "lattice_s": t1 - t0, "extract_s": t2 - t1, "ply": paths}))


if __name__ == "__main__":
    main()
