"""Time surface extraction on the GPU: the density lattice (`surface.density_lattice`) and the iso-surface (`abi.iso_surface`)
apart, at hidden_dim 420 (the released checkpoint's zero-padded path, legacy_mode) and 256 (the fused per-point kernel),
B = 1, lattice resolutions 128 / 256 / 512.
    python tools/surface_bench.py [--resolutions 128 256 512] [--rounds 5] [--out DIR]
Each round times every case once, lattice then iso-surface, so the cases alternate; the JSON line per case holds the median
and range over the rounds, the peak device memory of one extraction, V / F, and the card's name and power limit read in the
same process.  Parameters are seeded (sigma gain 200, bias 1, as the density tests use), the iso level is the lattice mean.
The last line is a summary; everything is also written to --out (a new temporary directory by default)."""
import argparse
import copy
import importlib
import json
import os
import subprocess
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    name, power = (q.stdout.strip().splitlines() or ["?, ?"])[0].split(", ")
    return {"gpu": name, "power_limit": power}


def generator(pkg, C):
    from oracle import port
    gen = importlib.import_module("3dhumangan_b200.modules.generator")
    if C == 420:
        cfg = pkg.configs.extract_metadata(copy.deepcopy(pkg.configs.MAP3DBN512L), 0)
        cfg.update(dataset_length=16, num_steps=32)
    else:
        cfg = pkg.configs.baseline_config("C2")
    G = gen.Map3DGenerator(**cfg).cuda()
    G.load_state_dict({k: v.cuda() for k, v in port.init_generator_params(cfg, seed=3, sigma_gain=200.0, sigma_bias=1.0).items()})
    G.set_device(torch.device("cuda:0"))
    G.eval()
    return G, cfg


def timed(fn):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    out = fn()
    e.record()
    torch.cuda.synchronize()
    return out, s.elapsed_time(e)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--resolutions", type=int, nargs="+", default=[128, 256, 512])
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("surface_bench: needs a CUDA device")
    pkg = importlib.import_module("3dhumangan_b200")
    surface = importlib.import_module("3dhumangan_b200.surface")
    abi = importlib.import_module("3dhumangan_b200.abi")
    out_dir = args.out or tempfile.mkdtemp(prefix="hg3d_surface_bench_")
    os.makedirs(out_dir, exist_ok=True)
    cond = {k: v.cuda() for k, v in pkg.synthetic.make_conditions(1, seed=1).items()}
    cases = []
    for C in (420, 256):
        G, cfg = generator(pkg, C)
        with torch.no_grad():
            freq, phase, _ = G.truncated_codes(torch.randn(1, cfg["latent_dim"], device="cuda"), 1.0, cfg)
        for res in args.resolutions:
            kw = dict(cfg, freq=freq, phase=phase, resolution=res)
            lat = surface.density_lattice(G, cond, **kw)[0]               # warm-up of every shape the rounds use
            level = float(lat["density"].mean())
            abi.iso_surface(lat["density"], level, lat["origin"], lat["spacing"])
            torch.cuda.synchronize()
            base = torch.cuda.memory_allocated()
            torch.cuda.reset_peak_memory_stats()
            lat = surface.density_lattice(G, cond, **kw)[0]
            v, n, f = abi.iso_surface(lat["density"], level, lat["origin"], lat["spacing"])
            torch.cuda.synchronize()
            peak = torch.cuda.max_memory_allocated() - base
            cases.append(dict(G=G, kw=kw, level=level, lat=lat, rec={
                "hidden_dim": C, "resolution": res, "lattice": list(lat["density"].shape), "points": lat["density"].numel(),
                "V": int(v.shape[0]), "F": int(f.shape[0]), "peak_mib": peak / 2 ** 20, "lattice_ms": [], "iso_ms": []}))
            del v, n, f
    for _ in range(args.rounds):
        for c in cases:
            lat, ms = timed(lambda: surface.density_lattice(c["G"], cond, **c["kw"])[0])
            c["rec"]["lattice_ms"].append(ms)
            _, ms = timed(lambda: abi.iso_surface(lat["density"], c["level"], lat["origin"], lat["spacing"]))
            c["rec"]["iso_ms"].append(ms)
            del lat
    info = card()
    lines = []
    for c in cases:
        r = c["rec"]
        for k in ("lattice_ms", "iso_ms"):
            t = sorted(r.pop(k))
            r[k] = {"median": t[len(t) // 2], "min": t[0], "max": t[-1]}
        r["lattice_ns_per_point"] = r["lattice_ms"]["median"] * 1e6 / r["points"]
        r.update(info)
        lines.append(json.dumps(r))
        print(lines[-1])
    summary = json.dumps({"cases": len(cases), "rounds": args.rounds, **info, "out": out_dir})
    print(summary)
    with open(os.path.join(out_dir, "surface_bench.jsonl"), "w") as fh:
        fh.write("\n".join(lines + [summary]) + "\n")


if __name__ == "__main__":
    main()
