"""Time the device preprocessor (view rotation + SMPL label-map rasterisation, 3dhumangan_b200/preprocess.py) at the sizes a
training step uses: B=32 at 256x128 (MAP3DBN) and B=16 at 512x512.  CUDA events around `forward_with_rotation` over many calls
after a warm-up, plus the three kernels alone; prints one JSON line per case with the device name and power limit.

    python tools/raster_bench.py [--iters 200]"""
import argparse
import importlib
import json
import math
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def device_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, IndexError, subprocess.SubprocessError):
        q = torch.cuda.get_device_name(0)
    return q


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("raster_bench: needs a CUDA device")
    importlib.import_module("3dhumangan_b200.build").build()
    smpl = importlib.import_module("3dhumangan_b200.smpl")
    pre = importlib.import_module("3dhumangan_b200.preprocess")
    model, faces = smpl.SMPLModel.synthetic_surface("cuda")
    labels = torch.randint(0, 24, (faces.shape[0],), generator=torch.Generator().manual_seed(0))
    info = device_info()
    for B, H, W in ((32, 256, 128), (16, 512, 512)):
        g = torch.Generator().manual_seed(1)
        out = smpl.lbs(torch.randn(B, 10, generator=g) * 0.5, torch.randn(B, 24, 3, generator=g) * 0.2, model)
        orig_cam = torch.stack([1.2 + 0.2 * torch.rand(B, generator=g), torch.ones(B), 0.1 * torch.randn(B, generator=g),
                                0.1 * torch.randn(B, generator=g)], 1)
        cond = smpl.conditions_fix_body(orig_cam, out, model)
        p = pre.Preprocessor(gen_height=H, gen_width=W).cuda()
        p.init_smpl(faces, labels)
        h, v, r = torch.randn(B, generator=g) * 0.4, torch.randn(B, generator=g) * 0.1, torch.zeros(B)
        full = lambda: p.forward_with_rotation(dict(cond), h, v, r)
        Rb = smpl.body_rotation(cond, h, v, r)
        T = cond["T"][:, :3, -1].clone()
        T[:, -1] = pre.FOCAL_RASTER / cond["scales"] * 0.5
        R = torch.inverse(Rb)
        kern = lambda: pre.rasterize_projected(pre.project(cond["vertices"], R, T, -pre.FOCAL_RASTER), p.smpl_faces,
                                               p.smpl_faces_to_labels, cond["tpose_vertices"][0], H, W)
        res = {"B": B, "H": H, "W": W, "device": info}
        for name, fn in (("forward_with_rotation_ms", full), ("kernels_ms", kern)):
            for _ in range(args.warmup):
                fn()
            torch.cuda.synchronize()
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            for _ in range(args.iters):
                fn()
            e.record()
            torch.cuda.synchronize()
            res[name] = round(s.elapsed_time(e) / args.iters, 4)
        seg = full()["rasterized_segments"]
        res["foreground_fraction"] = round(float((seg > 1).float().mean()), 4)
        res["images_per_s"] = round(B / (res["forward_with_rotation_ms"] * 1e-3), 1) if res["forward_with_rotation_ms"] > 0 else math.inf
        print(json.dumps(res))


if __name__ == "__main__":
    main()
