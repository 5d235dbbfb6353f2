"""CUDA-event time of each `hg_spade_conv` launch of one C2 generator forward (eager, B = 8 by default), labelled by variant,
next to what the launch has to move and compute:
    hbm    compulsory HBM bytes (read x [+ residual] [+ rgb_in], write out [+ rgb])
    w_l2   weight bytes streamed from L2 into shared memory (one 128-pixel tile fetches the whole packed image)
    flop   tensor FLOPs issued (3 bf16 products per fp32x3 MAC; pixel-style adds the [gamma | beta] GEMM)
and the floor those imply at the data-sheet rates (3.35 TB/s HBM3, 989 TFLOP/s dense bf16).  The card's name, power limit and
SM clock are printed with the numbers.
    python tools/spade_bench.py [--batch 8] [--reps 5] [--precision fp32x3] > spade.json"""
import argparse
import importlib
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402

HBM_BPS, TENSOR_FLOPS = 3.35e12, 989e12
C = 256


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm,clocks_throttle_reasons.active"
    try:
        row = subprocess.run(["nvidia-smi", "--id=0", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.TimeoutExpired):
        return {"name": torch.cuda.get_device_name(0), "nvidia_smi": None}
    return dict(zip(["name", "power_limit", "sm_clock", "sm_clock_max", "throttle_reasons"], [v.strip() for v in row.split(",")]))


def costs(tag, passes):
    """Bytes and FLOPs of one launch from its tag '<const|pixel>[ skip][ rgb][ stats][ xshared] HxW B<n>'."""
    words = tag.split()
    H, W = (int(v) for v in words[-2].split("x"))
    B = int(words[-1][1:])
    HW, tiles = H * W, B * ((H * W + 127) // 128)
    act = B * HW * C * 4
    hbm = act + (HW * C * 4 if "xshared" in words else act)
    hbm += act if "skip" in words else 0
    hbm += 2 * B * HW * 3 * 4 if "rgb" in words else 0        # rgb_in read + rgb_out write (the first ToRGB has no rgb_in)
    w_stage = C * C * 2 * (2 if passes == 3 else 1)            # packed conv image: hi (+ lo) bf16
    flop = tiles * 128 * C * C * 2 * passes
    w_l2 = tiles * w_stage
    if words[0] == "pixel":
        flop += tiles * 128 * 2 * C * 128 * 2 * passes         # [gamma | beta] (N = 512) from A1 (K = 128)
        w_l2 += tiles * 2 * C * 128 * 2 * (2 if passes == 3 else 1)
    return hbm, w_l2, flop


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--reps", type=int, default=5, help="timed forwards; each launch reports its median")
    ap.add_argument("--precision", default="fp32x3", choices=["fp32x3", "bf16"])
    args = ap.parse_args()
    pkg = importlib.import_module("3dhumangan_b200")
    abi = importlib.import_module("3dhumangan_b200.abi")
    gen = importlib.import_module("3dhumangan_b200.modules.generator")
    dev = torch.device("cuda", 0)
    abi.require_device()
    cfg = bench.workload_cfg(pkg, "C2")
    torch.manual_seed(0)
    G = gen.Map3DGenerator(**cfg).to(dev)
    G.set_device(dev)
    G.train()
    kw = dict(cfg, hg_precision=args.precision, hg_cuda_graph=False, hg_cuda_graph_nccl=False)
    B = args.batch
    cond = {k: v.to(dev) for k, v in pkg.synthetic.make_conditions(B, seed=1).items()}
    z = torch.randn(B, cfg["latent_dim"], generator=torch.Generator().manual_seed(2)).to(dev)
    passes = 3 if args.precision == "fp32x3" else 1
    with torch.no_grad():
        for _ in range(2):
            G(z, cond, **kw)
        torch.cuda.synchronize()
        abi.TIMING_TAGS = True
        runs = []
        for _ in range(args.reps):
            abi.TIMING = []
            G(z, cond, **kw)
            torch.cuda.synchronize()
            runs.append([(n, s.elapsed_time(e)) for n, s, e in abi.TIMING if n.startswith("hg_spade_conv")])
        abi.TIMING = None
    rows = []
    for i, (name, _) in enumerate(runs[0]):
        tag = name[len("hg_spade_conv["):-1]
        ms = statistics.median(r[i][1] for r in runs)
        hbm, w_l2, flop = costs(tag, passes)
        t_hbm, t_tc = hbm / HBM_BPS * 1e3, flop / TENSOR_FLOPS * 1e3
        rows.append({"launch": i, "variant": tag, "ms": round(ms, 3), "spread_ms": round(max(r[i][1] for r in runs) - min(r[i][1] for r in runs), 3),
                     "hbm_gb": round(hbm / 1e9, 3), "w_l2_gb": round(w_l2 / 1e9, 3), "tflop": round(flop / 1e12, 3),
                     "floor_ms": round(max(t_hbm, t_tc), 3), "floor_by": "hbm" if t_hbm >= t_tc else "tensor",
                     "hbm_frac_of_floor": round(t_hbm / ms, 3), "tensor_frac_of_floor": round(t_tc / ms, 3),
                     "w_l2_tb_per_s": round(w_l2 / ms / 1e9, 2)})
    total = sum(r["ms"] for r in rows)
    floor = sum(r["floor_ms"] for r in rows)
    print(json.dumps({"card": card(), "batch": B, "precision": args.precision, "reps": args.reps, "launches": len(rows),
                      "total_ms": round(total, 2), "floor_ms": round(floor, 2), "rows": rows}))


if __name__ == "__main__":
    main()
