"""Time the metrics of 3dhumangan_b200.metrics at evaluation sizes, in one invocation:
    python tools/metrics_bench.py [--batch 64] [--rounds 5] [--kid-n 50000] [--pr-n 10000 50000] [--out DIR]

  vgg16       VGG16Features.features on B uint8 images of 512x256 (the 420-wide generator's output size), ms per image
  inception   FIDInceptionV3.features on the same batch, for comparison, ms per image
  kid         kid() with 100 subsets of 1000 from --kid-n real / gen 2048-d seeded features, ms
  pr_<n>      precision_recall() at k = 3 on n real / n gen 4096-d seeded features (two radii passes and one coverage pass), ms

The parts run in alternating rounds (every part once per round, after one warm-up call each); each is reported as the median
and the range over --rounds of a CUDA-event-timed call, with the peak device memory of the part.  Achieved FP64 rates are
counted from shapes (the dot products only: 2 n_a n_b D per pass) against the data sheet's 67 TFLOP/s FP64 tensor rate.  The
card's name and power limit are read in the same run.  The detectors' weights are seeded (the real files are not needed for a
timing).  Prints one JSON line and writes it to --out (a new temporary directory by default)."""
import argparse
import importlib
import json
import os
import statistics
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

FP64_PEAK = 67e12
KID_SUBSETS, KID_M, KID_D, PR_D, PR_K = 100, 1000, 2048, 4096, 3


def kid_flop(S=KID_SUBSETS, m=KID_M, D=KID_D):
    return 3 * S * 2.0 * m * m * D


def pr_flop(n, D=PR_D):
    return 3 * 2.0 * n * n * D


def parts(metrics, fid, vgg, inc, args):
    """name -> (callable, FP64 FLOP or None)."""
    g = torch.Generator(device="cuda").manual_seed(0)
    imgs = torch.randint(0, 256, (args.batch, 3, 512, 256), generator=g, device="cuda", dtype=torch.uint8)
    out = {"vgg16": (lambda: vgg.features(imgs), None), "inception": (lambda: inc.features(imgs), None)}
    kr = torch.rand(args.kid_n, KID_D, generator=g, device="cuda")
    kg = torch.rand(args.kid_n, KID_D, generator=g, device="cuda") * 1.01
    out["kid"] = (lambda: metrics.kid(kr, kg, KID_SUBSETS, KID_M), kid_flop())
    for n in args.pr_n:
        pr = torch.relu(torch.randn(n, PR_D, generator=g, device="cuda"))
        pg = torch.relu(torch.randn(n, PR_D, generator=g, device="cuda") + 0.05)
        out[f"pr_{n}"] = ((lambda a=pr, b=pg: metrics.precision_recall(a, b, PR_K)), pr_flop(n))
    return out


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--kid-n", type=int, default=50000)
    ap.add_argument("--pr-n", type=int, nargs="+", default=[10000, 50000])
    ap.add_argument("--out")
    args = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("metrics_bench: needs a CUDA device")
    from fid_bench import card
    from oracle import inception_port as ip
    from oracle import metrics_port as mp
    fid = importlib.import_module("3dhumangan_b200.fid")
    metrics = importlib.import_module("3dhumangan_b200.metrics")
    inc = fid.FIDInceptionV3(weights=ip.seeded_fid_inception_state(0)).cuda()
    vgg = metrics.VGG16Features(weights=mp.seeded_vgg16_state(0)).cuda()
    todo = parts(metrics, fid, vgg, inc, args)
    times = {k: [] for k in todo}
    peak = {}
    for name, (fn, _) in todo.items():          # warm-up, and each part's peak memory on its own
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        fn()
        torch.cuda.synchronize()
        peak[name] = (torch.cuda.max_memory_allocated() - base) / 2**20
    for _ in range(args.rounds):
        for name, (fn, _) in todo.items():
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            fn()
            e.record()
            torch.cuda.synchronize()
            times[name].append(s.elapsed_time(e))
    r = {"batch": args.batch, "input": "512x256 uint8", "rounds": args.rounds, **card()}
    for name, (_, flop) in todo.items():
        t = times[name]
        med = statistics.median(t)
        row = {"ms": med, "ms_min": min(t), "ms_max": max(t), "peak_mib": peak[name]}
        if name in ("vgg16", "inception"):
            row.update(ms_per_image=med / args.batch, ms_per_image_min=min(t) / args.batch, ms_per_image_max=max(t) / args.batch)
        if flop:
            row.update(fp64_tflops=flop / (med * 1e-3) / 1e12, fp64_share_of_67=flop / (med * 1e-3) / FP64_PEAK)
        r[name] = row
    line = json.dumps(r)
    out_dir = args.out or tempfile.mkdtemp(prefix="hg3d_metrics_bench_")
    os.makedirs(out_dir, exist_ok=True)
    with open(os.path.join(out_dir, "metrics_bench.json"), "w") as fh:
        fh.write(line + "\n")
    print(line)


if __name__ == "__main__":
    main()
