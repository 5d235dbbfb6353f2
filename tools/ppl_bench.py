"""Time perceptual path length's parts at evaluation sizes, in one invocation:
    python tools/ppl_bench.py [--pairs 64] [--gen-batch 8] [--rounds 5] [--out DIR]

  lpips_256x128  LPIPS.distance on --pairs pairs at the PPL input size of 512x256 images (box-downsampled by 2 to 256x128)
  lpips_256x256  the same at the input size of C2's 512x512 images (256x256)
  pair_420       ppl.pair_images on --gen-batch pairs of the 420-wide generator at the sample-app setting (512x256 from a 96x48
                 render of 32 steps, last_back): both endpoints' renders and syntheses, without LPIPS

The parts run in alternating rounds (every part once per round, after one warm-up call each); each is reported as the median
and the range over --rounds of a CUDA-event-timed call.  In a separate pass, with CUDA events around every launch, the head
kernel's time (the five hg_lpips_level launches) is read per LPIPS call, and the render's time (`render_forward_wide`) per
pair batch; both are reported as shares of the part's median.  `ppl_50k_s_extrapolated` is 50 000 times the per-pair time of
pair_420 plus lpips_256x128: an extrapolation from these batches, not a measured 50k run.  The card's name and power limit are
read in the same run.  The VGG16 / lin weights are seeded and the generator randomly initialised (timings do not depend on
the values).  Prints one JSON line and writes it to --out (a new temporary directory by default)."""
import argparse
import importlib
import json
import os
import statistics
import sys
import tempfile

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))


def _images(n, H, W, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    low = torch.rand(n, 3, H // 8, W // 8, generator=g, device="cuda") * 2 - 1
    return F.interpolate(low, size=(H, W), mode="bilinear", align_corners=False)


def _event_ms(fn):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e)


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=64)
    ap.add_argument("--gen-batch", type=int, default=8)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out")
    args = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("ppl_bench: needs a CUDA device")
    from fid_bench import card
    from invert import released_like
    from oracle import metrics_port as mp
    from oracle import ppl_port as plp
    pkg = importlib.import_module("3dhumangan_b200")
    abi = importlib.import_module("3dhumangan_b200.abi")
    metrics = importlib.import_module("3dhumangan_b200.metrics")
    ppl = importlib.import_module("3dhumangan_b200.ppl")
    wide_ops = importlib.import_module("3dhumangan_b200.modules.wide_ops")
    lp = ppl.LPIPS(vgg=metrics.VGG16Features(weights=mp.seeded_vgg16_state(0)), lin=plp.seeded_lin_state(0)).cuda()
    G, cfg, _ = released_like(pkg, "420")
    P = args.pairs
    inputs = {"lpips_256x128": (_images(P, 512, 256, 1), _images(P, 512, 256, 2)),
              "lpips_256x256": (_images(P, 512, 512, 3), _images(P, 512, 512, 4))}
    todo = {name: (lambda a=a, b=b: lp.distance(a, b, ppl.downsample_factor(a.shape[2]))) for name, (a, b) in inputs.items()}
    todo["pair_420"] = lambda: ppl.pair_images(G, cfg, list(range(args.gen_batch)), seed=0, batch=0)
    for fn in todo.values():
        fn()
    torch.cuda.synchronize()
    times = {k: [] for k in todo}
    for _ in range(args.rounds):
        for name, fn in todo.items():
            times[name].append(_event_ms(fn))

    # one pass with events around every launch: the head kernel's share of an LPIPS call
    head = {}
    for name in ("lpips_256x128", "lpips_256x256"):
        abi.TIMING = []
        todo[name]()
        torch.cuda.synchronize()
        head[name] = sum(s.elapsed_time(e) for n, s, e in abi.TIMING if n == "hg_lpips_level")
        abi.TIMING = None
    # and the render's share of a pair batch
    render_ms = []
    orig = wide_ops.render_forward_wide

    def timed_render(*a, **k):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        out = orig(*a, **k)
        e.record()
        render_ms.append((s, e))
        return out
    wide_ops.render_forward_wide = timed_render
    try:
        todo["pair_420"]()
        torch.cuda.synchronize()
    finally:
        wide_ops.render_forward_wide = orig
    render = sum(s.elapsed_time(e) for s, e in render_ms)

    r = {"pairs": P, "gen_batch": args.gen_batch, "rounds": args.rounds, **card()}
    for name, t in times.items():
        med = statistics.median(t)
        n = args.gen_batch if name == "pair_420" else P
        row = {"ms": med, "ms_min": min(t), "ms_max": max(t), "ms_per_pair": med / n}
        if name in head:
            row.update(head_ms=head[name], head_share=head[name] / med)
        else:
            row.update(render_ms=render, render_share=render / med, renders=len(render_ms))
        r[name] = row
    per_pair = r["pair_420"]["ms_per_pair"] + r["lpips_256x128"]["ms_per_pair"]
    r["ppl_50k_s_extrapolated"] = 50000 * per_pair / 1e3
    line = json.dumps(r)
    out_dir = args.out or tempfile.mkdtemp(prefix="hg3d_ppl_bench_")
    os.makedirs(out_dir, exist_ok=True)
    with open(os.path.join(out_dir, "ppl_bench.json"), "w") as fh:
        fh.write(line + "\n")
    print(line)


if __name__ == "__main__":
    main()
