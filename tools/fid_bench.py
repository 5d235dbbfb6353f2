"""Time FID's parts against the generation they evaluate, in one invocation:
    python tools/fid_bench.py [--batch 64] [--gen-batch 8] [--rounds 5] [--out DIR]

  features    FIDInceptionV3.features on B uint8 images of 512x256 (the 420-wide generator's output size), ms per image
  moments     hg_feature_moments on one batch of B 2048-d features, ms per batch
  generate    staged_forward at the sample app's 420-wide setting (512x256 from a 96x48 render, last_back, eager launches),
              ms per image

Each is the median over --rounds of a CUDA-event-timed window after a warm-up; the card's name and power limit are read in
the same run.  The Inception weights are seeded (pytorch-fid's file is not needed for a timing).  Prints one JSON line and
writes it to --out (a new temporary directory by default)."""
import argparse
import importlib
import json
import os
import statistics
import subprocess
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    name, power = (q.stdout.strip().splitlines() or ["?, ?"])[0].split(", ")
    return {"gpu": name, "power_limit": power}


def timed(fn, rounds, reps=1):
    fn()
    torch.cuda.synchronize()
    out = []
    for _ in range(rounds):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        for _ in range(reps):
            fn()
        e.record()
        torch.cuda.synchronize()
        out.append(s.elapsed_time(e) / reps)
    return statistics.median(out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--gen-batch", type=int, default=8)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("fid_bench: needs a CUDA device")
    from oracle import inception_port as ip
    from invert import released_like
    pkg = importlib.import_module("3dhumangan_b200")
    fid = importlib.import_module("3dhumangan_b200.fid")
    net = fid.FIDInceptionV3(weights=ip.seeded_fid_inception_state(0)).cuda()
    g = torch.Generator(device="cuda").manual_seed(0)
    imgs = torch.randint(0, 256, (args.batch, 3, 512, 256), generator=g, device="cuda", dtype=torch.uint8)
    feat_ms = timed(lambda: net.features(imgs), args.rounds)
    feats = net.features(imgs)
    stats = fid.FeatureStats()
    mom_ms = timed(lambda: stats.update(feats), args.rounds, reps=10)

    G, cfg, _ = released_like(pkg, "420", batch=args.gen_batch)
    cond = {k: v.cuda() for k, v in pkg.synthetic.make_conditions(args.gen_batch, seed=1).items()}
    z = torch.randn(args.gen_batch, cfg["latent_dim"], device="cuda")
    run = dict(cfg, nerf_noise=0, last_back=True, truncation_psi=1.0)
    gen_ms = timed(lambda: G.staged_forward(z, cond, **run), args.rounds)

    r = {"features_ms_per_image": feat_ms / args.batch, "features_ms_per_batch": feat_ms, "batch": args.batch,
         "input": "512x256 uint8", "moments_ms_per_batch": mom_ms,
         "generate_ms_per_image": gen_ms / args.gen_batch, "gen_batch": args.gen_batch,
         "features_over_generate": feat_ms / args.batch / (gen_ms / args.gen_batch), "rounds": args.rounds, **card()}
    line = json.dumps(r)
    out_dir = args.out or tempfile.mkdtemp(prefix="hg3d_fid_bench_")
    os.makedirs(out_dir, exist_ok=True)
    with open(os.path.join(out_dir, "fid_bench.json"), "w") as fh:
        fh.write(line + "\n")
    print(line)


if __name__ == "__main__":
    main()
