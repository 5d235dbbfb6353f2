"""Training throughput of the zero-padded generator widths: `Trainer.iteration` (fp16 autocast + GradScaler) on the MAP3DBN
curriculum (hidden 384, 256x128, render 64x32) and on MAP3DBN512L (hidden 420, 512x256, render 96x48), each with the
curriculum's batch of 32 in `batch_split` micro-batches.  After warm-up, each step is timed with a
device-synchronised clock.  The default warm-up runs phases 0-2 and the timed window phases 3-6, so it holds one do_r1
phase (R1 on phases 3 and 7), which is reported apart.  Prints one JSON line.
    python tools/train_wide.py [--split384 4] [--split420 16] [--warmup 3] [--iters 4]"""
import argparse
import importlib
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def _power_limit():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                             text=True, timeout=30).stdout.strip()
        return out or None
    except (OSError, subprocess.SubprocessError):
        return None


def run(pkg, name, split, warmup, iters, dev):
    gen = importlib.import_module("3dhumangan_b200.modules.generator")
    disc = importlib.import_module("3dhumangan_b200.modules.discriminator")
    ts = importlib.import_module("3dhumangan_b200.train_step")
    cur = getattr(pkg.configs, name)
    cfg = pkg.configs.extract_metadata({k: v for k, v in cur.items()}, 0)
    cfg = {k: v for k, v in cfg.items() if isinstance(k, str)}
    cfg.update(nerf_noise=0.5, batch_split=split)
    B, Hg, Wg, C = cfg["batch_size"], cfg["gen_height"], cfg["gen_width"], cfg["hidden_dim"]
    torch.manual_seed(0)
    G = gen.Map3DGenerator(**cfg).to(dev).train()
    G.set_device(dev)
    D = disc.UNetDiscriminator(**cfg).to(dev).train()
    trainer = ts.Trainer(G, D, cfg, amp=True)
    g = torch.Generator().manual_seed(5)
    batch = dict(images=torch.randn(B, 3, Hg, Wg, generator=g).clamp_(-1, 1).to(dev),
                 labels=torch.randint(1, cfg["label_dim"], (B, Hg, Wg), generator=g).to(dev),
                 cond={k: v.to(dev) for k, v in pkg.synthetic.make_conditions(B, seed=1).items()})
    for _ in range(warmup):
        trainer.iteration(batch)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats(dev)
    d_ms, d_r1_ms, g_ms = [], [], []
    for _ in range(iters):
        r1 = bool(cfg["phases"][D.step % len(cfg["phases"])]["do_r1"])
        t0 = time.perf_counter()
        trainer.train_discriminator(batch)
        torch.cuda.synchronize()
        t1 = time.perf_counter()
        trainer.train_generator(batch)
        torch.cuda.synchronize()
        t2 = time.perf_counter()
        D.step += 1
        G.step += 1
        (d_r1_ms if r1 else d_ms).append((t1 - t0) * 1e3)
        g_ms.append((t2 - t1) * 1e3)
    total_s = (sum(d_ms) + sum(d_r1_ms) + sum(g_ms)) / 1e3
    mean = lambda v: round(sum(v) / len(v), 2) if v else None
    return {"curriculum": name, "hidden_dim": C, "gen": [Hg, Wg], "render": [cfg["render_height"], cfg["render_width"]],
            "num_steps": cfg["num_steps"], "batch": B, "batch_split": split,
            "images_per_s": round(B * iters / total_s, 2),
            "d_step_ms": mean(d_ms), "d_step_r1_ms": mean(d_r1_ms), "g_step_ms": mean(g_ms),
            "peak_mem_gib": round(torch.cuda.max_memory_allocated(dev) / 2 ** 30, 2),
            "padding_mma_factor": round((512 / C) ** 2, 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--split384", type=int, default=4)
    ap.add_argument("--split420", type=int, default=16)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--iters", type=int, default=4)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("train_wide: needs a CUDA device")
    pkg = importlib.import_module("3dhumangan_b200")
    dev = torch.device("cuda", 0)
    rows = [run(pkg, name, split, args.warmup, args.iters, dev)
            for name, split in (("MAP3DBN", args.split384), ("MAP3DBN512L", args.split420))]
    print(json.dumps({"gpu": torch.cuda.get_device_name(dev), "power_limit": _power_limit(), "amp": "fp16", "runs": rows}))


if __name__ == "__main__":
    main()
