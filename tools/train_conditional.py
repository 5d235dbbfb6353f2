"""Cost of a conditional (reconstruction) training iteration against the unconditional one, at the training size `bench.py`
times (C3: 512x512 images, render 96x96, 16 images per iteration in `batch_split` = 4 micro-batches, fp32, no autocast).

The conditional iteration runs a `uncond: False` phase with all three reconstruction terms (latent regression in both steps,
photometric and perceptual in the generator step, seeded VGG16 weights) and a latent pool of MAP3DBN512L's size
(`dataset_length` = 219047 rows of 256): its dense gradient, Adam and EMA are part of every generator step.  The unconditional
iteration runs the shipped curriculum's first phase on the same networks and the same pool.  The two alternate round by
round; each round times `--iters` iterations of each with a device-synchronised clock.

Also reported: peak memory of each kind, per-term times measured apart with CUDA events (perceptual forward + backward at one
micro-batch, the latent and photometric losses, the pool lookup and its dense gradient, one Adam + EMA step over the pool
alone), and the device time per kernel of one conditional iteration from `torch.profiler`.  Prints one JSON line; the line
and the profiler table are also written to `--out` (a new temporary directory by default, named in the line).
    python tools/train_conditional.py [--rounds 5] [--iters 2] [--warmup 2] [--out DIR]"""
import argparse
import importlib
import json
import os
import subprocess
import sys
import tempfile
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

POOL = 219047          # MAP3DBN512L's dataset_length


def _gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return out or None
    except (OSError, subprocess.SubprocessError):
        return None


def _events_ms(fn, n):
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(n):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / n


def _stats(v):
    v = sorted(v)
    return {"median": round(v[len(v) // 2], 2), "min": round(v[0], 2), "max": round(v[-1], 2), "n": len(v)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=2)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--split", type=int, default=4)
    ap.add_argument("--out", default=None, help="directory for the JSON line and the profiler table (default: a new temporary one)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("train_conditional: needs a CUDA device")
    pkg = importlib.import_module("3dhumangan_b200")
    gen = importlib.import_module("3dhumangan_b200.modules.generator")
    disc = importlib.import_module("3dhumangan_b200.modules.discriminator")
    ts = importlib.import_module("3dhumangan_b200.train_step")
    ops = importlib.import_module("3dhumangan_b200.ops.trainer_ops")
    perceptual = importlib.import_module("3dhumangan_b200.perceptual")
    from oracle import perceptual_port as pp
    dev = torch.device("cuda", 0)
    B, split = args.batch, args.split

    base = pkg.configs.baseline_config("C2")
    base.update(nerf_noise=0.5, batch_split=split, dataset_length=POOL)
    cond_meta = dict(base, latent_lambda=1.0, photometric_lambda=1.0, perceptual_lambda=[1.0, 1.0, 1.0, 1.0])
    cond_meta["phases"] = [{"name": "cond", "uncond": False, "rotate": False, "gen_modal": "rgbs", "do_r1": False}]
    uncond_meta = dict(base)
    uncond_meta["phases"] = [dict(base["phases"][0])]
    torch.manual_seed(0)
    G = gen.Map3DGenerator(**base).to(dev).train()
    G.set_device(dev)
    D = disc.UNetDiscriminator(**base).to(dev).train()
    codes, app = pkg.synthetic.make_appearance(B, POOL, base["latent_dim"], seed=2)
    vgg = perceptual.VGGPerceptualLoss(weights=pp.seeded_vgg16_state(0)).to(dev)
    trainer = ts.Trainer(G, D, cond_meta, amp=False, perceptual=vgg, appearance_codes=codes)
    Hg, Wg = base["gen_height"], base["gen_width"]
    g = torch.Generator().manual_seed(5)
    cond = {k: v.to(dev) for k, v in pkg.synthetic.make_conditions(B, seed=1).items()}
    cond.update({k: v.to(dev) for k, v in app.items()})
    batch = dict(z_d=torch.randn(B, base["latent_dim"], generator=g).to(dev), z_g=torch.randn(B, base["latent_dim"], generator=g).to(dev),
                 images=torch.randn(B, 3, Hg, Wg, generator=g).clamp_(-1, 1).to(dev),
                 labels=torch.randint(1, base["label_dim"], (B, Hg, Wg), generator=g).to(dev), cond=cond)
    metas = {"conditional": cond_meta, "unconditional": uncond_meta}

    def iterate(kind, n):
        trainer.meta = metas[kind]
        out = []
        for _ in range(n):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            trainer.iteration(batch)
            torch.cuda.synchronize()
            out.append((time.perf_counter() - t0) * 1e3)
        return out

    peak = {}
    for kind in metas:
        iterate(kind, args.warmup)
        torch.cuda.reset_peak_memory_stats(dev)
        iterate(kind, 1)
        peak[kind] = round(torch.cuda.max_memory_allocated(dev) / 2 ** 30, 2)
    times = {k: [] for k in metas}
    for r in range(args.rounds):
        order = list(metas) if r % 2 == 0 else list(metas)[::-1]
        for kind in order:
            times[kind] += iterate(kind, args.iters)

    # ---- per-term costs, measured apart at one micro-batch
    b = B // split
    rgbs = torch.rand(b, 3, Hg, Wg, device=dev, requires_grad=True)
    real = torch.rand(b, 3, Hg, Wg, device=dev)
    lat = torch.randn(b, base["latent_dim"], device=dev, requires_grad=True)
    lat_t = torch.randn(b, base["latent_dim"], device=dev)
    pool = G.latent_pool.latents
    idx = app["indices"][:b].to(dev)

    def perceptual_term():
        sum(vgg(rgbs, real)).backward()

    def photometric_term():
        ops.image_loss(rgbs, real, kind="smooth_l1", beta=0.1).backward()

    def latent_term():
        ops.latent_loss(lat, lat_t, beta=0.1).backward()

    dz = torch.randn(b, base["latent_dim"], device=dev)

    def pool_lookup_and_grad():
        pool.grad = None
        ops.latent_pool_gather(pool, idx).backward(dz)

    pool_grad = torch.randn_like(pool) * 1e-3
    probe = ts.ParameterEMA([pool])
    opt = ops.FusedAdam([{"params": [pool]}], lr=0.0, betas=(0.0, 0.9))

    def pool_adam_ema():
        pool.grad = pool_grad
        opt.step(clip_max_norm=1.0, ema=probe, ema_params=[pool])

    terms = {}
    for name, fn in (("perceptual_fwd_bwd", perceptual_term), ("photometric", photometric_term), ("latent_loss", latent_term),
                     ("pool_gather_and_dense_grad", pool_lookup_and_grad), ("pool_adam_ema", pool_adam_ema)):
        fn()
        terms[name] = round(_events_ms(fn, 10), 3)
    pool.grad = None
    pool_bytes = pool.numel() * 4
    # Adam + EMA with clipping over the pool: read p, g, m, v, shadow (5), write p, m, v, shadow (4); the norm pass reads g once
    terms["pool_adam_ema_bytes"] = 10 * pool_bytes
    terms["pool_adam_ema_GBps"] = round(10 * pool_bytes / (terms["pool_adam_ema"] * 1e-3) / 1e9, 1)

    # ---- device time per kernel of one conditional iteration
    trainer.meta = cond_meta
    out_dir = args.out or tempfile.mkdtemp(prefix="train_conditional_")
    os.makedirs(out_dir, exist_ok=True)
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        trainer.iteration(batch)
        torch.cuda.synchronize()
    table = prof.key_averages().table(sort_by="cuda_time_total", row_limit=60)
    with open(os.path.join(out_dir, "profile_conditional.txt"), "w") as f:
        f.write(table)
    new_kernels = {}
    for e in prof.key_averages():
        for key in ("latent_pool_gather", "latent_pool_grad", "latent_loss", "image_loss_kernel", "mt_adam", "mt_sumsq", "vgg"):
            if key in e.key:
                t = getattr(e, "device_time_total", None)
                if t is None:
                    t = getattr(e, "cuda_time_total", 0)
                new_kernels[e.key[:60]] = {"ms": round(t / 1e3, 3), "calls": e.count}
    line = {"gpu": _gpu_info(), "workload": f"C3 {Hg}x{Wg}, render {base['render_height']}, B={B} in {split} micro-batches, fp32",
            "pool": [POOL, base["latent_dim"]], "iteration_ms": {k: _stats(v) for k, v in times.items()},
            "ratio_median": round(_stats(times["conditional"])["median"] / _stats(times["unconditional"])["median"], 3),
            "peak_mem_gib": peak, "term_ms": terms, "profiled_kernels": new_kernels, "out_dir": out_dir}
    print(json.dumps(line))
    with open(os.path.join(out_dir, "train_conditional.json"), "w") as f:
        json.dump(line, f)


if __name__ == "__main__":
    main()
