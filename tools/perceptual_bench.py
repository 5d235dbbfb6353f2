"""Cost of the VGG16 perceptual loss (3dhumangan_b200/perceptual.py) on 512x256 inputs, seeded weights.
    loss_B1 / loss_B8     forward + input gradient with cached target features (`loss(x, target_features(t))`), B = 1 and 8
    inversion             one latent-inversion step at the sample app's setting (420 wide, 512x256 from a 96x48 render of 32
                          steps, last_back, B = 1, frozen generator, point records re-used as `inversion.invert` does), with and
                          without the perceptual term, alternating within a round as tools/inversion_bench.py does
For each: median and range over --reps rounds of --iters steps (CUDA events) and the peak device memory of one step.  The
card's name and power limit are printed with the numbers.
    python tools/perceptual_bench.py [--reps 5] [--iters 10] > perceptual.json
    python tools/perceptual_bench.py --profile [--batch 8]      per-kernel split of one loss step (torch.profiler)"""
import argparse
import importlib
import json
import os
import statistics
import sys
from collections import defaultdict

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
from hierarchical_bench import peak, timed  # noqa: E402
from invert import released_like  # noqa: E402
from spade_bench import card  # noqa: E402


def make_net():
    from oracle import perceptual_port as pp
    mod = importlib.import_module("3dhumangan_b200.perceptual")
    return mod.VGGPerceptualLoss(weights=pp.seeded_vgg16_state(0)).cuda()


def loss_step(net, B):
    g = torch.Generator().manual_seed(B)
    x = torch.rand(B, 3, 512, 256, generator=g).cuda().requires_grad_(True)
    tf = net.target_features(torch.rand(B, 3, 512, 256, generator=g).cuda())

    def step():
        sum(net.loss(x, tf)).backward()
        x.grad = None
    return step


def inversion_steps(pkg, net):
    ops = importlib.import_module("3dhumangan_b200.ops.trainer_ops")
    G, cfg, cond = released_like(pkg, "420")
    for p in G.parameters():
        p.requires_grad_(False)
    with torch.no_grad():
        target = G(torch.randn(1, cfg["latent_dim"], device="cuda"), cond, **cfg)["rgbs"]
    tf = net.target_features(0.5 * target + 0.5)
    z = torch.randn(1, cfg["latent_dim"], device="cuda")
    with torch.no_grad():
        freq, phase = G.neural_field_mapping_network(torch.zeros_like(z))
        styles = G.synthesis_mapping_network(z)[1]
    var = [t.clone().requires_grad_(True) for t in (freq, phase, styles)]
    state = {"records": None}

    def make(perceptual):
        def step():
            extra = {"hg_records": state["records"]} if state["records"] is not None else {}
            out = G.synthesize(*var, cond, **dict(cfg, **extra))
            state["records"] = out["hg_records"]
            value = ops.image_loss(out["rgbs"], target)
            if perceptual:
                value = value + net.loss(0.5 * out["rgbs"] + 0.5, tf, (1, 1, 1, 1))
            value.backward()
            for v in var:
                v.grad = None
        return step
    return {"inversion_pixel": make(False), "inversion_pixel_perceptual": make(True)}


def profile(net, B, reps=5):
    step = loss_step(net, B)
    for _ in range(3):
        step()
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            step()
        torch.cuda.synchronize()
    groups = {"conv": ("conv", "halo"), "relu (bias_act)": ("bias_act",), "maxpool": ("maxpool",),
              "level backward": ("vgg_level_bwd",), "input transform": ("vgg_input",), "smooth-L1": ("smooth_l1",),
              "packing": ("pack",)}
    us = defaultdict(float)
    for e in prof.key_averages():
        t = e.self_device_time_total
        if t <= 0:
            continue
        key = next((k for k, pats in groups.items() if any(p in e.key.lower() for p in pats)), "other")
        us[key] += t / reps
    total = sum(us.values())
    print(json.dumps({"profile_batch": B, "ms_per_step": round(total / 1e3, 3),
                      "share": {k: round(v / total, 4) for k, v in sorted(us.items(), key=lambda kv: -kv[1])},
                      "ms": {k: round(v / 1e3, 3) for k, v in us.items()}}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--batch", type=int, default=8)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("perceptual_bench: needs a CUDA device")
    print(json.dumps({"card": card()}), flush=True)
    net = make_net()
    if args.profile:
        profile(net, args.batch)
        return
    pkg = importlib.import_module("3dhumangan_b200")
    fns = {"loss_B1": loss_step(net, 1), "loss_B8": loss_step(net, 8)}
    fns.update(inversion_steps(pkg, net))
    for fn in fns.values():
        for _ in range(args.warmup):
            fn()
    ms = {name: [] for name in fns}
    for _ in range(args.reps):
        for name, fn in fns.items():
            ms[name].append(timed(fn, args.iters))
    for name, fn in fns.items():
        print(json.dumps({"variant": name, "ms_median": round(statistics.median(ms[name]), 3), "ms_min": round(min(ms[name]), 3),
                          "ms_max": round(max(ms[name]), 3), "peak_gib": round(peak(fn), 3)}), flush=True)
    print(json.dumps({"card": card()}), flush=True)


if __name__ == "__main__":
    main()
