"""Cost of hierarchical_sample=True: the same workload with the option off and on, in alternating runs.
    g_c2_graph     Map3DGenerator.forward at C2 (256 wide, 96x96 render, 32 steps), B = 8, CUDA graph
    g_420_b1/b8    the sample app's 420-wide setting (MAP3DBN512L: 96x48 render, last_back, nerf_noise 0), B = 1 and B = 8, eager
    train_c2_b2    one train_step.Trainer iteration (D step + G step) at C2, B = 2
For each: median and range of the per-call time over --reps alternating runs of --iters calls (CUDA events), and the peak
device memory of one call (for the graphed forward the captured graph's pool is allocated before, so only its
outputs count).  Then the per-launch time of hg_sample_fine / hg_merge_samples from a separate torch.profiler run
of one hierarchical C2 forward.  The card's name and power limit are printed with the numbers.
    python tools/hierarchical_bench.py [--reps 5] [--iters 10] > hierarchical.json"""
import argparse
import copy
import importlib
import json
import os
import statistics
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
from spade_bench import card  # noqa: E402


def setup(pkg, which, B, train=False):
    gen = importlib.import_module("3dhumangan_b200.modules.generator")
    if which == "420":                        # the released checkpoint's curriculum as apps/sample_from_generator.py runs it
        cfg = pkg.configs.extract_metadata(copy.deepcopy(pkg.configs.MAP3DBN512L), 0)
        cfg["last_back"] = True
    else:
        cfg = pkg.configs.baseline_config(which)
    cfg["nerf_noise"] = 0.5 if train else 0.0
    torch.manual_seed(0)
    G = gen.Map3DGenerator(**cfg).cuda()
    G.set_device(torch.device("cuda:0"))
    G.train() if train else G.eval()
    z = torch.randn(B, cfg["latent_dim"], device="cuda")
    cond = {k: v.cuda() for k, v in pkg.synthetic.make_conditions(B, seed=1).items()}
    return G, cfg, z, cond


def forward_fn(pkg, which, B, graph):
    G, cfg, z, cond = setup(pkg, which, B)

    def make(hier):
        kw = dict(cfg, hierarchical_sample=hier, hg_cuda_graph=graph)
        return lambda: G(z, cond, **kw)
    return make


def train_fn(pkg, B):
    disc = importlib.import_module("3dhumangan_b200.modules.discriminator")
    ts = importlib.import_module("3dhumangan_b200.train_step")
    trainers = {}
    for hier in (False, True):
        G, cfg, _, cond = setup(pkg, "C2", B, train=True)
        cfg["hierarchical_sample"] = hier
        D = disc.UNetDiscriminator(**cfg).cuda().train()
        Hg, Wg = cfg["gen_height"], cfg["gen_width"]
        batch = dict(cond=cond, images=torch.randn(B, 3, Hg, Wg, device="cuda").clamp_(-1, 1),
                     labels=torch.randint(1, cfg["label_dim"], (B, Hg, Wg), device="cuda"))
        trainers[hier] = (ts.Trainer(G, D, cfg, amp=False, ddp=False), batch)

    def make(hier):
        t, batch = trainers[hier]
        return lambda: t.iteration(batch)
    return make


def timed(fn, n):
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(n):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / n


def peak(fn):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    fn()
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() / 2 ** 30


def compare(name, make, reps, iters, warmup=3):
    fns = {h: make(h) for h in (False, True)}
    for fn in fns.values():
        for _ in range(warmup):
            fn()
    ms = {False: [], True: []}
    for _ in range(reps):
        for h in (False, True):
            ms[h].append(timed(fns[h], iters))
    row = {"workload": name}
    for h, key in ((False, "off"), (True, "on")):
        row[key] = {"ms_median": round(statistics.median(ms[h]), 3), "ms_min": round(min(ms[h]), 3),
                    "ms_max": round(max(ms[h]), 3), "peak_gib": round(peak(fns[h]), 3)}
    row["ratio_on_off"] = round(row["on"]["ms_median"] / row["off"]["ms_median"], 3)
    print(json.dumps(row), flush=True)


def kernel_profile(pkg):
    from torch.profiler import ProfilerActivity, profile
    fn = forward_fn(pkg, "C2", 8, graph=False)(True)
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        for k in ("sample_fine_kernel", "merge_samples_kernel"):
            if k in e.key:
                total = getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0)
                out[k] = {"calls": e.count, "us_per_call": round(total / max(e.count, 1), 1)}
    print(json.dumps({"kernels_c2_b8": out}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--iters", type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("hierarchical_bench: needs a CUDA device")
    pkg = importlib.import_module("3dhumangan_b200")
    print(json.dumps({"card": card()}), flush=True)
    with torch.no_grad():
        compare("g_c2_graph_b8", forward_fn(pkg, "C2", 8, graph=True), args.reps, args.iters)
        compare("g_420_b1", forward_fn(pkg, "420", 1, graph=False), args.reps, args.iters)
        compare("g_420_b8", forward_fn(pkg, "420", 8, graph=False), args.reps, args.iters)
        kernel_profile(pkg)
    compare("train_c2_b2", train_fn(pkg, 2), args.reps, max(1, args.iters // 5))


if __name__ == "__main__":
    main()
