"""Cost of one latent-inversion step at the sample app's setting (420 wide, 512x256 from a 96x48 render of 32 steps,
last_back, B = 1): forward through `Map3DGenerator.synthesize` in eval mode, `image_loss`, backward to freq / phase / style.
    frozen / unfrozen     every parameter frozen (no weight-gradient kernel) vs every parameter requiring grad
    records reuse / off   `hg_records` of the first render re-used vs ray sampling + nearest vertex + features every step
    hierarchical          hierarchical_sample on (2 x 32 samples per ray; its records cannot be re-used) vs off
For each variant: median and range of the per-step time over --reps rounds of --iters steps (CUDA events), the variants
alternating within a round, and the peak device memory of one step.  The card's name and power limit are printed with
the numbers.
    python tools/inversion_bench.py [--reps 5] [--iters 10] > inversion.json"""
import argparse
import importlib
import json
import os
import statistics
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
from hierarchical_bench import peak, timed  # noqa: E402
from invert import released_like  # noqa: E402
from spade_bench import card  # noqa: E402

VARIANTS = {            # name: (frozen, records re-used, hierarchical)
    "frozen_reuse": (True, True, False),
    "frozen": (True, False, False),
    "unfrozen_reuse": (False, True, False),
    "unfrozen": (False, False, False),
    "frozen_hierarchical": (True, False, True),
    "unfrozen_hierarchical": (False, False, True),
}


def step_fn(pkg, G, cfg, cond, target, frozen, reuse, hier):
    ops = importlib.import_module("3dhumangan_b200.ops.trainer_ops")
    kw = dict(cfg, hierarchical_sample=hier)
    z = torch.randn(1, cfg["latent_dim"], device="cuda")
    with torch.no_grad():
        freq, phase = G.neural_field_mapping_network(torch.zeros_like(z))
        styles = G.synthesis_mapping_network(z)[1]
    var = [t.clone().requires_grad_(True) for t in (freq, phase, styles)]
    state = {"records": None}

    def step():
        extra = {"hg_records": state["records"]} if reuse and state["records"] is not None else {}
        out = G.synthesize(*var, cond, **dict(kw, **extra))
        state["records"] = out["hg_records"]
        ops.image_loss(out["rgbs"], target).backward()
        for v in var:
            v.grad = None

    def freeze():           # before a run of steps, outside the timed region
        for p in G.parameters():
            p.requires_grad_(not frozen)
    return freeze, step


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("inversion_bench: needs a CUDA device")
    pkg = importlib.import_module("3dhumangan_b200")
    print(json.dumps({"card": card()}), flush=True)
    G, cfg, cond = released_like(pkg, "420")
    with torch.no_grad():
        target = G(torch.randn(1, cfg["latent_dim"], device="cuda"), cond, **cfg)["rgbs"]
    fns = {name: step_fn(pkg, G, cfg, cond, target, *v) for name, v in VARIANTS.items()}
    def run(name, call):
        freeze, step = fns[name]
        freeze()
        value = call(step)
        for p in G.parameters():      # the unfrozen variants leave parameter gradients behind
            p.grad = None
        return value

    for name in fns:
        run(name, lambda step: [step() for _ in range(args.warmup)])
    ms = {name: [] for name in fns}
    for _ in range(args.reps):
        for name in fns:
            ms[name].append(run(name, lambda step: timed(step, args.iters)))
    for name in fns:
        fn = lambda: run(name, lambda step: step())
        print(json.dumps({"variant": name, "ms_median": round(statistics.median(ms[name]), 2), "ms_min": round(min(ms[name]), 2),
                          "ms_max": round(max(ms[name]), 2), "peak_gib": round(peak(fn), 3)}), flush=True)


if __name__ == "__main__":
    main()
