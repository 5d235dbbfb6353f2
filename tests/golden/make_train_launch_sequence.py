"""The train-mode launch schedule of the generator, recorded for tests/test_gpu_train_launch_sequence.py.

    python tests/golden/make_train_launch_sequence.py [out.json]      # needs an H100; default tests/golden/train_launch_sequence.json

For hidden_dim 256 and 420, with and without hierarchical_sample: one train() forward + backward of `Map3DGenerator` at a
tiny size with every parameter requiring grad, recording every `abi.call`: the entry point's name, its scalar arguments
(ints and floats) and which pointer arguments are NULL.  The committed fixture was recorded at the commit BEFORE eval-mode
gradients were added (when `hg_render_composite_bwd` had no `last_back` argument); the test replays the same recipe on
the current code and requires the same schedule, so that work on the eval / frozen paths cannot move the training path.
Stored as {"calls": [distinct call strings], "cases": {name: [indices into calls]}}."""
import ctypes
import importlib
import json
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
CASES = {"h256": (256, False), "h256_hier": (256, True), "h420": (420, False), "h420_hier": (420, True)}


def describe(name, args):
    parts = []
    for a in args:
        if a is None:
            parts.append("NULL")
        elif isinstance(a, bool):
            parts.append(str(int(a)))
        elif isinstance(a, int):
            parts.append(str(a))
        elif isinstance(a, float):
            parts.append(repr(a))
        elif isinstance(a, ctypes.c_void_p):
            parts.append("p" if a.value else "NULL")
        else:
            parts.append("p")
    return name + "(" + ",".join(parts) + ")"


def record_case(pkg, C, hier):
    """-> the list of call strings of one train-mode forward + backward."""
    abi = importlib.import_module("3dhumangan_b200.abi")
    gen = importlib.import_module("3dhumangan_b200.modules.generator")
    cfg = pkg.configs.baseline_config("tiny")
    cfg.update(hidden_dim=C, feature_dim=C, map3d_mode="isolated" if C == 420 else "mixed", legacy_mode=C == 420, gen_height=16,
               gen_width=16, render_height=4, render_width=4, num_steps=32, nerf_noise=0.5, hierarchical_sample=hier)
    torch.manual_seed(0)
    G = gen.Map3DGenerator(**cfg).cuda().train()
    G.set_device(torch.device("cuda:0"))
    cond = {k: v.cuda() for k, v in pkg.synthetic.make_conditions(2, seed=22).items()}
    z = torch.randn(2, cfg["latent_dim"], device="cuda")
    calls = []
    orig = abi.call

    def spy(name, *args, **kw):
        calls.append(describe(name, args))
        return orig(name, *args, **kw)

    abi.call = spy
    try:
        out = G(z, cond, **cfg)
        (out["rgbs"].square().sum() + out["rgbs_render"].square().sum()).backward()
        torch.cuda.synchronize()
    finally:
        abi.call = orig
    return calls


def main():
    sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
    pkg = importlib.import_module("3dhumangan_b200")
    distinct, cases = {}, {}
    for name, (C, hier) in CASES.items():
        cases[name] = [distinct.setdefault(c, len(distinct)) for c in record_case(pkg, C, hier)]
    out = sys.argv[1] if len(sys.argv) > 1 else os.path.join(HERE, "train_launch_sequence.json")
    with open(out, "w") as f:
        json.dump({"calls": list(distinct), "cases": cases}, f, separators=(",", ":"))
    print({k: len(v) for k, v in cases.items()}, len(distinct), "distinct calls")


if __name__ == "__main__":
    main()
