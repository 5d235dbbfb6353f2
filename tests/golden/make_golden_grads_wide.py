"""Gradient fixtures at the padded widths from the UNMODIFIED reference (build container only; see make_golden.py).

    python tests/golden/make_golden_grads_wide.py      # writes tests/golden/g_h384_mixed_grads.npz,
                                                       #        tests/golden/g_h420_isolated_legacy_train_grads.npz

Same recipe and format as make_golden_grads.py (`summarise`), for the forward fixtures `g_h384_mixed` (MAP3DBN's width) and
`g_h420_isolated_legacy` (MAP3DBN512L's width, isolated style, legacy feature order) -- the latter with last_back=False, the
training setting, instead of the sample app's last_back.  `tests/test_oracle_pin_wide.py` checks autograd through the oracle
against them.  No other fixture is written.
"""
import copy
import importlib
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, HERE)
sys.path.insert(0, ROOT)
import make_golden  # noqa: E402
from make_golden_grads import FULL_G, loss_weights, summarise  # noqa: E402

# fixture name -> (forward case of make_golden.CASES, config overrides)
CASES = {"g_h384_mixed": ("g_h384_mixed", {}),
         "g_h420_isolated_legacy_train": ("g_h420_isolated_legacy", dict(last_back=False))}
SEED = 1234          # the forward fixtures' rng_seed (manifest.json)


def main():
    pkg = importlib.import_module("3dhumangan_b200")
    from oracle import port
    gens, _, impl = make_golden.reference_modules()
    for name, (case, over) in CASES.items():
        cfg, params, cond, z, _ = make_golden.build_case(pkg, port, case)
        cfg.update(over)
        meta = dict(cfg)
        meta["neural_field_cls"] = getattr(impl, meta["neural_field_cls"])
        G = gens.Map3DGenerator(**meta)
        G.load_state_dict(copy.deepcopy(params), strict=True)
        G.set_device("cpu")
        G.train()
        torch.manual_seed(SEED)
        out = G(z, cond, **meta)
        loss = (out["rgbs"] * loss_weights(out["rgbs"].shape, 1)).sum() + \
            (out["rgbs_render"] * loss_weights(out["rgbs_render"].shape, 2)).sum()
        loss.backward()
        grads = {n: p.grad.detach().clone() for n, p in G.named_parameters() if p.grad is not None}
        np.savez_compressed(os.path.join(HERE, name + "_grads.npz"), loss=np.array(float(loss)), **summarise(grads, FULL_G))
        print(name, "loss", float(loss), len(grads), "gradients")


if __name__ == "__main__":
    main()
