"""Eval-mode gradient fixture from the UNMODIFIED reference (build container only; see make_golden.py).

    python tests/golden/make_golden_eval_grads.py      # writes tests/golden/g_eval_grads.npz

The sample app's setting: `eval()`, `last_back=True`, `nerf_noise=0`.  For the forward cases `g_small_isolated_legacy`
(hidden 64) and `g_h420_isolated_legacy` (the released checkpoint's width): WARMUP train-mode forwards first, so that the
running statistics and the spectral-norm u / v are those of a trained module (at random initialisation the eval output is
~1e26, SURVEY.md 8c pitfall 1), then `eval()` and, under autograd with the forward fixtures' rng seed,
loss = sum(output * w) with the seeded weights of make_golden_grads.py.  Stored per case, under `<case>/`:
    loss, dz, dfreq, dphase                 the loss and its gradients w.r.t. the latent and the FiLM tables
    names, norms, dots, full:<name>         the parameter-gradient checksums of make_golden_grads.summarise
    buf:<name>                              every buffer after the warm-up = the state the eval pass starts from
    buffers_unchanged                       1 when the eval forward + backward left every buffer bit-identical
`tests/test_oracle_pin_eval_grads.py` checks eval-mode autograd through the oracle against them.
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

CASES = ("g_small_isolated_legacy", "g_h420_isolated_legacy")
SEED = 1234          # the forward fixtures' rng_seed (manifest.json)
WARMUP = 3           # train-mode forwards, seeds 500, 501, ...; latents seeded 600, 601, ...


def main():
    pkg = importlib.import_module("3dhumangan_b200")
    from oracle import port
    gens, _, impl = make_golden.reference_modules()
    out_all = {}
    for case in CASES:
        cfg, params, cond, z, B = make_golden.build_case(pkg, port, case)
        assert cfg["last_back"] and cfg["nerf_noise"] == 0.0
        meta = dict(cfg)
        meta["neural_field_cls"] = getattr(impl, meta["neural_field_cls"])
        G = gens.Map3DGenerator(**meta)
        G.load_state_dict(copy.deepcopy(params), strict=True)
        G.set_device("cpu")
        G.train()
        for i in range(WARMUP):
            torch.manual_seed(500 + i)
            with torch.no_grad():
                G(torch.randn(B, cfg["latent_dim"], generator=torch.Generator().manual_seed(600 + i)), cond, **meta)
        G.eval()
        bufs = {n: b.detach().clone() for n, b in G.named_buffers()}
        kept = {}

        def keep(module, inputs, output):          # (freq, phase): non-leaf, keep their gradients
            kept["freq"], kept["phase"] = output
            output[0].retain_grad()
            output[1].retain_grad()

        hook = G.neural_field_mapping_network.register_forward_hook(keep)
        zz = z.clone().requires_grad_(True)
        torch.manual_seed(SEED)
        out = G(zz, cond, **meta)
        hook.remove()
        loss = (out["rgbs"] * loss_weights(out["rgbs"].shape, 1)).sum() + \
            (out["rgbs_render"] * loss_weights(out["rgbs_render"].shape, 2)).sum()
        loss.backward()
        same = all(torch.equal(b, bufs[n]) for n, b in G.named_buffers())
        grads = {n: p.grad.detach().clone() for n, p in G.named_parameters() if p.grad is not None}
        rec = dict(loss=np.array(float(loss)), dz=zz.grad.numpy(), dfreq=kept["freq"].grad.numpy(), dphase=kept["phase"].grad.numpy(),
                   buffers_unchanged=np.array(int(same)), **summarise(grads, FULL_G))
        rec.update({"buf:" + n: b.numpy() for n, b in bufs.items()})
        out_all.update({f"{case}/{k}": v for k, v in rec.items()})
        print(case, "loss", float(loss), len(grads), "gradients; buffers unchanged:", same,
              "| rgbs abs max", float(out["rgbs"].abs().max()))
    np.savez_compressed(os.path.join(HERE, "g_eval_grads.npz"), **out_all)


if __name__ == "__main__":
    main()
