"""Pin the oracle's EVAL-MODE backward -- running-statistics BatchNorm, spectral norm from the stored u / v,
`last_back=True`, `nerf_noise=0`: the sample app's setting -- against gradients of the unmodified reference
(tests/golden/make_golden_eval_grads.py): d loss / d latent, d freq, d phase in full, the parameter-gradient checksums,
and the buffers, which neither side may touch.  The GPU tests (tests/test_gpu_eval_backward.py) compare the kernels with
eval-mode autograd through the oracle."""
import os

import numpy as np
import pytest
import torch

from golden_util import GOLD, generator_case, rel_l2
from test_oracle_pin import _check_grad_summary, _loss_weights

TOL = {"g_small_isolated_legacy": 2e-3, "g_h420_isolated_legacy": 1e-2}      # the train-mode pins' bounds at these widths


def _gold(case):
    raw = np.load(os.path.join(GOLD, "g_eval_grads.npz"))
    out = {k[len(case) + 1:]: raw[k] for k in raw.files if k.startswith(case + "/")}
    names = [str(n) for n in out.pop("names")]
    out = {k: torch.from_numpy(v) for k, v in out.items()}
    out["names_list"] = names
    return out


@pytest.mark.parametrize("case", sorted(TOL))
def test_oracle_eval_backward_matches_reference(port, case):
    cfg, params, cond, z, (u, noise), _ = generator_case(case)
    assert cfg["last_back"] and cfg["nerf_noise"] == 0.0
    gold = _gold(case)
    assert int(gold["buffers_unchanged"]) == 1
    bufs = {k[4:]: v for k, v in gold.items() if k.startswith("buf:")}
    assert bufs and all(n in params for n in bufs)
    pc = {n: (v.clone().requires_grad_(True) if v.is_floating_point() and n not in bufs else bufs.get(n, v).clone())
          for n, v in params.items()}
    zz = z.clone().requires_grad_(True)
    # d freq, d phase: the same forward from FiLM tables cut off the mapping network
    z_field = zz if cfg.get("neural_field_latent_input", True) else torch.zeros_like(zz)
    freq, phase = (t.detach().requires_grad_(True) for t in port.mapping_network(pc, z_field))
    orig = port.mapping_network
    port.mapping_network = lambda *a, **k: (freq, phase)
    try:
        out_f = port.generator_forward(pc, zz, cond, cfg, u, noise, training=False)
    finally:
        port.mapping_network = orig
    stats = {}
    out = port.generator_forward(pc, zz, cond, cfg, u, noise, training=False, stats_out=stats)
    weigh = lambda o: (o["rgbs"] * _loss_weights(o["rgbs"].shape, 1)).sum() + (o["rgbs_render"] * _loss_weights(o["rgbs_render"].shape, 2)).sum()
    loss = weigh(out)
    assert abs(float(loss) - float(gold["loss"])) < 1e-3 * abs(float(gold["loss"])) + 1e-4
    dfreq, dphase = torch.autograd.grad(weigh(out_f), [freq, phase])
    loss.backward()
    tol = TOL[case]
    assert rel_l2(zz.grad, gold["dz"]) < tol
    assert rel_l2(dfreq, gold["dfreq"]) < tol
    assert rel_l2(dphase, gold["dphase"]) < tol
    grads = {n: v.grad for n, v in pc.items() if torch.is_tensor(v) and v.is_floating_point() and v.requires_grad}
    assert len(gold["names_list"]) > 200
    assert _check_grad_summary(gold, grads, tol) < tol
    for k, v in gold.items():
        if k.startswith("full:"):
            assert rel_l2(grads[k[5:]], v) < tol, k
    # eval mode reads the buffers and returns them as they are
    for n, v in stats.items():
        assert torch.equal(v.detach(), bufs[n]), n
    for n, v in bufs.items():
        assert torch.equal(pc[n], v), n
