"""Pin the oracle's BACKWARD at the padded widths (384: MAP3DBN, 420: MAP3DBN512L) against gradient checksums of the
unmodified reference (tests/golden/make_golden_grads_wide.py).  The GPU tests (tests/test_gpu_train_wide.py) compare the
kernels with autograd through the oracle.

Bounds: every checksum within 1e-2 and the median within 1e-3 (test_oracle_pin.py holds every checksum to 2e-3 at 256).
Both sides are fp32 on the CPU, and at these widths fp32 rounding alone moves the gradients by more than 2e-3: the oracle
evaluated once in fp32 and once in fp64 (`generator_forward(dtype=torch.float64)`, mapping networks in fp32 as in the
reference), with the same inputs and draws, differs by more than 2e-3 on 11 % (384) / 19 % (420) of the parameters, by up
to 4.2e-3 / 6.0e-3.  Against the reference the oracle's fp32 checksums differ by a median of 2.5e-4 / 5.7e-4 and at most
2.4e-3 / 4.9e-3, i.e. within that rounding spread; the losses agree to 1e-4 relative.  (The reference itself cannot be run
in fp64 with the same random draws: it draws its jitter and noise in the default dtype.)"""
import pytest
import torch

from golden_util import generator_case, rel_l2
from test_oracle_pin import _check_grad_summary, _direction, _load_grads, _loss_weights

TOL = 1e-2            # per checksum: above the 6e-3 fp32 rounding spread
TOL_MEDIAN = 1e-3

# gradient fixture -> (forward fixture whose recipe it uses, config overrides)
CASES = {"g_h384_mixed": ("g_h384_mixed", {}),
         "g_h420_isolated_legacy_train": ("g_h420_isolated_legacy", dict(last_back=False))}


@pytest.mark.parametrize("name", sorted(CASES))
def test_generator_oracle_backward_matches_reference_gradients_wide(port, name):
    case, over = CASES[name]
    cfg, params, cond, z, (u, noise), _ = generator_case(case)
    cfg.update(over)
    gold = _load_grads(name)
    pc = {n: (v.clone().requires_grad_(True) if v.is_floating_point() else v.clone()) for n, v in params.items()}
    out = port.generator_forward(pc, z, cond, cfg, u, noise, training=True)
    loss = (out["rgbs"] * _loss_weights(out["rgbs"].shape, 1)).sum() + (out["rgbs_render"] * _loss_weights(out["rgbs_render"].shape, 2)).sum()
    assert abs(float(loss) - float(gold["loss"])) < 1e-3 * abs(float(gold["loss"])) + 1e-4
    loss.backward()
    grads = {n: v.grad for n, v in pc.items() if torch.is_tensor(v) and v.is_floating_point()}
    assert len(gold["names_list"]) > 200
    worst = _check_grad_summary(gold, grads, TOL)
    for k, v in gold.items():
        if k.startswith("full:"):
            assert rel_l2(grads[k[5:]], v) < TOL, k
    assert worst < TOL
    scale = float(gold["norms"].max())
    errs = []
    for i, n in enumerate(str(n) for n in gold["names_list"]):
        gn, gd = float(gold["norms"][i]), float(gold["dots"][i])
        if gn >= 1e-7 * scale:                     # analytic zeros are checked by _check_grad_summary
            g = grads[n].double()
            errs.append(max(abs(float(g.norm()) - gn), abs(float((g * _direction(n, g.shape).double()).sum()) - gd)) / gn)
    assert sorted(errs)[len(errs) // 2] < TOL_MEDIAN, sorted(errs)[len(errs) // 2]
