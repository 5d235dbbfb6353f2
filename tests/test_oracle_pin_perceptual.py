"""The fp64 perceptual-loss oracle (oracle/perceptual_port.py) against the reference's own VGGPerceptualLoss
(tests/golden/perceptual.npz, made by tests/golden/make_golden_perceptual.py with seeded weights).  CPU only."""
import json
import os

import numpy as np
import pytest
import torch

from oracle import perceptual_port as pp

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "perceptual.npz")
CASES = {"rgb64x32": True, "rgb60x44_noresize": False, "gray48": True}


@pytest.mark.parametrize("name", list(CASES))
def test_oracle_matches_reference_fixture(name):
    gold = np.load(GOLD)
    params = pp.module_params(pp.seeded_vgg16_state(0))
    x = torch.from_numpy(gold[f"{name}_input"]).double().requires_grad_(True)
    t = torch.from_numpy(gold[f"{name}_target"])
    losses = pp.losses(params, x, t, CASES[name])
    sum(losses).backward()
    want = gold[f"{name}_losses"]
    got = np.array([float(v.detach()) for v in losses])
    assert np.all(np.abs(got - want) <= 2e-5 * np.abs(want)), (got, want)
    # the reference ran in fp32: a few dozen pre-activations per layer lie within 1e-6 of zero at 224x224, and the ReLU masks
    # that flip between fp32 and fp64 bound the gradient's agreement (measured 7.5e-4 / 4.9e-4 with the resize, 2e-6 without)
    g, gw = x.grad.numpy(), gold[f"{name}_grad"].astype(np.float64)
    assert np.linalg.norm(g - gw) <= (1.5e-3 if CASES[name] else 1e-5) * np.linalg.norm(gw)
    with torch.no_grad():
        norms = [float(f.norm()) for f in pp.features(params, x, CASES[name])]
    assert np.allclose(norms, gold[f"{name}_feature_norms"], rtol=1e-5, atol=0)


def test_state_dict_keys_match_reference():
    mod = __import__("importlib").import_module("3dhumangan_b200.perceptual")
    gold = json.loads(str(np.load(GOLD)["state_dict_keys"]))
    m = mod.VGGPerceptualLoss(weights=pp.seeded_vgg16_state(0))
    assert [[k, list(v.shape)] for k, v in m.state_dict().items()] == gold
    assert [k for k, _ in gold if k.endswith(".weight")] == [f"blocks.{l}.{i}.weight" for l, idxs in enumerate(pp.BLOCKS) for i in idxs]
    # the module's own load_state_dict takes the reference's keys and gives the same weights as the torchvision loader
    ref = pp.module_params(pp.seeded_vgg16_state(0))
    assert all(torch.equal(m.state_dict()[k], v) for k, v in ref.items())
    m2 = mod.VGGPerceptualLoss(weights=pp.seeded_vgg16_state(1))
    m2.load_state_dict(m.state_dict(), strict=True)
    assert all(torch.equal(a, b) for a, b in zip(m2.state_dict().values(), m.state_dict().values()))
    assert not any(p.requires_grad for p in m.parameters())
