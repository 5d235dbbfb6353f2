"""CPU checks of perceptual path length (3dhumangan_b200/ppl.py) and its oracle (oracle/ppl_port.py): the fp64 LPIPS oracle
against a direct restatement on torchvision's VGG16 with nn.Conv2d lin layers, slerp against its formula, the pair draws,
the percentile filter against numpy with ties, the lin weights' names, shapes and loading, the batch -> rank -> seed
assignment, the refusals that need no device, and tools/evaluate.py's `ppl` parsing."""
import importlib
import math
import os
import sys

import numpy as np
import pytest
import torch

from oracle import metrics_port as mp
from oracle import ppl_port as plp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _ppl():
    return importlib.import_module("3dhumangan_b200.ppl")


# ------------------------------------------------------------------------------------------------------------------ LPIPS
def _lpips_restated(vgg_state, lin_state, a, b):
    """The lpips package's forward for net='vgg', version='0.1', restated on torchvision modules in fp64."""
    import torchvision
    net = torchvision.models.vgg16()
    net.load_state_dict(vgg_state)
    feats = net.features.double().eval()
    slices = [feats[0:4], feats[4:9], feats[9:16], feats[16:23], feats[23:30]]
    lins = []
    for k, C in enumerate(plp.LIN_CHANNELS):
        conv = torch.nn.Conv2d(C, 1, 1, stride=1, padding=0, bias=False).double()
        conv.weight.data.copy_(lin_state[f"lin{k}.model.1.weight"])
        lins.append(conv)
    shift = torch.tensor([-.030, -.088, -.188], dtype=torch.float64)[None, :, None, None]
    scale = torch.tensor([.458, .448, .450], dtype=torch.float64)[None, :, None, None]
    norm = lambda f: f / (torch.sqrt(torch.sum(f ** 2, dim=1, keepdim=True)) + 1e-10)
    ha, hb = (a.double() - shift) / scale, (b.double() - shift) / scale
    val = 0
    for s, lin in zip(slices, lins):
        ha, hb = s(ha), s(hb)
        val = val + lin((norm(ha) - norm(hb)) ** 2).mean([2, 3], keepdim=True)
    return val.reshape(-1)


@pytest.mark.parametrize("H,W", [(32, 32), (48, 80)])
def test_lpips_oracle_equals_the_lpips_definition_on_torchvision(H, W):
    vgg_state, lin_state = mp.seeded_vgg16_state(0), plp.seeded_lin_state(0)
    g = torch.Generator().manual_seed(H + W)
    a = torch.rand(3, 3, H, W, generator=g, dtype=torch.float64) * 2 - 1
    b = (a + 0.1 * torch.randn(3, 3, H, W, generator=g, dtype=torch.float64)).clamp(-1, 1)
    with torch.no_grad():
        got = plp.lpips(vgg_state, lin_state, a, b)
        want = _lpips_restated(vgg_state, lin_state, a, b)
        same = plp.lpips(vgg_state, lin_state, a, a.clone())
    print(f"{H}x{W}: LPIPS {got.tolist()}")
    assert got.shape == (3,) and (got > 0).all()
    assert torch.allclose(got, want, rtol=1e-12, atol=0)
    assert torch.equal(same, torch.zeros(3, dtype=torch.float64))


def test_input_stage_oracle_is_the_box_mean_then_the_scaling():
    x = torch.rand(2, 3, 8, 12, generator=torch.Generator().manual_seed(1), dtype=torch.float64) * 2 - 1
    got = plp.input_stage(x, 4)
    box = torch.nn.functional.avg_pool2d(x, 4)
    want = (box - torch.tensor(plp.SHIFT, dtype=torch.float64).view(1, 3, 1, 1)) / torch.tensor(plp.SCALE, dtype=torch.float64).view(1, 3, 1, 1)
    assert torch.allclose(got, want, rtol=1e-14, atol=1e-14)
    # the scaling is ImageNet's mean / std applied to (x + 1) / 2, to the three digits LPIPS states
    mean, std = np.array([0.485, 0.456, 0.406]), np.array([0.229, 0.224, 0.225])
    assert np.allclose(2 * mean - 1, plp.SHIFT, atol=1e-3) and np.allclose(2 * std, plp.SCALE, atol=1e-3)
    assert _ppl().SHIFT == plp.SHIFT and _ppl().SCALE == plp.SCALE


# ------------------------------------------------------------------------------------------------------------ sampling
def test_slerp_against_its_formula():
    ppl = _ppl()
    g = torch.Generator().manual_seed(0)
    a = torch.randn(5, 512, generator=g, dtype=torch.float64)
    b = torch.randn(5, 512, generator=g, dtype=torch.float64)
    t = torch.rand(5, 1, generator=g, dtype=torch.float64)
    got = ppl.slerp(a, b, t)
    an, bn = a / a.norm(dim=1, keepdim=True), b / b.norm(dim=1, keepdim=True)
    for i in range(5):
        om = math.acos(float(an[i] @ bn[i]))
        tt = float(t[i])
        # the textbook form: sin((1 - t) om) / sin om a + sin(t om) / sin om b
        want = math.sin((1 - tt) * om) / math.sin(om) * an[i] + math.sin(tt * om) / math.sin(om) * bn[i]
        assert torch.allclose(got[i], want, rtol=0, atol=1e-12)
    assert torch.allclose(got.norm(dim=1), torch.ones(5, dtype=torch.float64), rtol=0, atol=1e-14)
    assert torch.allclose(ppl.slerp(a, b, torch.zeros(5, 1, dtype=torch.float64)), an, rtol=0, atol=1e-14)
    assert torch.allclose(ppl.slerp(a, b, torch.ones(5, 1, dtype=torch.float64)), bn, rtol=0, atol=1e-12)
    assert torch.equal(got, plp.slerp(a, b, t))


def test_pair_draws_depend_on_seed_and_index_alone():
    ppl = _ppl()
    z0, z1, t = ppl.pair_draws(3, 7, 16, "end")
    assert t == 0.0 and z0.shape == z1.shape == (16,) and not torch.equal(z0, z1)
    f0, f1, tf = ppl.pair_draws(3, 7, 16, "full")
    assert torch.equal(z0, f0) and torch.equal(z1, f1) and 0.0 <= tf < 1.0
    again = ppl.pair_draws(3, 7, 16, "full")
    assert torch.equal(again[0], f0) and again[2] == tf
    assert ppl.pair_draws(3, 8, 16, "full")[2] != tf and not torch.equal(ppl.pair_draws(4, 7, 16, "end")[0], z0)
    # the draws ignore the global RNG
    torch.manual_seed(123)
    assert torch.equal(ppl.pair_draws(3, 7, 16, "end")[0], z0)


def test_batches_ranks_and_jitter_seeds():
    ppl = _ppl()
    one = ppl.batches(10, 4)
    assert one == [(0, [0, 1, 2, 3]), (1, [4, 5, 6, 7]), (2, [8, 9])]
    two = [ppl.batches(10, 4, r, 2) for r in range(2)]
    assert two == [[(0, [0, 1, 2, 3]), (2, [8, 9])], [(1, [4, 5, 6, 7])]]
    three = [ppl.batches(10, 4, r, 3) for r in range(3)]
    assert sorted(b for r in three for b in r) == one
    assert ppl.batches(10, 4, 3, 4) == []
    # a batch's jitter seed depends on (seed, k) alone, so the ranks render what one rank would
    seeds = {ppl.jitter_seed(s, k) for s in range(3) for k in range(50)}
    assert len(seeds) == 150
    assert ppl.jitter_seed(2, 5) == (2 << 32) + 5


@pytest.mark.parametrize("dist", [np.arange(200.0)[::-1], np.r_[np.zeros(5), np.ones(190), np.full(5, 9.0)],
                                  np.exp(np.random.default_rng(0).normal(size=1001)), np.array([3.0, 1.0]),
                                  np.r_[np.full(3, 2.0), np.arange(97.0)]])
def test_filtered_mean_against_numpy_with_ties(dist):
    ppl = _ppl()
    lo, hi, mean = ppl.filtered_mean(dist)
    assert lo == np.percentile(dist, 1, method="lower") and hi == np.percentile(dist, 99, method="higher")
    assert lo in dist and hi in dist
    keep = dist[(dist >= lo) & (dist <= hi)]
    assert mean == pytest.approx(keep.mean(), rel=1e-15)
    assert (lo, hi) == plp.filtered_mean(dist)[:2]
    assert (dist == lo).sum() <= (keep == lo).sum() and (dist == hi).sum() <= (keep == hi).sum()     # ties at lo / hi stay


# ------------------------------------------------------------------------------------------------------------ lin weights
def test_lin_state_names_shapes_and_loading(tmp_path):
    ppl = _ppl()
    state = plp.seeded_lin_state(0)
    assert sorted(state) == [f"lin{k}.model.1.weight" for k in range(5)]
    assert [tuple(state[f"lin{k}.model.1.weight"].shape) for k in range(5)] == [(1, C, 1, 1) for C in (64, 128, 256, 512, 512)]
    got = ppl.load_lin(state)
    assert all(torch.equal(got[k], state[k]) for k in state)
    path = tmp_path / "vgg.pth"
    torch.save(state, str(path))
    assert torch.equal(ppl.load_lin(str(path))["lin3.model.1.weight"], state["lin3.model.1.weight"])
    missing = tmp_path / "nothere" / "vgg.pth"
    with pytest.raises(RuntimeError, match=str(missing).replace(".", r"\.")):
        ppl.load_lin(str(missing))
    bad = dict(state)
    del bad["lin4.model.1.weight"]
    with pytest.raises(RuntimeError, match="lin4"):
        ppl.load_lin(bad)
    bad = dict(state, **{"lin1.model.1.weight": torch.rand(1, 64, 1, 1)})
    with pytest.raises(RuntimeError, match="shape"):
        ppl.load_lin(bad)
    bad = dict(state, **{"lin0.model.1.weight": -state["lin0.model.1.weight"]})
    with pytest.raises(RuntimeError, match="negative"):
        ppl.load_lin(bad)
    assert ppl.default_lin_path() == os.path.join(torch.hub.get_dir(), "checkpoints", "lpips_vgg_v0.1.pth")


def test_lpips_module_names():
    ppl, metrics = _ppl(), importlib.import_module("3dhumangan_b200.metrics")
    net = ppl.LPIPS(vgg=metrics.VGG16Features(weights=mp.seeded_vgg16_state(0)), lin=plp.seeded_lin_state(0))
    keys = set(net.state_dict())
    assert {k for k in keys if k.startswith("lin")} == {f"lin{k}.model.1.weight" for k in range(5)}
    assert torch.equal(net.state_dict()["lin2.model.1.weight"], plp.seeded_lin_state(0)["lin2.model.1.weight"])
    assert "vgg.features.28.weight" in keys


def test_refusals_without_a_device():
    ppl = _ppl()
    cfg = {"latent_dim": 8}
    for kw, match in ((dict(space="x"), "space"), (dict(sampling="mid"), "sampling"), (dict(epsilon=0.0), "epsilon"),
                      (dict(epsilon=-1e-4), "epsilon"), (dict(num_samples=1), "num_samples")):
        args = dict(num_samples=4, batch_size=2)
        args.update(kw)
        with pytest.raises(ValueError, match=match):
            ppl.path_length(None, cfg, **args)
    with pytest.raises(RuntimeError, match="fp32x3"):
        ppl.path_length(None, dict(cfg, hg_precision="bf16"), 4, 2)
    with pytest.raises(ValueError, match="epsilon"):
        ppl.pair_images(None, cfg, [0], epsilon=-1.0)
    assert ppl.downsample_factor(256) == 1 and ppl.downsample_factor(512) == 2 and ppl.downsample_factor(1024) == 4
    assert ppl.downsample_factor(64) == 1


# ---------------------------------------------------------------------------------------------------- tools/evaluate.py
def test_evaluate_ppl_parsing():
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    try:
        ev = importlib.import_module("evaluate")
    finally:
        sys.path.pop(0)
    a = ev.parser().parse_args(["ppl", "--config", "tiny"])
    assert (a.cmd, a.config, a.checkpoint, a.num, a.batch, a.seed, a.space, a.sampling, a.epsilon, a.truncation, a.vgg,
            a.lpips) == ("ppl", "tiny", None, 50000, 8, 0, "w", "end", 1e-4, 1.0, None, None)
    a = ev.parser().parse_args(["ppl", "--num", "100", "--batch", "4", "--seed", "2", "--space", "z", "--sampling", "full",
                                "--epsilon", "2e-4", "--truncation", "0.7", "--vgg", "v.pth", "--lpips", "l.pth",
                                "--checkpoint", "g.pth"])
    assert (a.config, a.num, a.batch, a.seed, a.space, a.sampling, a.epsilon, a.truncation, a.vgg, a.lpips, a.checkpoint) == \
        ("420", 100, 4, 2, "z", "full", 2e-4, 0.7, "v.pth", "l.pth", "g.pth")
    for bad in (["ppl", "--space", "q"], ["ppl", "--sampling", "mid"], ["ppl", "--config", "99"]):
        with pytest.raises(SystemExit):
            ev.parser().parse_args(bad)
