"""hierarchical_sample=True on the CPU: the oracle against the unmodified reference's render (fixture from
tests/golden/make_golden_hierarchical.py, draws replayed by `rng.draw_hierarchical_noise`, which pins the draw order),
and the argument checks of the two sampling entry points, which run before any device work."""
import ctypes
import importlib
import json
import os
import sys

import numpy as np
import pytest
import torch

from golden_util import GOLD, rel_l2

sys.path.insert(0, os.path.join(GOLD))
from make_golden_hierarchical import build_case  # noqa: E402

import hierarchical_oracle  # noqa: E402

FIXTURE = os.path.join(GOLD, "g_hierarchical.npz")


def _recipe():
    return json.loads(str(np.load(FIXTURE)["recipe"]))


def hierarchical_case(name, device="cpu"):
    """-> cfg, params, cond, z, (u, HierarchicalNoise), golden outputs of one fixture case."""
    pkg = importlib.import_module("3dhumangan_b200")
    from oracle import port
    cfg, params, cond, z = build_case(pkg, port, name)
    B, R, S = z.shape[0], cfg["render_width"] * cfg["render_height"], cfg["num_steps"]
    torch.manual_seed(_recipe()["seed"])
    u, noise = pkg.rng.draw_hierarchical_noise(B, R, S, device, cfg["sample_dist"])
    raw = np.load(FIXTURE)
    gold = {k.split(".", 1)[1]: torch.from_numpy(raw[k]) for k in raw.files if k.startswith(name + ".")}
    return cfg, params, cond, z, (u, noise), gold


CASES = sorted(_recipe()["cases"])


@pytest.mark.parametrize("name", CASES)
def test_oracle_matches_reference(port, name):
    cfg, params, cond, z, (u, noise), gold = hierarchical_case(name)
    with torch.no_grad():
        freq, phase = port.mapping_network(params, z)
        rgb, fmap, depth, w, idx, fz = hierarchical_oracle.render(params, freq, phase, cond, cfg, u, noise)
    assert rel_l2(rgb, gold["rgb_render"]) < 1e-5
    assert rel_l2(fmap, gold["feature_maps"]) < 1e-5
    assert rel_l2(depth, gold["depth"]) < 1e-5
    assert rel_l2(w, gold["weights"]) < 1e-5


def test_draw_order(pkg):
    # jitter, two camera draws, coarse noise, u_pdf, final noise: the one-pass draws are a prefix
    torch.manual_seed(5)
    u, n = pkg.rng.draw_hierarchical_noise(2, 3, 4, "cpu", "gaussian")
    torch.manual_seed(5)
    u1, n1 = pkg.rng.draw_render_noise(2, 3, 4, "cpu", "gaussian")
    u_pdf, final = torch.rand(6, 4), torch.randn(2, 3, 8, 1)
    assert torch.equal(u, u1) and torch.equal(n.coarse, n1)
    assert torch.equal(n.u_pdf, u_pdf) and torch.equal(n.final, final)
    cfg = dict(hierarchical_sample=False, sample_dist="gaussian")
    torch.manual_seed(5)
    a = pkg.rng.draw(2, 3, 4, "cpu", cfg)
    assert torch.equal(a[0], u1) and torch.equal(a[1], n1)


def test_sample_pdf_uniform_and_degenerate_bins():
    bins = torch.tensor([[0.0, 1.0, 2.0, 3.0]])
    u = torch.tensor([[0.0, 0.5, 1.0 / 3, 0.999]])
    s = hierarchical_oracle.sample_pdf(bins, torch.ones(1, 3), u)
    assert torch.allclose(s, torch.tensor([[0.0, 1.5, 1.0, 2.997]]), atol=1e-5)
    # a zero-width cdf bin is never chosen for u strictly inside a non-empty one
    s = hierarchical_oracle.sample_pdf(bins, torch.tensor([[1.0, 0.0, 1.0]]) * 1e6, torch.tensor([[0.25, 0.75]]))
    assert s[0, 0] < 1.0 and s[0, 1] > 2.0


@pytest.fixture(scope="module")
def lib():
    return importlib.import_module("3dhumangan_b200.abi").lib()


def _fine_args(**over):
    p = ctypes.c_void_p(16)
    a = dict(sigma=p, sigma_stride=1, z=p, noise=None, u_pdf=p, noise_std=0.0, softplus=0, xs=p, ys=p, focals=p, c2w=p, B=1, Rw=2,
             Rh=2, S=32, fz=p, pts=p, stream=None)
    a.update(over)
    return list(a.values())


@pytest.mark.parametrize("over, msg", [
    (dict(sigma=None), "null pointer"),
    (dict(u_pdf=None), "null pointer"),
    (dict(c2w=None), "null pointer"),
    (dict(S=2), "num_steps"),
    (dict(S=65), "num_steps"),
    (dict(B=0), "bad shape"),
    (dict(sigma_stride=0), "sigma_stride"),
    (dict(softplus=2), "clamp_softplus"),
])
def test_sample_fine_rejects_bad_arguments(lib, over, msg):
    assert lib.hg_sample_fine(*_fine_args(**over)) == 1
    assert msg in lib.hg_last_error().decode()


def test_merge_samples_rejects_bad_arguments(lib):
    p, odd = ctypes.c_void_p(16), ctypes.c_void_p(20)
    assert lib.hg_merge_samples(p, p, p, p, 1, 4, 65, p, p, None, None) == 1
    assert "samples per ray" in lib.hg_last_error().decode()
    assert lib.hg_merge_samples(p, p, odd, p, 1, 4, 32, p, p, None, None) == 1
    assert "16-byte aligned" in lib.hg_last_error().decode()
    assert lib.hg_merge_samples(None, p, p, p, 1, 4, 32, p, p, None, None) == 1


def test_steps_must_double_to_a_power_of_two(pkg):
    hier = importlib.import_module("3dhumangan_b200.modules.hierarchical")
    with pytest.raises(RuntimeError, match="power of two"):
        hier.check_steps(dict(num_steps=24, lock_view_dependence=True))
    with pytest.raises(RuntimeError, match="lock_view_dependence=False"):
        hier.check_steps(dict(num_steps=32, lock_view_dependence=False))
    assert hier.check_steps(dict(num_steps=32, lock_view_dependence=True)) == 32
