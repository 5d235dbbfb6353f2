"""CPU checks of the metrics (3dhumangan_b200/metrics.py) and their oracle (oracle/metrics_port.py): KID's formula against a
brute-force double loop and its subset draw, k-NN radii against scikit-learn and the coverage edge cases, the VGG16 fc7 oracle
against torchvision, the module's names and weight loading, argument refusals, and tools/evaluate.py's parsing and .npz round
trip."""
import importlib
import os
import sys

import numpy as np
import pytest
import torch

from oracle import metrics_port as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _metrics():
    return importlib.import_module("3dhumangan_b200.metrics")


def _feats(n, D, seed, shift=0.0):
    return torch.rand(n, D, generator=torch.Generator().manual_seed(seed), dtype=torch.float64) + shift


# ------------------------------------------------------------------------------------------------------------------ KID
@pytest.mark.parametrize("m,D", [(2, 3), (3, 5), (7, 16)])
def test_kid_oracle_equals_brute_force(m, D):
    g, r = _feats(11, D, 1), _feats(9, D, 2, 0.1)
    ig, ir = mp.kid_indices(11, 9, 4, m, seed=5)
    assert ig.shape == ir.shape == (4, m)
    a = mp.kid_terms(g, r, ig, ir)
    b = mp.kid_brute(g.numpy(), r.numpy(), ig, ir)
    assert np.allclose(a, b, rtol=1e-12, atol=1e-13 * np.abs(b).max())


def test_kid_oracle_near_zero_for_one_distribution_and_positive_when_shifted():
    g, r = _feats(400, 8, 3), _feats(400, 8, 4)
    ig, ir = mp.kid_indices(400, 400, 10, 200, seed=0)
    same = mp.kid_terms(g, r, ig, ir)
    shifted = mp.kid_terms(g + 0.5, r, ig, ir)
    kmean = float(((g @ r.T / 8 + 1) ** 3).mean())
    assert abs(same.mean()) < 1e-2 * kmean
    assert (shifted > 0).all() and shifted.mean() > 100 * abs(same.mean())


def test_kid_subset_draw_is_the_oracle_draw_and_reproducible():
    metrics = _metrics()
    ig, ir = metrics.kid_subsets(50, 40, num_subsets=6, max_subset_size=30, seed=7)
    og, orr = mp.kid_indices(50, 40, 6, 30, 7)
    assert np.array_equal(ig, og) and np.array_equal(ir, orr)
    ig2, ir2 = metrics.kid_subsets(50, 40, num_subsets=6, max_subset_size=30, seed=7)
    assert np.array_equal(ig, ig2) and np.array_equal(ir, ir2)
    ig3, _ = metrics.kid_subsets(50, 40, num_subsets=6, max_subset_size=30, seed=8)
    assert not np.array_equal(ig, ig3)
    for s in range(6):
        assert len(set(ig[s].tolist())) == 30 and len(set(ir[s].tolist())) == 30
        assert ig[s].max() < 50 and ir[s].max() < 40
    assert ig.dtype == np.int64


@pytest.mark.parametrize("n_gen,n_real,cap,m", [(50, 40, 1000, 40), (30, 40, 1000, 30), (50, 40, 25, 25), (2, 9, 1000, 2)])
def test_kid_subset_size_follows_the_min_rule(n_gen, n_real, cap, m):
    ig, ir = _metrics().kid_subsets(n_gen, n_real, 3, cap)
    assert ig.shape == ir.shape == (3, m)


def test_kid_refusals():
    metrics = _metrics()
    with pytest.raises(ValueError, match="below 2"):
        metrics.kid_subsets(1, 10, 3, 1000)
    with pytest.raises(ValueError, match="below 2"):
        metrics.kid_subsets(10, 10, 3, 1)
    for bad in (0, -1, 2.5, True):
        with pytest.raises(ValueError, match="num_subsets"):
            metrics.kid_subsets(10, 10, bad, 5)
    with pytest.raises(RuntimeError, match="differ in D"):
        metrics.kid(torch.rand(5, 3), torch.rand(5, 4))
    with pytest.raises(ValueError, match="below 2"):
        metrics.kid(torch.rand(1, 3), torch.rand(5, 3))
    with pytest.raises(RuntimeError, match="CUDA"):
        metrics.kid(torch.rand(5, 3), torch.rand(5, 3))


# ------------------------------------------------------------------------------------------------------- precision / recall
@pytest.mark.parametrize("k", range(1, 9))
def test_oracle_radii_equal_sklearn(k):
    from sklearn.neighbors import NearestNeighbors
    x = _feats(60, 7, k)
    x[5] = x[17]                          # a duplicate pair: each is the other's nearest neighbour at distance 0
    x[30] = x[17]
    got = mp.knn_radii(x, k).numpy()
    # the query set is the fitted set: sklearn returns each row itself first (its own index among zero-distance ties may be
    # any of them, so drop one zero-distance entry rather than the entry with the row's index)
    d, _ = NearestNeighbors(n_neighbors=k + 1).fit(x.numpy()).kneighbors(x.numpy())
    ref = d[:, k] ** 2
    assert np.allclose(got, ref, rtol=1e-12, atol=1e-14)
    assert got[5] == got[17] == got[30] and (k > 2 or got[17] == 0)


def test_coverage_edge_cases():
    x = _feats(40, 5, 1)
    assert mp.precision_recall(x, x.clone(), 3) == (1.0, 1.0)
    far = _feats(30, 5, 2, 100.0)
    assert mp.precision_recall(x, far, 3) == (0.0, 0.0)
    # unequal sizes: a gen set that is half of the real set plus far points
    g = torch.cat([x[:20], _feats(10, 5, 3, 100.0)])
    p, r = mp.precision_recall(x, g, 3)
    assert p == 20 / 30 and 0 < r <= 1
    with_dups = torch.cat([x[:10], x[:10]])
    rho = mp.knn_radii(with_dups, 1)
    assert (rho == 0).all()


def test_precision_recall_refusals():
    metrics = _metrics()
    a, b = torch.rand(5, 3), torch.rand(4, 3)
    for bad in (0, 9, 2.0, True):
        with pytest.raises(ValueError, match="k must be"):
            metrics.precision_recall(a, b, bad)
    with pytest.raises(ValueError, match="more than k"):
        metrics.precision_recall(a, b, 4)
    with pytest.raises(ValueError, match="more than k"):
        metrics.precision_recall(b, a, 4)
    with pytest.raises(RuntimeError, match="differ in D"):
        metrics.precision_recall(torch.rand(5, 3), torch.rand(5, 4))
    with pytest.raises(RuntimeError, match="CUDA"):
        metrics.precision_recall(a, b, 3)


# ------------------------------------------------------------------------------------------------------------- VGG16
@pytest.fixture(scope="module")
def vgg_state():
    return mp.seeded_vgg16_state(0)


def test_vgg16_oracle_equals_torchvision(vgg_state):
    import torchvision
    ref = torchvision.models.vgg16()
    ref.load_state_dict(vgg_state)
    ref = ref.double().eval()
    x = torch.rand(2, 3, 96, 80, generator=torch.Generator().manual_seed(1), dtype=torch.float64)
    with torch.no_grad():
        got = mp.vgg16_fc7(vgg_state, x)
        h = ref.avgpool(ref.features(mp.pp.transform(x, resize=True))).flatten(1)
        want = ref.classifier[:5](h)          # fc6, ReLU, dropout, fc7, ReLU
    assert got.shape == (2, 4096)
    assert float((got - want).abs().max() / want.abs().max()) < 1e-12
    # the seeded fan-in scaling keeps fc7 alive and bounded
    assert 0.2 < float((got > 0).double().mean()) < 0.8 and 1e-2 < float(got.abs().max()) < 1e3


def test_vgg16_module_names_and_loading(vgg_state, tmp_path):
    metrics = _metrics()
    net = metrics.VGG16Features(weights=vgg_state)
    keys = set(net.state_dict())
    want = {f"features.{i}.{p}" for i in (0, 2, 5, 7, 10, 12, 14, 17, 19, 21, 24, 26, 28) for p in ("weight", "bias")}
    want |= {f"classifier.{i}.{p}" for i in (0, 3) for p in ("weight", "bias")}
    assert len(want) == 30 and keys == want
    assert torch.equal(net.state_dict()["classifier.3.weight"], vgg_state["classifier.3.weight"])
    assert callable(net.features)
    path = tmp_path / "vgg16.pth"
    torch.save(vgg_state, str(path))
    assert torch.equal(metrics.VGG16Features(weights=str(path)).state_dict()["features.28.bias"], vgg_state["features.28.bias"])
    missing = tmp_path / "nothere" / "vgg16-397923af.pth"
    with pytest.raises(RuntimeError, match=str(missing).replace(".", r"\.")):
        metrics.VGG16Features(weights=str(missing))
    bad = dict(vgg_state)
    del bad["classifier.3.bias"]
    with pytest.raises(RuntimeError, match="classifier.3.bias"):
        metrics.VGG16Features(weights=bad)
    bad = dict(vgg_state)
    bad["classifier.0.weight"] = torch.zeros(4096, 100)
    with pytest.raises(RuntimeError, match="shape"):
        metrics.VGG16Features(weights=bad)


def test_vgg16_default_path_is_torchvisions_cache():
    metrics = _metrics()
    assert metrics.default_weights_path() == os.path.join(torch.hub.get_dir(), "checkpoints", "vgg16-397923af.pth")


# ---------------------------------------------------------------------------------------------------- tools/evaluate.py
def _evaluate():
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    try:
        return importlib.import_module("evaluate")
    finally:
        sys.path.pop(0)


def test_evaluate_parsing():
    ev = _evaluate()
    a = ev.parser().parse_args(["real", "--images", "d", "--out", "o.npz"])
    assert (a.cmd, a.images, a.out, a.batch, a.inception, a.vgg) == ("real", "d", "o.npz", 64, None, None)
    a = ev.parser().parse_args(["gen", "--config", "tiny", "--num", "7", "--out", "g.npz", "--seed", "3", "--truncation", "0.7"])
    assert (a.config, a.num, a.batch, a.seed, a.truncation, a.checkpoint) == ("tiny", 7, 8, 3, 0.7, None)
    a = ev.parser().parse_args(["score", "r.npz", "g.npz", "--subsets", "5", "--subset-size", "50", "--k", "4"])
    assert (a.real, a.gen, a.subsets, a.subset_size, a.k) == ("r.npz", "g.npz", 5, 50, 4)
    a = ev.parser().parse_args(["score", "r.npz", "g.npz"])
    assert (a.subsets, a.subset_size, a.k) == (100, 1000, 3)
    with pytest.raises(SystemExit):
        ev.parser().parse_args(["gen", "--config", "99", "--num", "1", "--out", "x"])
    with pytest.raises(SystemExit):
        ev.parser().parse_args(["score", "r.npz"])


def test_features_npz_round_trip(tmp_path):
    metrics = _metrics()
    f = {"inception": torch.randn(5, 2048), "vgg16": torch.rand(5, 4096)}
    p = str(tmp_path / "f.npz")
    metrics.save_features(p, f)
    with np.load(p) as z:
        assert sorted(z.files) == ["inception", "vgg16"] and z["vgg16"].dtype == np.float32
    g = metrics.load_features(p)
    assert torch.equal(g["inception"], f["inception"]) and torch.equal(g["vgg16"], f["vgg16"])
    with pytest.raises(RuntimeError, match="4096"):
        metrics.save_features(p, {"inception": torch.randn(5, 2048), "vgg16": torch.rand(5, 100)})
    with open(p, "wb") as fh:
        np.savez(fh, inception=np.zeros((3, 2048), np.float32), vgg16=np.zeros((4, 4096), np.float32))
    with pytest.raises(RuntimeError, match="rows"):
        metrics.load_features(p)
