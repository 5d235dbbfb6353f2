"""CPU checks of FID (3dhumangan_b200/fid.py): the fp64 oracle (oracle/inception_port.py) against torchvision's own Inception3
modules with pytorch-fid's pooling changes, the module's torchvision names and loading, the Frechet distance three ways, the
host moments of FeatureStats and its .npz files, and `to_uint8` against the sample app's expression."""
import importlib

import numpy as np
import pytest
import scipy.linalg
import torch
import torch.nn.functional as F

from oracle import inception_port as ip


def _fid():
    return importlib.import_module("3dhumangan_b200.fid")


@pytest.fixture(scope="module")
def state():
    return ip.seeded_fid_inception_state(0)


@pytest.fixture(scope="module")
def tv(state):
    torchvision = pytest.importorskip("torchvision")
    m = torchvision.models.inception.Inception3(num_classes=1008, aux_logits=False, init_weights=False).double().eval()
    missing, unexpected = m.load_state_dict(state, strict=False)
    assert not unexpected and all(k.startswith("fc.") or k.endswith("num_batches_tracked") for k in missing), missing
    return m


def _rel(a, b):
    return float((a - b).norm() / b.norm())


def test_oracle_stem_and_reduction_blocks_equal_torchvision(state, tv):
    g = torch.Generator().manual_seed(1)
    x = torch.rand(2, 3, 83, 79, generator=g, dtype=torch.float64) * 2 - 1
    with torch.no_grad():
        ref = x
        for name in ("Conv2d_1a_3x3", "Conv2d_2a_3x3", "Conv2d_2b_3x3", "maxpool1", "Conv2d_3b_1x1", "Conv2d_4a_3x3", "maxpool2"):
            ref = getattr(tv, name)(ref)
        got = ip.stem(ip._Graph(state), x)
        assert _rel(got, ref) < 1e-12
        for name, cin in (("Mixed_6a", 288), ("Mixed_7a", 768)):
            h = torch.relu(torch.randn(2, cin, 13, 11, generator=g, dtype=torch.float64))
            assert _rel(ip.block(ip._Graph(state), name, h), getattr(tv, name)(h)) < 1e-12, name


def _tv_fid_block(m, kind, x):
    """pytorch-fid's FIDInceptionA / C / E_1 / E_2 forward composed from torchvision's branch modules."""
    avg = lambda t: F.avg_pool2d(t, 3, 1, 1, count_include_pad=False)
    if kind == "A":
        b5 = m.branch5x5_2(m.branch5x5_1(x))
        b3 = m.branch3x3dbl_3(m.branch3x3dbl_2(m.branch3x3dbl_1(x)))
        return torch.cat([m.branch1x1(x), b5, b3, m.branch_pool(avg(x))], 1)
    if kind == "C":
        b7 = m.branch7x7_3(m.branch7x7_2(m.branch7x7_1(x)))
        bd = x
        for i in range(1, 6):
            bd = getattr(m, f"branch7x7dbl_{i}")(bd)
        return torch.cat([m.branch1x1(x), b7, bd, m.branch_pool(avg(x))], 1)
    b3 = m.branch3x3_1(x)
    b3 = torch.cat([m.branch3x3_2a(b3), m.branch3x3_2b(b3)], 1)
    bd = m.branch3x3dbl_2(m.branch3x3dbl_1(x))
    bd = torch.cat([m.branch3x3dbl_3a(bd), m.branch3x3dbl_3b(bd)], 1)
    pool = avg(x) if kind == "E1" else F.max_pool2d(x, 3, 1, 1)
    return torch.cat([m.branch1x1(x), b3, bd, m.branch_pool(pool)], 1)


@pytest.mark.parametrize("name,kind,cin", [("Mixed_5b", "A", 192), ("Mixed_5d", "A", 288), ("Mixed_6b", "C", 768),
                                           ("Mixed_6e", "C", 768), ("Mixed_7b", "E1", 1280), ("Mixed_7c", "E2", 2048)])
def test_oracle_fid_blocks_equal_torchvision_branches(state, tv, name, kind, cin):
    g = torch.Generator().manual_seed(cin)
    x = torch.randn(2, cin, 9, 7, generator=g, dtype=torch.float64)       # signed: the max-pool branch sees negatives
    with torch.no_grad():
        assert _rel(ip.block(ip._Graph(state), name, x), _tv_fid_block(getattr(tv, name), kind, x)) < 1e-12


def test_module_names_and_loading(state):
    torchvision = pytest.importorskip("torchvision")
    fid = _fid()
    ref = torchvision.models.inception.Inception3(num_classes=1008, aux_logits=False, init_weights=False).state_dict()
    want = {k: tuple(v.shape) for k, v in ref.items() if not k.startswith("fc.") and not k.endswith("num_batches_tracked")}
    m = fid.FIDInceptionV3(weights=state)
    assert {k: tuple(v.shape) for k, v in m.state_dict().items()} == want
    assert len(m.layers()) == 94
    for k, v in m.state_dict().items():
        assert torch.equal(v, state[k]), k
    # a full torchvision state_dict: fc.* and num_batches_tracked present
    full = dict(ref)
    full.update(state)
    fid.FIDInceptionV3(weights=full)
    broken = dict(state)
    del broken["Mixed_6c.branch7x7dbl_4.bn.running_var"]
    with pytest.raises(RuntimeError, match="Mixed_6c.branch7x7dbl_4.bn.running_var"):
        fid.FIDInceptionV3(weights=broken)


def test_missing_weight_file_names_the_path(tmp_path):
    fid = _fid()
    path = tmp_path / "nowhere" / fid.WEIGHTS_FILE
    with pytest.raises(RuntimeError, match="never downloaded") as e:
        fid.FIDInceptionV3(weights=str(path))
    assert str(path) in str(e.value)
    assert fid.default_weights_path().endswith(fid.WEIGHTS_FILE)


def _scipy_fid(mu1, s1, mu2, s2):
    covmean = scipy.linalg.sqrtm(s1 @ s2)
    covmean = covmean.real
    d = mu1 - mu2
    return float(d @ d + np.trace(s1) + np.trace(s2) - 2 * np.trace(covmean))


def test_frechet_distance_matches_scipy_sqrtm():
    fid = _fid()
    rng = np.random.default_rng(0)
    D, n = 2048, 6000
    stats = []
    for k in range(2):
        a = rng.standard_normal((D, D)) / np.sqrt(D) + (0.3 + k * 0.1) * np.eye(D)
        x = rng.standard_normal((n, D)) @ a.T + rng.standard_normal(D) * 0.1
        stats.append((x.mean(0), np.cov(x, rowvar=False)))
    got = fid.frechet_distance(*stats[0], *stats[1])
    ref = _scipy_fid(*stats[0], *stats[1])
    assert abs(got - ref) <= 1e-6 * abs(ref), (got, ref)


def test_frechet_distance_rank_deficient_equals_nuclear_norm_identity():
    fid = _fid()
    rng = np.random.default_rng(1)
    D, n1, n2 = 256, 40, 57
    x1 = rng.standard_normal((n1, D)) * rng.uniform(0.5, 2, D)
    x2 = rng.standard_normal((n2, D)) + 0.2
    c1, c2 = x1 - x1.mean(0), x2 - x2.mean(0)
    s1, s2 = np.cov(x1, rowvar=False), np.cov(x2, rowvar=False)
    tr_sqrt = np.linalg.svd(c1 @ c2.T, compute_uv=False).sum() / np.sqrt((n1 - 1) * (n2 - 1))
    d = x1.mean(0) - x2.mean(0)
    ref = float(d @ d + np.trace(s1) + np.trace(s2) - 2 * tr_sqrt)
    got = fid.frechet_distance(x1.mean(0), s1, x2.mean(0), s2)
    assert abs(got - ref) <= 1e-6 * abs(ref), (got, ref)


def test_frechet_distance_of_identical_statistics_is_zero():
    fid = _fid()
    rng = np.random.default_rng(2)
    x = rng.standard_normal((300, 2048)) * rng.uniform(0, 3, 2048)
    mu, s = x.mean(0), np.cov(x, rowvar=False)
    assert abs(fid.frechet_distance(mu, s, mu, s)) <= 1e-8 * np.trace(s)


def test_feature_stats_on_host_equal_numpy_and_round_trip(tmp_path):
    fid = _fid()
    rng = np.random.default_rng(3)
    x = np.abs(rng.standard_normal((101, 2048))).astype(np.float32)
    st = fid.FeatureStats(device="cpu")
    for a, b in ((0, 7), (7, 40), (40, 41), (41, 101)):
        st.update(torch.from_numpy(x[a:b]))
    mu, sigma = st.mean_cov()
    x64 = x.astype(np.float64)
    assert st.n == 101
    assert np.abs(mu - x64.mean(0)).max() <= 1e-12 * np.abs(x64.mean(0)).max()
    ref = np.cov(x64, rowvar=False)
    assert np.abs(sigma - ref).max() <= 1e-12 * np.abs(ref).max()
    path = str(tmp_path / "stats.npz")
    st.save(path)
    with np.load(path) as z:
        assert sorted(z.files) == ["mu", "sigma"]
    m2, s2 = fid.load_stats(path)
    assert np.array_equal(m2, mu) and np.array_equal(s2, sigma)
    other = str(tmp_path / "pytorch_fid.npz")
    np.savez(other, mu=mu.astype(np.float32), sigma=sigma)             # a file written by someone else
    m3, s3 = fid.load_stats(other)
    assert m3.dtype == np.float64 and np.array_equal(s3, sigma)
    with pytest.raises(RuntimeError):
        st.update(torch.zeros(3, 17))


def test_to_uint8_equals_the_sample_app_expression():
    fid = _fid()
    k = torch.arange(256, dtype=torch.float64)
    steps = (k / 255 * 2 - 1).float()
    vals = torch.cat([torch.tensor([-1.0, 1.0, 0.0, -0.0, -1.5, 1.5, -7.0, 3.0, float("inf"), -float("inf")]), steps,
                      torch.nextafter(steps, torch.full_like(steps, -2)), torch.nextafter(steps, torch.full_like(steps, 2))])
    x = vals.view(1, 1, 1, -1)
    frames = torch.clamp(x, -1, 1)                                          # apps/sample_from_generator.py:59-62
    frames = frames * 0.5 + 0.5
    ref = torch.clamp(frames * 255, 0, 255).to(torch.uint8)
    got = fid.to_uint8(x)
    assert got.dtype == torch.uint8 and torch.equal(got, ref)
    assert int(got.min()) == 0 and int(got.max()) == 255
