"""KID and k-NN precision / recall on sm_90a (3dhumangan_b200/metrics.py, csrc/metrics.cu) against the fp64 oracle
(oracle/metrics_port.py): the KID kernel over subset sizes and dimensions, with real features' cancellation; the k-NN radii on
ragged sizes with duplicates; the coverage flags; radii at 50 000 x 4096; VGG16 fc7 features; repeatability and no torch op on
the path; `generator_features` against explicit calls, FID and two ranks; and tools/evaluate.py end to end."""
import importlib
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import metrics_port as mp

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _abi():
    return importlib.import_module("3dhumangan_b200.abi")


def _metrics():
    return importlib.import_module("3dhumangan_b200.metrics")


def _fid():
    return importlib.import_module("3dhumangan_b200.fid")


# ------------------------------------------------------------------------------------------------------------------ KID
@pytest.mark.parametrize("m,D,S,n", [(2, 64, 5, 2), (3, 100, 7, 9), (17, 2048, 10, 40), (17, 64, 100, 17), (1000, 100, 20, 1300),
                                     (1000, 2048, 100, 1500)])
def test_kid_kernel_against_fp64(m, D, S, n):
    metrics = _metrics()
    g = torch.Generator(device="cuda").manual_seed(m * 7 + D)
    real = torch.rand(n, D, generator=g, device="cuda")
    gen = torch.rand(n + 3, D, generator=g, device="cuda") * 1.1
    mean, std, t = metrics.kid(real, gen, S, 1000, seed=m)
    ig, ir = mp.kid_indices(n + 3, n, S, 1000, m)
    ref = mp.kid_terms(gen.double(), real.double(), ig, ir)
    kmean = float(((gen.double() @ real.double().T) / D + 1).pow(3).mean())
    err = np.abs(t - ref).max()
    print(f"m={m} D={D} S={S}: max |t - t_oracle| = {err:.3e} = {err / kmean:.2e} x mean kernel value")
    assert t.dtype == np.float64 and t.shape == (S,)
    assert err <= 1e-11 * kmean, (err, kmean)
    assert mean == pytest.approx(ref.mean(), rel=0, abs=1e-11 * kmean) and std == pytest.approx(ref.std(), rel=0, abs=1e-11 * kmean)
    again = metrics.kid(real, gen, S, 1000, seed=m)[2]
    assert np.array_equal(t, again)


def test_kid_with_the_cancellation_of_real_features():
    """Two close distributions: KID is ~1e-3 of the kernel value, so the kernel sums cancel to three digits."""
    metrics = _metrics()
    g = torch.Generator(device="cuda").manual_seed(11)
    real = torch.rand(1200, 2048, generator=g, device="cuda")
    gen = torch.rand(1200, 2048, generator=g, device="cuda") * 1.035
    mean, _, t = metrics.kid(real, gen, 50, 1000, seed=1)
    ig, ir = mp.kid_indices(1200, 1200, 50, 1000, 1)
    ref = mp.kid_terms(gen.double(), real.double(), ig, ir)
    kmean = float(((gen.double() @ real.double().T) / 2048 + 1).pow(3).mean())
    ratio = mean / kmean
    err = np.abs(t - ref).max()
    print(f"KID / mean kernel value {ratio:.2e}; max |t - t_oracle| {err / kmean:.2e} x mean kernel value")
    assert 3e-4 < ratio < 3e-3
    assert err <= 1e-11 * kmean


def test_kid_refusals_in_the_library():
    abi = _abi()
    lib = abi.lib()
    p = torch.zeros(64, device="cuda")
    ptr = abi.ptr(p)
    assert lib.hg_kid(ptr, 4, ptr, 4, 4, ptr, ptr, 1, 1, ptr, ptr, 1 << 20, None) == 1
    assert b"subset size" in lib.hg_last_error()
    assert lib.hg_kid(ptr, 4, ptr, 3, 4, ptr, ptr, 1, 4, ptr, ptr, 1 << 20, None) == 1
    assert lib.hg_kid(ptr, 4, ptr, 4, 4, ptr, ptr, 1, 4, ptr, ptr, 8, None) == 1
    assert b"workspace" in lib.hg_last_error()
    assert lib.hg_knn_radii(ptr, ptr, 1, 4, 1, ptr, None) == 1
    assert lib.hg_knn_radii(ptr, ptr, 10, 4, 9, ptr, None) == 1
    assert lib.hg_knn_radii(ptr, ptr, 10, 4, 0, ptr, None) == 1
    assert lib.hg_ball_coverage(ptr, ptr, ptr, 0, ptr, ptr, ptr, 3, 4, ptr, ptr, ptr, None) == 1
    with pytest.raises(ValueError, match="more than k"):
        _metrics().precision_recall(torch.rand(1, 4, device="cuda"), torch.rand(5, 4, device="cuda"), 1)


# ------------------------------------------------------------------------------------------------------------ k-NN radii
def _radii(x, k):
    metrics = _metrics()
    x = x.float().contiguous()
    return metrics._radii(x, metrics._sqnorms(x), k)


@pytest.mark.parametrize("n,D", [(2, 1), (9, 4096), (63, 100), (65, 4096), (64, 1), (129, 100), (3000, 100), (3000, 1),
                                 (1000, 4096)])
def test_knn_radii_against_fp64(n, D):
    g = torch.Generator(device="cuda").manual_seed(n + D)
    x = torch.randn(n, D, generator=g, device="cuda")
    if n > 8:
        x[n // 2] = x[1]                                     # duplicates at other indices count at distance 0
        x[n - 1] = x[1]
    d = mp.sq_dists(x, x)
    d.fill_diagonal_(float("inf"))
    sq = x.double().pow(2).sum(1)
    for k in range(1, min(8, n - 1) + 1):
        ref, nb = d.kthvalue(k, dim=1)
        got = _radii(x, k)
        tol = 1e-12 * (sq + sq[nb])
        bad = int(((got - ref).abs() > tol).sum())
        print(f"n={n} D={D} k={k}: max |rho2 - oracle| / (|a|^2 + |b|^2) = {float(((got - ref).abs() / (sq + sq[nb])).max()):.2e}")
        assert bad == 0, (k, bad)
        if n > 8:
            assert float(got[1]) == float(got[n // 2]) and (k > 2 or float(got[1]) == 0.0)
        assert torch.equal(got, _radii(x, k))


def test_coverage_flags_equal_the_oracle():
    metrics = _metrics()
    abi = _abi()
    g = torch.Generator(device="cuda").manual_seed(3)
    real = torch.randn(700, 64, generator=g, device="cuda")
    gen = torch.randn(530, 64, generator=g, device="cuda") * 1.2 + 0.1
    k = 3
    rr, rg = mp.knn_radii(real, k), mp.knn_radii(gen, k)
    d = mp.sq_dists(gen, real)
    sg, sr = gen.double().pow(2).sum(1), real.double().pow(2).sum(1)
    band = 1e-10 * (sg[:, None] + sr[None, :])
    ambiguous = int(((d - rr[None, :]).abs() <= band).sum() + ((d - rg[:, None]).abs() <= band).sum())
    print(f"coverage: {ambiguous} pairs within 1e-10 (|g|^2 + |r|^2) of a radius")
    assert ambiguous == 0
    fg, fr = mp.coverage(gen, real, rg, rr)
    x_r, x_g = real.contiguous(), gen.contiguous()
    sq_r, sq_g = metrics._sqnorms(x_r), metrics._sqnorms(x_g)
    rho_r, rho_g = metrics._radii(x_r, sq_r, k), metrics._radii(x_g, sq_g, k)
    row = torch.full((530,), 7, dtype=torch.uint8, device="cuda")
    col = torch.full((700,), 7, dtype=torch.uint8, device="cuda")
    counts = torch.empty(2, dtype=torch.int64, device="cuda")
    abi.call("hg_ball_coverage", abi.ptr(x_g), abi.ptr(sq_g), abi.ptr(rho_g), 530, abi.ptr(x_r), abi.ptr(sq_r), abi.ptr(rho_r), 700,
             64, abi.ptr(row), abi.ptr(col), abi.ptr(counts), abi.stream())
    assert torch.equal(row.bool(), fg) and torch.equal(col.bool(), fr)
    assert set(row.unique().tolist()) <= {0, 1} and set(col.unique().tolist()) <= {0, 1}
    assert counts.tolist() == [int(fg.sum()), int(fr.sum())]
    p, r = metrics.precision_recall(real, gen, k)
    assert (p, r) == (int(fg.sum()) / 530, int(fr.sum()) / 700)
    assert 0 < p < 1 and 0 < r < 1
    assert metrics.precision_recall(real, gen, k) == (p, r)
    assert metrics.precision_recall(real, real.clone(), k) == (1.0, 1.0)
    assert metrics.precision_recall(real, real + 100, k) == (0.0, 0.0)


def test_radii_at_full_size():
    """50 000 x 4096: the radii of 512 sampled rows against a torch fp64 computation on the device."""
    g = torch.Generator(device="cuda").manual_seed(5)
    x = torch.relu(torch.randn(50000, 4096, generator=g, device="cuda"))
    k = 3
    got = _radii(x, k)
    rows = torch.randperm(50000, generator=torch.Generator().manual_seed(0))[:512].cuda()
    d = mp.sq_dists(x[rows], x)
    d[torch.arange(512, device="cuda"), rows] = float("inf")
    ref, nb = d.kthvalue(k, dim=1)
    sq = x.double().pow(2).sum(1)
    rel = ((got[rows] - ref).abs() / (sq[rows] + sq[nb])).max()
    print(f"50000 x 4096: max |rho2 - oracle| / (|a|^2 + |b|^2) over 512 rows = {float(rel):.2e}")
    assert float(rel) <= 1e-12


# ------------------------------------------------------------------------------------------------------------------ VGG16
@pytest.fixture(scope="module")
def vgg_state():
    return mp.seeded_vgg16_state(0)


@pytest.fixture(scope="module")
def vgg(vgg_state):
    return _metrics().VGG16Features(weights=vgg_state).cuda()


def _smooth_images(n, H, W, seed):
    g = torch.Generator().manual_seed(seed)
    low = torch.rand(n, 3, max(H // 8, 2), max(W // 8, 2), generator=g)
    return F.interpolate(low, size=(H, W), mode="bilinear", align_corners=False).clamp(0, 1)


# measured on an H100: 1.8e-4 per image at both input sizes and batch sizes (fp32x3 convolutions, and fc6's K = 25088 fp32
# tensor-core accumulation); the bound keeps a 2.5x margin under the 1e-3 contract
VGG_BOUND = 4.5e-4


@pytest.mark.parametrize("B", [1, 5])
@pytest.mark.parametrize("H,W", [(224, 224), (512, 256)])
def test_vgg16_features_against_fp64_oracle(vgg, vgg_state, B, H, W):
    imgs = (_smooth_images(B, H, W, H + W + B) * 255).round().to(torch.uint8)
    got = vgg.features(imgs.cuda())
    sd = {k: v.cuda() for k, v in vgg_state.items() if not k.startswith("classifier.6")}
    with torch.no_grad():
        ref = mp.vgg16_fc7(sd, imgs.double().cuda() / 255)
    assert got.shape == (B, 4096) and got.dtype == torch.float32
    errs = [float((got[i].double() - ref[i]).norm() / ref[i].norm()) for i in range(B)]
    print(f"VGG16 fc7 {H}x{W} B={B}: per-image rel-L2 {max(errs):.3e} (max)")
    assert max(errs) < VGG_BOUND, errs
    assert float((got > 0).float().mean()) > 0.1
    assert torch.equal(got, vgg.features(imgs.cuda()))


def test_gradients_refused(vgg):
    with pytest.raises(RuntimeError, match="gradients"):
        vgg.features(torch.rand(1, 3, 64, 32, device="cuda", requires_grad=True))


def test_no_torch_op_on_the_path(vgg):
    metrics = _metrics()
    imgs = (_smooth_images(2, 128, 64, 7) * 255).to(torch.uint8).cuda()
    real = torch.rand(300, 128, device="cuda")
    gen = torch.rand(200, 128, device="cuda")
    vgg.features(imgs)
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        vgg.features(imgs)
        metrics.kid(real, gen, 5, 100)
        metrics.precision_recall(real, gen, 3)
        torch.cuda.synchronize()
    names = {e.name for e in prof.events()}
    banned = [n for n in names if any(k in n for k in ("aten::mm", "aten::addmm", "aten::linear", "aten::convolution", "aten::cdist",
                                                         "aten::topk", "aten::kthvalue", "aten::matmul", "aten::bmm", "cudnn",
                                                         "upsample_bilinear2d", "max_pool2d"))]
    assert not banned, banned
    for kern in ("conv_general_kernel", "kid_blocks_kernel", "knn_radii_kernel", "ball_coverage_kernel"):
        assert any(kern in n for n in names), kern


# ------------------------------------------------------------------------------------------------------ generator_features
@pytest.fixture(scope="module")
def inception():
    from oracle import inception_port as ip
    return _fid().FIDInceptionV3(weights=ip.seeded_fid_inception_state(0)).cuda()


def _tiny_generator(pkg):
    gen = importlib.import_module("3dhumangan_b200.modules.generator")
    cfg = pkg.configs.baseline_config("tiny")
    cfg.update(gen_height=32, gen_width=32, render_height=8, render_width=8, num_steps=16)
    torch.manual_seed(0)
    G = gen.Map3DGenerator(**cfg).cuda()
    G.set_device(torch.device("cuda:0"))
    G.eval()
    return G, cfg


def test_generator_features_equal_explicit_calls_and_fid(pkg, vgg, inception):
    fid, metrics = _fid(), _metrics()
    G, cfg = _tiny_generator(pkg)
    torch.manual_seed(5)
    got = metrics.generator_features(G, cfg, 12, 5, seed=3, inception=inception, vgg=vgg)
    assert got["inception"].shape == (12, 2048) and got["vgg16"].shape == (12, 4096)
    conds = fid.synthetic_conditions(3)
    run = dict(cfg, nerf_noise=0, last_back=cfg.get("eval_last_back", False), truncation_psi=1.0)
    torch.manual_seed(5)
    inc, vg = [], []
    for idx in ([0, 1, 2, 3, 4], [5, 6, 7, 8, 9], [10, 11]):
        z = torch.stack([fid.latent(3, i, cfg["latent_dim"]) for i in idx]).cuda()
        c = {k: v.cuda() for k, v in conds(idx).items()}
        with torch.no_grad():
            u8 = fid.to_uint8(G.staged_forward(z, c, **run)["rgbs"])
        inc.append(inception.features(u8))
        vg.append(vgg.features(u8))
    assert torch.equal(got["inception"], torch.cat(inc)) and torch.equal(got["vgg16"], torch.cat(vg))

    torch.manual_seed(5)
    stats = fid.generator_statistics(G, cfg, 12, 5, seed=3, inception=inception)
    bank = fid.FeatureStats()
    bank.update(got["inception"])
    other = fid.FeatureStats()
    other.update(got["inception"].flip(0) * 1.05 + 0.01)
    d_stats = fid.frechet_distance(*stats.mean_cov(), *other.mean_cov())
    d_bank = fid.frechet_distance(*bank.mean_cov(), *other.mean_cov())
    print(f"FID from generator_statistics {d_stats:.12g}, from the feature bank {d_bank:.12g}")
    assert abs(d_bank - d_stats) <= 1e-9 * abs(d_stats)


def _rank_worker(rank, world, port_no, out_path):
    sys.path.insert(0, ROOT)
    import torch.distributed as dist
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    pkg = importlib.import_module("3dhumangan_b200")
    rng = importlib.import_module("3dhumangan_b200.rng")
    metrics = importlib.import_module("3dhumangan_b200.metrics")
    fid = importlib.import_module("3dhumangan_b200.fid")
    from oracle import inception_port as ip
    # fixed ray jitter: the renderer's draws would otherwise differ between the per-rank and the single-rank batches
    rng.draw = lambda batch, rays, steps, device, cfg: (torch.full((batch, rays, steps, 1), 0.5, device=device),
                                                         torch.zeros(batch, rays, steps, 1, device=device))
    G, cfg = _tiny_generator(pkg)
    inc = fid.FIDInceptionV3(weights=ip.seeded_fid_inception_state(0)).to(dev)
    vgg = metrics.VGG16Features(weights=mp.seeded_vgg16_state(0)).to(dev)
    if rank == 0:
        one = metrics.generator_features(G, cfg, 5, 1, seed=2, inception=inc, vgg=vgg)
    dist.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{port_no}", rank=rank, world_size=world)
    got = metrics.generator_features(G, cfg, 5, 1, seed=2, inception=inc, vgg=vgg)
    gathered = [None] * world
    dist.all_gather_object(gathered, {k: v.cpu() for k, v in got.items()})
    dist.barrier()
    dist.destroy_process_group()
    if rank == 0:
        torch.save({"ranks": gathered, "one": {k: v.cpu() for k, v in one.items()}}, out_path)


def test_two_ranks_equal_one_rank(tmp_path):
    import torch.multiprocessing as tmp
    out = str(tmp_path / "res.pt")
    tmp.spawn(_rank_worker, args=(2, 29800 + os.getpid() % 90, out), nprocs=2, join=True)
    r = torch.load(out)
    for got in r["ranks"]:
        for key in ("inception", "vgg16"):
            assert got[key].shape[0] == 5
            assert torch.equal(got[key], r["one"][key]), key


# ------------------------------------------------------------------------------------------------------------------ tool
def test_evaluate_tool_end_to_end(tmp_path, vgg_state):
    import torchvision.io as tio
    from oracle import inception_port as ip
    ipath, vpath = str(tmp_path / "inception.pth"), str(tmp_path / "vgg16.pth")
    torch.save(ip.seeded_fid_inception_state(0), ipath)
    torch.save(vgg_state, vpath)
    imgdir = tmp_path / "imgs"
    imgdir.mkdir()
    for i, im in enumerate((_smooth_images(6, 32, 32, 1) * 255).to(torch.uint8)):
        tio.write_png(im, str(imgdir / f"{i}.png"))
    ev, fd = os.path.join(ROOT, "tools", "evaluate.py"), os.path.join(ROOT, "tools", "fid.py")
    run = lambda tool, *a: subprocess.run([sys.executable, tool, *a], capture_output=True, text=True, timeout=900)
    rs = [run(ev, "real", "--images", str(imgdir), "--out", str(tmp_path / "real.npz"), "--inception", ipath, "--vgg", vpath),
          run(ev, "gen", "--config", "tiny", "--num", "7", "--batch", "4", "--out", str(tmp_path / "gen.npz"), "--inception", ipath,
              "--vgg", vpath),
          run(fd, "real", "--images", str(imgdir), "--out", str(tmp_path / "real_stats.npz"), "--inception", ipath),
          run(fd, "gen", "--config", "tiny", "--num", "7", "--batch", "4", "--out", str(tmp_path / "gen_stats.npz"), "--inception",
              ipath)]
    for r in rs:
        assert r.returncode == 0, r.stderr[-3000:]
    s = run(ev, "score", str(tmp_path / "real.npz"), str(tmp_path / "gen.npz"), "--subsets", "10", "--subset-size", "5", "--k", "2")
    assert s.returncode == 0, s.stderr[-3000:]
    res = json.loads(s.stdout.strip().splitlines()[-1])
    assert set(res) == {"fid", "kid", "kid_std", "precision", "recall", "n_real", "n_gen", "k", "subsets", "subset_size"}
    assert (res["n_real"], res["n_gen"], res["k"], res["subsets"], res["subset_size"]) == (6, 7, 2, 10, 5)
    assert 0 <= res["precision"] <= 1 and 0 <= res["recall"] <= 1 and np.isfinite(res["kid"])
    f = run(fd, "fid", str(tmp_path / "real_stats.npz"), str(tmp_path / "gen_stats.npz"))
    assert f.returncode == 0, f.stderr[-3000:]
    fid = _fid()
    ref = fid.frechet_distance(*fid.load_stats(str(tmp_path / "real_stats.npz")), *fid.load_stats(str(tmp_path / "gen_stats.npz")))
    print(f"evaluate.py fid {res['fid']:.12g}, fid.py fid {f.stdout.strip()} ({ref:.12g} unrounded)")
    assert abs(float(f.stdout.strip()) - ref) <= 1e-6          # fid.py prints six decimals
    assert abs(res["fid"] - ref) <= 1e-9 * abs(ref)
