"""CPU-only checks of the drop-in boundary: the C-ABI library loads and exports every symbol that
include/hg3d.h declares, the module surfaces carry the reference's state_dict schema, the drop-in
import paths resolve, and the product path fails loudly without a GPU (no fallback)."""
import copy
import importlib
import json
import os
import re
import subprocess
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _header_symbols():
    text = open(os.path.join(ROOT, "include", "hg3d.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(hg_[a-z0-9_]+)\s*\(", text)))


def test_library_exports_every_declared_symbol():
    abi = importlib.import_module("3dhumangan_b200.abi")
    build = importlib.import_module("3dhumangan_b200.build")
    build.build()
    lib = abi.lib()
    syms = _header_symbols()
    assert len(syms) >= 14
    for s in syms:
        assert hasattr(lib, s), f"{s} declared in include/hg3d.h but not exported"
        assert s in abi.SIGNATURES, f"{s} has no ctypes signature in abi.py"
    assert set(abi.SIGNATURES) == set(syms), set(abi.SIGNATURES) ^ set(syms)
    assert lib.hg_abi_version() == 1
    assert lib.hg_packed_weight_bytes(256, 256, 256) == 4 * 2 * 256 * 128
    assert lib.hg_render_weight_blob_bytes() == 60 * 256 * 128


def test_argument_validation_reports_errors_without_a_gpu():
    abi = importlib.import_module("3dhumangan_b200.abi")
    lib = abi.lib()
    rc = lib.hg_pack_weight(None, 256, 256, 256, None, 1.0, 256, None, 0, None)
    assert rc != 0 and b"null pointer" in lib.hg_last_error()
    rc = lib.hg_render_mlp(*([None] * 12), 1, 1, 24, 256, 0.0, 0, 0, 0, 3, None)
    assert rc != 0


@pytest.mark.parametrize("name", ["MAP3DBN", "MAP3DBN512", "MAP3DBN512L"])
def test_state_dict_schema_matches_reference(pkg, name):
    schema = json.load(open(os.path.join(ROOT, "tests", "golden", "state_dict_schema.json")))[name]
    gen = importlib.import_module("3dhumangan_b200.modules.generator")
    disc = importlib.import_module("3dhumangan_b200.modules.discriminator")
    meta = pkg.configs.extract_metadata(getattr(pkg.configs, name), 0)
    if name == "MAP3DBN512L":
        meta["dataset_length"] = 16
    G = gen.Map3DGenerator(**meta)
    D = disc.UNetDiscriminator(**meta)
    got_g = [[k, list(v.shape), str(v.dtype)] for k, v in G.state_dict().items()]
    got_d = [[k, list(v.shape), str(v.dtype)] for k, v in D.state_dict().items()]
    assert got_g == schema["G"]          # names, shapes, dtypes AND order (EMA zips parameters() in order)
    assert got_d == schema["D"]
    assert [k for k, _ in G.named_parameters()] == schema["G_params"]
    assert [k for k, _ in D.named_parameters()] == schema["D_params"]


def test_oracle_params_load_strictly(pkg, port):
    gen = importlib.import_module("3dhumangan_b200.modules.generator")
    cfg = pkg.configs.baseline_config("tiny")
    G = gen.Map3DGenerator(**cfg)
    G.load_state_dict(port.init_generator_params(cfg, seed=0), strict=True)
    G.set_device("cpu")
    assert G.device == "cpu" and G.neural_field.device == "cpu"
    assert G.step == 0 and G.epoch == 0
    G.latent_pool.init(torch.ones(cfg["dataset_length"], cfg["latent_dim"]))


def test_forward_fails_loudly_without_gpu(pkg, port):
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    gen = importlib.import_module("3dhumangan_b200.modules.generator")
    cfg = pkg.configs.baseline_config("tiny")
    G = gen.Map3DGenerator(**cfg)
    G.set_device("cpu")
    cond = pkg.synthetic.make_conditions(1)
    with pytest.raises(RuntimeError):
        with torch.no_grad():
            G(torch.randn(1, cfg["latent_dim"]), cond, **cfg)
    bias_act = importlib.import_module("3dhumangan_b200.ops.bias_act")
    with pytest.raises(RuntimeError):
        bias_act.bias_act(torch.randn(4, 8), torch.zeros(8), act="lrelu")


def test_training_forward_has_no_cpu_path_either(pkg):
    """With autograd enabled the generator takes the training kernels; on a CPU tensor that must raise, not fall back."""
    gen = importlib.import_module("3dhumangan_b200.modules.generator")
    cfg = pkg.configs.baseline_config("tiny")
    G = gen.Map3DGenerator(**cfg)
    G.set_device("cpu")
    with pytest.raises(RuntimeError, match="CUDA|sm_90a|no CPU path"):
        G(torch.randn(1, cfg["latent_dim"]), pkg.synthetic.make_conditions(1), **cfg)
    D = importlib.import_module("3dhumangan_b200.modules.discriminator").UNetDiscriminator(**cfg)
    with pytest.raises(RuntimeError, match="CUDA|sm_90a|no CPU path"):
        D(torch.randn(1, 3, 64, 64, requires_grad=True), None, 1.0)


def test_dropin_import_paths():
    code = "\n".join([
        "import sys",
        "sys.path.insert(0, %r); sys.path.insert(0, %r)" % (os.path.join(ROOT, "3dhumangan_b200", "dropin"), ROOT),
        "import configs, lib.generators, lib.discriminators, lib.implicit_funcitions",
        "from lib.components.ops import bias_act, upfirdn2d",
        "class O:",
        "    config = 'MAP3DBN512'; tune = ''; variant = 0",
        "c = configs.get_config(O); c = configs.get_config(O)",
        "m = configs.extract_metadata(c, 0)",
        "G = getattr(lib.generators, m['generator'])(**m)",
        "assert m['neural_field_cls'] is lib.implicit_funcitions.COORDCONCATSIREN",
        "print('ok')"])
    out = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0 and "ok" in out.stdout, out.stderr[-2000:]


def test_config_semantics(pkg):
    c = pkg.configs
    m0 = c.extract_metadata(c.MAP3DBN, 0)
    m1 = c.extract_metadata(c.MAP3DBN, 200000)
    assert m0["gen_lr"] == 1e-4 and m1["gen_lr"] == 5e-5 and m0["hidden_dim"] == 384 and m0["r1_lambda"] == 0.25
    assert [p["do_r1"] for p in c.MAP3DBN512["phases"]] == [False, False, False, True, False, False, False, True]
    big = c.extract_metadata(c.MAP3DBN512L, 0)
    assert big["hidden_dim"] == 420 and big["legacy_mode"] and big["map3d_mode"] == "isolated"


def test_synthetic_conditions_are_consistent(pkg):
    cond = pkg.synthetic.make_conditions(2, seed=3)
    assert cond["vertices"].shape == (2, 6890, 3) and cond["lbs_weights"].shape == (2, 6890, 24)
    assert torch.allclose(cond["lbs_weights"].sum(-1), torch.ones(2, 6890), atol=1e-5)
    assert (cond["lbs_weights"] > 0).sum(-1).max() <= 4
    # skinning identity: vertices == sum_j w_j fk_j [tpose - (0,.35,0); 1]
    tp = cond["tpose_vertices"].clone()
    tp[..., 1] -= 0.35
    hom = torch.cat([tp, torch.ones(2, 6890, 1)], -1)
    vfk = torch.einsum("bvj,bjkl->bvkl", cond["lbs_weights"], cond["fk_matrices"])
    v = torch.einsum("bvij,bvj->bvi", vfk, hom)[..., :3]
    assert (v - cond["vertices"]).abs().max() < 1e-4
    again = pkg.synthetic.make_conditions(2, seed=3)
    assert all(torch.equal(cond[k], again[k]) for k in cond)


def test_segmentation_loss_matches_reference_trainer():
    """train_step.segmentation_loss against values of the reference's own method (tests/golden/make_golden_loss.py)."""
    import numpy as np
    sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
    import make_golden_loss
    ts = importlib.import_module("3dhumangan_b200.train_step")
    gold = np.load(os.path.join(ROOT, "tests", "golden", "seg_loss.npz"))
    for i, (seg, gt, L) in enumerate(make_golden_loss.cases()):
        s = seg.clone().requires_grad_(True)
        loss = ts.segmentation_loss(s, gt, L)
        loss.backward()
        assert abs(float(loss) - gold["loss"][i]) < 1e-5 * max(1.0, abs(gold["loss"][i])), i
        assert abs(float(s.grad.double().norm()) - gold["grad_norm"][i]) < 1e-5 * gold["grad_norm"][i], i


def test_initialisation_statistics_match_reference(pkg):
    """From-scratch training must start from the reference's distributions: per-tensor std / abs-max of every parameter
    (3-seed averages) against the unmodified reference modules (tests/golden/make_init_stats.py).  Catches e.g. the
    spectral-normed discriminator convolutions, whose `weight_orig` the reference re-draws with kaiming-normal through
    the aliased `.weight` (unet_discriminators.py:74-78,121)."""
    gen = importlib.import_module("3dhumangan_b200.modules.generator")
    disc = importlib.import_module("3dhumangan_b200.modules.discriminator")
    ref = json.load(open(os.path.join(ROOT, "tests", "golden", "init_stats.json")))
    cfg = pkg.configs.extract_metadata(copy.deepcopy(pkg.configs.MAP3DBN512), 0)
    seeds = 3
    got = {"G": {}, "D": {}}
    numel = {}
    for seed in range(seeds):
        torch.manual_seed(100 + seed)
        for key, m in (("G", gen.Map3DGenerator(**cfg)), ("D", disc.UNetDiscriminator(**cfg))):
            for n, p in m.named_parameters():
                r = got[key].setdefault(n, [0.0, 0.0])
                numel[key, n] = p.numel()
                r[0] += (float(p.detach().std()) if p.numel() > 1 else 0.0) / seeds
                r[1] += float(p.detach().abs().max()) / seeds
    bad = []
    checked = 0
    for key in ("G", "D"):
        assert set(got[key]) == set(ref[key])
        for n, (mean, std, amax) in ref[key].items():
            s, a = got[key][n]
            if amax == 0 or (std == 0 and numel[key, n] > 1):      # constant initialisation (zeros / ones)
                if abs(a - amax) > 1e-6:
                    bad.append((key, n, "absmax", a, amax))
                continue
            if numel[key, n] < 64:                 # 1-3 element tensors: sample statistics say nothing
                continue
            tol = max(0.03, 6.0 / (2 * numel[key, n] * seeds) ** 0.5)      # ~6 sigma of the sample std, both sides
            checked += 1
            if abs(s - std) > tol * std:
                bad.append((key, n, "std", s, std, tol))
    assert checked > 250 and not bad, bad[:10]
