"""CPU checks of the perceptual loss's boundary: the new C entry points agree between include/hg3d.h, abi.py and the
library; the weights are never downloaded; the reference's import path binds to this package's class; no CPU path."""
import importlib
import os
import re
import subprocess
import sys

import pytest
import torch

from oracle import perceptual_port as pp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ENTRIES = ("hg_vgg_input", "hg_vgg_input_adjoint", "hg_maxpool2x2", "hg_vgg_level_bwd", "hg_smooth_l1")


def test_entry_points_agree_between_header_bindings_and_library():
    abi = importlib.import_module("3dhumangan_b200.abi")
    importlib.import_module("3dhumangan_b200.build").build()
    text = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "hg3d.h")).read(), flags=re.S)
    lib = abi.lib()
    for name in ENTRIES:
        m = re.search(r"\bint\s+" + name + r"\s*\(([^)]*)\)", text)
        assert m, name
        nargs = len([a for a in m.group(1).split(",") if a.strip()])
        assert len(abi.SIGNATURES[name][1]) == nargs, name
        assert hasattr(lib, name)
    p = abi.c_void_p(16)
    assert lib.hg_vgg_input(p, 2, 1, 8, 8, p, p, p, 8, 8, None) == 1 and b"channels" in lib.hg_last_error()
    assert lib.hg_vgg_level_bwd(p, p, None, None, 1.0, p, 4, 8, 8, None) == 1
    assert lib.hg_maxpool2x2(p, p, 4, 1, 8, None) == 1
    assert lib.hg_smooth_l1(p, p, 0, p, p, None) == 1


def test_missing_weight_file_raises_and_never_downloads(monkeypatch, tmp_path):
    mod = importlib.import_module("3dhumangan_b200.perceptual")

    def no_download(*a, **k):
        pytest.fail("torch.hub.load_state_dict_from_url was called")
    monkeypatch.setattr(torch.hub, "load_state_dict_from_url", no_download)
    monkeypatch.setattr(torch.hub, "get_dir", lambda: str(tmp_path / "hub"))
    want = os.path.join(str(tmp_path / "hub"), "checkpoints", "vgg16-397923af.pth")
    assert mod.default_weights_path() == want
    with pytest.raises(RuntimeError, match=re.escape(want)):
        mod.VGGPerceptualLoss()
    with pytest.raises(RuntimeError, match="not found"):
        mod.VGGPerceptualLoss(weights=str(tmp_path / "elsewhere.pth"))
    # the cached file in torchvision's keys (with the classifier a real file carries) is read from there
    os.makedirs(os.path.dirname(want))
    sd = dict(pp.seeded_vgg16_state(2), **{"classifier.0.weight": torch.zeros(2, 2)})
    torch.save(sd, want)
    m = mod.VGGPerceptualLoss(resize=False)
    assert torch.equal(m.blocks[3]._modules["21"].weight, sd["features.21.weight"]) and m.resize is False


def test_product_path_has_no_cpu_fallback():
    mod = importlib.import_module("3dhumangan_b200.perceptual")
    m = mod.VGGPerceptualLoss(weights=pp.seeded_vgg16_state(0))
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(RuntimeError, match="CUDA|sm_90a|no CPU path"):
        m(torch.rand(1, 3, 32, 32, requires_grad=True), torch.rand(1, 3, 32, 32))


def test_dropin_import_binds_this_package():
    code = "\n".join([
        "import sys",
        "sys.path.insert(0, %r); sys.path.insert(0, %r)" % (os.path.join(ROOT, "3dhumangan_b200", "dropin"), ROOT),
        "import importlib",
        "from lib.components.perceptual_loss import VGGPerceptualLoss",
        "assert VGGPerceptualLoss is importlib.import_module('3dhumangan_b200.perceptual').VGGPerceptualLoss",
        "print('ok')"])
    out = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0 and "ok" in out.stdout, out.stderr[-2000:]
