"""SPADE synthesis network on the wgmma kernels vs the oracle (train-mode BatchNorm, fp32 contract 1e-3)."""
from importlib import import_module

import pytest
import torch
import torch.nn.functional as F

from golden_util import rel_l2

pytestmark = pytest.mark.gpu


def _case(pkg, port, over, seed, B):
    cfg = pkg.configs.baseline_config("C2")
    cfg.update(over)
    params = port.init_generator_params(cfg, seed=seed)
    g = torch.Generator().manual_seed(seed)
    fmap = torch.rand(B, 256, cfg["render_height"], cfg["render_width"], generator=g) * 2 - 0.5
    fstyle = torch.randn(B, 1, 256, generator=g)
    return cfg, params, fmap, fstyle


@pytest.mark.parametrize("over,B,mode,passes,tol", [
    (dict(gen_height=32, gen_width=32, render_height=8, render_width=8), 2, "mixed", 3, 1e-3),
    (dict(gen_height=32, gen_width=32, render_height=8, render_width=8), 2, "isolated", 3, 1e-3),
    (dict(gen_height=32, gen_width=32, render_height=8, render_width=8), 1, "all", 3, 1e-3),
    (dict(gen_height=128, gen_width=96, render_height=24, render_width=18), 2, "mixed", 3, 1e-3),   # >148 tiles
    (dict(gen_height=40, gen_width=25, render_height=8, render_width=5), 2, "mixed", 3, 1e-3),       # ragged tiles
    (dict(gen_height=32, gen_width=32, render_height=8, render_width=8), 2, "mixed", 1, 6e-2),       # plain bf16 mode
])
def test_synthesis_matches_oracle(pkg, port, over, B, mode, passes, tol):
    syn = import_module("3dhumangan_b200.modules.synthesis_ops")
    over = dict(over, map3d_mode=mode)
    cfg, params, fmap, fstyle = _case(pkg, port, over, 21, B)
    Hg, Wg = cfg["gen_height"], cfg["gen_width"]
    stats = {}
    with torch.no_grad():
        style = F.interpolate(fmap, (Hg, Wg), mode="bilinear")
        x0 = port.synthesis_input(params, B, Hg, Wg)
        ref_rgb, ref_int = port.synthesis_network(params, x0, style, fstyle, cfg, training=True, stats_out=stats,
                                                  return_internal=True)
    gp = {k: v.cuda() for k, v in params.items()}
    feat_lr = fmap.permute(0, 2, 3, 1).reshape(B, -1, 256).contiguous().cuda()
    rgb, internal = syn.synthesis_forward(gp, feat_lr, fstyle.cuda(), cfg, training=True, passes=passes, return_internal=True)
    torch.cuda.synchronize()
    for k in range(cfg["synthesis_blocks"]):
        e = rel_l2(internal[f"m3d_{k}"].cpu(), ref_int[f"m3d_{k}"])
        assert e < tol, f"block {k}: rel-L2 {e:.3e}"
    assert rel_l2(rgb.cpu(), ref_rgb) < tol
    if passes == 3:
        # buffers updated like the reference modules do in train mode
        for name in ("synthesis_network.network.m3d_0.spade_0.first_norm.running_mean",
                     "synthesis_network.network.m3d_4.spade_1.first_norm.running_var",
                     "synthesis_network.network.m3d_8.conv_1.weight_u"):
            assert rel_l2(gp[name].cpu(), stats[name]) < 1e-4, name
        assert int(gp["synthesis_network.network.m3d_0.spade_0.first_norm.num_batches_tracked"]) == 1


def test_synthesis_eval_mode_uses_running_stats(pkg, port):
    syn = import_module("3dhumangan_b200.modules.synthesis_ops")
    over = dict(gen_height=32, gen_width=32, render_height=8, render_width=8)
    cfg, params, fmap, fstyle = _case(pkg, port, over, 22, 2)
    # populate plausible running statistics so that eval-mode activations stay O(1)
    for k, v in params.items():
        if k.endswith("running_var"):
            v.fill_(0.5)
        if k.endswith("running_mean"):
            v.fill_(0.1)
    with torch.no_grad():
        style = F.interpolate(fmap, (32, 32), mode="bilinear")
        x0 = port.synthesis_input(params, 2, 32, 32)
        ref = port.synthesis_network(params, x0, style, fstyle, cfg, training=False)
    gp = {k: v.cuda() for k, v in params.items()}
    feat_lr = fmap.permute(0, 2, 3, 1).reshape(2, -1, 256).contiguous().cuda()
    rgb = syn.synthesis_forward(gp, feat_lr, fstyle.cuda(), cfg, training=False, passes=3)
    assert rel_l2(rgb.cpu(), ref) < 1e-3
    assert torch.equal(gp["synthesis_network.network.m3d_0.conv_0.weight_u"].cpu(),
                       params["synthesis_network.network.m3d_0.conv_0.weight_u"])
