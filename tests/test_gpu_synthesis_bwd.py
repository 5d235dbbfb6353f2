"""The synthesis network's backward (modules/synthesis_train.py::synthesis_backward) against fp64 autograd through the
restated reference (SPADE2d/SPADEBlock, map3d_layers.py:176-238).  Its kernels are tested launch by launch in
tests/test_gpu_synthesis_bwd_kernels.py."""
import importlib

import pytest
import torch

pytestmark = pytest.mark.gpu

C = 256


def _planar(t, HW):
    B, T, Cc, _ = t.shape
    return t.permute(0, 2, 1, 3).reshape(B, Cc, T * 128)[:, :, :HW]


def _network_case(port, monkeypatch, mod_blocks, mode, Rh, Rw, seed, C=C):
    """Whole-network gradients against fp64 autograd through the restated reference on the CPU, at hidden_dim 256
    (synthesis_train's forward) or a zero-padded width (wide_ops' forward); one backward serves both.

    The gradient is DISCONTINUOUS in the LeakyReLU masks: a pre-activation that rounds to the other side of zero
    changes its contribution by a factor 5, so even torch-fp32 vs torch-fp64 gradients of this network differ by
    1e-3 (block 0) although the forwards agree to 3e-6.  To test the backward kernels rather than that
    sensitivity, the fp64 reference is evaluated with the masks OUR backward differentiates through (rebuilt from
    the saved half-block inputs / exported by the pixel-style branch); the forward itself is compared without help."""
    import torch.nn.functional as TF
    pkg = importlib.import_module("3dhumangan_b200")
    st = importlib.import_module("3dhumangan_b200.modules.synthesis_train")
    wo = importlib.import_module("3dhumangan_b200.modules.wide_ops")
    cfg = pkg.configs.baseline_config("tiny")
    cfg.update(hidden_dim=C, feature_dim=C, gen_height=16, gen_width=24, render_height=Rh, render_width=Rw, mod_blocks=mod_blocks,
               map3d_mode=mode)
    B, Hg, Wg = 2, cfg["gen_height"], cfg["gen_width"]
    HW = Hg * Wg
    params = port.init_generator_params(cfg, seed=seed)
    names = [n for n in params if n.startswith(("synthesis_network.", "synthesis_input."))]
    learn = [n for n in names if not n.endswith(("weight_u", "weight_v", "running_mean", "running_var", "num_batches_tracked"))]
    g = torch.Generator().manual_seed(seed + 1)
    fixed = torch.randn(B, 1, C, generator=g) * 0.5
    fmap = torch.randn(B, C, Rh, Rw, generator=g) * 0.7
    wgt = torch.randn(B, 3, Hg, Wg, generator=g)

    # ---- kernels
    pg = {n: params[n].clone().cuda() for n in names}
    for n in learn:
        pg[n].requires_grad_(True)
    feat_lr = fmap.permute(0, 2, 3, 1).reshape(B, Rh * Rw, C).contiguous().cuda()
    if C == 256:
        rgb, tape = st.synthesis_forward_train(pg, feat_lr, fixed.cuda(), cfg)
    else:
        tape = st.SynthesisTape()
        rgb = wo.synthesis_forward_wide(pg, feat_lr, fixed.cuda(), cfg, training=True, tape=tape)
    tape.keep_masks = True
    dfs, dfeat = st.synthesis_backward(pg, tape, wgt.cuda())
    torch.cuda.synchronize()

    def planar(halves):
        """Per-half tile-blocked activations (batch-shared ones expanded) -> [B,C,HW] without the padded channels."""
        return torch.cat([_planar(t.expand(B, -1, -1, -1), HW) for t in halves], 1)[:, :C].cpu()

    masks, relu_masks = [], []
    for rec in tape.halves:
        if rec["pixel"]:
            masks.append(torch.where(planar(rec["mask"]), 1.0, 0.2).double().reshape(B, C, Hg, Wg))
            relu_masks.append(_planar(rec["mask_a1"], HW).cpu().double().reshape(B, 128, Hg, Wg))     # ReLU of the gamma/beta MLP
            continue
        relu_masks.append(None)
        xp = planar(rec["x"]).double()
        m = torch.cat(rec["mod_d"], -1)[..., :C].double().cpu()
        pre = xp * m[:, 0, :, None] + m[:, 1, :, None]
        masks.append(torch.where(pre > 0, 1.0, 0.2).reshape(B, C, Hg, Wg))

    def oracle(mask_list):
        pc = {n: (params[n].clone().double() if params[n].is_floating_point() else params[n].clone()) for n in names}
        for n in learn:
            pc[n].requires_grad_(True)
        fc = fixed.clone().double().requires_grad_(True)
        fm = fmap.clone().double().requires_grad_(True)
        ii, jj = torch.linspace(-1, 1, Hg).double(), torch.linspace(-1, 1, Wg).double()
        coords = torch.stack([ii[:, None].expand(Hg, Wg), jj[None, :].expand(Hg, Wg)], 0)[None].repeat(B, 1, 1, 1)
        x0 = torch.sin(TF.conv2d(coords, pc["synthesis_input.network.0.weight"], pc["synthesis_input.network.0.bias"]))
        style = TF.interpolate(fm, (Hg, Wg), mode="bilinear")
        with monkeypatch.context() as mp:
            if mask_list is not None:
                it = iter(mask_list)
                mp.setattr(port.F, "leaky_relu", lambda v, slope: v * next(it))
                rit, real_relu = iter(relu_masks), TF.relu

                def relu(v):
                    mk = next(rit)
                    return real_relu(v) if mk is None else v * mk
                mp.setattr(port.F, "relu", relu)
            out = port.synthesis_network(pc, x0, style, fc, cfg, training=True)
        return out, pc, fc, fm

    with torch.no_grad():
        rgb_plain = oracle(None)[0]
    assert (rgb.cpu().double() - rgb_plain).abs().max() / rgb_plain.abs().max() < 2e-4
    rgb_ref, pc, fc, fm = oracle(masks)
    (rgb_ref * wgt.double()).sum().backward()

    def rel(a, b):
        return ((a - b).norm() / b.norm()).item()

    scale = max(pc[n].grad.norm().item() for n in learn if pc[n].grad is not None)
    bad = {}
    for n in learn:
        if pc[n].grad is None:         # e.g. the ToRGB layers of blocks 0-2, which the forward never uses
            assert pg[n].grad is None or float(pg[n].grad.abs().max()) == 0.0, n
            continue
        assert pg[n].grad is not None and pg[n].grad.shape == pg[n].shape, n
        a, b = pg[n].grad.cpu().double(), pc[n].grad.double()
        if b.norm().item() < 1e-9 * scale:      # analytic zeros (a conv bias in front of a BatchNorm)
            err = a.norm().item() / scale
        else:
            err = rel(a, b)
        if err > 5e-4:
            bad[n] = err
    assert not bad, sorted(bad.items(), key=lambda t: -t[1])[:8]
    assert rel(dfs.cpu().double().reshape(-1), fc.grad.reshape(-1)) < 5e-4
    if mod_blocks or mode == "all":
        ref = fm.grad.permute(0, 2, 3, 1).reshape(B, Rh * Rw, C)
        assert rel(dfeat.cpu().double(), ref) < 5e-4
    else:
        assert dfeat is None


def test_synthesis_network_backward_const_style(port, monkeypatch):
    """Block 0 const-style at 256: its data gradient reads the batch-shared synthesis input."""
    _network_case(port, monkeypatch, [], "mixed", 4, 6, 5)


@pytest.mark.parametrize("C", [256, 384, 420])
@pytest.mark.parametrize("mode", ["mixed", "isolated"])
def test_synthesis_network_backward_mixed(port, monkeypatch, mode, C):
    """Blocks 0-2 pixel-style (per-pixel gamma/beta from the up-sampled render features), 3-8 const-style."""
    _network_case(port, monkeypatch, [0, 1, 2], mode, 5, 7, 7, C)
