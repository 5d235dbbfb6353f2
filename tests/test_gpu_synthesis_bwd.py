"""Backward kernels of the const-style SPADE half-block (csrc/synth.cu kBwd, csrc/synth_bwd.cu) against the
same gradients written with plain torch ops in fp64 (autograd through SPADE2d/SPADEBlock, map3d_layers.py:176-238)."""
import importlib

import pytest
import torch

pytestmark = pytest.mark.gpu

C = 256


def _blocked(t, fill=0.0):
    """[B,C,HW] -> tile-blocked [B,T,C,128]; the rows past the image hold `fill` (zero; NaN = what an uninitialised
    activation buffer may hold there in production: nothing may leak from them)."""
    B, Cc, HW = t.shape
    T = (HW + 127) // 128
    pad = torch.full((B, Cc, T * 128), fill, dtype=t.dtype, device=t.device)
    pad[:, :, :HW] = t
    return pad.reshape(B, Cc, T, 128).permute(0, 2, 1, 3).contiguous()


def _planar(t, HW):
    B, T, Cc, _ = t.shape
    return t.permute(0, 2, 1, 3).reshape(B, Cc, T * 128)[:, :, :HW]


def _case(B, Hg, Wg, seed):
    g = torch.Generator().manual_seed(seed)
    HW = Hg * Wg
    x = torch.randn(B, C, HW, generator=g)
    dout = torch.randn(B, C, HW, generator=g)
    mod = torch.stack([1.0 + 0.5 * torch.randn(B, C, generator=g), 0.5 * torch.randn(B, C, generator=g)], dim=1)   # [B,2,C]
    W = torch.randn(C, C, generator=g) / 16
    return x, dout, mod, W


@pytest.mark.parametrize("B,Hg,Wg", [(2, 24, 20), (3, 32, 32)])
@pytest.mark.parametrize("passes,tol", [(3, 2e-5), (1, 2e-2)])
def test_dgrad(B, Hg, Wg, passes, tol):
    abi = importlib.import_module("3dhumangan_b200.abi")
    x, dout, mod, W = _case(B, Hg, Wg, 1)
    HW = Hg * Wg
    xd, dd = x.double(), dout.double()
    pre = xd * mod[:, 0, :, None].double() + mod[:, 1, :, None].double()
    dy = torch.einsum("oc,bop->bcp", W.double(), dd)
    dpre_ref = dy * torch.where(pre > 0, 1.0, 0.2)
    s1_ref, s2_ref = dpre_ref.sum(2), (dpre_ref * xd).sum(2)

    wimg_t, _ = abi.pack_weight(W.t().contiguous().cuda(), Nb=256)
    xb, db_ = _blocked(x, float("nan")).cuda(), _blocked(dout, float("nan")).cuda()
    dpre = torch.full_like(xb, float("nan"))
    sums = torch.zeros(B, 2, C, dtype=torch.float64, device="cuda")
    T = xb.shape[1]
    abi.spade_bwd_dgrad(db_, xb, T * C * 128, mod.cuda().contiguous(), wimg_t, dpre, sums, B=B, Hg=Hg, Wg=Wg, passes=passes)
    torch.cuda.synchronize()
    got = _planar(dpre, HW).cpu().double()
    # pre-activations within rounding distance of zero may legitimately pick the other slope
    safe = pre.abs() > 1e-5
    err = ((got - dpre_ref) * safe).abs().max() / dpre_ref.abs().max()
    assert err < tol, err
    assert (sums[:, 0].cpu() - s1_ref).abs().max() / s1_ref.abs().max() < 10 * tol
    assert (sums[:, 1].cpu() - s2_ref).abs().max() / s2_ref.abs().max() < 10 * tol


def test_dgrad_shared_input():
    """x with batch stride 0 (the synthesis input is shared by the batch)."""
    abi = importlib.import_module("3dhumangan_b200.abi")
    B, Hg, Wg = 2, 16, 24
    x, dout, mod, W = _case(B, Hg, Wg, 2)
    x = x[:1]
    HW = Hg * Wg
    pre = x.double() * mod[:, 0, :, None].double() + mod[:, 1, :, None].double()
    ref = torch.einsum("oc,bop->bcp", W.double(), dout.double()) * torch.where(pre > 0, 1.0, 0.2)
    wimg_t, _ = abi.pack_weight(W.t().contiguous().cuda(), Nb=256)
    dpre = torch.empty(B, (HW + 127) // 128, C, 128, device="cuda")
    sums = torch.zeros(B, 2, C, dtype=torch.float64, device="cuda")
    abi.spade_bwd_dgrad(_blocked(dout).cuda(), _blocked(x).cuda()[0], 0, mod.cuda().contiguous(), wimg_t, dpre, sums, B=B, Hg=Hg, Wg=Wg)
    got = _planar(dpre, HW).cpu().double()
    assert ((got - ref) * (pre.abs() > 1e-5)).abs().max() / ref.abs().max() < 2e-5


@pytest.mark.parametrize("B,Hg,Wg", [(2, 24, 20), (3, 64, 48)])
@pytest.mark.parametrize("passes,tol", [(3, 2e-5), (1, 2e-2)])
def test_wgrad(B, Hg, Wg, passes, tol):
    abi = importlib.import_module("3dhumangan_b200.abi")
    x, dout, mod, _ = _case(B, Hg, Wg, 3)
    pre = x.double() * mod[:, 0, :, None].double() + mod[:, 1, :, None].double()
    y = torch.where(pre > 0, pre, 0.2 * pre)
    dw_ref = torch.einsum("bop,bcp->oc", dout.double(), y)
    db_ref = dout.double().sum((0, 2))
    xb = _blocked(x, float("nan")).cuda()
    dw, db = abi.spade_bwd_wgrad(_blocked(dout, float("nan")).cuda(), xb, xb.shape[1] * C * 128, mod.cuda().contiguous(), B=B, Hg=Hg,
                                 Wg=Wg, passes=passes)
    torch.cuda.synchronize()
    assert (dw.cpu().double() - dw_ref).abs().max() / dw_ref.abs().max() < tol
    assert (db.cpu().double() - db_ref).abs().max() / db_ref.abs().max() < 1e-5


@pytest.mark.parametrize("with_rgb,with_skip,with_dpre", [(True, True, True), (False, False, True), (True, False, False),
                                                          (False, True, True)])
def test_combine(with_rgb, with_skip, with_dpre):
    abi = importlib.import_module("3dhumangan_b200.abi")
    B, Hg, Wg = 2, 20, 18          # HW = 360: last tile partial, multiple of 4
    HW = Hg * Wg
    g = torch.Generator().manual_seed(4)
    x = torch.randn(B, C, HW, generator=g)
    dpre = torch.randn(B, C, HW, generator=g)
    dskip = torch.randn(B, C, HW, generator=g)
    drgb = torch.randn(B, 3, HW, generator=g)
    rgb_w = torch.randn(3, C, generator=g)
    g1 = torch.randn(B, 2, C, generator=g)
    ak = torch.randn(2, C, generator=g)
    ref = torch.zeros(B, C, HW, dtype=torch.float64)
    if with_dpre:
        ref += dpre.double() * g1[:, 0, :, None].double() + ak[0, None, :, None].double() + ak[1, None, :, None].double() * x.double()
    if with_skip:
        ref += dskip.double()
    if with_rgb:
        ref += torch.einsum("jc,bjp->bcp", rgb_w.double(), drgb.double())
    dw_ref = torch.einsum("bjp,bcp->jc", drgb.double(), x.double())
    xb = _blocked(x).cuda()
    dx = torch.full_like(xb, float("nan"))
    dwrgb = torch.zeros(3, C, dtype=torch.float64, device="cuda")
    abi.spade_bwd_combine(dx, B=B, Hg=Hg, Wg=Wg, dpre=_blocked(dpre).cuda() if with_dpre else None, x=xb,
                          x_bstride=xb.shape[1] * C * 128, g1=g1.cuda() if with_dpre else None, ak=ak.cuda() if with_dpre else None,
                          dskip=_blocked(dskip).cuda() if with_skip else None, drgb=drgb.cuda() if with_rgb else None,
                          rgb_w=rgb_w.cuda() if with_rgb else None, dwrgb=dwrgb if with_rgb else None)
    torch.cuda.synchronize()
    assert torch.isfinite(dx).all()
    assert (dx[:, -1, :, HW % 128:] == 0).all()          # padding pixels of the last tile stay zero
    assert (_planar(dx, HW).cpu().double() - ref).abs().max() < 1e-4
    if with_rgb:
        assert (dwrgb.cpu() - dw_ref).abs().max() / dw_ref.abs().max() < 1e-5


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
