"""bias_act / upfirdn2d (sm_90a) against the restated reference implementations."""
import importlib

import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("act", ["linear", "relu", "lrelu", "tanh", "sigmoid", "elu", "selu", "softplus", "swish"])
@pytest.mark.parametrize("shape,dim", [((7, 256), 1), ((3, 5, 11, 13), 1), ((4, 9, 6), 2)])
def test_bias_act(port, act, shape, dim):
    ba = importlib.import_module("3dhumangan_b200.ops.bias_act")
    g = torch.Generator().manual_seed(1)
    x = torch.randn(*shape, generator=g) * 3
    b = torch.randn(shape[dim], generator=g)
    for clamp in (None, 0.7):
        ref = port.bias_act_ref(x, b, dim=dim, act=act, clamp=clamp)
        with torch.no_grad():
            got = ba.bias_act(x.cuda(), b.cuda(), dim=dim, act=act, clamp=clamp).cpu()
        assert torch.allclose(got, ref, rtol=2e-6, atol=2e-6), (act, clamp, (got - ref).abs().max())
    with torch.no_grad():
        got = ba.bias_act(x.cuda(), None, act=act, gain=0.5, alpha=0.1).cpu()
    assert torch.allclose(got, port.bias_act_ref(x, None, act=act, gain=0.5, alpha=0.1), rtol=2e-6, atol=2e-6)


def test_upfirdn2d_matches_reference_semantics(port):
    uf = importlib.import_module("3dhumangan_b200.ops.upfirdn2d")
    g = torch.Generator().manual_seed(2)
    x = torch.randn(2, 3, 17, 13, generator=g)
    f2 = uf.setup_filter([1, 3, 3, 1])
    f1 = uf.setup_filter([0.1, 0.2, 0.3, 0.25, 0.1, 0.05, 0.0, 0.0, 0.1, 0.2, 0.05, 0.02])   # 12 taps -> separable
    assert f2.ndim == 2 and f1.ndim == 1
    cases = [dict(f=f2), dict(f=f2, up=2, padding=[2, 1, 2, 1], gain=4), dict(f=f2, down=2, padding=1),
             dict(f=f2, up=(2, 1), down=(1, 2), padding=[1, 2, 0, 3], flip_filter=True),
             dict(f=f1, up=2, padding=[6, 5, 6, 5], gain=4), dict(f=f1, down=2, padding=[1, 2, 5, 5], flip_filter=True), dict(f=f2, down=2, padding=[-1, -2, 0, -3]),
             dict(f=None, up=1)]
    for kw in cases:
        ref = port.upfirdn2d_ref(x, **kw)
        with torch.no_grad():
            got = uf.upfirdn2d(x.cuda(), **{k: (v.cuda() if torch.is_tensor(v) else v) for k, v in kw.items()}).cpu()
        assert got.shape == ref.shape, (kw, got.shape, ref.shape)
        assert torch.allclose(got, ref, rtol=1e-5, atol=1e-5), kw


def test_upsample_downsample_wrappers(port):
    """The only call shapes of the reference: augment.py:314,325 (sym6 filter, up=2 / down=2 with negative padding)."""
    uf = importlib.import_module("3dhumangan_b200.ops.upfirdn2d")
    sym6 = [0.015404109327027373, 0.0034907120842174702, -0.11799011114819057, -0.048311742585633, 0.4910559419267466,
            0.787641141030194]
    f = uf.setup_filter(sym6 + sym6[::-1])
    x = torch.randn(2, 3, 40, 24, generator=torch.Generator().manual_seed(3))
    with torch.no_grad():
        up = uf.upsample2d(x.cuda(), f.cuda(), up=2)
        dn = uf.downsample2d(up, f.cuda(), down=2, padding=-6, flip_filter=True)
    fw = f.numel()
    p_up = [(fw + 1) // 2, (fw - 2) // 2] * 2
    ref_up = port.upfirdn2d_ref(x, f, up=2, padding=p_up, gain=4)
    assert torch.allclose(up.cpu(), ref_up, rtol=1e-5, atol=1e-5)
    p_dn = [-6 + (fw - 1) // 2, -6 + (fw - 2) // 2] * 2
    ref_dn = port.upfirdn2d_ref(ref_up, f, down=2, padding=p_dn, flip_filter=True)
    assert torch.allclose(dn.cpu(), ref_dn, rtol=1e-5, atol=1e-5)


@pytest.mark.parametrize("act", ["linear", "relu", "lrelu", "tanh", "sigmoid", "elu", "selu", "softplus", "swish"])
def test_bias_act_gradients(port, act):
    """First- and second-order gradients (bias_act.py:124-207) against autograd through the restated reference."""
    ba = importlib.import_module("3dhumangan_b200.ops.bias_act")
    g = torch.Generator().manual_seed(4)
    x0 = torch.randn(3, 5, 7, 4, generator=g) * 1.5
    if act in ("relu", "lrelu", "elu", "selu"):          # keep away from the kink, where one-sided derivatives differ
        x0 = torch.where(x0.abs() < 0.05, torch.full_like(x0, 0.3), x0)
    b0 = torch.randn(5, generator=g) * 0.1
    w = torch.randn(3, 5, 7, 4, generator=g)
    for clamp in (None, 0.9):
        outs = []
        for dev, fn in (("cpu", port.bias_act_ref), ("cuda", ba.bias_act)):
            x = x0.to(dev).requires_grad_(True)
            b = b0.to(dev).requires_grad_(True)
            y = fn(x, b, dim=1, act=act, clamp=clamp)
            gx, gb = torch.autograd.grad((y * w.to(dev)).sum(), (x, b), create_graph=True)
            # a scalar of the first-order gradients -> second-order terms towards x, b (R1-style penalty)
            pen = (gx * gx).sum() + (gb * gb).sum()
            hx, hb = torch.autograd.grad(pen, (x, b), allow_unused=True) if pen.requires_grad else (None, None)
            hx = torch.zeros_like(x) if hx is None else hx
            hb = torch.zeros_like(b) if hb is None else hb
            outs.append([t.detach().cpu() for t in (y, gx, gb, hx, hb)])
        for name, r, c in zip(("y", "dx", "db", "d2x", "d2b"), *outs):
            assert torch.allclose(c, r, rtol=2e-4, atol=2e-5), (act, clamp, name, (c - r).abs().max())


def test_upfirdn2d_gradients(port):
    """The adjoint pass (and its own adjoint) against autograd through the restated reference."""
    uf = importlib.import_module("3dhumangan_b200.ops.upfirdn2d")
    g = torch.Generator().manual_seed(5)
    x0 = torch.randn(2, 3, 14, 10, generator=g)
    f2 = uf.setup_filter([1, 3, 3, 1])
    f1 = uf.setup_filter([0.1, 0.2, 0.3, 0.25, 0.1, 0.05, 0.0, 0.0, 0.1, 0.2, 0.05, 0.02])
    cases = [dict(f=f2), dict(f=f2, up=2, padding=[2, 1, 2, 1], gain=4), dict(f=f2, down=2, padding=1),
             dict(f=f2, up=(2, 1), down=(1, 2), padding=[1, 2, 0, 3], flip_filter=True),
             dict(f=f1, up=2, padding=[6, 5, 6, 5], gain=4), dict(f=f1, down=2, padding=[1, 2, 5, 5], flip_filter=True),
             dict(f=f2, down=2, padding=[-1, -2, 0, -3]), dict(f=f2, up=3, down=2, padding=[2, 0, 1, 3])]
    for kw in cases:
        res = []
        for dev, fn in (("cpu", port.upfirdn2d_ref), ("cuda", uf.upfirdn2d)):
            x = x0.to(dev).requires_grad_(True)
            y = fn(x, **{k: (v.to(dev) if torch.is_tensor(v) else v) for k, v in kw.items()})
            w = torch.randn(y.shape, generator=torch.Generator().manual_seed(6)).to(dev).requires_grad_(True)
            (gx,) = torch.autograd.grad((y * w).sum(), x, create_graph=True)
            (gw,) = torch.autograd.grad((gx * gx).sum(), w)       # double backward: adjoint of the adjoint
            res.append((gx.detach().cpu(), gw.detach().cpu()))
        assert torch.allclose(res[1][0], res[0][0], rtol=1e-5, atol=1e-5), kw
        assert torch.allclose(res[1][1], res[0][1], rtol=1e-4, atol=1e-4), kw


def test_spectral_norm_kernel_matches_torch():
    """hg_spectral_norm: a table of matrices of different shapes in one launch vs torch.nn.utils.spectral_norm's arithmetic
    (one power iteration in training mode with in-place buffer updates; stored vectors in eval mode)."""
    import importlib
    import torch.nn.functional as F
    abi = importlib.import_module("3dhumangan_b200.abi")
    g = torch.Generator().manual_seed(0)
    shapes = [(256, 256), (128, 27), (512, 4608), (64, 2304), (3, 64), (256, 1152)]
    ws = [torch.randn(n, k, generator=g).cuda() / k ** 0.5 for n, k in shapes]
    us = [F.normalize(torch.randn(n, generator=g), dim=0).cuda() for n, _ in shapes]
    vs = [F.normalize(torch.randn(k, generator=g), dim=0).cuda() for _, k in shapes]
    for training in (True, False, True):
        ref = []
        for w, u, v in zip(ws, us, vs):
            wd, ud, vd = w.double(), u.double(), v.double()
            if training:
                vd = F.normalize(wd.t() @ ud, dim=0, eps=1e-12)
                ud = F.normalize(wd @ vd, dim=0, eps=1e-12)
            ref.append((ud, vd, torch.dot(ud, wd @ vd)))
        inv = abi.spectral_norm(ws, us, vs, training)
        torch.cuda.synchronize()
        for i, (ud, vd, sig) in enumerate(ref):
            assert abs(float(inv[i]) * float(sig) - 1.0) < 2e-6, (i, training)
            assert float((us[i].double() - ud).norm()) < 2e-6 and float((vs[i].double() - vd).norm()) < 2e-6, (i, training)
    a = abi.spectral_norm(ws, us, vs, False)
    b = abi.spectral_norm(ws, us, vs, False)
    assert torch.equal(a, b)                                 # deterministic summation order


def test_dense_forward_backward_matches_torch():
    """ops.dense (the mapping networks' layers on hg_linear): value, dX, dW, db vs fp64 torch, incl. contraction > 256."""
    import importlib
    dn = importlib.import_module("3dhumangan_b200.ops.dense")
    g = torch.Generator().manual_seed(1)
    for (M, K, N, gain) in [(8, 256, 256, 1.0), (1, 256, 256, 1.0), (5, 256, 2048, 0.01 / 16), (16, 420, 420, 1.0), (300, 64, 96, 2.0)]:
        x = torch.randn(M, K, generator=g)
        w = torch.randn(N, K, generator=g) / K ** 0.5
        b = torch.randn(N, generator=g)
        gy = torch.randn(M, N, generator=g)
        xr, wr, br = (t.double().requires_grad_(True) for t in (x, w, b))
        yr = xr @ (wr * gain).t() + br
        yr.backward(gy.double())
        xc, wc, bc = (t.cuda().requires_grad_(True) for t in (x, w, b))
        y = dn.dense(xc, wc, bc, gain=gain)
        y.backward(gy.cuda())
        torch.cuda.synchronize()
        rel = lambda a_, r_: float((a_.detach().cpu().double() - r_).norm() / r_.norm())
        assert rel(y, yr.detach()) < 2e-5, (M, K, N)
        assert rel(xc.grad, xr.grad) < 2e-5 and rel(wc.grad, wr.grad) < 2e-5 and rel(bc.grad, br.grad) < 1e-5, (M, K, N)


@pytest.mark.parametrize("width", [201, 204])
@pytest.mark.parametrize("taps", [4, 8, 12, 16])
def test_upfirdn2d_fused_separable_multi_tile(port, taps, width):
    """The fused two-axis kernel (hg_upfirdn2d_sep2) over many tiles, both padding parities, negative padding (crop),
    flip on / off, sizes that are not multiples of the tile -- against the reference's zero-insert / pad / conv / decimate.
    width 204: rows are 16-byte aligned, the input tiles are staged by TMA (out-of-bounds zero fill = the padding);
    width 201: the 4-byte cp.async staging."""
    uf = importlib.import_module("3dhumangan_b200.ops.upfirdn2d")
    g = torch.Generator().manual_seed(10 + taps)
    f = uf.setup_filter(torch.rand(taps, generator=g) - 0.3, separable=True)
    assert f.ndim == 1
    x = torch.randn(2, 3, 150, width, generator=g)
    cases = []
    for pad in ([taps // 2, taps // 2 - 1] * 2, [taps // 2 + 1, taps // 2, taps // 2 - 2, taps // 2 + 3], [-3, taps, taps - 1, -2]):
        for flip in (False, True):
            cases.append(dict(f=f, up=2, padding=pad, flip_filter=flip, gain=4))
            cases.append(dict(f=f, down=2, padding=pad, flip_filter=flip, gain=1.5))
    for kw in cases:
        ref = port.upfirdn2d_ref(x, **kw)
        with torch.no_grad():
            got = uf.upfirdn2d(x.cuda(), **{k: (v.cuda() if torch.is_tensor(v) else v) for k, v in kw.items()}).cpu()
        assert got.shape == ref.shape, (kw, got.shape, ref.shape)
        assert torch.allclose(got, ref, rtol=2e-5, atol=2e-5), (kw["padding"], kw.get("up"), kw["flip_filter"], (got - ref).abs().max())


@pytest.mark.parametrize("case", ["balanced", "background_only", "prior"])
def test_seg_ce_balanced_matches_trainer_formula(case):
    """hg_seg_ce (one pass: loss + gradient) vs the torch restatement of PhaseTrainer._calculate_segmentation_loss
    (train_step.segmentation_loss, itself pinned to the reference's values by tests/golden/seg_loss.npz on the CPU)."""
    ts = importlib.import_module("3dhumangan_b200.train_step")
    to = importlib.import_module("3dhumangan_b200.ops.trainer_ops")
    g = torch.Generator().manual_seed(11)
    B, L, H, W = 3, 26, 40, 56
    logits = (torch.randn(B, L, H, W, generator=g) * 3).cuda()
    if case == "background_only":
        gt = torch.zeros(B, H, W, dtype=torch.int64).cuda()
    else:
        gt = torch.randint(0, L, (B, H, W), generator=g)
        gt[gt == 7] = 0                                    # a class that never occurs
        gt = gt.cuda()
    prior = [1.0 + 0.1 * i for i in range(L)] if case == "prior" else None
    a = logits.clone().requires_grad_(True)
    ref = ts.segmentation_loss(a, gt, L, prior)
    ref.backward()
    b = logits.clone().requires_grad_(True)
    got = to.seg_ce_balanced(b, gt, L, prior)
    (got * 1.7).backward()
    torch.cuda.synchronize()
    assert abs(float(got) - float(ref)) < 2e-6 * max(1.0, abs(float(ref))), (float(got), float(ref))
    assert float((b.grad / 1.7 - a.grad).abs().max()) < 2e-6 * float(a.grad.abs().max()) + 1e-12


@pytest.mark.parametrize("betas,wd", [((0.0, 0.9), 0.0), ((0.9, 0.999), 0.01)])
def test_fused_adam_clip_ema_matches_torch(betas, wd):
    """FusedAdam.step(clip_max_norm, ema) vs clip_grad_norm_ + torch.optim.Adam + the reference's EMA update, two parameter
    groups with different learning rates, tensors larger than one chunk, a parameter without gradient; state_dict interchange."""
    to = importlib.import_module("3dhumangan_b200.ops.trainer_ops")
    ts = importlib.import_module("3dhumangan_b200.train_step")
    g = torch.Generator().manual_seed(12)
    shapes = [(300, 41), (7,), (5000, 3), (64, 64, 1, 1), (3,)]
    p_ref = [torch.nn.Parameter(torch.randn(*s, generator=g).cuda()) for s in shapes]
    p_fus = [torch.nn.Parameter(p.detach().clone()) for p in p_ref]
    groups = lambda ps: [{"params": ps[:2], "name": "a"}, {"params": ps[2:], "name": "b", "lr": 3e-3}]
    o_ref = torch.optim.Adam(groups(p_ref), lr=1e-3, betas=betas, weight_decay=wd)
    o_fus = to.FusedAdam(groups(p_fus), lr=1e-3, betas=betas, weight_decay=wd)
    e_ref = ts.ParameterEMA(p_ref[::-1], decay=0.999)       # the EMA's own order differs from the optimiser's group order
    e_fus = ts.ParameterEMA(p_fus[::-1], decay=0.999)
    for it in range(4):
        for i, (a, b) in enumerate(zip(p_ref, p_fus)):
            if i == 4 and it % 2 == 0:                    # a parameter that gets no gradient in some steps
                a.grad = b.grad = None
                continue
            gr = torch.randn(a.shape, generator=g).cuda() * (10.0 if it == 1 else 0.1)
            a.grad, b.grad = gr.clone(), gr.clone()
        n_ref = torch.nn.utils.clip_grad_norm_(p_ref, 1.0)
        o_ref.step()
        e_ref.update(p_ref[::-1])
        o_fus.step(clip_max_norm=1.0, ema=e_fus, ema_params=p_fus[::-1])
        torch.cuda.synchronize()
        assert abs(float(o_fus.last_grad_norm) - float(n_ref)) < 1e-5 * float(n_ref)
        for a, b in zip(p_ref, p_fus):
            assert float((a - b).abs().max()) < 2e-6 * float(a.abs().max()), it
            if a.grad is not None:
                assert torch.allclose(a.grad, b.grad, rtol=1e-5, atol=1e-8)           # clipped in place on both sides
        for a, b in zip(e_ref.shadow_params, e_fus.shadow_params):
            assert float((a - b).abs().max()) < 2e-6 * float(a.abs().max())
    assert e_ref.num_updates == e_fus.num_updates == 4
    sd = o_ref.state_dict()
    o_fus.load_state_dict(sd)                              # same schema: step / exp_avg / exp_avg_sq, param_groups with names
    assert [g_["name"] for g_ in o_fus.param_groups] == ["a", "b"]
    for k, v in o_fus.state_dict()["state"].items():
        assert set(v) == {"step", "exp_avg", "exp_avg_sq"}
