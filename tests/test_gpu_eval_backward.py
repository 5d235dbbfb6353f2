"""Gradients through the generator in eval() mode: running-statistics BatchNorm, spectral norm from the stored u / v,
`last_back=True`, a frozen generator differentiated w.r.t. its input alone -- against eval-mode autograd through the
oracle (the whole generator; tests/test_oracle_pin_eval_grads.py pins that to the reference).  The compositing kernels'
`last_back` forward and gradient are checked launch by launch in tests/test_gpu_render_kernels.py."""
import importlib

import pytest
import torch

import hierarchical_oracle

pytestmark = pytest.mark.gpu

WGRAD = ("hg_wgrad_blocked", "hg_act_wgrad_blocked", "hg_spade_bwd_wgrad", "hg_synth_input_bwd", "hg_render_heads_bwd")


def _rel(a, b):
    return ((a - b).norm() / b.norm().clamp_min(1e-30)).item()


# ----------------------------------------------------------------------------------------------------------------------
# 1.-3. whole generator
# ----------------------------------------------------------------------------------------------------------------------
def _generator(pkg, port, C, mode, legacy, last_back, hier=False, seed=21):
    """An eval-mode generator whose running statistics and u / v come from three train-mode forwards (at random
    initialisation the eval output overflows: the running variance is still 1)."""
    gen = importlib.import_module("3dhumangan_b200.modules.generator")
    cfg = pkg.configs.baseline_config("tiny")
    cfg.update(hidden_dim=C, feature_dim=C, map3d_mode=mode, legacy_mode=legacy, gen_height=16, gen_width=16, render_height=4,
               render_width=4, num_steps=32, nerf_noise=0.0, last_back=last_back, hierarchical_sample=hier)
    G = gen.Map3DGenerator(**cfg).cuda()
    G.load_state_dict(port.init_generator_params(cfg, seed=seed, sigma_gain=200.0, sigma_bias=1.0), strict=True)
    G.set_device(torch.device("cuda:0"))
    G.train()
    cond = pkg.synthetic.make_conditions(2, seed=22)
    cg = {k: v.cuda() for k, v in cond.items()}
    torch.manual_seed(5)
    with torch.no_grad():
        for _ in range(3):
            G(torch.randn(2, cfg["latent_dim"], device="cuda"), cg, **dict(cfg, last_back=False))
    G.eval()
    return G, cfg, cond, cg


def _record(monkeypatch, abi):
    names = []
    orig = abi.call
    monkeypatch.setattr(abi, "call", lambda name, *a, **k: (names.append(name), orig(name, *a, **k))[1])
    return names


@pytest.mark.parametrize("C,mode,legacy,last_back,hier", [
    (256, "mixed", False, True, False), (256, "isolated", True, False, False), (384, "mixed", False, True, False),
    (420, "isolated", True, True, False), (256, "mixed", False, True, True), (420, "isolated", True, True, True)])
def test_generator_eval_backward_matches_oracle(pkg, port, monkeypatch, C, mode, legacy, last_back, hier):
    rng = importlib.import_module("3dhumangan_b200.rng")
    G, cfg, cond, cg = _generator(pkg, port, C, mode, legacy, last_back, hier=hier)
    B = 2
    params = {k: v.detach().cpu().clone() for k, v in G.state_dict().items()}
    z = torch.randn(B, cfg["latent_dim"], generator=torch.Generator().manual_seed(23))
    wgt = torch.randn(B, 3, 16, 16, generator=torch.Generator().manual_seed(24))
    wgt_r = torch.randn(B, 3, 4, 4, generator=torch.Generator().manual_seed(25))
    torch.manual_seed(3)
    if hier:
        u, noise = rng.draw_hierarchical_noise(B, 16, 32, "cpu", cfg["sample_dist"])
        nd = rng.HierarchicalNoise(noise.coarse.cuda(), noise.u_pdf.cuda(), noise.final.cuda())
        monkeypatch.setattr(rng, "draw_hierarchical_noise", lambda *a, **k: (u.cuda(), nd))
    else:
        u, noise = rng.draw_render_noise(B, 16, 32, "cpu", cfg["sample_dist"])
        monkeypatch.setattr(rng, "draw_render_noise", lambda *a, **k: (u.cuda(), noise.cuda()))
    loss_of = lambda o, dev: (o["rgbs"] * wgt.to(dev)).sum() + (o["rgbs_render"] * wgt_r.to(dev)).sum()

    # through the mapped space, so that d freq / d phase / d style are visible next to d z
    zc = z.cuda().requires_grad_(True)
    freq, phase = G.neural_field_mapping_network(zc if cfg.get("neural_field_latent_input", True) else torch.zeros_like(zc))
    styles = G.synthesis_mapping_network(zc)[1]
    for t in (freq, phase, styles):
        t.retain_grad()
    out = G.synthesize(freq, phase, styles, cg, **cfg)
    assert out["rgbs"].requires_grad and out["rgbs_render"].requires_grad
    loss_of(out, "cuda").backward()
    with torch.no_grad():
        out_ng = G(z.cuda(), cg, **cfg)
    torch.cuda.synchronize()
    # the same image as the inference path: at 256 its fused kernels sum in another order (1e-4); on the padded path the
    # kernels are the same and only the BatchNorm tables differ, hg_bn_finalize folding them in fp32 where the taped
    # forward folds them in fp64 (measured 1.6e-5 / 1.9e-5 at 384 / 420, hence 3e-5 rather than 1e-5)
    tol_fwd = 1e-4 if C == 256 else 3e-5
    assert _rel(out["rgbs"].detach(), out_ng["rgbs"]) < tol_fwd
    assert _rel(out["rgbs_render"].detach(), out_ng["rgbs_render"]) < tol_fwd
    # no buffer moved
    for k, v in G.state_dict().items():
        assert torch.equal(v.cpu(), params[k]), k

    trainable = {n for n, _ in G.named_parameters()}
    pc = {n: (v.clone().requires_grad_(True) if n in trainable else v.clone()) for n, v in params.items()}
    zr = z.clone().requires_grad_(True)
    fr, pr = (t.detach().requires_grad_(True) for t in
              port.mapping_network(pc, zr if cfg.get("neural_field_latent_input", True) else torch.zeros_like(zr)))
    sr = port.synthesis_mapping(pc, zr)
    sr.retain_grad()
    monkeypatch.setattr(port, "mapping_network", lambda *a, **k: (fr, pr))
    monkeypatch.setattr(port, "synthesis_mapping", lambda *a, **k: sr)
    if hier:        # the oracle's hierarchical render at the device's own fine depths (they carry no gradient)
        merged = importlib.import_module("3dhumangan_b200.modules.hierarchical").merged_records
        fz = merged(G._params(), freq.detach(), phase.detach(), cg, G._cfg_for(cfg, 4, 4), u.cuda(), nd, want_fine=True)["fine_z"].cpu()
        monkeypatch.setattr(port, "render", lambda p, f, ph, c, k, uu, nn, dtype=None:
                            hierarchical_oracle.render(p, f, ph, c, k, uu, nn, fine_z=fz, dtype=dtype)[:5])
    ref = port.generator_forward(pc, zr, cond, cfg, u, noise, training=False)
    assert (out["rgbs"].detach().cpu() - ref["rgbs"].detach()).abs().max() / ref["rgbs"].abs().max() < 1e-3
    loss_of(ref, "cpu").backward()
    assert _rel(freq.grad.cpu(), fr.grad) < 2e-2
    assert _rel(phase.grad.cpu(), pr.grad) < 2e-2
    assert _rel(styles.grad.cpu().reshape(sr.grad.shape), sr.grad) < 2e-2
    assert _rel(zc.grad.cpu(), zr.grad) < 2e-2
    worst = {}
    for n, p in G.named_parameters():
        if n.startswith(("neural_field_mapping", "synthesis_mapping")) or pc[n].grad is None or pc[n].grad.norm() == 0:
            continue          # the mapping networks were cut off the oracle's graph above
        assert p.grad is not None and p.grad.shape == p.shape, n
        worst[n] = _rel(p.grad.cpu().double(), pc[n].grad.double())
    assert len(worst) > 100
    med = sorted(worst.values())[len(worst) // 2]
    top = max(pc[n].grad.norm() for n in worst)
    # the sigma bias sums dsig over every ray sample, its terms cancel: see tests/test_gpu_train_wide.py
    over = {n: e for n, e in worst.items() if e > 0.1 and pc[n].grad.norm() > 1e-6 * top and n != "neural_field.sigma_layer.bias"}
    print(f"hidden {C} eval{' hierarchical' if hier else ''}: median {med:.2e}, over 0.1: {sorted(over.items(), key=lambda t: -t[1])[:6]}")
    assert med < 2e-2 and not over, (med, over)


@pytest.mark.parametrize("C,hier", [(256, False), (420, False), (420, True)])
def test_frozen_generator_launches_no_weight_gradient(pkg, port, monkeypatch, C, hier):
    abi = importlib.import_module("3dhumangan_b200.abi")
    G, cfg, cond, cg = _generator(pkg, port, C, "isolated", True, True, hier=hier)
    bufs = {k: v.clone() for k, v in G.named_buffers()}
    z = torch.randn(2, cfg["latent_dim"], generator=torch.Generator().manual_seed(23)).cuda()
    wgt = torch.randn(2, 3, 16, 16, generator=torch.Generator().manual_seed(24)).cuda()

    def run(frozen_prefixes):
        for n, p in G.named_parameters():
            p.requires_grad_(not n.startswith(frozen_prefixes))
            p.grad = None
        zc = z.clone().requires_grad_(True)
        torch.manual_seed(9)
        out = G(zc, cg, **cfg)
        assert out["rgbs"].grad_fn is not None
        names = _record(monkeypatch, abi)
        (out["rgbs"] * wgt).sum().backward()
        monkeypatch.undo()
        torch.cuda.synchronize()
        return zc.grad, [n for n in names if n in WGRAD]

    dz_all, w_all = run(("no such prefix",))
    dz_frozen, w_frozen = run(("",))
    assert w_all and not w_frozen, w_frozen
    assert all(p.grad is None for p in G.parameters())
    assert torch.isfinite(dz_all).all() and dz_all.abs().max() > 0
    assert _rel(dz_frozen, dz_all) < 1e-4      # the same launches on the data path; their atomic sums differ from run to run
    dz_part, w_part = run(("neural_field.",))
    renderer = [n for n in w_all if n in ("hg_act_wgrad_blocked", "hg_render_heads_bwd")]
    assert renderer and sorted(w_part) == sorted(n for n in w_all if n not in ("hg_act_wgrad_blocked", "hg_render_heads_bwd"))
    assert all(p.grad is None for n, p in G.named_parameters() if n.startswith("neural_field."))
    assert sum(p.grad is not None for n, p in G.named_parameters() if n.startswith("synthesis_network.")) > 100
    for k, v in G.named_buffers():
        assert torch.equal(v, bufs[k]), k


def test_eval_backward_issues_no_collective(pkg, port, monkeypatch):
    """Eval-mode BatchNorm is local: with a 2-rank process group visible, forward and backward issue no collective -- neither
    through torch.distributed nor through the statistics helper the modules import by name."""
    import torch.distributed as dist
    G, cfg, cond, cg = _generator(pkg, port, 384, "mixed", False, True)
    monkeypatch.setattr(dist, "is_initialized", lambda: True)
    monkeypatch.setattr(dist, "get_world_size", lambda group=None: 2)

    def refuse(*a, **k):
        raise AssertionError("collective issued in eval mode")
    for name in ("all_reduce", "all_gather", "all_gather_into_tensor", "reduce_scatter", "broadcast", "reduce", "barrier"):
        monkeypatch.setattr(dist, name, refuse)
    for module in ("synthesis_ops", "synthesis_train", "wide_ops"):      # the helper is imported by name into these
        monkeypatch.setattr(importlib.import_module("3dhumangan_b200.modules." + module), "all_reduce_stats", refuse)
    z = torch.randn(2, cfg["latent_dim"], device="cuda", requires_grad=True)
    out = G(z, cg, **cfg)
    out["rgbs"].square().sum().backward()
    torch.cuda.synchronize()
    assert torch.isfinite(z.grad).all()


def test_eval_mode_refusals(pkg, port):
    """What is still not built raises: a second backward on a released tape, records re-used across sizes; train() mode keeps
    refusing `last_back` (tests/test_gpu_train_wide.py::test_wide_surface_guards)."""
    G, cfg, cond, cg = _generator(pkg, port, 256, "mixed", False, True)
    z = torch.randn(2, cfg["latent_dim"], device="cuda", requires_grad=True)
    out = G(z, cg, **cfg)
    out["rgbs"].sum().backward(retain_graph=True)
    with pytest.raises(RuntimeError, match="released by a previous backward"):
        out["rgbs"].sum().backward()
    freq, phase = G.neural_field_mapping_network(torch.zeros_like(z))
    styles = G.synthesis_mapping_network(z)[1]
    rec = G.synthesize(freq, phase, styles, cg, **cfg)["hg_records"]
    with pytest.raises(RuntimeError, match="hg_records"):
        G.synthesize(freq, phase, styles, cg, **dict(cfg, num_steps=16, hg_records=rec))
    with pytest.raises(RuntimeError, match="hg_records"):
        G.synthesize(freq, phase, styles, cg, **dict(cfg, hierarchical_sample=True, hg_records=rec))
    again = G.synthesize(freq, phase, styles, cg, **dict(cfg, hg_records=rec))
    assert again["hg_records"][0].data_ptr() == rec[0].data_ptr()
    G.train()
    with pytest.raises(RuntimeError, match="last_back=True is an inference-only setting"):
        G(z, cg, **cfg)
