"""Host-side trainer logic pinned against the reference's own code: the five Adam parameter groups of
`PhaseTrainer.init_optimizer` (phase_trainer.py:57-76), the EMA update of `lib/components/ema.py:29-48` and the rest below,
executed by the unmodified reference functions on THIS package's modules (same parameter names by the state_dict contract).
Their results were recorded by tests/golden/make_golden_trainer.py (`golden_util.reference_result`), so the tests need no
reference checkout."""
import copy
import importlib
import os
import sys
import types

import pytest
import torch

from golden_util import reference_result

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.environ.get("HG_REFERENCE", "")


def _reference(modname):
    for p in (os.path.join(ROOT, "oracle", "shims"), REF):
        if p not in sys.path:
            sys.path.insert(0, p)
    return importlib.import_module(modname)


def _modules(pkg):
    gen = importlib.import_module("3dhumangan_b200.modules.generator")
    disc = importlib.import_module("3dhumangan_b200.modules.discriminator")
    cfg = pkg.configs.baseline_config("tiny")
    torch.manual_seed(0)
    return gen.Map3DGenerator(**cfg), disc.UNetDiscriminator(**cfg), cfg


def test_optimizer_groups_match_phase_trainer_init_optimizer(pkg, tmp_path):
    ts = importlib.import_module("3dhumangan_b200.train_step")
    G, D, cfg = _modules(pkg)
    meta = dict(cfg, gen_lr=2e-5, disc_lr=2e-4, betas=(0.0, 0.9),      # (0, 0.9) in configs/map3d.py; this torch wants two floats
                weight_decay=0, appearance_codes_lr_mul=3.0, mapping_net_lr_mul=0.5,
                neural_field_lr_mul=0.25)
    names = {id(p): n for n, p in list(G.named_parameters()) + list(D.named_parameters())}

    def reference():
        me = types.SimpleNamespace(generator_ddp=G, discriminator_ddp=D, output_dir=str(tmp_path), device="cpu")
        _reference("lib.trainers.phase_trainer").PhaseTrainer.init_optimizer(me, meta)    # the reference's own method
        return [[dict(g, params=[names[id(p)] for p in g["params"]]) for g in o.param_groups] for o in (me.optimizer_G, me.optimizer_D)]
    ref_G, ref_D = reference_result("init_optimizer", reference)
    og, od = ts.make_optimizers(G, D, meta, fused=False)
    og_f, od_f = ts.make_optimizers(G, D, meta, fused=True)         # the multi-tensor optimiser keeps the same groups
    for mine in (og, og_f):
        assert len(mine.param_groups) == len(ref_G) == 5
        for a, b in zip(mine.param_groups, ref_G):
            assert a["name"] == b["name"]
            assert a["lr"] == pytest.approx(b["lr"], rel=0, abs=0) and tuple(a["betas"]) == tuple(b["betas"])
            assert a["weight_decay"] == b["weight_decay"] and a["eps"] == b["eps"]
            assert [names[id(p)] for p in a["params"]] == b["params"], a["name"]      # same tensors, same order
    for mine in (od, od_f):
        a, b = mine.param_groups[0], ref_D[0]
        assert len(mine.param_groups) == 1 and a["lr"] == b["lr"] and tuple(a["betas"]) == tuple(b["betas"])
        assert [names[id(p)] for p in a["params"]] == b["params"]
    # every generator parameter is in exactly one group
    ids = [id(p) for g in og.param_groups for p in g["params"]]
    assert len(ids) == len(set(ids)) == len(list(G.parameters()))


def _stats(t):
    """(norm, dot, |dot|) of a tensor with a direction seeded by its size, in fp64."""
    x = t.detach().double().reshape(-1)
    d = torch.randn(x.numel(), generator=torch.Generator().manual_seed(x.numel() % 100003), dtype=torch.float64)
    return [float(x.norm()), float((x * d).sum()), float((x * d).abs().sum())]


def test_parameter_ema_matches_reference_ema(pkg):
    ts = importlib.import_module("3dhumangan_b200.train_step")
    G, _, _ = _modules(pkg)

    def reference():       # the reference's EMA on a copy: num_updates per step, then every shadow tensor as _stats
        G2 = copy.deepcopy(G)
        b = _reference("lib.components.ema").ExponentialMovingAverage(G2.parameters(), decay=0.999)
        gen, nums = torch.Generator().manual_seed(3), []
        for step in range(12):
            with torch.no_grad():
                for q in G2.parameters():
                    q.add_(torch.randn(q.shape, generator=gen) * 0.01)
            b.update(list(G2.parameters()))
            nums.append(b.num_updates)
        return nums, torch.tensor([_stats(t) for t in b.shadow_params], dtype=torch.float64)
    nums, ref = reference_result("ema", reference)
    a = ts.ParameterEMA(G.parameters(), decay=0.999)
    gen = torch.Generator().manual_seed(3)
    for step in range(12):                                          # the num_updates ramp (1+n)/(10+n) and the plateau
        with torch.no_grad():
            for p in G.parameters():
                p.add_(torch.randn(p.shape, generator=gen) * 0.01)
        a.update(list(G.parameters()))
        assert a.num_updates == nums[step]
    assert len(a.shadow_params) == ref.shape[0]

    def check(tensors):    # the elementwise rtol 1e-6 / atol 1e-8 bound, carried over to the norm and the dot product
        for t, (norm, dot, absdot) in zip(tensors, ref.tolist()):
            n, d, _ = _stats(t)
            assert abs(n - norm) <= 1e-6 * norm + 1e-8 * t.numel() ** 0.5, (n, norm)
            assert abs(d - dot) <= 1e-6 * absdot + 1e-8 * 0.8 * t.numel(), (d, dot)       # E|N(0,1)| ~ 0.8 per entry
    check(a.shadow_params)
    # copy_to writes the averages into the parameters that require grad, in order
    a.copy_to(G.parameters())
    check(list(G.parameters()))


@pytest.mark.parametrize("gan_lambda", [1.0, 0.0])
def test_r1_penalty_matches_phase_trainer(gan_lambda):
    """`train_step.r1_penalty` against the reference's `_calculate_r1_regularization` (phase_trainer.py:259-294) on a small
    differentiable stand-in for the discriminator: value and the gradient the penalty sends into the parameters (the double
    backward), with an enabled-style scale factor going through `scaler.scale` / `get_scale`."""
    ts = importlib.import_module("3dhumangan_b200.train_step")

    class Scaler:                     # GradScaler's two calls used there, with a non-trivial scale
        def scale(self, t):
            return t * 1024.0

        def get_scale(self):
            return 1024.0

    g = torch.Generator().manual_seed(9)
    w1 = torch.randn(6, 3, 3, 3, generator=g, dtype=torch.float64) * 0.3
    w2 = torch.randn(5, 6, 1, 1, generator=g, dtype=torch.float64) * 0.3
    x0 = torch.randn(3, 3, 8, 8, generator=g, dtype=torch.float64)
    meta = dict(gan_lambda=gan_lambda, segmentation_lambda=1.0, r1_lambda=0.25)

    def run(fn):
        a, b = w1.clone().requires_grad_(True), w2.clone().requires_grad_(True)
        x = x0.clone().requires_grad_(True)
        h = torch.nn.functional.leaky_relu(torch.nn.functional.conv2d(x, a, padding=1), 0.2)
        seg = torch.nn.functional.conv2d(torch.tanh(h), b)
        out = {"prediction": (h * h).mean(dim=(1, 2, 3)), "segments": seg}
        pen = fn(x, out)
        pen.backward()
        return float(pen), a.grad.clone(), b.grad.clone() if b.grad is not None else torch.zeros_like(b)

    me = types.SimpleNamespace(scaler=Scaler(), amp=False)
    ref = reference_result(f"r1_{gan_lambda}", lambda: run(lambda x, out: _reference(
        "lib.trainers.phase_trainer").PhaseTrainer._calculate_r1_regularization(me, x, out, {"do_r1": True}, meta)))
    got = run(lambda x, out: ts.r1_penalty(x, out, Scaler(), meta))
    assert got[0] == pytest.approx(ref[0], rel=1e-12, abs=1e-18)
    assert torch.allclose(got[1], ref[1], rtol=1e-10, atol=1e-16) and torch.allclose(got[2], ref[2], rtol=1e-10, atol=1e-16)
    if gan_lambda > 0:
        assert ref[0] > 0


# ----------------------------------------------------------------------------------------------------------------------
# the composition of the two steps: the reference's own `_train_discriminator` / `_train_generator` (phase_trainer.py:344-560),
# unmodified, against `train_step.Trainer.train_discriminator / train_generator` on the same stand-in networks
# ----------------------------------------------------------------------------------------------------------------------
class _StandInG(torch.nn.Module):
    """A generator with the call signature the trainer uses (z, conditions, latent_indices=..., **meta) -> {'rgbs', 'rgbs_render'}."""

    def __init__(self, L):
        super().__init__()
        g = torch.Generator().manual_seed(21)
        self.neural_field_mapping_network = torch.nn.Linear(L, 6)
        self.synthesis_network = torch.nn.Conv2d(6, 3, 3, padding=1)
        with torch.no_grad():
            for p in self.parameters():
                p.copy_(torch.randn(p.shape, generator=g) * 0.3)

    def forward(self, z, conditions, latent_indices=None, disable_synthesis=False, **kwargs):
        h = torch.tanh(self.neural_field_mapping_network(z))[:, :, None, None] + conditions["x"]
        rgb = torch.tanh(self.synthesis_network(h))
        return {"rgbs": rgb, "rgbs_render": torch.nn.functional.avg_pool2d(rgb, 2)}


class _StandInD(torch.nn.Module):
    def __init__(self, label_dim):
        super().__init__()
        g = torch.Generator().manual_seed(22)
        self.c1 = torch.nn.Conv2d(3, 8, 3, padding=1)
        self.seg = torch.nn.Conv2d(8, label_dim, 1)
        self.pred = torch.nn.Linear(8, 1)
        self.step = 0
        with torch.no_grad():
            for p in self.parameters():
                p.copy_(torch.randn(p.shape, generator=g) * 0.3)

    def forward(self, x, conditions, alpha=1.0, mode="real", **kwargs):
        h = torch.nn.functional.leaky_relu(self.c1(x), 0.2) + (0.1 if mode == "real" else -0.1) * conditions["x"][:, :1]
        return {"prediction": self.pred(h.mean(dim=(2, 3))), "segments": self.seg(h), "latents": h.mean(dim=(2, 3))}


@pytest.mark.parametrize("gan_lambda,do_r1", [(0.0, False), (0.0, True), (1.0, True)])
def test_step_composition_matches_phase_trainer(pkg, gan_lambda, do_r1, monkeypatch):
    ts = importlib.import_module("3dhumangan_b200.train_step")
    L, LD, B, H = 5, 7, 4, 8
    phase = {"name": "uncond", "uncond": True, "rotate": True, "gen_modal": "rgbs", "do_r1": do_r1}
    meta = dict(latent_dim=L, label_dim=LD, z_dist="gaussian", gan_lambda=gan_lambda, segmentation_lambda=1.0, latent_lambda=0,
                perceptual_lambda=[0, 0, 0, 0], photometric_lambda=0, r1_lambda=0.25, grad_clip=1e9, gen_lr=0.0, disc_lr=0.0,
                betas=(0.0, 0.9), weight_decay=0, appearance_codes_lr_mul=1.0, mapping_net_lr_mul=1.0, neural_field_lr_mul=1.0,
                batch_split=2, phases=[phase], render_height=4, render_width=4, gen_height=H, gen_width=H)
    g = torch.Generator().manual_seed(23)
    images = torch.randn(B, 3, H, H, generator=g).clamp_(-1, 1)
    labels = torch.randint(0, LD, (B, H, H), generator=g)
    x = torch.randn(B, 6, H, H, generator=g) * 0.2
    z_d, z_g = torch.randn(B, L, generator=g), torch.randn(B, L, generator=g)

    Gr, Dr = _StandInG(L), _StandInD(LD)

    def reference():        # ---- the reference's methods on a bare namespace
        pt = _reference("lib.trainers.phase_trainer")
        me = types.SimpleNamespace(amp=False, device="cpu", batch_split=2, rank=0, generator_ddp=Gr, discriminator_ddp=Dr, discriminator=Dr,
                                   scaler=torch.amp.GradScaler("cuda", enabled=False))
        for name in ("_train_discriminator", "_train_generator", "_get_disc_input_real", "_get_disc_input_gen",
                     "_calculate_r1_regularization", "_calculate_segmentation_loss"):
            setattr(me, name, types.MethodType(getattr(pt.PhaseTrainer, name), me))
        zs = [z_d, z_g]
        monkeypatch.setattr(pt, "z_sampler", lambda *a, **k: zs.pop(0))
        monkeypatch.setattr(pt.training_stats, "report", lambda *a, **k: None)
        data = {"images": images, "body_segments": labels, "rasterized_segments": labels, "latents": torch.zeros(B, L), "x": x}
        d_ref = me._train_discriminator(data, 1.0, meta, phase)
        d_ref.backward()
        dgrads = [p.grad.clone() for p in Dr.parameters()]
        Gr.zero_grad()
        Dr.zero_grad()
        g_ref, _ = me._train_generator(data, 1.0, meta, phase)
        ggrads = [p.grad.clone() for p in Gr.parameters()]
        return float(d_ref), dgrads, float(g_ref), ggrads
    d_ref, dgrads, g_ref, ggrads = reference_result(f"step_{gan_lambda}_{do_r1}", reference)

    # ---- this package's trainer on identical stand-ins
    Gm, Dm = _StandInG(L), _StandInD(LD)
    t = ts.Trainer(Gm, Dm, meta, amp=False, ddp=False, fused=False)
    batch = dict(images=images, labels=labels, cond={"x": x}, z_d=z_d, z_g=z_g)
    d_mine = t.train_discriminator(batch)
    for p, r in zip(Dm.parameters(), dgrads):
        assert torch.allclose(p.grad, r, rtol=1e-5, atol=1e-7), float((p.grad - r).abs().max())
    assert float(d_mine) == pytest.approx(float(d_ref), rel=1e-6)
    g_mine = t.train_generator(batch)
    for p, r in zip(Gm.parameters(), ggrads):
        assert torch.allclose(p.grad, r, rtol=1e-5, atol=1e-7), float((p.grad - r).abs().max())
    assert float(g_mine) == pytest.approx(float(g_ref), rel=1e-6, abs=1e-12)
    # learning rate 0, no clipping: both steps ran their optimiser / EMA tail without moving a parameter
    for p, q in zip(list(Gm.parameters()) + list(Dm.parameters()), list(Gr.parameters()) + list(Dr.parameters())):
        assert torch.equal(p.detach(), q.detach())


@pytest.mark.parametrize("name", ["MAP3DBN", "MAP3DBN512", "MAP3DBN512L"])
def test_curricula_match_reference_configs(pkg, name):
    """`3dhumangan_b200.configs` (the drop-in `configs` package) against the reference's `configs/map3d.py` + `extract_metadata`
    (configs/__init__.py) for every shipped curriculum at steps on both sides of every schedule boundary."""
    mine = pkg.configs
    cur_m = getattr(mine, name)

    def reference():
        ref = _reference("configs")
        cur_r = getattr(ref, name)
        steps = sorted({0, 1, 999, 1000, 200000, 200001, 300000, 300001, 300002, 10 ** 6} | {int(k) for k in cur_r if isinstance(k, int)} |
                       {int(k) + 1 for k in cur_r if isinstance(k, int)})
        return {step: ref.extract_metadata(cur_r, step) for step in steps}
    for step, a in reference_result(f"curriculum_{name}", reference).items():
        b = mine.extract_metadata(cur_m, step)
        for k, v in a.items():
            assert k in b, (name, step, k)
            if k == "neural_field_cls":
                assert (v if isinstance(v, str) else v.__name__) == (b[k] if isinstance(b[k], str) else b[k].__name__)
            else:
                assert b[k] == v, (name, step, k, v, b[k])
        extra = set(b) - set(a)
        assert all(k.startswith("hg_") for k in extra), (name, step, extra)


def test_trainer_refuses_the_branches_it_does_not_mirror():
    ts = importlib.import_module("3dhumangan_b200.train_step")
    meta = dict(latent_dim=5, label_dim=7, gan_lambda=0.0, segmentation_lambda=1.0, r1_lambda=0.0, grad_clip=1.0, gen_lr=0.0, disc_lr=0.0,
                betas=(0.0, 0.9), weight_decay=0, appearance_codes_lr_mul=1.0, mapping_net_lr_mul=1.0, neural_field_lr_mul=1.0,
                phases=[{"name": "uncond", "uncond": True, "rotate": True, "gen_modal": "rgbs_render", "do_r1": False}])
    t = ts.Trainer(_StandInG(5), _StandInD(7), meta, amp=False, ddp=False, fused=False)
    batch = dict(images=torch.zeros(2, 3, 8, 8), labels=torch.zeros(2, 8, 8, dtype=torch.long), cond={"x": torch.zeros(2, 6, 8, 8)})
    with pytest.raises(RuntimeError, match="not built"):
        t.train_discriminator(batch)
    with pytest.raises(RuntimeError, match="not built"):
        t.train_generator(batch)


def test_activation_table_matches_reference_bias_act():
    """ops/bias_act.ACTIVATIONS (id, default alpha, default gain, which tensor the backward keeps, second derivative) against the
    reference's `activation_funcs` (lib/components/ops/bias_act.py:22-32) -- the ids are what the C ABI's `act` argument means."""
    mine = importlib.import_module("3dhumangan_b200.ops.bias_act").ACTIVATIONS
    cuda_acts = reference_result("activation_funcs", lambda: {
        k: (v.cuda_idx, v.def_alpha, float(v.def_gain), v.ref, v.has_2nd_grad)
        for k, v in _reference("lib.components.ops.bias_act").activation_funcs.items() if v.cuda_idx is not None})
    assert set(mine) == set(cuda_acts)
    for k, (cuda_idx, def_alpha, def_gain, ref, has_2nd_grad) in cuda_acts.items():
        aid, alpha, gain, keep, second = mine[k]
        assert aid == cuda_idx and alpha == pytest.approx(def_alpha) and gain == pytest.approx(def_gain)
        assert keep == ref and second == has_2nd_grad


@pytest.mark.parametrize("tune,variant", [("", 0), ("lr", 0), ("lr", 3), ("map3d_mode", 0), ("map3d_mode", 2)])
def test_get_config_matches_reference(pkg, tune, variant):
    """`configs.get_config(opt)` (configs/__init__.py:49-76: curriculum lookup, neural-field class resolution, the two `--tune`
    sweeps) on deep copies of both packages' curricula."""
    mine = pkg.configs
    name = "MAP3DBN512"
    opt = types.SimpleNamespace(config=name, tune=tune, variant=variant)

    def reference():
        ref = _reference("configs")
        saved_r = copy.deepcopy(getattr(ref, name))
        try:
            a = ref.get_config(opt)
            return {k: v for k, v in a.items() if isinstance(k, int) or k in ("name", "map3d_mode", "neural_field_cls")}
        finally:
            setattr(ref, name, saved_r)
            ref.__dict__[name] = saved_r
    a = reference_result(f"get_config_{tune}_{variant}", reference)
    saved_m = copy.deepcopy(getattr(mine, name))
    try:
        b = mine.get_config(opt)
        assert a["name"] == b["name"] and a["map3d_mode"] == b["map3d_mode"]
        assert a["neural_field_cls"].__name__ == b["neural_field_cls"].__name__
        for k in a:
            if isinstance(k, int):
                assert a[k] == b[k], (k, a[k], b[k])
    finally:
        setattr(mine, name, saved_m)
