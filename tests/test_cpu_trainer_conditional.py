"""The reference's conditional (reconstruction) training mode pinned against its own step functions: the unmodified
`_train_discriminator` / `_train_generator` (lib/trainers/phase_trainer.py:344-553) on a bare namespace against
`train_step.Trainer(fused=False)`, on identical stand-in networks -- a generator that looks its latents up in a `LatentPool` when
given `latent_indices`, a discriminator with a live `latents` head and one four-level perceptual module injected on both sides.

Covered: the latent regression of both steps (`latent_lambda > 0`) in an unconditional phase, and a conditional phase with the
latent, photometric and perceptual terms (`gan_lambda` zeroed in the generator step), with distinct and with repeated indices.
The reference side was recorded by tests/golden/make_golden_conditional.py into tests/golden/conditional_phases.npz, so the
tests need no reference checkout."""
import importlib
import json
import os
import random
import sys
import types

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import golden_util

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.environ.get("HG_REFERENCE", "")
RESULTS = os.path.join(ROOT, "tests", "golden", "conditional_phases.npz")
RECORDING = None      # {key: value} while make_golden_conditional.py runs this file against a reference checkout


def _reference_result(key, compute):
    if RECORDING is not None:
        RECORDING[key] = value = compute()
        return value
    raw = np.load(RESULTS)
    index = json.loads(str(raw["index"]))
    return golden_util._decode(index[key], {k: raw[k] for k in raw.files if k != "index"})


def save_results():
    arrays = {}
    index = {k: golden_util._encode(v, arrays) for k, v in RECORDING.items()}
    np.savez_compressed(RESULTS, index=np.array(json.dumps(index, sort_keys=True)), **arrays)


def _phase_trainer():
    for p in (os.path.join(ROOT, "oracle", "shims"), REF):
        if p not in sys.path:
            sys.path.insert(0, p)
    return importlib.import_module("lib.trainers.phase_trainer")


def _seeded(module, seed):
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for p in module.parameters():
            p.copy_(torch.randn(p.shape, generator=g) * 0.3)
    return module


class _StandInG(torch.nn.Module):
    """(z, conditions, latent_indices=None, **meta) -> {'rgbs', 'rgbs_render'}; with indices the latent is the pool's row."""

    def __init__(self, L, P):
        super().__init__()
        gen = importlib.import_module("3dhumangan_b200.modules.generator")
        self.latent_pool = gen.LatentPool(P, L)
        self.neural_field_mapping_network = torch.nn.Linear(L, 6)
        self.synthesis_network = torch.nn.Conv2d(6, 3, 3, padding=1)
        _seeded(self, 31)

    def forward(self, z, conditions, latent_indices=None, disable_synthesis=False, **kwargs):
        if latent_indices is not None:
            z = self.latent_pool(latent_indices)
        h = torch.tanh(self.neural_field_mapping_network(z))[:, :, None, None] + conditions["x"]
        rgb = torch.tanh(self.synthesis_network(h))
        return {"rgbs": rgb, "rgbs_render": F.avg_pool2d(rgb, 2)}


class _StandInD(torch.nn.Module):
    def __init__(self, label_dim, L):
        super().__init__()
        self.c1 = torch.nn.Conv2d(3, 8, 3, padding=1)
        self.seg = torch.nn.Conv2d(8, label_dim, 1)
        self.pred = torch.nn.Linear(8, 1)
        self.latent_layer = torch.nn.Linear(8, L)
        self.step = 0
        _seeded(self, 32)

    def forward(self, x, conditions, alpha=1.0, mode="real", **kwargs):
        h = F.leaky_relu(self.c1(x), 0.2) + (0.1 if mode == "real" else -0.1) * conditions["x"][:, :1]
        pooled = h.mean(dim=(2, 3))
        return {"prediction": self.pred(pooled), "segments": self.seg(h), "latents": self.latent_layer(torch.tanh(pooled))}


class _StandInPerceptual(torch.nn.Module):
    """Four frozen levels, forward(input, target) -> four smooth-L1 losses, as VGGPerceptualLoss."""

    def __init__(self):
        super().__init__()
        self.convs = torch.nn.ModuleList([torch.nn.Conv2d(a, b, 3, padding=1) for a, b in ((3, 4), (4, 4), (4, 6), (6, 6))])
        _seeded(self, 33)
        for p in self.parameters():
            p.requires_grad_(False)

    def forward(self, input, target):
        x, y, losses = input, target, []
        for i, c in enumerate(self.convs):
            if i > 0:
                x, y = F.avg_pool2d(x, 2), F.avg_pool2d(y, 2)
            x, y = F.relu(c(x)), F.relu(c(y))
            losses.append(F.smooth_l1_loss(x, y))
        return losses


class _Wrapped:
    """What the reference reaches through `generator_ddp.module`."""

    def __init__(self, m):
        self.module = m

    def __call__(self, *a, **k):
        return self.module(*a, **k)


CASES = {
    "uncond_latent": dict(uncond=True, rotate=True, latent_lambda=0.5, photometric_lambda=0, perceptual_lambda=[0, 0, 0, 0],
                          indices=[3, 7, 1, 5]),
    "cond": dict(uncond=False, rotate=False, latent_lambda=0.5, photometric_lambda=2.0, perceptual_lambda=[1.0, 0.5, 0.25, 0.1],
                 indices=[3, 7, 1, 5]),
    "cond_repeated": dict(uncond=False, rotate=False, latent_lambda=0.5, photometric_lambda=2.0,
                          perceptual_lambda=[1.0, 0.5, 0.25, 0.1], indices=[4, 2, 4, 4]),
}


@pytest.mark.parametrize("case", sorted(CASES))
def test_conditional_steps_match_phase_trainer(pkg, case, monkeypatch):
    ts = importlib.import_module("3dhumangan_b200.train_step")
    c = CASES[case]
    L, LD, B, H, P = 5, 7, 4, 8, 10
    phase = {"name": case, "uncond": c["uncond"], "rotate": c["rotate"], "gen_modal": "rgbs", "do_r1": False}
    meta = dict(latent_dim=L, label_dim=LD, z_dist="gaussian", gan_lambda=1.0, segmentation_lambda=1.0, latent_lambda=c["latent_lambda"],
                perceptual_lambda=c["perceptual_lambda"], photometric_lambda=c["photometric_lambda"], r1_lambda=0.25, grad_clip=1e9,
                gen_lr=0.0, disc_lr=0.0, betas=(0.0, 0.9), weight_decay=0, appearance_codes_lr_mul=1.0, mapping_net_lr_mul=1.0,
                neural_field_lr_mul=1.0, batch_split=2, phases=[phase], render_height=4, render_width=4, gen_height=H, gen_width=H)
    g = torch.Generator().manual_seed(41)
    images = torch.randn(B, 3, H, H, generator=g).clamp_(-1, 1)
    labels = torch.randint(0, LD, (B, H, H), generator=g)
    x = torch.randn(B, 6, H, H, generator=g) * 0.2
    z_d, z_g = torch.randn(B, L, generator=g), torch.randn(B, L, generator=g)
    codes = torch.randn(P, L, generator=g)
    indices = torch.tensor(c["indices"], dtype=torch.int64)
    latents = torch.randn(B, L, generator=g)
    monkeypatch.setattr(random, "random", lambda: 0.9)      # disc_mode "real" / "gen", body_segments as the target

    def reference():
        pt = _phase_trainer()
        Gr, Dr = _StandInG(L, P), _StandInD(LD, L)
        Gr.latent_pool.init(codes)                 # PhaseTrainer.__init__ (:29-32)
        me = types.SimpleNamespace(amp=False, device="cpu", batch_split=2, rank=0, generator_ddp=_Wrapped(Gr), discriminator_ddp=Dr,
                                   discriminator=Dr, scaler=torch.amp.GradScaler("cuda", enabled=False),
                                   perceptual_loss=_StandInPerceptual())
        for name in ("_train_discriminator", "_train_generator", "_get_disc_input_real", "_get_disc_input_gen",
                     "_calculate_r1_regularization", "_calculate_segmentation_loss"):
            setattr(me, name, types.MethodType(getattr(pt.PhaseTrainer, name), me))
        zs = [z_d, z_g]
        monkeypatch.setattr(pt, "z_sampler", lambda *a, **k: zs.pop(0))
        monkeypatch.setattr(pt.training_stats, "report", lambda *a, **k: None)
        data = {"images": images, "body_segments": labels, "rasterized_segments": labels, "latents": latents, "indices": indices, "x": x}
        d_ref = me._train_discriminator(data, 1.0, meta, phase)
        d_ref.backward()
        dgrads = [p.grad.clone() for p in Dr.parameters()]
        Gr.zero_grad()
        Dr.zero_grad()
        g_ref, _ = me._train_generator(data, 1.0, meta, phase)
        ggrads = [p.grad.clone() if p.grad is not None else None for p in Gr.parameters()]
        return float(d_ref.detach()), dgrads, float(g_ref), ggrads
    d_ref, dgrads, g_ref, ggrads = _reference_result(case, reference)

    Gm, Dm = _StandInG(L, P), _StandInD(LD, L)
    t = ts.Trainer(Gm, Dm, meta, amp=False, ddp=False, fused=False, perceptual=_StandInPerceptual(), appearance_codes=codes)
    assert torch.equal(Gm.latent_pool.latents.detach(), codes)
    batch = dict(images=images, labels=labels, cond={"x": x, "indices": indices, "latents": latents}, z_d=z_d, z_g=z_g)
    d_mine = t.train_discriminator(batch)
    assert float(d_mine) == pytest.approx(d_ref, rel=1e-6)
    for p, r in zip(Dm.parameters(), dgrads):
        assert torch.allclose(p.grad, r, rtol=1e-5, atol=1e-7), float((p.grad - r).abs().max())
    assert float(Dm.latent_layer.weight.grad.abs().max()) > 0       # the latent head takes part
    g_mine = t.train_generator(batch)
    assert float(g_mine) == pytest.approx(g_ref, rel=1e-6, abs=1e-12)
    for (n, p), r in zip(Gm.named_parameters(), ggrads):
        if r is None:
            assert p.grad is None or not p.grad.any(), n
            continue
        assert torch.allclose(p.grad, r, rtol=1e-5, atol=1e-7), (n, float((p.grad - r).abs().max()))
    pool = Gm.latent_pool.latents.grad
    touched = torch.zeros(P, dtype=torch.bool)
    touched[indices] = True
    if c["uncond"]:
        assert pool is None or not pool.any()
    else:
        assert bool((pool[touched].abs().sum(1) > 0).all()) and not pool[~touched].any()
