"""Latent inversion: fit the generator's input to a target image under a known pose and camera.

The generator stays as released -- `eval()`, every parameter frozen, no buffer written -- and only its input moves:
`space="z"` optimises the latent [B, latent_dim]; `space="film"` optimises the mapped tensors directly (freq / phase of
`neural_field_mapping_network`, the style of `synthesis_mapping_network`), the larger space GAN projection usually wants.
Each step is `Map3DGenerator.synthesize` (modules/render_train.GeneratorCore in eval mode: running-statistics BatchNorm,
no weight-gradient kernel for the frozen parameters), `ops.trainer_ops.image_loss` and one `FusedAdam` launch.  The ray
jitter is drawn once: the point records of the first render (ray samples, nearest vertices, geometry features) are re-used
by every later step, so every step differentiates one fixed function; a given seed repeats the run up to the order of the
atomic sums in the data-gradient kernels (the last bits of a gradient).
With `hierarchical_sample=True` the fine samples follow the density and every step redraws them from a per-step seed.

`perceptual` (a `perceptual.VGGPerceptualLoss`) adds the reference trainer's feature-space term (phase_trainer.py:515-520):
sum_i perceptual_lambda[i] * L_i(0.5 * rgbs + 0.5, 0.5 * target + 0.5), the target's VGG features computed once before the
loop.  `loss=None` drops the pixel term.  A merged training config passed through **kwargs carries its own `perceptual_lambda`
(zeros in every shipped configuration), which then takes this argument's place; all-zero weights with a `perceptual`
module raise rather than silently drop the term.
"""
from __future__ import annotations

import torch

from . import abi
from .ops.trainer_ops import FusedAdam, image_loss


def invert(G, target, conditions, *, space="film", steps=100, lr=0.01, mask=None, seed=0, loss="l2", perceptual=None,
           perceptual_lambda=(1, 1, 1, 1), **kwargs):
    """target [B,3,gen_height,gen_width] in [-1,1]; conditions: the SMPL / camera dict of `Map3DGenerator.forward`;
    kwargs: the merged config that `forward` takes (render_height, render_width, num_steps, last_back, ...).
    -> dict(variables={name: tensor}, losses=[float per step], image=[B,3,H,W] of the optimised variables).
    Without hierarchical_sample `losses` and `image` are values of one function (the jitter of the first render).  With it
    every step and the final image draw their own samples (seed + step), so the curve is that of a stochastic objective.
    The objective is image_loss(kind=loss) (`mask` weights this pixel term only; `loss=None` drops it) plus, with
    `perceptual`, the perceptual term above."""
    if space not in ("z", "film"):
        raise RuntimeError(f"hg3d: inversion space {space!r} is not built ('z' or 'film')")
    if loss is None and perceptual is None:
        raise RuntimeError("hg3d: inversion needs a pixel loss, a perceptual loss or both")
    if perceptual is not None and not any(float(w) for w in perceptual_lambda):
        raise RuntimeError(f"hg3d: perceptual_lambda {list(perceptual_lambda)} switches the perceptual term off; pass non-zero "
                           "weights (a merged config's own perceptual_lambda overrides the default)")
    abi.require_device()
    dev = target.device
    B = target.shape[0]
    hier = kwargs.get("hierarchical_sample", False)
    field_latent = kwargs.get("neural_field_latent_input", G._cfg.get("neural_field_latent_input", True))
    was_training = G.training
    frozen = [(p, p.requires_grad) for p in G.parameters()]
    G.eval()
    for p, _ in frozen:
        p.requires_grad_(False)
    try:
        target_features = None
        if perceptual is not None:
            target_features = perceptual.target_features(0.5 * target + 0.5)
        z = torch.randn(B, G.latent_dim, generator=torch.Generator(device=dev).manual_seed(seed), device=dev)
        if space == "z":
            variables = {"z": z.requires_grad_(True)}
        else:
            with torch.no_grad():
                freq, phase = G.neural_field_mapping_network(z if field_latent else torch.zeros_like(z))
                _, styles = G.synthesis_mapping_network(z)
            variables = {"freq": freq.clone().requires_grad_(True), "phase": phase.clone().requires_grad_(True),
                         "styles": styles.clone().requires_grad_(True)}

        def mapped():
            if space == "film":
                return variables["freq"], variables["phase"], variables["styles"]
            zz = variables["z"]
            freq, phase = G.neural_field_mapping_network(zz if field_latent else torch.zeros_like(zz))
            return freq, phase, G.synthesis_mapping_network(zz)[1]

        opt = FusedAdam(list(variables.values()), lr=lr)
        records = None
        losses = []
        with torch.random.fork_rng(devices=[torch.cuda.current_device()]):
            for step in range(steps + 1):
                torch.manual_seed(seed + (step if hier else 0))
                last = step == steps                      # the final render of the optimised variables, no update
                with torch.set_grad_enabled(not last):
                    extra = {} if records is None or last else {"hg_records": records}
                    out = G.synthesize(*mapped(), conditions, **dict(kwargs, **extra))
                    if last:
                        break
                    if not hier:
                        records = out["hg_records"]
                    value = 0.0 if loss is None else image_loss(out["rgbs"], target, mask, kind=loss)
                    if perceptual is not None:
                        value = value + perceptual.loss(0.5 * out["rgbs"] + 0.5, target_features, perceptual_lambda)
                for v in variables.values():
                    v.grad = None
                value.backward()
                opt.step()
                losses.append(value.detach())
        losses = [float(v) for v in torch.stack(losses).cpu()] if losses else []
        return {"variables": {k: v.detach() for k, v in variables.items()}, "losses": losses, "image": out["rgbs"].detach()}
    finally:
        for p, flag in frozen:
            p.requires_grad_(flag)
        G.train(was_training)
