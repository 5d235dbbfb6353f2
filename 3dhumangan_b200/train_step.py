"""One training iteration of the reference's trainer over this library's modules: the host-side mirror of
`PhaseTrainer.train_discriminator / train_generator` (lib/trainers/phase_trainer.py:297-344, `_train_discriminator`
:344-444, `_train_generator` :446-560), `init_optimizer` (:57-76), `_calculate_segmentation_loss` (:203-256),
`_calculate_r1_regularization` (:259-294), `BaseTrainer.init_model`'s DDP wrapping (base_trainer.py:102-104) and
`ExponentialMovingAverage.update` (lib/components/ema.py:29-48).

It exists for two reasons: (1) the reference's trainer cannot travel to the GPU box (it needs the dataset, the
pytorch3d rasteriser and tensorboard), so THIS is what exercises the module surfaces exactly the way that trainer
does -- `DistributedDataParallel(find_unused_parameters=True, broadcast_buffers=False)`, fp16 autocast +
`GradScaler`, `disc_input_real.requires_grad = True`, `torch.autograd.grad(..., create_graph=True)` on the do_r1 phases,
`backward(retain_graph=True)`, `unscale_` / `clip_grad_norm_` / `scaler.step`, EMA over `parameters()`; (2) it is the
G+D step that `bench.py` times (BASELINE.json's second metric).

Everything between the inputs and the two losses runs on the sm_90a kernels (generator: fused inference kernels under
no_grad in the discriminator step, training kernels in the generator step; discriminator: the autograd graph of
modules/discriminator_train.py).  Loss reduction, clipping, Adam and EMA are multi-tensor torch calls (SURVEY.md §8f-1).
"""
from __future__ import annotations

import math
import random

import torch
import torch.nn.functional as F


# ----------------------------------------------------------------------------------------------------------------------
# losses
# ----------------------------------------------------------------------------------------------------------------------
def segmentation_loss(segments, gt, label_dim, prior_weights=None, with_stats=False):
    """`cross_entropy_balanced` of PhaseTrainer._calculate_segmentation_loss (phase_trainer.py:203-256): per-class weights
    ~ 1 / occurrence (background excluded), normalised by the number of classes present."""
    if gt.shape[1:] != segments.shape[2:]:
        with torch.no_grad():
            gt = F.interpolate(gt[:, None].float(), segments.shape[2:], mode="nearest")[:, 0].long()
    if not bool((gt > 0).any()):
        loss = F.cross_entropy(segments, gt)
    else:
        pw = torch.ones(label_dim, dtype=segments.dtype, device=segments.device) if prior_weights is None else \
            torch.as_tensor(prior_weights, dtype=segments.dtype, device=segments.device)
        pw = pw / pw.mean()
        occ = torch.bincount(gt.reshape(-1), minlength=label_dim)[:label_dim].clone()
        occ[0] = 0
        n_occ = torch.count_nonzero(occ)
        coef = torch.reciprocal(occ.to(segments.dtype)) * (gt.numel() * label_dim) / (n_occ * label_dim)
        coef[0] = 0
        coef[torch.isinf(coef)] = 0
        coef = coef * pw
        loss = (F.cross_entropy(segments, gt, reduction="none") * coef[gt]).mean()
    if not with_stats:
        return loss
    with torch.no_grad():
        real_prob = (1 - torch.softmax(segments, dim=1)[:, 0]).mean()
        acc = ((torch.argmax(segments[:, 1:], dim=1) + 1) == gt).float().mean()
    return loss, acc, real_prob


def normalize_2nd_moment(x, dim=1, eps=1e-8):
    """lib/components/util.py:58."""
    return x * (x.square().mean(dim=dim, keepdim=True) + eps).rsqrt()


def latent_regression_loss(pred, target):
    """The latent term of phase_trainer.py:425-437 and :493-506 for one side: SL1_0.1(n(pred), n(target)), the target under
    no_grad."""
    with torch.no_grad():
        target = normalize_2nd_moment(target)
    return F.smooth_l1_loss(normalize_2nd_moment(pred), target, beta=0.1)


def r1_penalty(disc_input_real, out_real, scaler, meta):
    """phase_trainer.py:259-294, arithmetic as the reference EXECUTES it: the gradient of f = sum(prediction) (gan_lambda > 0) or
    sum(softmax(segments)) (segmentation only) w.r.t. the real images is taken for the whole batch, but
    `[p * inv_scale for p in grad_real][0]` (:281-282) iterates over the batch dimension of that tensor and keeps entry 0, and
    `grad_real.view(grad_real.size(0), -1).pow(2).sum(dim=1).mean()` (:287-288) then averages over its CHANNELS:
        penalty = 0.5 * r1_lambda * |d f / d x_0|^2 / C          (first sample of the batch, C = 3)
    -- not the batch mean of the textbook R1.  Pinned against the reference's method by tests/test_cpu_trainer_pin.py.
    Differentiated again by `d_loss.backward()` (create_graph=True)."""
    if meta["gan_lambda"] > 0:
        target = out_real["prediction"].sum()
    elif meta["segmentation_lambda"] > 0:
        target = torch.softmax(out_real["segments"], dim=1).sum()
    else:
        raise RuntimeError("cannot do r1 regularization when segmentation_lambda == 0 and gan_lambda == 0")
    grad_real = torch.autograd.grad(outputs=scaler.scale(target), inputs=disc_input_real, create_graph=True)[0]
    grad_real = grad_real[0] * (1.0 / scaler.get_scale())
    pen = grad_real.reshape(grad_real.shape[0], -1).pow(2).sum(dim=1).mean()
    pen = 0.5 * meta["r1_lambda"] * pen
    if bool(torch.isnan(pen).any()):
        return 0.0
    return pen


# ----------------------------------------------------------------------------------------------------------------------
# optimisers, EMA
# ----------------------------------------------------------------------------------------------------------------------
def generator_param_groups(named_params, meta):
    """The five Adam groups of PhaseTrainer.init_optimizer (phase_trainer.py:57-76), selected by the same name substrings
    in the same precedence: neural_field_mapping_network, synthesis_mapping_network, latent_pool, neural_field, rest."""
    named = list(named_params)
    nf_map = {n: p for n, p in named if "neural_field_mapping_network" in n}
    syn_map = {n: p for n, p in named if "synthesis_mapping_network" in n}
    codes = {n: p for n, p in named if "latent_pool" in n}
    field = {n: p for n, p in named if "neural_field" in n and n not in nf_map}
    taken = {**codes, **field, **nf_map, **syn_map}
    rest = {n: p for n, p in named if n not in taken}
    lr = meta["gen_lr"]
    return [
        {"params": list(rest.values()), "name": "generator"},
        {"params": list(codes.values()), "name": "appearance_codes", "lr": lr * meta["appearance_codes_lr_mul"]},
        {"params": list(nf_map.values()), "name": "neural_field_mapping", "lr": lr * meta["mapping_net_lr_mul"]},
        {"params": list(syn_map.values()), "name": "synthesis_mapping", "lr": lr},
        {"params": list(field.values()), "name": "neural_field", "lr": lr * meta["neural_field_lr_mul"]},
    ]


def make_optimizers(G, D, meta, fused=True):
    """Adam for G (five groups with the curriculum's learning-rate multipliers) and D, as PhaseTrainer.init_optimizer.
    fused=True: `ops.trainer_ops.FusedAdam` (same state_dict and arithmetic as torch.optim.Adam, one multi-tensor launch that
    also carries the gradient clipping and the EMA); fused=False: torch.optim.Adam."""
    betas = tuple(float(b) for b in meta.get("betas", (0, 0.9)))
    wd = meta.get("weight_decay", 0)
    if fused:
        from .ops.trainer_ops import FusedAdam as Adam
    else:
        Adam = torch.optim.Adam
    og = Adam(generator_param_groups(G.named_parameters(), meta), lr=meta["gen_lr"], betas=betas, weight_decay=wd)
    od = Adam(D.parameters(), lr=meta["disc_lr"], betas=betas, weight_decay=wd)
    return og, od


class ParameterEMA:
    """lib/components/ema.py:8-48: shadow copies of the parameters that require grad, decay = min(decay, (1+n)/(10+n)),
    updated with one multi-tensor call per step."""

    def __init__(self, parameters, decay=0.999, use_num_updates=True):
        if not 0.0 <= decay <= 1.0:
            raise ValueError("Decay must be between 0 and 1")
        self.decay = decay
        self.num_updates = 0 if use_num_updates else None
        self.shadow_params = [p.clone().detach() for p in parameters if p.requires_grad]

    @torch.no_grad()
    def update(self, parameters):
        decay = self.decay
        if self.num_updates is not None:
            self.num_updates += 1
            decay = min(decay, (1 + self.num_updates) / (10 + self.num_updates))
        params = [p.detach() for p in parameters if p.requires_grad]
        torch._foreach_lerp_(self.shadow_params, params, 1.0 - decay)          # s -= (1 - decay) * (s - p)

    @torch.no_grad()
    def copy_to(self, parameters):
        for s, p in zip(self.shadow_params, [p for p in parameters if p.requires_grad]):
            p.data.copy_(s.data)


def average_gradients(module, group=None, _cache={}):
    """Optional fast path WITHOUT DistributedDataParallel: one flat NCCL all-reduce over every parameter that requires
    grad (a missing gradient counts as zeros, so all ranks always reduce the same number of elements), through a cached
    flat buffer.  The module surfaces work under real DDP (tests/test_gpu_multi.py); this is only for callers that want to
    place the collective themselves."""
    import torch.distributed as dist
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size(group) == 1:
        return
    params = [p for p in module.parameters() if p.requires_grad]
    if not params:
        return
    n = sum(p.numel() for p in params)
    key = (id(module), n, params[0].device)
    flat = _cache.get(key)
    if flat is None:
        flat = _cache[key] = torch.empty(n, dtype=torch.float32, device=params[0].device)
    off = 0
    for p in params:
        seg = flat[off:off + p.numel()]
        if p.grad is None:
            seg.zero_()
        else:
            seg.copy_(p.grad.reshape(-1))
        off += p.numel()
    dist.all_reduce(flat, group=group)
    flat /= dist.get_world_size(group)
    off = 0
    for p in params:
        seg = flat[off:off + p.numel()].view_as(p)
        if p.grad is None:
            p.grad = seg.clone()
        else:
            p.grad.copy_(seg)
        off += p.numel()


# ----------------------------------------------------------------------------------------------------------------------
# the iteration
# ----------------------------------------------------------------------------------------------------------------------
class Trainer:
    """Drives (generator, discriminator) through the reference's two step functions.

    `batch`: dict(images [B,3,H,W], labels [B,H,W] int64 (the real segmentation map), cond = the pose conditions,
    optional z_d / z_g latents (drawn like `z_sampler` otherwise)).  `meta` is the merged curriculum dict that the
    reference splats into every call.  Conditional phases (`uncond: False`) and `latent_lambda > 0` also read
    `cond["indices"]` (int64 [B], the images' rows of `generator.latent_pool`) and `cond["latents"]` ([B, latent_dim], their
    inversion codes), the `indices` / `latents` of the reference's dataset (lib/data/datasets.py:291)."""

    def __init__(self, G, D, meta, *, amp=None, ddp=None, amp_dtype=torch.float16, ema_decay=0.999, fused=True, preprocessor=None,
                 perceptual=None, appearance_codes=None):
        """fused=True: the loss / clipping / Adam / EMA tail on the sm_90a kernels of csrc/trainer.cu (ops.trainer_ops);
        fused=False: the same steps as torch calls (F.cross_entropy, clip_grad_norm_, torch.optim.Adam, foreach lerp).
        preprocessor: a `preprocess.Preprocessor`.  With one, each step draws a view for `batch["cond"]` as
        phase_trainer.py:305,329 do, and the segmentation targets follow :350-353 and :533 -- the rasterised map on rotate phases,
        otherwise the rasterised map or `batch["labels"]` (the dataset's body_segments) with probability 1/2 each, drawn with
        `random.random()`.  Without one, `batch["cond"]` is used as given and `batch["labels"]` is the target in every phase.
        perceptual: the module of the perceptual term of conditional phases (`perceptual.VGGPerceptualLoss` or any module with
        its `forward(input, target)` -> 4 losses); built from torchvision's cached VGG16 weights when `sum(perceptual_lambda) > 0`
        and none is given (phase_trainer.py:51-54; raises when the weights are missing, nothing is downloaded).
        appearance_codes: [P, latent_dim] initial `generator.latent_pool` rows, the dataset's inversion codes
        (phase_trainer.py:29-32)."""
        self.preprocessor = preprocessor
        if appearance_codes is not None:
            G.latent_pool.init(torch.as_tensor(appearance_codes))
        if perceptual is None and sum(meta.get("perceptual_lambda", [0])) > 0:
            from .perceptual import VGGPerceptualLoss
            perceptual = VGGPerceptualLoss().to(next(G.parameters()).device)
        self.perceptual = perceptual
        import torch.distributed as dist
        self.meta = dict(meta)
        self.fused = bool(fused)
        self.amp = bool(self.meta.get("use_mixed_precision", False)) if amp is None else bool(amp)
        self.amp_dtype = amp_dtype
        self.scaler = torch.amp.GradScaler("cuda", enabled=self.amp and amp_dtype == torch.float16)
        multi = dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1
        self.use_ddp = multi if ddp is None else bool(ddp)
        if self.use_ddp:      # base_trainer.py:102-104
            from torch.nn.parallel import DistributedDataParallel as DDP
            dev = next(G.parameters()).device
            ids = [dev] if dist.get_backend() == "nccl" else None
            self.generator_ddp = DDP(G, device_ids=ids, find_unused_parameters=True, broadcast_buffers=False)
            self.discriminator_ddp = DDP(D, device_ids=ids, find_unused_parameters=True, broadcast_buffers=False)
        else:
            self.generator_ddp, self.discriminator_ddp = G, D
        self.generator, self.discriminator = G, D
        # groups are selected by name substrings, which survive DDP's "module." prefix (the reference builds them from
        # `generator_ddp.named_parameters()`, phase_trainer.py:59)
        self.optimizer_G, self.optimizer_D = make_optimizers(self.generator_ddp, self.discriminator_ddp, self.meta, fused=self.fused)
        self.ema = ParameterEMA(G.parameters(), decay=ema_decay)
        self.batch_split = int(self.meta.get("batch_split", 1))

    # -- helpers
    def _seg_loss(self, segments, gt):
        if self.fused:
            from .ops.trainer_ops import seg_ce_balanced
            return seg_ce_balanced(segments, gt, self.meta["label_dim"], self.meta.get("segmentation_weights"))
        return segmentation_loss(segments, gt, self.meta["label_dim"], self.meta.get("segmentation_weights"))

    def _latent_loss(self, pred, target):
        if self.fused:
            from .ops.trainer_ops import latent_loss
            return latent_loss(pred, target, beta=0.1)
        return latent_regression_loss(pred, target)

    def _photometric_loss(self, rgbs, images):
        if self.fused:
            from .ops.trainer_ops import image_loss
            return image_loss(rgbs, images.detach(), kind="smooth_l1", beta=0.1)
        return F.smooth_l1_loss(rgbs, images.detach(), beta=0.1)

    def _optimizer_step(self, opt, params, ema=None):
        """unscale_ -> clip_grad_norm_ -> scaler.step (-> EMA): phase_trainer.py:313-316, 335-339."""
        self.scaler.unscale_(opt)
        if self.fused:
            opt._stepped = False
            self.scaler.step(opt, clip_max_norm=self.meta["grad_clip"], ema=ema, ema_params=params if ema is not None else None)
            if ema is not None and not opt._stepped:          # GradScaler skipped the step (inf / nan): the EMA still follows
                ema.update(params)
        else:
            torch.nn.utils.clip_grad_norm_(params, self.meta["grad_clip"])
            self.scaler.step(opt)
            if ema is not None:
                ema.update(params)

    def _autocast(self):
        return torch.autocast("cuda", dtype=self.amp_dtype, enabled=self.amp)

    def _phase(self):
        phases = self.meta["phases"]
        return phases[self.discriminator.step % len(phases)]

    def _z(self, batch, key, B, device):
        if key in batch:
            return batch[key]
        if self.meta.get("z_dist", "gaussian") == "gaussian":
            return torch.randn(B, self.meta["latent_dim"], device=device)
        return torch.rand(B, self.meta["latent_dim"], device=device) * 2 - 1

    # -- phase_trainer.py:297-318 + :344-444
    def _check_phase(self, phase):
        """The input selection of `_get_disc_input_real / _gen` (phase_trainer.py:162-200) has two more branches (dual discrimination,
        render-resolution modalities) that no shipped curriculum reaches: refuse them instead of training on the wrong tensors."""
        if self.meta.get("dual_discrimination", False) or "render" in phase["gen_modal"]:
            raise RuntimeError("hg3d: dual_discrimination / gen_modal '%s' are not used by any shipped curriculum and are not "
                               "built" % phase["gen_modal"])

    def train_discriminator(self, batch, alpha=1.0):
        meta, phase = self.meta, self._phase()
        self._check_phase(phase)
        self.optimizer_D.zero_grad()
        real_images, labels, cond = batch["images"], batch["labels"], batch["cond"]
        if self.preprocessor is not None:
            cond = self.preprocessor(dict(cond), phase["rotate"], **meta)
            if phase["rotate"] or random.random() < 0.5:
                labels = cond["rasterized_segments"]
        B = real_images.shape[0]
        uncond = phase.get("uncond", True)
        with self._autocast():
            with torch.no_grad():
                z = self._z(batch, "z_d", B, real_images.device)
                split = B // self.batch_split
                outs = []
                for s in range(self.batch_split):
                    sl = slice(s * split, (s + 1) * split)
                    sub = {k: v[sl] for k, v in cond.items()}
                    outs.append(self.generator_ddp(z[sl], sub, latent_indices=None if uncond else sub["indices"], **meta))
                gen_outputs = {k: torch.cat([o[k] for o in outs], 0) for k in outs[0]}
            disc_input_real = real_images.detach().clone() if real_images.requires_grad else real_images
            disc_input_real.requires_grad = True
            out_real = self.discriminator_ddp(disc_input_real, cond, alpha=alpha, mode="real", **meta)
            pred_real = out_real["prediction"]
        grad_penalty = 4 * r1_penalty(disc_input_real, out_real, self.scaler, meta) if phase["do_r1"] else 0.0
        with self._autocast():
            disc_input_gen = gen_outputs[phase["gen_modal"]]
            out_gen = self.discriminator_ddp(disc_input_gen, cond, alpha=alpha, mode="gen", **meta)
            pred_gen = out_gen["prediction"]
            if meta["gan_lambda"] > 0:
                gan_loss = meta["gan_lambda"] * (F.softplus(pred_gen).mean() + F.softplus(-pred_real).mean())
            else:
                gan_loss = pred_gen.sum() * 0 + pred_real.sum() * 0
            if meta["segmentation_lambda"] > 0:
                seg = (self._seg_loss(out_real["segments"], labels)
                       + self._seg_loss(out_gen["segments"], torch.zeros_like(labels))) * meta["segmentation_lambda"]
            else:
                seg = (out_real["segments"].sum() + out_gen["segments"].sum()) * 0
            if meta.get("latent_lambda", 0) > 0:          # phase_trainer.py:425-437
                with torch.no_grad():
                    gt_gen = z if uncond else self.generator.latent_pool(cond["indices"])
                latent_loss = (self._latent_loss(out_gen["latents"], gt_gen)
                               + self._latent_loss(out_real["latents"], cond["latents"])) * meta["latent_lambda"]
            else:
                latent_loss = (out_real["latents"].sum() + out_gen["latents"].sum()) * 0
            d_loss = gan_loss + grad_penalty + seg + latent_loss
        self.scaler.scale(d_loss).backward()
        self._optimizer_step(self.optimizer_D, list(self.discriminator_ddp.parameters()))
        return d_loss.detach()

    # -- phase_trainer.py:321-341 + :446-560
    def train_generator(self, batch, alpha=1.0):
        meta, phase = self.meta, self._phase()
        self._check_phase(phase)
        self.optimizer_G.zero_grad()
        real_images, labels, cond = batch["images"], batch["labels"], batch["cond"]
        if self.preprocessor is not None:
            cond = self.preprocessor(dict(cond), phase["rotate"], **meta)
        B = real_images.shape[0]
        uncond = phase.get("uncond", True)
        z = self._z(batch, "z_g", B, real_images.device)
        split = B // self.batch_split
        total = 0.0
        # The reference leaves the discriminator's parameters trainable here and lets autograd fill (and DDP all-reduce)
        # gradients that `optimizer_D.zero_grad()` throws away at the start of the next discriminator step
        # (phase_trainer.py:301, 474).  Same parameter updates without that work: freeze them for this step and call the
        # bare module (no reducer bookkeeping, no weight-gradient kernels, no all-reduce of unused gradients).
        d_params = list(self.discriminator.parameters())
        flags = [p.requires_grad for p in d_params]
        for p in d_params:
            p.requires_grad_(False)
        try:
            for s in range(self.batch_split):
                sl = slice(s * split, (s + 1) * split)
                with self._autocast():
                    sub = {k: v[sl] for k, v in cond.items()}
                    gen_outputs = self.generator_ddp(z[sl], sub, latent_indices=None if uncond else sub["indices"], **meta)
                    rgbs = gen_outputs[phase["gen_modal"]]
                    out = self.discriminator(rgbs, sub, alpha=alpha, mode="gen", **meta)
                    pred_gen = out["prediction"]
                    gan_lambda = meta["gan_lambda"] if uncond else 0
                    gan_loss = gan_lambda * F.softplus(-pred_gen).mean() if gan_lambda > 0 else 0 * pred_gen.sum()
                    if meta.get("latent_lambda", 0) > 0:          # phase_trainer.py:493-506
                        with torch.no_grad():
                            gt = z[sl] if uncond else self.generator.latent_pool(sub["indices"])
                        latent_loss = self._latent_loss(out["latents"], gt)
                        if not uncond:        # depends on no parameter; part of the reported loss as in the reference
                            latent_loss = latent_loss + F.smooth_l1_loss(z[sl], sub["latents"].detach(), beta=0.1)
                        latent_loss = latent_loss * meta["latent_lambda"]
                    else:
                        latent_loss = out["latents"].sum() * 0
                    g_loss = gan_loss          # + the perceptual and photometric terms of conditional phases (:509-527)
                    if not uncond and sum(meta.get("perceptual_lambda", [0])) > 0:
                        losses = self.perceptual(0.5 * rgbs + 0.5, (0.5 * real_images[sl] + 0.5).detach())
                        g_loss = g_loss + sum(meta["perceptual_lambda"][i] * losses[i] for i in range(4))
                    if not uncond and meta.get("photometric_lambda", 0) > 0:
                        g_loss = g_loss + self._photometric_loss(rgbs, real_images[sl]) * meta["photometric_lambda"]
                    if meta["segmentation_lambda"] > 0:
                        gt = labels[sl]
                        if self.preprocessor is not None and (phase["rotate"] or random.random() < 0.5):
                            gt = sub["rasterized_segments"]
                        seg = self._seg_loss(out["segments"], gt) * meta["segmentation_lambda"]
                    else:
                        seg = out["segments"].sum() * 0
                    g_loss = (g_loss + latent_loss + seg) / self.batch_split
                    self.scaler.scale(g_loss).backward()
                total = total + g_loss.detach()
        finally:
            for p, f in zip(d_params, flags):
                p.requires_grad_(f)
        self._optimizer_step_g(list(self.generator_ddp.parameters()))
        return total

    def _optimizer_step_g(self, gparams):
        """phase_trainer.py:335-339: unscale_, clip, step, scaler.update(), EMA."""
        self.scaler.unscale_(self.optimizer_G)
        if self.fused:
            self.optimizer_G._stepped = False
            self.scaler.step(self.optimizer_G, clip_max_norm=self.meta["grad_clip"], ema=self.ema, ema_params=gparams)
            self.scaler.update()
            if not self.optimizer_G._stepped:
                self.ema.update(gparams)
        else:
            torch.nn.utils.clip_grad_norm_(gparams, self.meta["grad_clip"])
            self.scaler.step(self.optimizer_G)
            self.scaler.update()
            self.ema.update(gparams)

    def iteration(self, batch, alpha=1.0):
        """base_trainer.py:366-446: discriminator step, generator step, step counters."""
        d = self.train_discriminator(batch, alpha)
        g = self.train_generator(batch, alpha)
        self.discriminator.step += 1
        self.generator.step += 1
        return d, g


# ----------------------------------------------------------------------------------------------------------------------
# functional form (bench.py, tests): fp32, no AMP, R1 on its schedule
# ----------------------------------------------------------------------------------------------------------------------
def train_iteration(G, D, opt_g, opt_d, batch, cfg, trainer=None):
    """batch: dict(z_d, z_g, cond, images, labels).  Returns (d_loss, g_loss).  Kept for callers that own their optimisers;
    builds a `Trainer` around them once (cached on G)."""
    t = trainer or getattr(G, "_hg_trainer", None)
    if t is None or t.discriminator is not D:
        from .ops.trainer_ops import FusedAdam
        t = Trainer(G, D, cfg, amp=False, fused=isinstance(opt_g, FusedAdam) and isinstance(opt_d, FusedAdam))
        t.optimizer_G, t.optimizer_D = opt_g, opt_d
        G._hg_trainer = t
    return t.iteration(batch)
