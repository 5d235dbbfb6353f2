"""Loss + optimiser tail of the reference's training iteration on sm_90a kernels (csrc/trainer.cu; SURVEY.md 8f-1).

  seg_ce_balanced   PhaseTrainer._calculate_segmentation_loss, mode 'cross_entropy_balanced' (phase_trainer.py:203-256):
                    label histogram -> per-class coefficients -> ONE pass over the logits that yields the loss and its gradient.
  image_loss        reconstruction loss of latent inversion (inversion.py) and the photometric loss of conditional phases
                    (phase_trainer.py:525-527): weighted L2, Charbonnier or smooth L1 over an image, value and gradient in one pass.
  latent_pool_gather  `LatentPool.forward` (lib/components/util.py:18-29) with the dense [P,L] gradient of `latents[indices]`.
  latent_loss       the latent regression of phase_trainer.py:425-437, :493-506: mean SL1_beta(n(pred) - n(target)),
                    n = normalize_2nd_moment.
  FusedAdam         torch.optim.Adam (same state_dict: step / exp_avg / exp_avg_sq, same arithmetic) for the reference's
                    parameter groups (phase_trainer.py:57-76) with global-norm clipping (clip_grad_norm_, :314,336) and the
                    generator's EMA (lib/components/ema.py:29-48) folded into the same multi-tensor launch.
"""
from __future__ import annotations

import ctypes
import math

import numpy as np
import torch

from .. import abi


# ----------------------------------------------------------------------------------------------------------------------
# class-balanced cross entropy
# ----------------------------------------------------------------------------------------------------------------------
class _SegCE(torch.autograd.Function):
    @staticmethod
    @torch.amp.custom_fwd(device_type="cuda", cast_inputs=torch.float32)
    def forward(ctx, logits, labels, prior, label_dim):
        abi.require_device()
        logits = logits.contiguous()
        labels = labels.contiguous()
        B, L = logits.shape[0], logits.shape[1]
        HW = logits.numel() // (B * L)
        if L != label_dim or labels.numel() != B * HW or labels.dtype != torch.int64:
            raise RuntimeError("hg3d: seg_ce_balanced expects logits [B,L,H,W] and int64 labels [B,H,W]")
        dev = logits.device
        hist = torch.empty(L, dtype=torch.int32, device=dev)
        coef = torch.empty(L, dtype=torch.float32, device=dev)
        loss = torch.empty(1, dtype=torch.float32, device=dev)
        ws = torch.empty(2 * 160 * 2, dtype=torch.float64, device=dev)
        need_grad = ctx.needs_input_grad[0]
        dlog = torch.empty_like(logits) if need_grad else None
        with torch.cuda.device_of(logits):
            abi.call("hg_label_histogram", abi.ptr(labels), labels.numel(), L, abi.ptr(hist), abi.stream())
            abi.call("hg_seg_ce_coef", abi.ptr(hist), abi.ptr(prior), L, float(labels.numel()), abi.ptr(coef), abi.stream())
            abi.call("hg_seg_ce", abi.ptr(logits), abi.ptr(labels), abi.ptr(coef), abi.ptr(dlog), abi.ptr(loss), abi.ptr(ws), B, L, HW,
                     abi.stream())
        ctx.save_for_backward(dlog)
        return loss.reshape(())

    @staticmethod
    @torch.amp.custom_bwd(device_type="cuda")
    @torch.autograd.function.once_differentiable
    def backward(ctx, g):
        (dlog,) = ctx.saved_tensors
        return (dlog * g if dlog is not None else None), None, None, None


def seg_ce_balanced(segments, gt, label_dim, prior_weights=None):
    """`cross_entropy_balanced` (phase_trainer.py:203-256) -> scalar loss; differentiable w.r.t. `segments` (first order)."""
    if gt.shape[1:] != segments.shape[2:]:
        with torch.no_grad():
            gt = torch.nn.functional.interpolate(gt[:, None].float(), segments.shape[2:], mode="nearest")[:, 0].long()
    prior = None
    if prior_weights is not None:
        prior = torch.as_tensor(prior_weights, dtype=torch.float32, device=segments.device).contiguous()
    return _SegCE.apply(segments, gt, prior, int(label_dim))


# ----------------------------------------------------------------------------------------------------------------------
# image reconstruction loss
# ----------------------------------------------------------------------------------------------------------------------
class _ImageLoss(torch.autograd.Function):
    @staticmethod
    @torch.amp.custom_fwd(device_type="cuda", cast_inputs=torch.float32)
    def forward(ctx, pred, target, mask, mode, eps):
        abi.require_device()
        B = pred.shape[0]
        if pred.dim() != 4 or pred.shape[1] != 3 or target.shape != pred.shape:
            raise RuntimeError("hg3d: image_loss expects prediction and target [B,3,H,W] of one shape")
        HW = pred.shape[2] * pred.shape[3]
        if mask is not None and mask.numel() != B * HW:
            raise RuntimeError("hg3d: image_loss expects a weight mask [B,1,H,W]")
        pred, target = pred.contiguous(), target.contiguous()
        mask = None if mask is None else mask.contiguous()
        dev = pred.device
        loss = torch.empty(1, dtype=torch.float32, device=dev)
        ws = torch.empty(2 * torch.cuda.get_device_properties(dev).multi_processor_count, dtype=torch.float64, device=dev)
        dpred = torch.empty_like(pred) if ctx.needs_input_grad[0] else None
        with torch.cuda.device_of(pred):
            abi.call("hg_image_loss", abi.ptr(pred), abi.ptr(target), abi.ptr(mask), abi.ptr(dpred), abi.ptr(loss), abi.ptr(ws), B, HW,
                     mode, float(eps), abi.stream())
        ctx.save_for_backward(dpred)
        return loss.reshape(())

    @staticmethod
    @torch.amp.custom_bwd(device_type="cuda")
    @torch.autograd.function.once_differentiable
    def backward(ctx, g):
        (dpred,) = ctx.saved_tensors
        return (dpred * g if dpred is not None else None), None, None, None, None


def image_loss(pred, target, mask=None, kind="l2", eps=1e-3, beta=1.0):
    """mean over the B*3*H*W elements of mask * rho(pred - target): rho(d) = d^2 (`kind="l2"`), the Charbonnier
    sqrt(d^2 + eps^2) (`kind="charbonnier"`) or `F.smooth_l1_loss`'s rho with `beta` (`kind="smooth_l1"`, the photometric
    loss of phase_trainer.py:525-527 with beta = 0.1).  `mask` [B,1,H,W] fp32 weights each pixel (the person's
    silhouette: `preprocess.Preprocessor` labels != background) or None.  Differentiable w.r.t. `pred` (first order); the
    value repeats bit for bit (fp64 partial sums in a fixed order)."""
    modes = {"l2": (0, eps), "charbonnier": (1, eps), "smooth_l1": (2, beta)}
    if kind not in modes:
        raise RuntimeError(f"hg3d: image_loss kind {kind!r} is not built ('l2', 'charbonnier' or 'smooth_l1')")
    if mask is not None:
        mask = mask.to(torch.float32)
    mode, e = modes[kind]
    return _ImageLoss.apply(pred, target, mask, mode, e)


# ----------------------------------------------------------------------------------------------------------------------
# latent pool lookup and latent regression
# ----------------------------------------------------------------------------------------------------------------------
class _LatentPoolGather(torch.autograd.Function):
    @staticmethod
    @torch.amp.custom_fwd(device_type="cuda", cast_inputs=torch.float32)
    def forward(ctx, pool, indices):
        abi.require_device()
        if pool.dim() != 2 or indices.dim() != 1 or indices.dtype != torch.int64:
            raise RuntimeError("hg3d: latent_pool_gather expects a pool [P,L] and int64 indices [B]")
        pool = pool.contiguous()
        indices = indices.to(pool.device).contiguous()
        P, L = pool.shape
        B = indices.shape[0]
        out = torch.empty(B, L, dtype=torch.float32, device=pool.device)
        if B > 0:
            with torch.cuda.device_of(pool):
                abi.call("hg_latent_pool_gather", abi.ptr(pool), P, L, abi.ptr(indices), B, abi.ptr(out), abi.stream())
        ctx.save_for_backward(indices)
        ctx.pool_shape = (P, L)
        return out

    @staticmethod
    @torch.amp.custom_bwd(device_type="cuda")
    @torch.autograd.function.once_differentiable
    def backward(ctx, dz):
        (indices,) = ctx.saved_tensors
        P, L = ctx.pool_shape
        dz = dz.float().contiguous()
        dpool = torch.empty(P, L, dtype=torch.float32, device=dz.device)
        with torch.cuda.device_of(dz):
            if indices.shape[0] > 0:
                abi.call("hg_latent_pool_grad", abi.ptr(dz), abi.ptr(indices), indices.shape[0], L, P, abi.ptr(dpool), abi.stream())
            else:
                dpool.zero_()
        return dpool, None


def latent_pool_gather(pool, indices):
    """`pool[indices]` for a pool [P,L] (the `latent_pool.latents` parameter) and integer indices [B] -> [B,L].  The backward
    returns the dense [P,L] gradient that the reference's `self.latents[indices]` produces -- zero rows except the indexed
    ones, each the sum of its rows of the incoming gradient in batch order -- to autograd, so accumulation over micro-batches
    and DDP's reducer hooks treat it as any other parameter's gradient.  An index outside [0, P) gives a NaN row."""
    idx = indices.long()
    return _LatentPoolGather.apply(pool, idx.reshape(-1)).reshape(*idx.shape, pool.shape[-1])


class _LatentLoss(torch.autograd.Function):
    @staticmethod
    @torch.amp.custom_fwd(device_type="cuda", cast_inputs=torch.float32)
    def forward(ctx, pred, target, beta):
        abi.require_device()
        if pred.dim() != 2 or target.shape != pred.shape:
            raise RuntimeError("hg3d: latent_loss expects prediction and target [B,L] of one shape")
        pred, target = pred.contiguous(), target.contiguous()
        loss = torch.empty(1, dtype=torch.float32, device=pred.device)
        with torch.cuda.device_of(pred):
            abi.call("hg_latent_loss", abi.ptr(pred), abi.ptr(target), pred.shape[0], pred.shape[1], float(beta), None, None, abi.ptr(loss),
                     abi.stream())
        ctx.save_for_backward(pred, target)
        ctx.beta = beta
        return loss.reshape(())

    @staticmethod
    @torch.amp.custom_bwd(device_type="cuda")
    @torch.autograd.function.once_differentiable
    def backward(ctx, g):
        pred, target = ctx.saved_tensors
        if not ctx.needs_input_grad[0]:
            return None, None, None
        dpred = torch.empty_like(pred)
        g = g.float().reshape(1).contiguous()
        with torch.cuda.device_of(pred):
            abi.call("hg_latent_loss", abi.ptr(pred), abi.ptr(target), pred.shape[0], pred.shape[1], float(ctx.beta), abi.ptr(g),
                     abi.ptr(dpred), None, abi.stream())
        return dpred, None, None


def latent_loss(pred, target, beta=0.1):
    """`F.smooth_l1_loss(normalize_2nd_moment(pred), normalize_2nd_moment(target), beta=beta)` for [B,L] latents
    (phase_trainer.py:425-437, :493-506) -> scalar; differentiable w.r.t. `pred` (first order), `target` is a constant.
    The value repeats bit for bit (fp64 row sums in a fixed order)."""
    return _LatentLoss.apply(pred, target.detach(), beta)


# ----------------------------------------------------------------------------------------------------------------------
# multi-tensor Adam + clip + EMA
# ----------------------------------------------------------------------------------------------------------------------
class FusedAdam(torch.optim.Optimizer):
    """Drop-in for `torch.optim.Adam(params, lr, betas, eps, weight_decay)` (no amsgrad / maximize): identical state
    (`step`, `exp_avg`, `exp_avg_sq`) and update arithmetic, executed for ALL tensors of all groups in one launch.
    `step(clip_max_norm=..., ema=...)` folds `clip_grad_norm_` over the optimiser's parameters and the EMA update in."""

    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0):
        super().__init__(params, dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay))
        self._chunks = None
        self._key = None
        self.last_grad_norm = None
        self._stepped = False

    def _flat(self):
        return [(gi, p) for gi, grp in enumerate(self.param_groups) for p in grp["params"]]

    @torch.no_grad()
    def step(self, closure=None, clip_max_norm=None, ema=None, ema_params=None):
        """ema: an object with `shadow_params` / `decay` / `num_updates` (train_step.ParameterEMA = lib/components/ema.py);
        ema_params: the parameter list the EMA was built from, in ITS order (`generator.parameters()`, ema.py:25 -- not the
        order of the optimiser's groups).  Defaults to this optimiser's parameters in group order."""
        if closure is not None:
            raise RuntimeError("hg3d: FusedAdam does not take a closure")
        abi.require_device()
        flat = self._flat()
        dev = flat[0][1].device
        shadow = None
        if ema is not None:      # shadow copies exist for the parameters that require grad, in parameters() order (ema.py:25)
            req = [p for p in (ema_params if ema_params is not None else [q for _, q in flat]) if p.requires_grad]
            if len(req) != len(ema.shadow_params) or any(p.shape != s.shape for p, s in zip(req, ema.shadow_params)):
                raise RuntimeError("hg3d: the EMA's shadow parameters do not line up with `ema_params`")
            shadow = {id(p): s for p, s in zip(req, ema.shadow_params)}
            if any(id(p) not in shadow for _, p in flat if p.requires_grad):
                raise RuntimeError("hg3d: the EMA does not cover this optimiser's parameters")
        # refuse before any state changes: a refused call must leave `step` (and so every later bias correction) as it was
        pairs = {(gi, int(self.state[p]["step"]) + 1 if len(self.state[p]) else 1) for gi, p in flat if p.grad is not None}
        if len(pairs) > 8:
            raise RuntimeError("hg3d: FusedAdam handles at most 8 distinct (group, step) pairs per call")
        # per-(group, step) scalars
        sgroups, sidx = [], {}
        ents = np.zeros((len(flat), 6), dtype=np.int64)
        chunk_rows = []
        CH = int(abi.lib().hg_mt_chunk_elems())
        for ti, (gi, p) in enumerate(flat):
            if p.dtype != torch.float32 or not p.is_contiguous():
                raise RuntimeError("hg3d: FusedAdam takes contiguous fp32 parameters")
            g = p.grad
            st = self.state[p]
            sg = 0
            if g is not None:
                if g.is_sparse or g.dtype != torch.float32:
                    raise RuntimeError("hg3d: FusedAdam takes dense fp32 gradients")
                if not g.is_contiguous():
                    g = p.grad = g.contiguous()
                if len(st) == 0:
                    st["step"] = torch.tensor(0.0, dtype=torch.float32)
                    st["exp_avg"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                    st["exp_avg_sq"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                st["step"] += 1
                t = int(st["step"])
                key = (gi, t)
                if key not in sidx:
                    grp = self.param_groups[gi]
                    b1, b2 = (float(b) for b in grp["betas"])
                    sidx[key] = len(sgroups)
                    sgroups.append((float(grp["lr"]), b1, b2, float(grp["eps"]), float(grp["weight_decay"]), 1.0 - b1 ** t,
                                    math.sqrt(1.0 - b2 ** t)))
                sg = sidx[key]
                ents[ti] = (p.data_ptr(), g.data_ptr(), st["exp_avg"].data_ptr(), st["exp_avg_sq"].data_ptr(),
                            shadow[id(p)].data_ptr() if shadow is not None and id(p) in shadow else 0, p.numel())
            else:
                ents[ti] = (p.data_ptr(), 0, 0, 0, shadow[id(p)].data_ptr() if shadow is not None and id(p) in shadow else 0, p.numel())
            for off in range(0, p.numel(), CH):
                chunk_rows.append((ti, sg, off))
        if not sgroups:
            sgroups.append((0.0, 0.0, 0.0, 1.0, 0.0, 1.0, 1.0))          # nothing to step; the EMA (if any) still runs
        assert len(sgroups) == max(1, len(pairs))
        assert int(abi.lib().hg_mt_entry_bytes()) == 48 and int(abi.lib().hg_mt_chunk_bytes()) == 16
        table = torch.from_numpy(ents).to(dev, non_blocking=True)
        ch = np.zeros((len(chunk_rows), 2), dtype=np.int64)
        for i, (ti, sg, off) in enumerate(chunk_rows):
            ch[i, 0] = ti | (sg << 32)
            ch[i, 1] = off
        chunks = torch.from_numpy(ch).to(dev, non_blocking=True)
        n = len(chunk_rows)
        norm_clip = None
        with torch.cuda.device_of(table):
            if clip_max_norm is not None:
                partials = torch.empty(n, dtype=torch.float64, device=dev)
                norm_clip = torch.empty(2, dtype=torch.float32, device=dev)
                abi.call("hg_mt_grad_norm", abi.ptr(table), abi.ptr(chunks), n, float(clip_max_norm), abi.ptr(partials), abi.ptr(norm_clip),
                         abi.stream())
                self.last_grad_norm = norm_clip[0]
            ng = len(sgroups)
            sc = (ctypes.c_float * (7 * ng))(*[sgroups[i][k] for k in range(7) for i in range(ng)])
            omd = 0.0
            if ema is not None:
                decay = ema.decay
                if ema.num_updates is not None:
                    ema.num_updates += 1
                    decay = min(decay, (1 + ema.num_updates) / (10 + ema.num_updates))
                omd = 1.0 - decay
            abi.call("hg_mt_adam", abi.ptr(table), abi.ptr(chunks), n, abi.ptr(norm_clip), ctypes.cast(sc, ctypes.c_void_p), ng, float(omd),
                     int(clip_max_norm is not None), abi.stream())
        self._keep = (table, chunks)          # keep the tables alive until the launches have been issued
        self._stepped = True
        return None
