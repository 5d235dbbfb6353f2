"""Host-side schedule of the SPADE synthesis network on top of the C ABI (csrc/synth.cu).

Mirrors `SynthesisNetwork.forward` (lib/generators/map3d_generator.py:58-97) +
`SynthesisInput` (lib/components/map3d_layers.py:260-275) + the bilinear feature up-sample of
`Map3DGenerator.forward` (:244-245), restructured around 18 fused half-block launches:

  * the up-sampled style map is never materialised: `mlp_shared` is applied to the render-resolution
    feature map (one wgmma GEMM, `hg_linear`) and interpolated inside the half-block kernel;
  * half-blocks whose style is spatially constant get per-sample (1+gamma, beta) vectors and skip
    the gamma/beta GEMMs entirely;
  * BatchNorm statistics of every activation are produced by the epilogue of the kernel that
    writes it; `hg_bn_finalize` turns them into scale/shift (+ running-stat update); with a process
    group the [sum, sumsq, count] vector is all-reduced over NCCL first (SyncBatchNorm semantics).

`params` is any mapping from the reference's state_dict names to CUDA fp32 tensors (a module's
`state_dict(keep_vars=True)` or a plain dict).  Buffers (`running_*`, `weight_u/v`,
`num_batches_tracked`) are updated in place when `training` is true, like the reference modules.
"""
from __future__ import annotations

import torch
import torch.distributed as dist
import torch.nn.functional as F

from .. import abi

STAT_STRIDE = 520  # doubles per statistics row: [0:256] sum, [256:512] sumsq, [512] count, pad


def spectral_sigma_batched(w_list, u_list, v_list, training, eps=1e-12):
    """One power iteration per training forward for a list of weights (torch.nn.utils.spectral_norm semantics,
    map3d_layers.py:205-206) in ONE launch of `hg_spectral_norm`; u / v are updated in place.  Returns 1/sigma [n]."""
    return abi.spectral_norm(list(w_list), list(u_list), list(v_list), training, eps)


class SpectralScale(torch.autograd.Function):
    """W / sigma with sigma = u^T W v (u, v constants): forward = W * inv_sigma (inv_sigma from hg_spectral_norm), backward
    dW = g / sigma - <g, W> / sigma^2 * u v^T -- elementwise torch ops only, differentiable again."""

    @staticmethod
    def forward(ctx, w, u, v, inv_sigma):
        ctx.save_for_backward(w, u, v, inv_sigma)
        return w * inv_sigma

    @staticmethod
    def backward(ctx, g):
        w, u, v, inv_sigma = ctx.saved_tensors
        wm = w.reshape(w.shape[0], -1)
        gm = g.reshape(w.shape[0], -1)
        coef = (gm * wm).sum() * inv_sigma * inv_sigma
        dw = gm * inv_sigma - coef * (u[:, None] * v[None, :])
        return dw.reshape(w.shape), None, None, None


def sn_weights(P, names, training, suffix=""):
    """{name: W/sigma with autograd history to weight_orig} for a list of spectral-normed layers: ONE batched
    power-iteration launch, then a differentiable scale per layer.  `names` are state_dict prefixes ending in '.'."""
    ws = [P[n + "weight_orig"] for n in names]
    us = [P[n + "weight_u"] for n in names]
    vs = [P[n + "weight_v"] for n in names]
    with torch.no_grad():
        inv = abi.spectral_norm([w.detach() for w in ws], us, vs, training)
    out = {}
    for i, n in enumerate(names):
        # clones: the buffers are overwritten by the next forward's power iteration while this graph may still be alive
        out[n] = SpectralScale.apply(ws[i], us[i].detach().clone(), vs[i].detach().clone(), inv[i])
    return out


def _gamma_beta_interleaved(wg, bg, wb, bb):
    """[512,128] weight / [512] bias in the accumulator order of spade_pixel_kernel:
    N-block nbk, 64-column group sub: even = gamma, odd = beta, channels nbk*128 + (sub//2)*64 + [0,64).
    The '+1' of `gamma = 1 + mlp_gamma(actv)` (map3d_layers.py:181) is folded into the bias."""
    wg = wg.reshape(256, 128)
    wb = wb.reshape(256, 128)
    Ws, bs = [], []
    for nbk in range(2):
        for half in range(2):
            c0 = nbk * 128 + half * 64
            Ws += [wg[c0:c0 + 64], wb[c0:c0 + 64]]
            bs += [bg[c0:c0 + 64] + 1.0, bb[c0:c0 + 64]]
    return torch.cat(Ws).contiguous(), torch.cat(bs).contiguous()


def all_reduce_stats(row, process_group=None):
    """SyncBatchNorm across ranks (map3d_layers.py:162): SUM-all-reduce one statistics row
    [sum(256) | sumsq(256) | count | pad] in fp64.  No-op without an initialised process group."""
    if dist.is_available() and dist.is_initialized() and dist.get_world_size(process_group) > 1:
        dist.all_reduce(row, group=process_group)
    return row


def is_pixel_style(cfg, k):
    mode = cfg.get("map3d_mode", "isolated")
    return mode == "all" or k in cfg["mod_blocks"]


@torch.no_grad()
def synthesis_forward(params, feat_lr, fixed_style, cfg, *, training=True, passes=3, prefix="synthesis_network.",
                      input_prefix="synthesis_input.", return_internal=False, process_group=None):
    """feat_lr: [B, Rh*Rw, ld>=256] render-resolution features (first 256 columns), fixed_style [B,256].
    Returns rgb [B,3,Hg,Wg] (and, optionally, the activation after every block)."""
    abi.require_device()
    P = params
    dev = feat_lr.device
    B = feat_lr.shape[0]
    Hg, Wg, Rh, Rw = cfg["gen_height"], cfg["gen_width"], cfg["render_height"], cfg["render_width"]
    C = cfg["hidden_dim"]
    if C != 256 or cfg["feature_dim"] != 256:
        raise RuntimeError("hg3d: the sm_90a synthesis kernels are built for hidden_dim == feature_dim == 256")
    HW = Hg * Wg
    nb = cfg["synthesis_blocks"]
    mode = cfg.get("map3d_mode", "isolated")
    world = dist.get_world_size(process_group) if (dist.is_available() and dist.is_initialized()) else 1
    f32 = dict(dtype=torch.float32, device=dev)

    halves = [(k, j) for k in range(nb) for j in range(2)]
    blk = lambda k: f"{prefix}network.m3d_{k}."

    # ---- spectral-normalised conv weights -> packed bf16 operand images
    conv_names = [blk(k) + f"conv_{j}." for k, j in halves]
    inv_sigma = spectral_sigma_batched([P[n + "weight_orig"] for n in conv_names], [P[n + "weight_u"] for n in conv_names],
                                       [P[n + "weight_v"] for n in conv_names], training)
    wimgs = [abi.pack_weight(P[n + "weight_orig"].reshape(C, C), Nb=256, scale_dev=inv_sigma[i:i + 1])[0]
             for i, n in enumerate(conv_names)]

    # ---- SPADE modulation inputs
    px = [(k, j) for k, j in halves if is_pixel_style(cfg, k)]
    cs = [(k, j) for k, j in halves if not is_pixel_style(cfg, k)]
    fs = fixed_style.reshape(B, C).float()
    sp = lambda k, j: blk(k) + f"spade_{j}."
    p_lr = p_bias = None
    wgb, bgb = {}, {}
    if px:
        Ws = torch.cat([P[sp(k, j) + "mlp_shared.0.weight"].reshape(128, C) for k, j in px])       # [n*128, 256]
        bsh = torch.stack([P[sp(k, j) + "mlp_shared.0.bias"] for k, j in px])                       # [n,128]
        img, Nb = abi.pack_weight(Ws.contiguous(), Nb=256)
        X = feat_lr.reshape(B * Rh * Rw, feat_lr.shape[-1])[:, :C]
        p_lr = abi.linear(X, img, Nb, Ws.shape[0], passes=passes)                                   # [B*Rhw, n*128]
        if mode in ("mixed", "all"):      # style = up(f) + fixed_style  => constant W_s.fs + b_s per sample
            p_bias = (fs @ Ws.t()).reshape(B, len(px), 128).permute(1, 0, 2) + bsh[:, None, :]
        else:                             # 'isolated': style = up(f)
            p_bias = bsh[:, None, :].expand(len(px), B, 128)
        p_bias = p_bias.contiguous()
        for k, j in px:
            w, b_ = _gamma_beta_interleaved(P[sp(k, j) + "mlp_gamma.weight"], P[sp(k, j) + "mlp_gamma.bias"],
                                            P[sp(k, j) + "mlp_beta.weight"], P[sp(k, j) + "mlp_beta.bias"])
            wgb[(k, j)] = abi.pack_weight(w, Nb=256)[0]
            bgb[(k, j)] = b_
    gb = {}
    if cs:
        Wsh = torch.stack([P[sp(k, j) + "mlp_shared.0.weight"].reshape(128, C) for k, j in cs])     # [m,128,256]
        bsh = torch.stack([P[sp(k, j) + "mlp_shared.0.bias"] for k, j in cs])
        actv = torch.relu(torch.einsum("bc,mhc->mbh", fs, Wsh) + bsh[:, None, :])                   # [m,B,128]
        Wg_ = torch.stack([P[sp(k, j) + "mlp_gamma.weight"].reshape(C, 128) for k, j in cs])
        Wb_ = torch.stack([P[sp(k, j) + "mlp_beta.weight"].reshape(C, 128) for k, j in cs])
        bg_ = torch.stack([P[sp(k, j) + "mlp_gamma.bias"] for k, j in cs])
        bb_ = torch.stack([P[sp(k, j) + "mlp_beta.bias"] for k, j in cs])
        G = 1.0 + torch.einsum("mbh,mch->mbc", actv, Wg_) + bg_[:, None, :]
        Bt = torch.einsum("mbh,mch->mbc", actv, Wb_) + bb_[:, None, :]
        GB = torch.stack([G, Bt], dim=2).contiguous()                                               # [m,B,2,C]
        for i, key in enumerate(cs):
            gb[key] = GB[i]

    # ---- synthesis input + its statistics
    stats = torch.zeros(len(halves) + 1, STAT_STRIDE, dtype=torch.float64, device=dev)
    stats[:, 512] = float(B * HW)
    ic = torch.linspace(-1, 1, Hg, **f32)
    jc = torch.linspace(-1, 1, Wg, **f32)
    T = (HW + 127) // 128                      # activations are tile-blocked: [B, T, C, 128] (csrc/synth.cu)
    x0 = torch.empty(T, C, 128, **f32)
    abi.synth_input(P[input_prefix + "network.0.weight"].reshape(C, 2).contiguous(), P[input_prefix + "network.0.bias"],
                    ic, jc, x0, stats[0] if training else None, B)

    bufs = [torch.empty(B, T, C, 128, **f32) for _ in range(3)]
    rgb = [torch.empty(B, 3, HW, **f32) for _ in range(2)]
    rgb_cur = None
    scsh = torch.empty(2, C, **f32)
    mod = torch.empty(B, 2, C, **f32)
    cur, cur_bstride = x0, 0
    free = [0, 1, 2]
    block_in = None
    internal = {}
    pxi = {key: i for i, key in enumerate(px)}
    for idx, (k, j) in enumerate(halves):
        bn = sp(k, j) + "first_norm."
        srow = stats[idx]
        if training and world > 1:
            all_reduce_stats(srow, process_group)
        pixel = (k, j) in pxi
        abi.bn_finalize(srow if training else None, P[bn + "weight"], P[bn + "bias"], P[bn + "running_mean"],
                        P[bn + "running_var"], training, count_dev=srow[512:513] if training else None,
                        gb=None if pixel else gb[(k, j)], B=B, scsh=scsh if pixel else None, mod=None if pixel else mod)
        if training and (bn + "num_batches_tracked") in P:
            P[bn + "num_batches_tracked"] += 1
        if j == 0:
            block_in = (cur, cur_bstride)
        out_i = next(i for i in free if bufs[i] is not cur and (block_in is None or bufs[i] is not block_in[0]))
        out = bufs[out_i]
        last_half = j == 1
        use_skip = last_half and k >= nb // 2 and block_in[1] != 0
        use_rgb = last_half and k >= nb // 2 - 1
        kw = {}
        if use_rgb:
            rgb_next = rgb[0] if rgb_cur is not rgb[0] else rgb[1]
            kw = dict(rgb_w=P[f"{prefix}to_rgbs.m3d_{k}.linear.weight"].reshape(3, C).contiguous(),
                      rgb_b=P[f"{prefix}to_rgbs.m3d_{k}.linear.bias"], rgb_in=rgb_cur, rgb_out=rgb_next)
        if pixel:
            i = pxi[(k, j)]
            kw.update(scsh=scsh, p_lr=p_lr[:, i * 128:], p_stride=p_lr.shape[1], p_bias=p_bias[i], wgb=wgb[(k, j)],
                      bgb=bgb[(k, j)], Rh=Rh, Rw=Rw)
        else:
            kw.update(mod=mod)
        _spade(cur, cur_bstride, wimgs[idx], P[blk(k) + f"conv_{j}.bias"], out, B, Hg, Wg, passes,
               skip=block_in[0] if use_skip else None, stats=stats[idx + 1] if training else None, **kw)
        if use_rgb:
            rgb_cur = rgb_next
        cur, cur_bstride = out, T * C * 128
        if return_internal and last_half:
            internal[f"m3d_{k}"] = cur.permute(0, 2, 1, 3).reshape(B, C, T * 128)[:, :, :HW].reshape(B, C, Hg, Wg).clone()
    out_rgb = rgb_cur.reshape(B, 3, Hg, Wg)
    return (out_rgb, internal) if return_internal else out_rgb


def _spade(x, x_bstride, wimg, bias, out, B, Hg, Wg, passes, p_lr=None, **kw):
    if p_lr is not None:
        # a column slice of the [M, n*128] projection: pass the base pointer of the slice explicitly
        view = p_lr
        kw["p_lr"] = _PtrView(view)
    abi.spade_conv(x, x_bstride, wimg, bias, out, B=B, Hg=Hg, Wg=Wg, passes=passes, **kw)


class _PtrView:
    """Minimal tensor stand-in so a non-contiguous column slice can be handed to the ABI by pointer."""

    def __init__(self, t):
        self._t = t
        self.is_cuda = t.is_cuda

    def is_contiguous(self):
        return True

    def data_ptr(self):
        return self._t.data_ptr()
