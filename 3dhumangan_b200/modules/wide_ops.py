"""Forward path for every hidden_dim / feature_dim <= 512 other than 256 -- the 256-pixel curriculum MAP3DBN (384,
configs/map3d.py:3-95) and the released checkpoint's MAP3DBN512L (420, configs/map3d.py:194-290, doc/GET_STARTED.md:17-22).

The fused kernels (csrc/render.cu, csrc/synth.cu's pixel-style kernel) are laid out for exactly 256 channels (register
accumulators, shared-memory budget).  Wider networks run on the library's GENERAL blocked-GEMM engine instead: every channel dimension is
zero-padded to 512 = two tile-blocked halves [B,T,256,128], and a 512 -> 512 layer is two launches of
`hg_blocked_conv_wide` (K = 512 from two sources with a modulation table per source, N = 256 outputs each), with the same
fused prologue (BatchNorm x SPADE modulation x LeakyReLU, or FiLM sine) and epilogue (bias, residual, ToRGB, next-layer
BatchNorm statistics) as the 256-channel path.  Zero padding is exact: padded channels carry zero weights, zero BatchNorm
affine and zero FiLM tables, so they stay zero through every layer.

  renderer   layer by layer over tile-blocked points (the training path's schedule, modules/render_train.py), compositing
             per 256-feature half;
  synthesis  const-style half-blocks: bn_finalize per half + 2 launches; pixel-style half-blocks: A1 = relu(up(P_lr) + c),
             gamma / beta by `hg_conv1x1_blocked`, pre = BN(x) * gamma + beta (`hg_spade_pixel_pre`), then the wide conv with
             an identity table -- the decomposition the 256-channel BACKWARD already uses.

Inference and train-mode forward (batch statistics, running-stat and spectral-norm buffer updates).  Given a `tape`
(train mode, or eval mode with the running statistics and the stored spectral-norm u / v as constants),
each forward also keeps what the backward of every width needs (render_train.mlp_backward,
synthesis_train.synthesis_backward, over two 256-channel halves here), and builds the small tables that carry
parameter gradients (FiLM, SPADE / BatchNorm, W / sigma) with autograd history.  Mirrors Map3DGenerator.render / forward (map3d_generator.py:208-280, 381-523),
COORDCONCATSIREN.forward (modulated.py:41-75), SynthesisNetwork.forward (map3d_generator.py:58-97).
"""
from __future__ import annotations

import torch
import torch.distributed as dist
import torch.nn.functional as F

from .. import abi
from ..ops.dense import _gemm_nt
from .synthesis_ops import STAT_STRIDE, _PtrView, all_reduce_stats, is_pixel_style, sn_weights, spectral_sigma_batched

HALF = 256


def _pad2(w, rows, cols):
    """Zero-pad a matrix to [rows, cols]."""
    out = torch.zeros(rows, cols, dtype=torch.float32, device=w.device)
    out[:w.shape[0], :w.shape[1]] = w
    return out


def _pad1(v, n, fill=0.0):
    out = torch.full((n,), float(fill), dtype=torch.float32, device=v.device)
    out[:v.shape[0]] = v
    return out


def _halves(v):
    return v[:HALF].contiguous(), v[HALF:].contiguous()


def _pack_rows(W512, oh):
    """Operand image of output half `oh` of a zero-padded [512, K] weight (K a multiple of 64, <= 512)."""
    return abi.pack_weight(W512[oh * HALF:(oh + 1) * HALF].contiguous(), Nb=256)[0]


def wide_layer(xs, W512, b512, *, mods=None, act=0, slope=0.2, skips=None, stats=None, rgb=None, B, Hg, Wg, passes):
    """One 512 -> 512 layer over two tile-blocked halves.  xs = (lo, hi) [B,T,256,128]; mods = (table_lo, table_hi) [B,2,256]
    or None (identity); skips = (lo, hi) or None; stats = (row_lo, row_hi) float64 views or None;
    rgb = dict(w [3,512], b [3], rgb_in, out0, out1) accumulates ToRGB over both halves.  Returns (out_lo, out_hi)."""
    outs = []
    T = xs[0].shape[1]
    for oh in (0, 1):
        out = torch.empty(B, T, HALF, 128, dtype=torch.float32, device=xs[0].device)
        kw = {}
        if rgb is not None:       # rgb_out(oh) = rgb_in(oh) + W_rgb[:, half] . out_half (+ bias once)
            kw = dict(rgb_w=rgb["w"][:, oh * HALF:(oh + 1) * HALF].contiguous(), rgb_b=rgb["b"] if oh == 0 else torch.zeros_like(rgb["b"]),
                      rgb_in=rgb["rgb_in"] if oh == 0 else rgb["out0"], rgb_out=rgb["out0"] if oh == 0 else rgb["out1"])
        with torch.cuda.device_of(out):
            abi.call("hg_blocked_conv_wide", abi.ptr(xs[0]), abi.ptr(xs[1]), abi.ptr(None if mods is None else mods[0]),
                     abi.ptr(None if mods is None else mods[1]), int(act), float(slope), abi.ptr(_pack_rows(W512, oh)),
                     abi.ptr(b512[oh * HALF:(oh + 1) * HALF].contiguous()), abi.ptr(None if skips is None else skips[oh]), abi.ptr(out),
                     abi.ptr(None if stats is None else stats[oh]), abi.ptr(kw.get("rgb_w")), abi.ptr(kw.get("rgb_b")),
                     abi.ptr(kw.get("rgb_in")), abi.ptr(kw.get("rgb_out")), B, Hg, Wg, passes, abi.stream())
        outs.append(out)
    return tuple(outs)


# ----------------------------------------------------------------------------------------------------------------------
# renderer
# ----------------------------------------------------------------------------------------------------------------------
@torch.no_grad()
def render_forward_wide(P, freq, phase, cond, cfg, u, noise, *, passes=3, prefix="neural_field.", tape=None, records=None,
                        sigma_only=False, point_rgb=False, training=True):
    """-> ray features [B,R,C], rgb [B,R,3] (in [0,1], before the *2-1), depth [B,R,1].
    `tape` (a dict) receives what `render_train.mlp_backward` needs, in the format its docstring describes: per half the
    linear outputs lin_a, lin_b, out_0..3, lin_c, feat, then sig, rgbp and the FiLM tables built from freq / phase
    leaves with autograd history.
    `records` (rec [B,N,36], z_vals [B,N]) replaces the ray stage (hierarchical_sample: the merged samples, with
    cfg["num_steps"] the samples per ray).  `sigma_only` stops after the sigma head and returns the raw sigma [B,N];
    `point_rgb` stops after the heads and returns the per-point colour [B,N,3] (the sigmoid of the rgb head, before compositing).
    `training` matters with a tape only: `last_back=True` is differentiated for an eval-mode module, refused in train mode."""
    from . import render_train
    abi.require_device()
    g = lambda n: P[prefix + n].detach().float()
    C = cfg["hidden_dim"]
    Fd = cfg["feature_dim"]
    if not (C <= 2 * HALF and Fd <= 2 * HALF):
        raise RuntimeError("hg3d: the zero-padded path serves hidden_dim <= 512")
    if cfg.get("neural_field_blocks", 4) != 4:
        raise RuntimeError("hg3d: the renderer is built for neural_field_blocks == 4 (all shipped curricula)")
    if tape is not None and training and cfg.get("last_back", False):
        raise RuntimeError("hg3d: last_back=True is an inference-only setting (eval_last_back); the training renderer does not build it")
    if records is None and cfg.get("hierarchical_sample", False):
        from . import hierarchical
        h = hierarchical.merged_records(P, freq, phase, cond, cfg, u, noise, passes=passes)
        records, cfg, noise = (h["rec"], h["z_vals"]), h["cfg"], h["noise"]
    dev = freq.device
    B = freq.shape[0]
    S = cfg["num_steps"]
    geo_dim = cfg["geo_feature_dim"]
    rec, z_vals = render_train.geo_records(cond, cfg, u) if records is None else records
    N = rec.shape[1]
    R = N // S
    if N % 128:
        raise RuntimeError("hg3d: the wide renderer needs render_height * render_width * num_steps to be a multiple of 128")
    f32 = dict(dtype=torch.float32, device=dev)
    kw = dict(B=B, Hg=1, Wg=N, passes=passes)
    T = N // 128
    new = lambda: torch.empty(B, T, HALF, 128, **f32)
    rec_b = render_train.blocked_points(rec[..., :3 + geo_dim], 128)

    # FiLM tables per half [B,2,256]: (f, phi), zero in the padded channels so that sin(0 * x + 0) = 0
    taped = tape is not None
    with torch.set_grad_enabled(taped):
        fq = freq.detach().float().requires_grad_(taped)
        ph = phase.detach().float().requires_grad_(taped)
        f = fq * 15 + 30

        def table(fv, pv):
            t = torch.zeros(B, 2, 2 * HALF, **f32)
            t[:, 0, :C] = fv
            t[:, 1, :C] = pv
            return t[:, :, :HALF].contiguous(), t[:, :, HALF:].contiguous()

        mods_h = [table(f[:, i * C:(i + 1) * C], ph[:, i * C:(i + 1) * C]) for i in range(4)]
    mods = [(lo.detach(), hi.detach()) for lo, hi in mods_h]
    m30 = table(torch.full((B, C), 30.0, **f32), torch.zeros(B, C, **f32))

    # first layers: K = 3 / 31 zero-padded to 128 input channels
    Wa = torch.zeros(2 * HALF, 128, **f32)
    Wb = torch.zeros(2 * HALF, 128, **f32)
    Wa[:C, :3] = g("first_layer_coord.layer.weight")
    Wb[:C, 3:3 + geo_dim] = g("first_layer_mod.layer.weight")
    ba, bb = _pad1(g("first_layer_coord.layer.bias"), 2 * HALF), _pad1(g("first_layer_mod.layer.bias"), 2 * HALF)
    lin_a = tuple(abi.conv1x1_blocked(rec_b, 128, _pack_rows(Wa, h), ba[h * HALF:(h + 1) * HALF].contiguous(), new(), **kw) for h in (0, 1))
    lin_b = tuple(abi.conv1x1_blocked(rec_b, 128, _pack_rows(Wb, h), bb[h * HALF:(h + 1) * HALF].contiguous(), new(), **kw) for h in (0, 1))
    # network.0: K = 2C = [sin(30 lin_a) | sin(30 lin_b)]: two K = 512 launches per output half, chained through the residual
    w0 = g("network.0.layer.weight")
    zero_b = torch.zeros(2 * HALF, **f32)
    part = wide_layer(lin_a, _pad2(w0[:, :C], 2 * HALF, 2 * HALF), _pad1(g("network.0.layer.bias"), 2 * HALF), mods=m30, act=1, **kw)
    x = wide_layer(lin_b, _pad2(w0[:, C:], 2 * HALF, 2 * HALF), zero_b, mods=m30, act=1, skips=part, **kw)
    if taped:
        tape.update(rec_b=rec_b, lin_a=lin_a, lin_b=lin_b, m30=m30)
    del part, lin_a, lin_b
    outs = []
    for i in range(1, 4):
        if taped:
            outs.append(x)
        x = wide_layer(x, _pad2(g(f"network.{i}.layer.weight"), 2 * HALF, 2 * HALF), _pad1(g(f"network.{i}.layer.bias"), 2 * HALF),
                       mods=mods[i - 1], act=1, **kw)
    out3 = x
    w_sigma = _pad1(g("sigma_layer.weight").reshape(-1), 2 * HALF)
    heads_b = torch.cat([g("sigma_layer.bias").reshape(1), g("color_layer_linear.bias").reshape(3)]).contiguous()
    if sigma_only:
        # hg_render_heads also forms the rgb head from its `linc` operand; out3 stands in for it and that output is dropped
        sig = None
        for h in (0, 1):
            s_h, _ = abi.render_heads(out3[h], out3[h], mods[3][h], w_sigma[h * HALF:(h + 1) * HALF].contiguous(),
                                      torch.zeros(3, HALF, **f32), heads_b if h == 0 else torch.zeros_like(heads_b), B=B, N=N)
            sig = s_h if sig is None else sig + s_h
        return sig
    wcol = g("color_layer_sine.layer.weight")
    dvec = torch.tensor((0.0, 0.0, -1.0), **f32)            # locked view direction (map3d_generator.py:418-420)
    bcol = g("color_layer_sine.layer.bias") + wcol[:, :3] @ dvec
    lin_c = wide_layer(out3, _pad2(wcol[:, 3:], 2 * HALF, 2 * HALF), _pad1(bcol, 2 * HALF), mods=mods[3], act=1, **kw)
    feat = wide_layer(lin_c, _pad2(g("feature_layer_linear.weight"), 2 * HALF, 2 * HALF), _pad1(g("feature_layer_linear.bias"), 2 * HALF),
                      mods=mods[3], act=1, **kw)
    # heads: sigma = w_s . sin(f3 out3 + phi3) + b, rgb_pre = W_rgb . sin(f3 lin_c + phi3) + b, summed over the halves
    w_rgb = _pad2(g("color_layer_linear.weight"), 3, 2 * HALF)
    sig = rgbp = None
    for h in (0, 1):
        s_h, r_h = abi.render_heads(out3[h], lin_c[h], mods[3][h], w_sigma[h * HALF:(h + 1) * HALF].contiguous(),
                                    w_rgb[:, h * HALF:(h + 1) * HALF].contiguous(), heads_b if h == 0 else torch.zeros_like(heads_b),
                                    B=B, N=N)
        sig = s_h if sig is None else sig + s_h
        rgbp = r_h if rgbp is None else rgbp + r_h
    if point_rgb:
        return torch.sigmoid(rgbp).transpose(1, 2).contiguous()
    nz = None if noise is None else noise.reshape(B, N).float().contiguous()
    comp = dict(B=B, R=R, S=S, noise_std=cfg["nerf_noise"], white_back=cfg.get("white_back", False),
                softplus=cfg["clamp_mode"] == "softplus", last_back=cfg.get("last_back", False))
    ray0, _ = abi.render_composite(sig, z_vals, nz, rgbp, feat[0], **comp)
    ray1, _ = abi.render_composite(sig, z_vals, nz, rgbp, feat[1], **comp)
    if taped:
        with torch.enable_grad():      # colour bias and direction columns, with history (cf. render_train.mlp_forward_train)
            bcol_t = P[prefix + "color_layer_sine.layer.bias"] + P[prefix + "color_layer_sine.layer.weight"][:, :3] @ dvec
        tape.update(P=P, prefix=prefix, C=C, Fd=Fd, B=B, N=N, R=R, geo_dim=geo_dim, kw=kw, fq=fq, ph=ph, mods_h=mods_h, mods=mods,
                    outs=outs + [out3], lin_c=lin_c, feat=feat, sig=sig, rgbp=rgbp, z=z_vals, noise=nz, comp=comp, bcol=bcol_t,
                    w_sigma=w_sigma, w_rgb=w_rgb)
    feats = torch.cat([ray0[..., :HALF], ray1[..., :HALF]], -1)[..., :Fd].contiguous()
    return feats, ray0[..., 256:259].contiguous(), ray0[..., 259:260].contiguous()


# ----------------------------------------------------------------------------------------------------------------------
# synthesis network
# ----------------------------------------------------------------------------------------------------------------------
@torch.no_grad()
def synthesis_forward_wide(P, feats, fixed_style, cfg, *, training=True, passes=3, prefix="synthesis_network.",
                           input_prefix="synthesis_input.", process_group=None, tape=None):
    """feats [B, Rh*Rw, C] render-resolution features, fixed_style [B,C] -> rgb [B,3,Hg,Wg].
    `tape` (a `synthesis_train.SynthesisTape`) receives what `synthesis_train.synthesis_backward` needs:
    per half-block its input halves, the SPADE tables built with autograd from sum(x) / sum(x^2) leaves (instead of
    hg_bn_finalize), W / sigma with history and the skip / ToRGB bookkeeping, in the format of that class.  With
    `training=False` the taped tables come from the running statistics (no leaves) and no buffer is written."""
    abi.require_device()
    dev = feats.device
    B = feats.shape[0]
    Hg, Wg, Rh, Rw = cfg["gen_height"], cfg["gen_width"], cfg["render_height"], cfg["render_width"]
    C = cfg["hidden_dim"]
    if cfg["feature_dim"] != C:
        raise RuntimeError("hg3d: the synthesis network is built for feature_dim == hidden_dim (all shipped curricula)")
    HW = Hg * Wg
    T = (HW + 127) // 128
    nb = cfg["synthesis_blocks"]
    mode = cfg.get("map3d_mode", "isolated")
    world = dist.get_world_size(process_group) if (training and dist.is_available() and dist.is_initialized()) else 1
    f32 = dict(dtype=torch.float32, device=dev)
    halves = [(k, j) for k in range(nb) for j in range(2)]
    blk = lambda k: f"{prefix}network.m3d_{k}."
    sp = lambda k, j: blk(k) + f"spade_{j}."
    W2 = 2 * HALF
    kw = dict(B=B, Hg=Hg, Wg=Wg, passes=passes)

    conv_names = [blk(k) + f"conv_{j}." for k, j in halves]
    fs = fixed_style.reshape(B, C).float()
    px = [(k, j) for k, j in halves if is_pixel_style(cfg, k)]
    pxi = {key: i for i, key in enumerate(px)}
    taped = tape is not None
    if taped:
        with torch.enable_grad():
            w_sns = sn_weights(P, conv_names, training)
        fs = fs.detach().requires_grad_(True)           # leaf: its gradient is returned by the backward
        tape.cfg, tape.B, tape.fixed_style, tape.px = cfg, B, fs, px
        tape.process_group, tape.world = process_group, world
    else:
        inv_sigma = spectral_sigma_batched([P[n + "weight_orig"] for n in conv_names], [P[n + "weight_u"] for n in conv_names],
                                           [P[n + "weight_v"] for n in conv_names], training)
    p_lr = None
    if px:
        Ws = torch.cat([P[sp(k, j) + "mlp_shared.0.weight"].reshape(128, C) for k, j in px]).float()      # [n*128, C]
        bsh = torch.stack([P[sp(k, j) + "mlp_shared.0.bias"] for k, j in px]).float()
        X = feats.reshape(B * Rh * Rw, feats.shape[-1])[:, :C]
        p_lr = _gemm_nt(X, Ws, passes=passes)                                                              # [B*Rhw, n*128]
        if taped:       # the per-sample constant after the up-sample, with history (cf. synthesis_train)
            with torch.enable_grad():
                PB = [F.linear(fs, P[sp(k, j) + "mlp_shared.0.weight"].reshape(128, C), P[sp(k, j) + "mlp_shared.0.bias"])
                      if mode in ("mixed", "all") else P[sp(k, j) + "mlp_shared.0.bias"][None, :].expand(B, 128) for k, j in px]
            p_bias = torch.stack([t.detach().float() for t in PB])
            tape.p = dict(Ws=Ws, X=X, p_lr=p_lr)
        elif mode in ("mixed", "all"):
            p_bias = (_gemm_nt(fs, Ws, passes=passes)).reshape(B, len(px), 128).permute(1, 0, 2) + bsh[:, None, :]
        else:
            p_bias = bsh[:, None, :].expand(len(px), B, 128)
        p_bias = p_bias.contiguous()

    # ---- synthesis input, per half, materialised per sample (the wide kernel strides both sources by sample)
    stats = torch.zeros(len(halves) + 1, 2, STAT_STRIDE, dtype=torch.float64, device=dev)
    stats[:, :, 512] = float(B * HW)
    ic = torch.linspace(-1, 1, Hg, **f32)
    jc = torch.linspace(-1, 1, Wg, **f32)
    w_in = _pad2(P[input_prefix + "network.0.weight"].reshape(C, 2).float(), W2, 2)
    b_in = _pad1(P[input_prefix + "network.0.bias"].float(), W2)
    cur = []
    for h in (0, 1):
        x0 = torch.empty(T, HALF, 128, **f32)
        abi.synth_input(w_in[h * HALF:(h + 1) * HALF].contiguous(), b_in[h * HALF:(h + 1) * HALF].contiguous(), ic, jc, x0,
                        stats[0, h] if training else None, B)
        cur.append(x0[None].expand(B, T, HALF, 128).contiguous())
    cur = tuple(cur)
    if taped:
        tape.input = dict(w=w_in, b=b_in, ic=ic, jc=jc, prefix=input_prefix)

    rgb_cur = None
    block_in = None
    full = T * HALF * 128
    for idx, (k, j) in enumerate(halves):
        bn = sp(k, j) + "first_norm."
        pixel = (k, j) in pxi
        if training and world > 1:
            for h in (0, 1):
                all_reduce_stats(stats[idx, h], process_group)
        if taped:
            mod, tables, ssum, ssq = _taped_tables(P, stats[idx] if training else None, bn, sp(k, j), fs, pixel, C,
                                                   float(B * HW * world))
        else:
            tables = _tables(P, stats[idx], bn, sp(k, j), fs, pixel, C, B, training, passes)
        if j == 0:
            block_in = (cur, idx)
        last_half = j == 1
        use_skip = last_half and k >= nb // 2 and block_in[1] != 0
        use_rgb = last_half and k >= nb // 2 - 1
        conv = blk(k) + f"conv_{j}."
        if taped:
            Wc = _pad2(w_sns[conv].detach().reshape(C, C), W2, W2)
        else:
            Wc = _pad2(P[conv + "weight_orig"].reshape(C, C).float() * inv_sigma[idx], W2, W2)
        bc = _pad1(P[conv + "bias"].float(), W2)
        rgb = name = None
        if use_rgb:
            name = f"{prefix}to_rgbs.m3d_{k}.linear."
            rgb = dict(w=_pad2(P[name + "weight"].reshape(3, C).float(), 3, W2), b=P[name + "bias"].float().contiguous(), rgb_in=rgb_cur,
                       out0=torch.empty(B, 3, HW, **f32), out1=torch.empty(B, 3, HW, **f32))
        srows = (stats[idx + 1, 0], stats[idx + 1, 1]) if training else None
        if taped:
            rec = dict(x=cur, x_bstride=full, mod=mod, mod_d=tuple(tables), w_sn=w_sns[conv], ssum=ssum, ssq=ssq, conv=conv,
                       pixel=pixel, skip_from=block_in[1] if use_skip else None, rgb=name, rgb_w=None if rgb is None else rgb["w"])
            tape.halves.append(rec)
        if pixel:
            i = pxi[(k, j)]
            s_ = sp(k, j)
            a1 = torch.empty(B, T, 128, 128, **f32)
            abi.spade_a1(_PtrView(p_lr[:, i * 128:]), p_lr.shape[1], p_bias[i].contiguous(), a1, B=B, Hg=Hg, Wg=Wg, Rh=Rh, Rw=Rw)
            wg = _pad2(P[s_ + "mlp_gamma.weight"].reshape(C, 128).float(), W2, 128)
            wb = _pad2(P[s_ + "mlp_beta.weight"].reshape(C, 128).float(), W2, 128)
            bg1 = _pad1(P[s_ + "mlp_gamma.bias"].float() + 1.0, W2)
            bb = _pad1(P[s_ + "mlp_beta.bias"].float(), W2)
            if taped:
                rec.update(i=i, spade=s_, p_bias=PB[i], p_bias_d=p_bias[i].contiguous(), wg=wg, wb=wb, bg1=bg1, bb=bb)
            pres = []
            for h in (0, 1):
                sl = slice(h * HALF, (h + 1) * HALF)
                gam = abi.conv1x1_blocked(a1, 128, _pack_rows(wg, h), bg1[sl].contiguous(), torch.empty(B, T, HALF, 128, **f32), **kw)
                pre = abi.conv1x1_blocked(a1, 128, _pack_rows(wb, h), bb[sl].contiguous(), torch.empty(B, T, HALF, 128, **f32), **kw)
                abi.spade_pixel_pre(cur[h], full, tables[h], gam, pre, B=B, Hg=Hg, Wg=Wg)        # pre = (x*sc+sh)*gam + bet
                pres.append(pre)
                del gam
            out = wide_layer(tuple(pres), Wc, bc, mods=None, act=0, slope=0.2, skips=block_in[0] if use_skip else None, stats=srows,
                             rgb=rgb, **kw)
            del pres, a1
        else:
            out = wide_layer(cur, Wc, bc, mods=tuple(tables), act=0, slope=0.2, skips=block_in[0] if use_skip else None, stats=srows,
                             rgb=rgb, **kw)
        if taped:
            rec["out"] = out
        if use_rgb:
            rgb_cur = rgb["out1"]
        cur = out
    rgb_cur = rgb_cur.reshape(B, 3, Hg, Wg)
    if taped:
        tape.rgb = rgb_cur
    return rgb_cur


def _taped_tables(P, srow, bn, s, fs, pixel, C, count):
    """Forward with a tape: the SPADE table of one half-block by `synthesis_train.spade_table` from the leaves
    sum(x), sum(x^2) [512] of its batch statistics (both halves), zero-padded to 512 channels; srow None (eval mode):
    by `spade_table_eval` from the running statistics, without leaves.
    -> (table [(B,)2,512] with history, its two detached halves, ssum, ssq)."""
    from .synthesis_train import const_gamma_beta, spade_table, spade_table_eval
    ssum = ssq = None
    if srow is not None:
        ssum = srow[:, :HALF].reshape(2 * HALF).clone().requires_grad_(True)
        ssq = srow[:, HALF:2 * HALF].reshape(2 * HALF).clone().requires_grad_(True)
    with torch.enable_grad():
        gb = None if pixel else const_gamma_beta(P, s, fs, C)
        mod = spade_table(P, bn, ssum[:C], ssq[:C], count, gb) if srow is not None else spade_table_eval(P, bn, gb)
        mod = F.pad(mod, (0, 2 * HALF - C))          # padded channels: g1 = g0 = 0
    return mod, [mod[..., :HALF].detach().contiguous(), mod[..., HALF:].detach().contiguous()], ssum, ssq


def _tables(P, srow, bn, s, fs, pixel, C, B, training, passes):
    """BatchNorm (+ per-sample SPADE vectors for const style) per half by hg_bn_finalize; padded channels get
    weight = bias = 0.  -> [table_lo, table_hi]: scsh [2,256] (pixel style) or [B,2,256]."""
    f32 = dict(dtype=torch.float32, device=fs.device)
    W2 = 2 * HALF
    bw, bbias = _pad1(P[bn + "weight"].float(), W2), _pad1(P[bn + "bias"].float(), W2)
    rm, rv = _pad1(P[bn + "running_mean"].float(), W2), _pad1(P[bn + "running_var"].float(), W2, fill=1.0)
    if not pixel:
        actv = torch.relu(_gemm_nt(fs, P[s + "mlp_shared.0.weight"].reshape(128, C).float(), passes=passes)
                          + P[s + "mlp_shared.0.bias"].float())
        G = 1.0 + _gemm_nt(actv, P[s + "mlp_gamma.weight"].reshape(C, 128).float(), passes=passes) + P[s + "mlp_gamma.bias"].float()
        Bt = _gemm_nt(actv, P[s + "mlp_beta.weight"].reshape(C, 128).float(), passes=passes) + P[s + "mlp_beta.bias"].float()
        GB = torch.zeros(B, 2, W2, **f32)
        GB[:, 0, :C] = G
        GB[:, 1, :C] = Bt
    tables = []
    for h in (0, 1):
        sl = slice(h * HALF, (h + 1) * HALF)
        rm_h, rv_h = rm[sl].contiguous(), rv[sl].contiguous()
        scsh = torch.empty(2, HALF, **f32) if pixel else None
        mod = None if pixel else torch.empty(B, 2, HALF, **f32)
        abi.bn_finalize(srow[h] if training else None, bw[sl].contiguous(), bbias[sl].contiguous(), rm_h, rv_h, training,
                        count_dev=srow[h, 512:513] if training else None, gb=None if pixel else GB[:, :, sl].contiguous(), B=B,
                        scsh=scsh, mod=mod)
        if training:
            rm[sl], rv[sl] = rm_h, rv_h
        tables.append(scsh if pixel else mod)
    if training:
        P[bn + "running_mean"].copy_(rm[:C])
        P[bn + "running_var"].copy_(rv[:C])
        if (bn + "num_batches_tracked") in P:
            P[bn + "num_batches_tracked"] += 1
    return tables
