"""Training-mode forward + backward of the FiLM-SIREN renderer (COORDCONCATSIREN.forward modulated.py:41-75 +
vr.ray_integration volume_rendering.py:12-56) on the sm_90a kernels.

The inference path is ONE fused kernel (csrc/render.cu) that keeps every activation on chip.  Training needs the
pre-activations back, so here the MLP runs layer by layer over tile-blocked points [B, T, 256, 128] (the layout of the
synthesis network; a "pixel" is a sample point p = ray*S + s) and keeps the 8 linear outputs:

    lin_a = Wc x + bc, lin_b = Wg g + bg                         hg_conv1x1_blocked        (K = 3 / 31, zero padded)
    out_0 = W0 [sin(30 lin_a); sin(30 lin_b)] + b0               hg_act_conv1x1_blocked    (sine operand, K = 512)
    out_i = W_i sin(f_{i-1} out_{i-1} + phi_{i-1}) + b_i         i = 1..3
    lin_c = Wcol[:,3:] sin(f_3 out_3 + phi_3) + (bcol + Wcol[:,:3] dir)
    feat  = Wf sin(f_3 lin_c + phi_3) + bf
    sigma, rgb_pre                                               hg_render_heads
    ray_out = composite(...)                                     hg_render_composite

Backward (`mlp_backward`, one for every width): the tape holds each activation as nh 256-channel halves -- nh = 1 here,
nh = 2 from the zero-padded forward of modules/wide_ops.py at hidden_dim 384 / 420.  Per feature half
hg_render_composite_bwd and hg_render_heads_bwd, then per layer and input half the blocked data-gradient kernel with
the cosine mask (K = nh*256 from the output-half gradients; the sigma / rgb heads enter as rank-1 / rank-3 terms of
its epilogue, the FiLM frequency of the consumer as a per-(sample, channel) scale of its operand) and per (output
half, input half) the blocked weight-gradient kernel with the sine operand.  d freq / d phase come from the per-(b,c)
sums S1 = sum dpre, S2 = sum dpre*x of the data-gradient kernels through torch autograd on the [B,256] tables.
Geometry features carry no gradient (wrapped in no_grad in the reference, map3d_generator.py:196-205).
"""
from __future__ import annotations

import torch

from .. import abi
from .wide_ops import _pad2

H = 256


def blocked_points(t, C):
    """[B,N,c] point-major -> tile-blocked [B,T,C,128] (channels zero padded to C)."""
    B, N, c = t.shape
    assert N % 128 == 0
    out = torch.zeros(B, N // 128, C, 128, dtype=torch.float32, device=t.device)
    out[:, :, :c] = t.reshape(B, N // 128, 128, c).permute(0, 1, 3, 2)
    return out


def mlp_forward_train(P, freq, phase, rec, z_vals, noise, cfg, *, geo_dim=31, locked_dir=(0.0, 0.0, -1.0), passes=3,
                      prefix="neural_field.", training=True):
    """rec [B,N,>=3+geo_dim] (scaled coordinates, geometry features), z_vals [B,N], noise [B,N] or None.
    Returns (ray_out [B,R,260] without autograd history, tape).  `last_back=True` is differentiated for an eval-mode
    module only (`training=False`): it is the sample app's compositing rule, no curriculum trains with it."""
    abi.require_device()
    g = lambda n: P[prefix + n]
    dev = rec.device
    B, N = rec.shape[0], rec.shape[1]
    S = cfg["num_steps"]
    R = N // S
    if training and cfg.get("last_back", False):
        raise RuntimeError("hg3d: last_back=True is an inference-only setting (eval_last_back); the training renderer does not build it")
    if g("network.0.layer.weight").shape[0] != H:
        raise RuntimeError("hg3d: the sm_90a render kernels are built for hidden_dim == 256")
    f32 = dict(dtype=torch.float32, device=dev)
    kw = dict(B=B, Hg=1, Wg=N, passes=passes)
    pack = lambda w: abi.pack_weight(w.detach().float().contiguous(), Nb=256)[0]

    # FiLM tables with autograd history: f = 15*freq + 30 (modulated.py:43); the colour layer re-uses the last slice
    fq = freq.detach().float().requires_grad_(True)
    ph = phase.detach().float().requires_grad_(True)
    f = fq * 15 + 30
    mods_h = [torch.stack([f[:, i * H:(i + 1) * H], ph[:, i * H:(i + 1) * H]], dim=1) for i in range(4)]    # [B,2,256] each
    mod30 = torch.stack([torch.full((B, H), 30.0, **f32), torch.zeros(B, H, **f32)], dim=1).contiguous()
    mods = [m.detach().contiguous() for m in mods_h]

    rec_b = blocked_points(rec[..., :3 + geo_dim], 128)
    Wa = torch.zeros(H, 128, **f32)
    Wb = torch.zeros(H, 128, **f32)
    Wa[:, :3] = g("first_layer_coord.layer.weight").detach()
    Wb[:, 3:3 + geo_dim] = g("first_layer_mod.layer.weight").detach()
    new = lambda: torch.empty(B, N // 128, H, 128, **f32)
    lin_a = abi.conv1x1_blocked(rec_b, 128, pack(Wa), g("first_layer_coord.layer.bias").detach(), new(), **kw)
    lin_b = abi.conv1x1_blocked(rec_b, 128, pack(Wb), g("first_layer_mod.layer.bias").detach(), new(), **kw)
    outs = [abi.act_conv1x1_blocked(lin_a, mod30, pack(g("network.0.layer.weight")), g("network.0.layer.bias").detach(), new(),
                                    x2=lin_b, **kw)]
    for i in range(1, 4):
        outs.append(abi.act_conv1x1_blocked(outs[-1], mods[i - 1], pack(g(f"network.{i}.layer.weight")),
                                            g(f"network.{i}.layer.bias").detach(), new(), **kw))
    wcol = g("color_layer_sine.layer.weight")
    dvec = torch.tensor(locked_dir, **f32)
    bcol = g("color_layer_sine.layer.bias") + wcol[:, :3] @ dvec            # autograd: bias and the direction columns
    lin_c = abi.act_conv1x1_blocked(outs[3], mods[3], pack(wcol[:, 3:]), bcol.detach().contiguous(), new(), **kw)
    feat = abi.act_conv1x1_blocked(lin_c, mods[3], pack(g("feature_layer_linear.weight")),
                                   g("feature_layer_linear.bias").detach(), new(), **kw)
    w_sigma = g("sigma_layer.weight").detach().reshape(-1).float().contiguous()
    w_rgb = g("color_layer_linear.weight").detach().float().contiguous()
    heads_b = torch.cat([g("sigma_layer.bias").detach().reshape(1), g("color_layer_linear.bias").detach().reshape(3)]).float().contiguous()
    sig, rgbp = abi.render_heads(outs[3], lin_c, mods[3], w_sigma, w_rgb, heads_b, B=B, N=N)
    noise = None if noise is None else noise.reshape(B, N).float().contiguous()
    comp = dict(B=B, R=R, S=S, noise_std=cfg["nerf_noise"], white_back=cfg.get("white_back", False),
                softplus=cfg["clamp_mode"] == "softplus", last_back=cfg.get("last_back", False))
    ray_out, _ = abi.render_composite(sig, z_vals, noise, rgbp, feat, **comp)
    tape = dict(P=P, prefix=prefix, C=H, Fd=H, geo_dim=geo_dim, fq=fq, ph=ph, mods=[(m,) for m in mods], mods_h=[(m,) for m in mods_h],
                m30=(mod30,), rec_b=rec_b, lin_a=(lin_a,), lin_b=(lin_b,), outs=[(o,) for o in outs], lin_c=(lin_c,), feat=(feat,),
                sig=sig, rgbp=rgbp, z=z_vals, noise=noise, comp=comp, kw=kw, bcol=bcol, w_sigma=w_sigma, w_rgb=w_rgb, B=B, N=N)
    return ray_out, tape


def mlp_backward(tape, dfeat, drgb, grads=None):
    """Backward of the training renderer at every width.  dfeat [B,R,Fd] and drgb [B,R,3] (either may be None) are the
    gradients w.r.t. the ray features and rgb.  Adds the gradients of the neural-field parameters to `grads` (name ->
    tensor; to `.grad` when grads is None) and returns (d freq, d phase) [B,4*C] each.

    The tape is the dict `mlp_forward_train` (hidden_dim 256) or `wide_ops.render_forward_wide(..., tape=tape)` (the
    zero-padded widths) fills.  Every point activation is a tuple of nh tile-blocked halves [B,T,256,128], nh = 1 at
    256 and 2 at the padded widths:
        lin_a, lin_b, outs[0..3], lin_c, feat   the linear outputs
        mods[0..3], m30     the detached FiLM tables (f, phi) [B,2,256] per half; m30 = (30, 0) of the first layers
        mods_h[0..3]        the same tables with autograd history from the leaves fq, ph
    and w_sigma [nh*256], w_rgb [3,nh*256] zero-padded, bcol (colour bias + direction columns) with history, the
    compositing inputs sig, rgbp, z, noise, comp, and rec_b, C, Fd, geo_dim, B, N, kw, P, prefix.  Padded channels
    carry zero weights and zero FiLM tables, so their gradients are zero up to the trimming to each parameter's shape."""
    from .synthesis_train import _packT, grad_accumulator
    P, prefix = tape["P"], tape["prefix"]
    g = lambda n: P[prefix + n]
    need = lambda *names: any(g(n).requires_grad for n in names)      # a weight-gradient kernel runs only for these
    acc_ = grad_accumulator(P, grads)
    acc = lambda n, gr: acc_(prefix + n, gr)
    B, N, C, Fd, kw = tape["B"], tape["N"], tape["C"], tape["Fd"], tape["kw"]
    mods, m30, outs, lin_c = tape["mods"], tape["m30"], tape["outs"], tape["lin_c"]
    nh = len(lin_c)
    halves = range(nh)
    W = nh * H
    sl = lambda h: slice(h * H, (h + 1) * H)
    dev = tape["sig"].device
    f32 = dict(dtype=torch.float32, device=dev)
    T = N // 128
    full = T * H * 128
    new = lambda: torch.empty(B, T, H, 128, **f32)
    scale = lambda m: torch.cat([t[:, 0] for t in m], -1).contiguous()        # FiLM frequency [B,nh*256] of a consumer
    pscale = lambda m: [t[:, 0].contiguous() for t in m]

    # ---- compositing per feature half: the rgb gradient enters once; dsig is linear in dray, so the halves' terms add
    dfh, drgbp, dsig = [], None, None
    for h in halves:
        dray = torch.zeros(B, tape["comp"]["R"], 260, **f32)
        if dfeat is not None:
            part = dfeat[..., sl(h)]
            dray[..., :part.shape[-1]] = part
        if h == 0 and drgb is not None:
            dray[..., 256:259] = drgb
        df, dp, ds = abi.render_composite_bwd(tape["sig"], tape["z"], tape["noise"], tape["rgbp"], tape["feat"][h], dray, **tape["comp"])
        dfh.append(df)
        drgbp = dp if h == 0 else drgbp
        dsig = ds if dsig is None else dsig + ds
        del dray
    # ---- heads (the biases once)
    if need("sigma_layer.weight", "color_layer_linear.weight", "sigma_layer.bias", "color_layer_linear.bias"):
        hb = [abi.render_heads_bwd(outs[3][h], lin_c[h], mods[3][h], dsig, drgbp, B=B, N=N) for h in halves]
        acc("sigma_layer.weight", torch.cat([t[:H] for t in hb])[:C].float())
        acc("color_layer_linear.weight", torch.cat([t[H:4 * H].reshape(3, H) for t in hb], -1)[:, :C].float())
        acc("sigma_layer.bias", hb[0][4 * H:4 * H + 1].float())
        acc("color_layer_linear.bias", hb[0][4 * H + 1:].float())

    dmods = [[torch.zeros(B, 2, H, **f32) for _ in halves] for _ in range(4)]

    def dgrad(gs, xs, Wp, mods_in, film=None, ascale=None, rk_w=None, rk_v=None):
        """Data gradient of one zero-padded layer per input half, K = nh*256 from the output halves' gradients gs; its
        S1 / S2 sums go to FiLM slice `film`."""
        res = []
        for ih in halves:
            s = torch.zeros(B, 2, H, dtype=torch.float64, device=dev)
            res.append(abi.conv1x1_blocked_bwd(gs[0], xs[ih], _packT(Wp, ih), new(), s, g2=gs[1] if nh == 2 else None, mod=mods_in[ih],
                                               act=1, ascale=ascale, rk_w=None if rk_w is None else rk_w[:, sl(ih)].contiguous(),
                                               rk_v=rk_v, **kw))
            if film is not None:        # d g1 = sum dpre*x, d g0 = sum dpre
                dmods[film][ih] += torch.stack([s[:, 1], s[:, 0]], dim=1).float()
        return tuple(res)

    def wgrad(gs, xs, mods_in, ps):
        """[nh*256, nh*256] weight gradient block by block, [nh*256] bias gradient."""
        dW = torch.empty(W, W, **f32)
        dbs = []
        for oh in halves:
            for ih in halves:
                dw, db = abi.act_wgrad_blocked(gs[oh], xs[ih], full, mods_in[ih], act=1, pscale=None if ps is None else ps[oh], **kw)
                dW[sl(oh), sl(ih)] = dw
                if ih == 0:
                    dbs.append(db)
        return dW, torch.cat(dbs)

    rk1 = torch.zeros(3, W, **f32)
    rk1[0] = tape["w_sigma"]
    # ---- feature layer: feat = Wf sin(f3 lin_c + phi3) + bf;  the rgb head feeds back through the same activation (rank 3)
    dpre_c = dgrad(dfh, lin_c, _pad2(g("feature_layer_linear.weight").detach().float(), W, W), mods[3], film=3,
                   rk_w=tape["w_rgb"], rk_v=drgbp)
    if need("feature_layer_linear.weight", "feature_layer_linear.bias"):
        dW, db = wgrad(dfh, lin_c, mods[3], None)
        acc("feature_layer_linear.weight", dW[:Fd, :C])
        acc("feature_layer_linear.bias", db[:Fd])
    del dfh
    # ---- colour layer: lin_c = Wcol' sin(f3 out3 + phi3) + bcol';  the sigma head feeds back through h4 (rank 1)
    wcol = g("color_layer_sine.layer.weight")
    dpre = dgrad(dpre_c, outs[3], _pad2(wcol[:, 3:].detach().float(), W, W), mods[3], film=3, ascale=scale(mods[3]),
                 rk_w=rk1, rk_v=dsig.reshape(B, 1, N))
    small = []
    if need("color_layer_sine.layer.weight", "color_layer_sine.layer.bias"):
        dW, db = wgrad(dpre_c, outs[3], mods[3], pscale(mods[3]))
        gw = torch.zeros_like(wcol)
        gw[:, 3:] = dW[:C, :C]
        acc("color_layer_sine.layer.weight", gw)
        small = [(tape["bcol"], db[:C])]                                      # bias + direction columns via autograd
    del dpre_c
    # ---- network.3 .. network.1: out_i = W_i sin(f_{i-1} out_{i-1} + phi_{i-1}) + b_i
    for i in (3, 2, 1):
        wi = _pad2(g(f"network.{i}.layer.weight").detach().float(), W, W)
        nxt = dgrad(dpre, outs[i - 1], wi, mods[i - 1], film=i - 1, ascale=scale(mods[i]))
        if need(f"network.{i}.layer.weight", f"network.{i}.layer.bias"):
            dW, db = wgrad(dpre, outs[i - 1], mods[i - 1], pscale(mods[i]))
            acc(f"network.{i}.layer.weight", dW[:C, :C])
            acc(f"network.{i}.layer.bias", db[:C])
        dpre = nxt
    # ---- network.0 (K = 2C: coordinate part, geometry part) and the two first layers
    w0 = g("network.0.layer.weight").detach().float()
    gw0 = torch.empty(C, 2 * C, **f32)
    need0 = need("network.0.layer.weight", "network.0.layer.bias")
    for part, lin, first, cols in ((0, tape["lin_a"], "first_layer_coord.layer.", slice(0, 3)),
                                   (1, tape["lin_b"], "first_layer_mod.layer.", slice(3, 3 + tape["geo_dim"]))):
        need_first = need(first + "weight", first + "bias")      # the coordinates and geometry features carry no gradient
        if need_first:
            dlin = dgrad(dpre, lin, _pad2(w0[:, part * C:(part + 1) * C], W, W), m30, ascale=scale(mods[0]))
        if need0:
            dW, db0 = wgrad(dpre, lin, m30, pscale(mods[0]))
            gw0[:, part * C:(part + 1) * C] = dW[:C, :C]
        if not need_first:
            continue
        # first layer: lin = W x + b with the sine's factor 30 folded into the incoming gradient
        dwf, dbf = zip(*[abi.act_wgrad_blocked(dlin[h], tape["rec_b"], T * 128 * 128, None, act=2, pscale=m30[h][:, 0].contiguous(),
                                               Cx=128, **kw) for h in halves])
        acc(first + "weight", torch.cat(dwf)[:C, cols])
        acc(first + "bias", torch.cat(dbf)[:C])
        del dlin
    if need0:
        acc("network.0.layer.weight", gw0)
        acc("network.0.layer.bias", db0[:C])
    # ---- FiLM tables, colour bias / direction columns: tiny autograd graphs
    outs_ = [t for m in tape["mods_h"] for t in m]
    grads_ = [t for m in dmods for t in m]
    for t, gr in small:
        if t.requires_grad:
            outs_.append(t)
            grads_.append(gr)
    leaves = [n for n in ("color_layer_sine.layer.bias", "color_layer_sine.layer.weight") if g(n).requires_grad]
    res = torch.autograd.grad(outs_, [tape["fq"], tape["ph"]] + [g(n) for n in leaves], grads_, allow_unused=True)
    for n, r in zip(leaves, res[2:]):
        if r is not None:
            acc(n, r)
    return res[0], res[1]


@torch.no_grad()
def geo_records(cond, cfg, u):
    """Ray sampling + jitter + camera transform + exact nearest vertex + 31-d features (no gradient, as in the
    reference: map3d_generator.py:196-205) -> (rec [B,N,36], z_vals [B,N]); same launches as render_ops.render_forward."""
    dev = cond["vertices"].device
    B = cond["vertices"].shape[0]
    Rw, Rh, S = cfg["render_width"], cfg["render_height"], cfg["num_steps"]
    f32 = dict(dtype=torch.float32, device=dev)
    xs = torch.linspace(-Rw / Rh, Rw / Rh, Rw, **f32)
    ys = torch.linspace(-1, 1, Rh, **f32)
    zs = torch.linspace(cfg["ray_start"], cfg["ray_end"], S, **f32)
    vik = abi.vertex_ik(cond["fk_matrices"], cond["lbs_weights"])
    geo = abi.geo_features(cond["vertices"], cond["tpose_vertices"], cond["skeletons_xyz"], vik,
                           input_scaler=2.0 / cfg["side_length"], legacy_mode=cfg.get("legacy_mode", False),
                           xs=xs, ys=ys, zs=zs, focals=cond["intrinsics"][:, 0, 0], scales=cond["scales"],
                           cam2world=cond["cam2world_matrices"], jitter=u.reshape(B, Rw * Rh * S) if u is not None else None)
    return geo["rec"], geo["z_vals"]


CORE_PREFIXES = ("neural_field.", "synthesis_network.", "synthesis_input.")


def core_parameters(module):
    """(names, tensors): the renderer / synthesis parameters that enter `GeneratorCore` as autograd inputs."""
    names, tensors = [], []
    for n, p in module.named_parameters():
        if n.startswith(CORE_PREFIXES):
            names.append(n)
            tensors.append(p)
    return names, tensors


class GeneratorCore(torch.autograd.Function):
    """(freq, phase, fixed style, *renderer and synthesis parameters) -> (rgbs, rgbs_render, depth, rec, z_vals) on the sm_90a
    kernels; rec / z_vals are the point records of the render (no gradient), which `cfg["hg_records"]` of a later call re-uses.

    EVERY parameter the kernels read is an input of this node and its gradient is RETURNED by `backward`, so the
    reference trainer's machinery sees them like any other autograd node's: `DistributedDataParallel` reducer hooks fire
    (base_trainer.py:102-104, find_unused_parameters=True walks the graph to them), `torch.autograd.grad(loss, params)`
    works, `GradScaler.unscale_` finds fp32 `.grad`s.  Under `torch.autocast` the inputs are taken as fp32 (the kernels
    compute in fp32 / bf16x3 whatever the ambient autocast dtype; phase_trainer.py:355,396,462 run the models under
    fp16 autocast).  First-order only: the reference never differentiates the generator twice (R1 acts on real images)."""

    @staticmethod
    @torch.amp.custom_fwd(device_type="cuda", cast_inputs=torch.float32)
    def forward(ctx, module, cond, cfg, u, noise, passes, names, freq, phase, styles, *tensors):
        from . import synthesis_train
        P = module._params()
        for n, t in zip(names, tensors):           # the tensors autograd tracks (identical objects unless a caller wraps them)
            P[n] = t
        B = freq.shape[0]
        Rh, Rw = cfg["render_height"], cfg["render_width"]
        if not cfg.get("lock_view_dependence", False):
            raise RuntimeError("hg3d: the training renderer is built for lock_view_dependence=True")
        if cfg.get("neural_field_blocks", 4) != 4:
            raise RuntimeError("hg3d: the training renderer is built for neural_field_blocks == 4 (all shipped curricula)")
        training = module.training      # eval: running statistics, stored u / v, last_back allowed, no buffer written
        # the point records: the 2S merged samples of hierarchical_sample, the ray stage's, or a previous render's
        if cfg.get("hierarchical_sample", False):
            if cfg.get("hg_records") is not None:
                raise RuntimeError("hg3d: hg_records cannot be re-used with hierarchical_sample=True (the fine samples "
                                   "follow the density, which moves with freq / phase)")
            from . import hierarchical
            h = hierarchical.merged_records(P, freq, phase, cond, cfg, u, noise, passes=passes)
            rec, z_vals, rcfg, rnoise = h["rec"], h["z_vals"], h["cfg"], h["noise"]
        else:
            rec, z_vals = cfg["hg_records"] if cfg.get("hg_records") is not None else geo_records(cond, cfg, u)
            rcfg, rnoise = cfg, noise
        if rec.shape[:2] != (B, Rh * Rw * rcfg["num_steps"]) or z_vals.shape != rec.shape[:2]:
            raise RuntimeError("hg3d: hg_records do not belong to this batch / render size / num_steps")
        if cfg["hidden_dim"] != H:      # 384 / 420: the zero-padded forward of wide_ops, with tapes
            from . import wide_ops
            rtape, stape = {}, synthesis_train.SynthesisTape()
            feats, rgb01, depth = wide_ops.render_forward_wide(P, freq, phase, cond, rcfg, u, rnoise, passes=passes, tape=rtape,
                                                               records=(rec, z_vals), training=training)
            rgb = wide_ops.synthesis_forward_wide(P, feats, styles.reshape(B, -1), cfg, training=training, passes=passes, tape=stape)
            rgb_render = (rgb01 * 2 - 1).reshape(B, Rh, Rw, 3).permute(0, 3, 1, 2).contiguous()
        else:
            with torch.enable_grad():
                ray, rtape = mlp_forward_train(P, freq, phase, rec, z_vals, rnoise, rcfg, geo_dim=cfg["geo_feature_dim"],
                                               passes=passes, training=training)
                rgb, stape = synthesis_train.synthesis_forward_train(P, ray, styles.reshape(B, -1), cfg, passes=passes,
                                                                     training=training)
            rgb_render = (ray[..., 256:259] * 2 - 1).reshape(B, Rh, Rw, 3).permute(0, 3, 1, 2).contiguous()
            depth = ray[..., 259:260].contiguous()
        ctx.tapes = (P, rtape, stape, cfg, passes, names)
        ctx.mark_non_differentiable(depth, rec, z_vals)
        return rgb, rgb_render, depth, rec, z_vals

    @staticmethod
    @torch.amp.custom_bwd(device_type="cuda")
    @torch.autograd.function.once_differentiable
    def backward(ctx, d_rgb, d_rgb_render, d_depth, d_rec, d_z_vals):
        from . import synthesis_train
        if ctx.tapes is None:
            raise RuntimeError("hg3d: the generator's activation tape was released by a previous backward pass "
                               "(one backward per forward; retain_graph=True keeps the graph, not the tape)")
        P, rtape, stape, cfg, passes, names = ctx.tapes
        B = stape.B
        Rh, Rw = cfg["render_height"], cfg["render_width"]
        grads = {}
        with torch.enable_grad():
            dfs, dfeat = synthesis_train.synthesis_backward(P, stape, d_rgb, passes=passes, grads=grads)
            drgb = None if d_rgb_render is None else 2.0 * d_rgb_render.permute(0, 2, 3, 1).reshape(B, Rh * Rw, 3)
            dfreq, dphase = mlp_backward(rtape, dfeat, drgb, grads=grads)
        ctx.tapes = None
        # Every returned gradient must own its storage: autograd's AccumulateGrad steals a returned tensor as `.grad` when
        # nobody else holds the TensorImpl, so two parameters whose gradients are views of one buffer (the nine ToRGB biases
        # all receive sum(d_rgb)) would end up with ALIASED `.grad`s -- and every in-place pass over the gradients
        # (GradScaler.unscale_, clip_grad_norm_) would then hit that buffer once per alias, concurrently in the foreach kernels.
        out, seen = [], set()
        for n in names:
            g = grads.get(n)
            if g is not None:
                g = g.detach()
                key = g.untyped_storage().data_ptr()
                if key in seen or g.untyped_storage().nbytes() != g.numel() * g.element_size():
                    g = g.clone()
                seen.add(g.untyped_storage().data_ptr())
            out.append(g)
        return (None, None, None, None, None, None, None, dfreq.detach(), dphase.detach(), dfs.detach().reshape(B, -1), *out)
