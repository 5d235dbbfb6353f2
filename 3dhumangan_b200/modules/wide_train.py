"""Backward of the zero-padded generator (hidden_dim <= 512 other than 256: MAP3DBN's 384, MAP3DBN512L's 420).

The training forward is the inference schedule of modules/wide_ops.py with a tape.  Every channel dimension is padded to
512 = two tile-blocked halves [B,T,256,128], so the backward of a 512 -> 512 layer is a composition of the blocked
kernels the 256-channel backward uses (render_train.mlp_backward, synthesis_train.synthesis_backward), over halves:

  data gradient     one hg_conv1x1_blocked_bwd per INPUT half, K = 512 from the two output-half gradients (g, g2); the
                    consumer's FiLM frequency is the [B,512] operand scale (columns 0..255 scale g, 256..511 g2)
  weight gradient   one hg_act_wgrad_blocked / hg_wgrad_blocked per (output half, input half) block
  per-half kernels  hg_render_composite_bwd, hg_render_heads_bwd, hg_spade_bwd_combine, hg_spade_pixel_mod_bwd,
                    hg_synth_input_bwd: once per half

Padded channels carry zero weights and zero tables, so their gradients are zero up to the trimming to each parameter's
true shape.  The [C]- and [B,C]-sized chains (FiLM tables, SPADE / BatchNorm tables, W / sigma, colour bias and view
direction) go through the same small autograd graphs as at 256.
"""
from __future__ import annotations

import torch
import torch.distributed as dist

from .. import abi
from ..ops.dense import _gemm_nt
from .synthesis_ops import _PtrView
from .synthesis_train import grad_accumulator
from .wide_ops import HALF, _pad2

W2 = 2 * HALF


def _sl(h):
    return slice(h * HALF, (h + 1) * HALF)


def _packT(W512, ih):
    """Operand image of the transposed input-half `ih` columns of a padded [512,512] weight: [256 x K = 512]."""
    return abi.pack_weight(W512[:, _sl(ih)].t().contiguous(), Nb=256)[0]


def _cat2(a, b):
    """[..., 256] halves -> [..., 512] (f32)."""
    return torch.cat([a, b], -1).float()


# ----------------------------------------------------------------------------------------------------------------------
# renderer
# ----------------------------------------------------------------------------------------------------------------------
def render_backward_wide(tape, dfeat, drgb, grads=None):
    """dfeat [B,R,Fd] (or None), drgb [B,R,3] (or None): gradients w.r.t. the ray features and rgb of
    `wide_ops.render_forward_wide(..., tape=tape)`.  Adds the neural-field parameter gradients to `grads` (`.grad` when
    None) and returns (d freq, d phase) [B, 4*C]."""
    P, prefix = tape["P"], tape["prefix"]
    g = lambda n: P[prefix + n]
    acc_ = grad_accumulator(P, grads)
    acc = lambda n, gr: acc_(prefix + n, gr)
    B, N, R, C, Fd, kw = tape["B"], tape["N"], tape["R"], tape["C"], tape["Fd"], tape["kw"]
    dev = tape["sig"].device
    f32 = dict(dtype=torch.float32, device=dev)
    T = N // 128
    full = T * HALF * 128
    new = lambda: torch.empty(B, T, HALF, 128, **f32)
    mods, m30, outs, lin_c = tape["mods"], tape["m30"], tape["outs"], tape["lin_c"]
    scale = lambda m: _cat2(m[0][:, 0], m[1][:, 0]).contiguous()               # FiLM frequency [B,512] of a table pair
    pscale = lambda m: (m[0][:, 0].contiguous(), m[1][:, 0].contiguous())

    # ---- compositing per feature half: the rgb gradient enters once; dsig is linear in dray, so the two calls add
    dfp = torch.zeros(B, R, W2, **f32)
    if dfeat is not None:
        dfp[..., :Fd] = dfeat
    dfh, drgbp, dsig = [], None, None
    for h in (0, 1):
        dray = torch.zeros(B, R, 260, **f32)
        dray[..., :HALF] = dfp[..., _sl(h)]
        if h == 0 and drgb is not None:
            dray[..., 256:259] = drgb
        df, dp, ds = abi.render_composite_bwd(tape["sig"], tape["z"], tape["noise"], tape["rgbp"], tape["feat"][h], dray, **tape["comp"])
        dfh.append(df)
        drgbp = dp if h == 0 else drgbp
        dsig = ds if dsig is None else dsig + ds
    del dfp
    # ---- heads (the biases once)
    hb = [abi.render_heads_bwd(outs[3][h], lin_c[h], mods[3][h], dsig, drgbp, B=B, N=N) for h in (0, 1)]
    acc("sigma_layer.weight", torch.cat([hb[0][:HALF], hb[1][:HALF]])[:C].float())
    acc("color_layer_linear.weight", _cat2(hb[0][HALF:4 * HALF].reshape(3, HALF), hb[1][HALF:4 * HALF].reshape(3, HALF))[:, :C])
    acc("sigma_layer.bias", hb[0][4 * HALF:4 * HALF + 1].float())
    acc("color_layer_linear.bias", hb[0][4 * HALF + 1:].float())

    dmods = [[torch.zeros(B, 2, HALF, **f32) for _ in (0, 1)] for _ in range(4)]

    def dgrad(gs, xs, W512, mods_in, film=None, ascale=None, rk_w=None, rk_v=None):
        """Data gradient of one padded layer per input half; its S1 / S2 sums go to FiLM slice `film`."""
        res = []
        for ih in (0, 1):
            s = torch.zeros(B, 2, HALF, dtype=torch.float64, device=dev)
            res.append(abi.conv1x1_blocked_bwd(gs[0], xs[ih], _packT(W512, ih), new(), s, g2=gs[1], mod=mods_in[ih], act=1,
                                               ascale=ascale, rk_w=None if rk_w is None else rk_w[:, _sl(ih)].contiguous(),
                                               rk_v=rk_v, **kw))
            if film is not None:        # d g1 = sum dpre*x, d g0 = sum dpre
                dmods[film][ih] += torch.stack([s[:, 1], s[:, 0]], dim=1).float()
        return tuple(res)

    def wgrad(gs, xs, mods_in, ps):
        """[512,512] weight gradient block by block, [512] bias gradient."""
        dW = torch.empty(W2, W2, **f32)
        dbs = []
        for oh in (0, 1):
            for ih in (0, 1):
                dw, db = abi.act_wgrad_blocked(gs[oh], xs[ih], full, mods_in[ih], act=1, pscale=None if ps is None else ps[oh], **kw)
                dW[_sl(oh), _sl(ih)] = dw
                if ih == 0:
                    dbs.append(db)
        return dW, torch.cat(dbs)

    w_rgb = tape["w_rgb"]                                                      # [3,512]
    rk1 = torch.zeros(3, W2, **f32)
    rk1[0] = tape["w_sigma"]
    # ---- feature layer; the rgb head feeds back through the same activation (rank 3)
    dfh = tuple(dfh)
    dpre_c = dgrad(dfh, lin_c, _pad2(g("feature_layer_linear.weight").detach().float(), W2, W2), mods[3], film=3,
                   rk_w=w_rgb, rk_v=drgbp)
    dW, db = wgrad(dfh, lin_c, mods[3], None)
    acc("feature_layer_linear.weight", dW[:Fd, :C])
    acc("feature_layer_linear.bias", db[:Fd])
    del dfh
    # ---- colour layer; the sigma head feeds back through the same activation (rank 1)
    wcol = g("color_layer_sine.layer.weight")
    dpre = dgrad(dpre_c, outs[3], _pad2(wcol[:, 3:].detach().float(), W2, W2), mods[3], film=3, ascale=scale(mods[3]),
                 rk_w=rk1, rk_v=dsig.reshape(B, 1, N))
    dW, db = wgrad(dpre_c, outs[3], mods[3], pscale(mods[3]))
    gw = torch.zeros_like(wcol)
    gw[:, 3:] = dW[:C, :C]
    acc("color_layer_sine.layer.weight", gw)
    small = [(tape["bcol"], db[:C])]
    del dpre_c
    # ---- network.3 .. network.1
    for i in (3, 2, 1):
        wi = _pad2(g(f"network.{i}.layer.weight").detach().float(), W2, W2)
        nxt = dgrad(dpre, outs[i - 1], wi, mods[i - 1], film=i - 1, ascale=scale(mods[i]))
        dW, db = wgrad(dpre, outs[i - 1], mods[i - 1], pscale(mods[i]))
        acc(f"network.{i}.layer.weight", dW[:C, :C])
        acc(f"network.{i}.layer.bias", db[:C])
        dpre = nxt
    # ---- network.0 (K = 2C: coordinate part, geometry part) and the two first layers (sine factor 30 folded in)
    w0 = g("network.0.layer.weight").detach().float()
    gw0 = torch.empty(C, 2 * C, **f32)
    for part, lin, first, cols in ((0, tape["lin_a"], "first_layer_coord.layer.", slice(0, 3)),
                                   (1, tape["lin_b"], "first_layer_mod.layer.", slice(3, 3 + tape["geo_dim"]))):
        dlin = dgrad(dpre, lin, _pad2(w0[:, part * C:(part + 1) * C], W2, W2), m30, ascale=scale(mods[0]))
        dW, db0 = wgrad(dpre, lin, m30, pscale(mods[0]))
        gw0[:, part * C:(part + 1) * C] = dW[:C, :C]
        dwf, dbf = zip(*[abi.act_wgrad_blocked(dlin[h], tape["rec_b"], T * 128 * 128, None, act=2, pscale=m30[h][:, 0].contiguous(),
                                               Cx=128, **kw) for h in (0, 1)])
        acc(first + "weight", torch.cat(dwf)[:C, cols])
        acc(first + "bias", torch.cat(dbf)[:C])
        del dlin
    acc("network.0.layer.weight", gw0)
    acc("network.0.layer.bias", db0[:C])
    # ---- FiLM tables, colour bias / direction columns: tiny autograd graphs
    outs_ = [t for pair in tape["mods_h"] for t in pair]
    grads_ = [t for pair in dmods for t in pair]
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


# ----------------------------------------------------------------------------------------------------------------------
# synthesis network
# ----------------------------------------------------------------------------------------------------------------------
def synthesis_backward_wide(params, tape, drgb, *, passes=3, grads=None):
    """Backward of `wide_ops.synthesis_forward_wide(..., tape=tape)`: gradients of every synthesis parameter into `grads`
    (`.grad` when None); returns (d fixed_style [B,C], d feats [B,Rh*Rw,C] or None without pixel-style half-blocks)."""
    P = params
    cfg, B = tape.cfg, tape.B
    C = cfg["hidden_dim"]
    Hg, Wg = cfg["gen_height"], cfg["gen_width"]
    HW = Hg * Wg
    T = (HW + 127) // 128
    dev = drgb.device
    f32 = dict(dtype=torch.float32, device=dev)
    kw = dict(B=B, Hg=Hg, Wg=Wg, passes=passes)
    drgb = drgb.reshape(B, 3, HW).float().contiguous()
    H = tape.halves
    n = len(H)
    full = T * HALF * 128
    new = lambda: torch.empty(B, T, HALF, 128, **f32)
    acc = grad_accumulator(P, grads)

    drgb_sum = drgb.sum((0, 2))
    small_out, small_grad = [], []
    dout = {}
    nxt = None                  # (dpre halves, g1 table halves, ak halves) of half-block h+1
    for h in range(n - 1, -1, -1):
        rec = H[h]
        # ---- dL/d(out_h) per half: next half-block, residual skip, ToRGB
        dskip = dout[h + 2] if (h + 2 < n and H[h + 2]["skip_from"] == h + 1) else (None, None)
        d, dwrgb = [], []
        for c in (0, 1):
            dc = new()
            ckw = {}
            if rec["rgb"] is not None:
                dwrgb.append(torch.zeros(3, HALF, dtype=torch.float64, device=dev))
                ckw = dict(drgb=drgb, rgb_w=rec["rgb_w"][:, _sl(c)].contiguous(), dwrgb=dwrgb[c])
            if nxt is not None:
                ckw.update(dpre=nxt[0][c], g1=nxt[1][c], ak=nxt[2][c])
            abi.spade_bwd_combine(dc, B=B, Hg=Hg, Wg=Wg, x=rec["out"][c], x_bstride=full, dskip=dskip[c], **ckw)
            d.append(dc)
        d = tuple(d)
        if rec["rgb"] is not None:
            acc(rec["rgb"] + "weight", _cat2(dwrgb[0], dwrgb[1])[:, :C])
            acc(rec["rgb"] + "bias", drgb_sum)
        dout[h] = d
        dout.pop(h + 3, None)
        # ---- this half-block: const style acts on x through its table, pixel style on the rebuilt `pre`
        Wsn = _pad2(rec["w_sn"].detach().reshape(C, C), W2, W2)
        sums = [torch.zeros(B, 2, HALF, dtype=torch.float64, device=dev) for _ in (0, 1)]
        dW = torch.empty(W2, W2, **f32)
        if rec["pixel"]:
            Rh, Rw = cfg["render_height"], cfg["render_width"]
            i = rec["i"]
            p_lr = tape.p["p_lr"]
            a1 = torch.empty(B, T, 128, 128, **f32)
            abi.spade_a1(_PtrView(p_lr[:, i * 128:]), p_lr.shape[1], rec["p_bias_d"], a1, B=B, Hg=Hg, Wg=Wg, Rh=Rh, Rw=Rw)
            gam, pre = [], []
            for c in (0, 1):
                gam.append(abi.conv1x1_blocked(a1, 128, abi.pack_weight(rec["wg"][_sl(c)].contiguous(), Nb=256)[0],
                                               rec["bg1"][_sl(c)].contiguous(), new(), **kw))
                pre.append(abi.conv1x1_blocked(a1, 128, abi.pack_weight(rec["wb"][_sl(c)].contiguous(), Nb=256)[0],
                                               rec["bb"][_sl(c)].contiguous(), new(), **kw))
                abi.spade_pixel_pre(rec["x"][c], full, rec["mod_d"][c], gam[c], pre[c], B=B, Hg=Hg, Wg=Wg)
            if getattr(tape, "keep_masks", False):      # tests: the masks this backward differentiates through
                rec["mask"] = [p > 0 for p in pre]
                rec["mask_a1"] = a1 > 0
            dpre = tuple(abi.conv1x1_blocked_bwd(d[0], pre[c], _packT(Wsn, c), new(), sums[c], g2=d[1], **kw) for c in (0, 1))
            for oh in (0, 1):
                for ih in (0, 1):
                    dw, db = abi.spade_bwd_wgrad(d[oh], pre[ih], full, None, want_bias=ih == 0, **kw)
                    dW[_sl(oh), _sl(ih)] = dw
                    if ih == 0:
                        acc_db = db if oh == 0 else torch.cat([acc_db, db])
            # modulation: dxn (over pre), dgam (over gam), BatchNorm scale / shift sums
            s3 = [torch.zeros(3, HALF, dtype=torch.float64, device=dev) for _ in (0, 1)]
            for c in (0, 1):
                abi.spade_pixel_mod_bwd(dpre[c], rec["x"][c], full, rec["mod_d"][c], gam[c], pre[c], s3[c], B=B, Hg=Hg, Wg=Wg)
            dxn, dgam = tuple(pre), tuple(gam)
            # gamma/beta MLP: dA1 = K 1024 over [dgam | dpre] as two K = 512 launches (the ReLU mask comes from A1)
            s7 = torch.zeros(B, 2, 128, dtype=torch.float64, device=dev)
            da1 = None
            for gs, wmat in ((dgam, rec["wg"]), (dpre, rec["wb"])):
                w7 = torch.zeros(256, W2, **f32)
                w7[:128] = wmat.t()
                part = abi.conv1x1_blocked_bwd(gs[0], a1, abi.pack_weight(w7, Nb=256)[0], torch.empty(B, HW, 128, **f32), s7, g2=gs[1],
                                               Cout=128, slope=0.0, pixel_major=True, **kw)
                da1 = part if da1 is None else da1.add_(part)
            sp_ = rec["spade"]
            for gs, nm in ((dgam, "mlp_gamma."), (dpre, "mlp_beta.")):
                dws, dbs = zip(*[abi.spade_bwd_wgrad(gs[c], a1, T * 128 * 128, None, Cx=128, **kw) for c in (0, 1)])
                acc(sp_ + nm + "weight", torch.cat(dws)[:C])
                acc(sp_ + nm + "bias", torch.cat(dbs)[:C])
            if "dp" not in tape.p:
                tape.p["dp"] = torch.zeros_like(p_lr)
            dp = tape.p["dp"]
            abi.bilinear_adjoint(da1, _PtrView(dp[:, i * 128:]), dp.shape[1], B=B, Hg=Hg, Wg=Wg, Rh=Rh, Rw=Rw)
            if rec["p_bias"].requires_grad:
                small_out.append(rec["p_bias"])
                small_grad.append(s7[:, 0].float())
            dmod = torch.stack([_cat2(s3[0][0], s3[1][0]), _cat2(s3[0][1], s3[1][1])])     # d sc = sum dxn*x, d sh = sum dxn
            dpre = dxn
            g1_tab = [m[0][None, None, :].expand(B, 2, HALF).contiguous() for m in rec["mod_d"]]
            del a1, da1, gam
        else:
            dpre = tuple(abi.conv1x1_blocked_bwd(d[0], rec["x"][c], _packT(Wsn, c), new(), sums[c], g2=d[1], mod=rec["mod_d"][c],
                                                 slope=0.2, **kw) for c in (0, 1))
            for oh in (0, 1):
                for ih in (0, 1):
                    dw, db = abi.spade_bwd_wgrad(d[oh], rec["x"][ih], full, rec["mod_d"][ih], want_bias=ih == 0, **kw)
                    dW[_sl(oh), _sl(ih)] = dw
                    if ih == 0:
                        acc_db = db if oh == 0 else torch.cat([acc_db, db])
            dmod = torch.stack([_cat2(sums[0][:, 1], sums[1][:, 1]), _cat2(sums[0][:, 0], sums[1][:, 0])], dim=1)   # d g1, d g0
            g1_tab = rec["mod_d"]
        acc(rec["conv"] + "bias", acc_db[:C])
        small_out.append(rec["w_sn"])
        small_grad.append(dW[:C, :C].reshape(rec["w_sn"].shape))
        ga, gk = torch.autograd.grad(rec["mod"], [rec["ssum"], rec["ssq"]], grad_outputs=dmod, retain_graph=True)
        ak = torch.stack([ga, gk])
        if tape.world > 1:          # SyncBatchNorm: every rank's loss depends on the global statistics
            dist.all_reduce(ak, group=tape.process_group)
        ak = torch.stack([ak[0], 2.0 * ak[1]]).float()                     # d(sum x)/dx = 1, d(sum x^2)/dx = 2x
        small_out.append(rec["mod"])
        small_grad.append(dmod)
        nxt = (dpre, g1_tab, [ak[:, _sl(c)].contiguous() for c in (0, 1)])
    # ---- synthesis input (materialised per sample), per half
    ip = tape.input["prefix"]
    dw_in, db_in = [], []
    for c in (0, 1):
        dx0 = new()
        abi.spade_bwd_combine(dx0, B=B, Hg=Hg, Wg=Wg, x=H[0]["x"][c], x_bstride=full, dpre=nxt[0][c], g1=nxt[1][c], ak=nxt[2][c])
        dw, db = abi.synth_input_bwd(dx0, tape.input["w"][_sl(c)].contiguous(), tape.input["b"][_sl(c)].contiguous(),
                                     tape.input["ic"], tape.input["jc"], B)
        dw_in.append(dw)
        db_in.append(db)
    acc(ip + "network.0.weight", torch.cat(dw_in)[:C])
    acc(ip + "network.0.bias", torch.cat(db_in)[:C])
    # ---- all [C]- and [B,C]-sized chains in one autograd pass
    fs = tape.fixed_style
    leaves = [t for t in small_out if t.requires_grad]
    small = [g for t, g in zip(small_out, small_grad) if t.requires_grad]
    names = [k for k, p in P.items() if isinstance(p, torch.Tensor) and p.requires_grad and p.is_leaf]
    res = torch.autograd.grad(leaves, [P[k] for k in names] + [fs], small, allow_unused=True)
    for k, r in zip(names, res[:-1]):
        if r is not None:
            acc(k, r)
    dfs = res[-1] if res[-1] is not None else torch.zeros_like(fs)
    # ---- render-resolution projection P_lr = X . W_shared^T: feature-map and weight gradients
    dfeat = None
    if tape.px and "dp" in tape.p:
        dp, Ws, X = tape.p["dp"], tape.p["Ws"], tape.p["X"]
        dfeat = _gemm_nt(dp, Ws.t().contiguous(), passes=passes).reshape(B, -1, C)
        prev = torch.backends.cuda.matmul.allow_tf32
        torch.backends.cuda.matmul.allow_tf32 = False
        dWs = dp.t() @ X                                                             # [n*128, C]  (plain library GEMM, as at 256)
        torch.backends.cuda.matmul.allow_tf32 = prev
        for rec in H:
            if rec["pixel"]:
                acc(rec["spade"] + "mlp_shared.0.weight", dWs[rec["i"] * 128:(rec["i"] + 1) * 128])
    return dfs, dfeat
