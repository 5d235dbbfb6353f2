"""Training-mode forward + backward of the SPADE synthesis network on the sm_90a kernels.

Forward: the same 18 fused half-block launches as `synthesis_ops.synthesis_forward`, but every half-block
input is kept (18 activations of B*HW*256 fp32 -- 2.1 GB each at the C2 workload; sized for 180 GB of HBM)
and every [B,C]- / [C]-sized quantity the kernels consume (folded BatchNorm+SPADE tables, spectrally
normalised weights) is built with torch autograd from its leaves.

Backward (autograd through SynthesisNetwork.forward map3d_generator.py:58-97, SPADEBlock.forward
map3d_layers.py:218-238, SPADE2d.forward :176-190, ToRGB :346-352, SynthesisInput :260-275), walking the
half-blocks in reverse; per half-block
    hg_spade_bwd_combine  dL/dout   from the next half-block's dpre (+ skip gradient, + ToRGB^T drgb)
    hg_spade_bwd_dgrad    dpre = (W^T dL/dout) * lrelu'(pre), S1 = sum dpre, S2 = sum dpre*x     (wgmma)
    hg_spade_bwd_wgrad    dW = dL/dout . y^T, dbias                                              (wgmma)
and the small chains on the host side: d(g1,g0) = (S2,S1) -> BatchNorm weight/bias, gamma/beta MLP, fixed style,
and -- through the leaves sum(x), sum(x^2) of the batch statistics -- the a[c] + k[c]*x term of dL/dx
(SyncBatchNorm: those two leaf gradients are SUM-all-reduced, like the statistics themselves).

Pixel-style half-blocks (per-pixel gamma/beta from the up-sampled render features; blocks in `mod_blocks`)
keep the fused forward kernel and, in backward, REBUILD their per-pixel quantities instead of storing them:
    hg_spade_a1            A1 = relu(bilinear_up(P_lr) + c)                      [B,T,128,128]
    hg_conv1x1_blocked x2  gam = Wg A1 + bg + 1,  bet = Wb A1 + bb               (wgmma)
    hg_spade_pixel_pre     pre = (x*sc + sh)*gam + bet
then the same dgrad / wgrad kernels run on `pre`, followed by
    hg_spade_pixel_mod_bwd dxn = dpre*gam, dgam = dpre*xn (+ the BatchNorm / bias sums)
    hg_conv1x1_blocked_bwd dA1 = ([dgam | dpre] . [Wg | Wb]) * relu'(A1)        (wgmma, K = 512, pixel-major out)
    hg_wgrad_blocked   x2  dWg = dgam . A1^T,  dWb = dpre . A1^T                 (wgmma)
    hg_bilinear_adjoint    dP_lr (render resolution)
and once, at the end, d(feature maps) = dP_lr . W_shared (wgmma `hg_linear`) and dW_shared = dP_lr^T . features
(a plain library GEMM through torch.matmul).
"""
from __future__ import annotations

import torch
import torch.distributed as dist
import torch.nn.functional as F

from .. import abi
from .synthesis_ops import STAT_STRIDE, _PtrView, _gamma_beta_interleaved, _spade, all_reduce_stats, is_pixel_style, sn_weights

C = 256


class SynthesisTape:
    """Everything `synthesis_backward` needs from one training forward."""

    def __init__(self):
        self.halves = []      # per half-block: dict(x, x_bstride, mod, w_sn, ssum, ssq, conv, skip_from, rgb_w ...)
        self.cfg = None
        self.B = 0
        self.rgb = None


def synthesis_forward_train(params, feat_lr, fixed_style, cfg, *, passes=3, prefix="synthesis_network.",
                            input_prefix="synthesis_input.", process_group=None):
    """-> (rgb [B,3,Hg,Wg] (no autograd history), tape).  `params`: name -> tensor (Parameters keep their .grad)."""
    abi.require_device()
    P = params
    dev = fixed_style.device
    B = fixed_style.shape[0]
    Hg, Wg = cfg["gen_height"], cfg["gen_width"]
    if cfg["hidden_dim"] != C or cfg["feature_dim"] != C:
        raise RuntimeError("hg3d: the sm_90a synthesis kernels are built for hidden_dim == feature_dim == 256")
    HW = Hg * Wg
    T = (HW + 127) // 128
    nb = cfg["synthesis_blocks"]
    halves = [(k, j) for k in range(nb) for j in range(2)]
    world = dist.get_world_size(process_group) if (dist.is_available() and dist.is_initialized()) else 1
    f32 = dict(dtype=torch.float32, device=dev)
    blk = lambda k: f"{prefix}network.m3d_{k}."
    sp = lambda k, j: blk(k) + f"spade_{j}."
    fs = fixed_style.detach().reshape(B, C).float().requires_grad_(True)     # leaf: its .grad is returned by backward

    tape = SynthesisTape()
    tape.cfg, tape.B, tape.fixed_style = cfg, B, fs
    tape.process_group, tape.world = process_group, world

    mode = cfg.get("map3d_mode", "isolated")
    Rh, Rw = cfg["render_height"], cfg["render_width"]
    px = [(k, j) for k, j in halves if is_pixel_style(cfg, k)]
    pxi = {key: i for i, key in enumerate(px)}
    tape.px = px
    p_lr = None
    PB = {}
    if px:
        # P_lr = W_shared . features at render resolution for all pixel-style half-blocks at once (no autograd: its
        # gradient comes back explicitly through the bilinear adjoint), and the per-sample constant added after the
        # up-sample: 'mixed'/'all' style = up(f) + fixed_style  =>  c = W_s fs + b_s;  'isolated': c = b_s
        Ws = torch.cat([P[sp(k, j) + "mlp_shared.0.weight"].detach().reshape(128, C) for k, j in px]).contiguous()   # [n*128,256]
        img, Nb = abi.pack_weight(Ws, Nb=256)
        X = feat_lr.detach().reshape(B * Rh * Rw, feat_lr.shape[-1])[:, :C]
        p_lr = abi.linear(X, img, Nb, Ws.shape[0], passes=passes)                                    # [B*Rhw, n*128]
        tape.p = dict(Ws=Ws, X=X, p_lr=p_lr, ld=feat_lr.shape[-1])
        for k, j in px:
            s = sp(k, j)
            w_s, b_s = P[s + "mlp_shared.0.weight"].reshape(128, C), P[s + "mlp_shared.0.bias"]
            PB[(k, j)] = (F.linear(fs, w_s, b_s) if mode in ("mixed", "all") else b_s[None, :].expand(B, 128))

    # ---- per-sample (1+gamma, beta) of every const-style half-block, with autograd history (tiny)
    GB = {}
    for k, j in halves:
        if (k, j) in pxi:
            continue
        GB[(k, j)] = const_gamma_beta(P, sp(k, j), fs, C)

    # ---- synthesis input (shared by the batch) + its statistics
    stats = torch.zeros(len(halves) + 1, STAT_STRIDE, dtype=torch.float64, device=dev)
    stats[:, 512] = float(B * HW)
    ic = torch.linspace(-1, 1, Hg, **f32)
    jc = torch.linspace(-1, 1, Wg, **f32)
    x0 = torch.empty(T, C, 128, **f32)
    w_in = P[input_prefix + "network.0.weight"].detach().reshape(C, 2).contiguous()
    abi.synth_input(w_in, P[input_prefix + "network.0.bias"].detach(), ic, jc, x0, stats[0], B)
    tape.input = dict(w=w_in, ic=ic, jc=jc, prefix=input_prefix)

    # spectral normalisation of the 18 convolutions: one launch (power iteration, buffers in place), W / sigma with history
    w_sns = sn_weights(P, [blk(k) + f"conv_{j}." for k, j in halves], True)

    rgb_cur = None
    cur, cur_bstride = x0, 0
    block_in = None
    for idx, (k, j) in enumerate(halves):
        bn = sp(k, j) + "first_norm."
        srow = stats[idx]
        if world > 1:
            all_reduce_stats(srow, process_group)
        count = float(B * HW * world)
        # leaves of the batch statistics: their gradients are the a[c], k[c] of dL/dx
        ssum = srow[:C].clone().requires_grad_(True)
        ssq = srow[C:2 * C].clone().requires_grad_(True)
        pixel = (k, j) in pxi
        mod = spade_table(P, bn, ssum, ssq, count, None if pixel else GB[(k, j)])
        conv = blk(k) + f"conv_{j}."
        w_sn = w_sns[conv].reshape(C, C)
        wimg = abi.pack_weight(w_sn.detach().contiguous(), Nb=256)[0]
        if j == 0:
            block_in = (cur, cur_bstride, idx)
        out = torch.empty(B, T, C, 128, **f32)
        last_half = j == 1
        use_skip = last_half and k >= nb // 2 and block_in[1] != 0
        use_rgb = last_half and k >= nb // 2 - 1
        kw = {}
        rgb_name = None
        if use_rgb:
            rgb_name = f"{prefix}to_rgbs.m3d_{k}.linear."
            rgb_next = torch.empty(B, 3, HW, **f32)
            kw = dict(rgb_w=P[rgb_name + "weight"].detach().reshape(3, C).contiguous(), rgb_b=P[rgb_name + "bias"].detach(),
                      rgb_in=rgb_cur, rgb_out=rgb_next)
        mod_d = mod.detach().contiguous()
        rec = dict(x=cur, x_bstride=cur_bstride, mod=mod, mod_d=mod_d, w_sn=w_sn, ssum=ssum, ssq=ssq, conv=conv,
                   skip_from=block_in[2] if use_skip else None, rgb=rgb_name, out=out, pixel=pixel)
        if pixel:
            i = pxi[(k, j)]
            s_ = sp(k, j)
            wg, bg = P[s_ + "mlp_gamma.weight"].detach().reshape(C, 128), P[s_ + "mlp_gamma.bias"].detach()
            wb, bb = P[s_ + "mlp_beta.weight"].detach().reshape(C, 128), P[s_ + "mlp_beta.bias"].detach()
            w_il, b_il = _gamma_beta_interleaved(wg, bg, wb, bb)
            p_bias = PB[(k, j)]
            p_bias_d = p_bias.detach().float().contiguous()
            rec.update(i=i, spade=s_, p_bias=p_bias, p_bias_d=p_bias_d, wg=wg, wb=wb, bg1=(bg + 1.0).contiguous(), bb=bb)
            _spade(cur, cur_bstride, wimg, P[conv + "bias"].detach(), out, B, Hg, Wg, passes, scsh=mod_d,
                   p_lr=p_lr[:, i * 128:], p_stride=p_lr.shape[1], p_bias=p_bias_d, wgb=abi.pack_weight(w_il, Nb=256)[0],
                   bgb=b_il, Rh=Rh, Rw=Rw, skip=block_in[0] if use_skip else None, stats=stats[idx + 1], **kw)
        else:
            _spade(cur, cur_bstride, wimg, P[conv + "bias"].detach(), out, B, Hg, Wg, passes, mod=mod_d,
                   skip=block_in[0] if use_skip else None, stats=stats[idx + 1], **kw)
        if use_rgb:
            rgb_cur = rgb_next
        tape.halves.append(rec)
        cur, cur_bstride = out, T * C * 128
    tape.rgb = rgb_cur.reshape(B, 3, Hg, Wg)
    return tape.rgb, tape


def const_gamma_beta(P, s, fs, C):
    """(1 + gamma, beta) [B,C] of a const-style SPADE from the fixed style fs [B,C], with autograd history
    (SPADE2d.forward, map3d_layers.py:176-190)."""
    actv = torch.relu(F.linear(fs, P[s + "mlp_shared.0.weight"].reshape(128, C), P[s + "mlp_shared.0.bias"]))
    G = 1.0 + F.linear(actv, P[s + "mlp_gamma.weight"].reshape(C, 128), P[s + "mlp_gamma.bias"])
    Bt = F.linear(actv, P[s + "mlp_beta.weight"].reshape(C, 128), P[s + "mlp_beta.bias"])
    return G, Bt


def spade_table(P, bn, ssum, ssq, count, gb=None):
    """The folded BatchNorm (+ SPADE) table of one half-block with autograd history from the batch-statistics leaves
    ssum = sum(x), ssq = sum(x^2) [C]: [2,C] = (sc, sh) for pixel style (gb None), else [B,2,C] = (sc*G, sh*G + beta) with
    gb = (G, beta) from `const_gamma_beta`.  Updates the running statistics (momentum 0.1, unbiased variance,
    map3d_layers.py:162)."""
    mean = ssum / count
    var = (ssq / count - mean * mean).clamp_min(0.0)
    rstd = torch.rsqrt(var + 1e-5)
    sc = P[bn + "weight"].double() * rstd
    sh = P[bn + "bias"].double() - mean * sc
    if gb is None:      # BatchNorm scale/shift only; gamma/beta are per pixel
        mod = torch.stack([sc, sh]).float()
    else:
        G, Bt = gb
        mod = torch.stack([sc[None, :] * G.double(), sh[None, :] * G.double() + Bt.double()], dim=1).float()
    with torch.no_grad():
        P[bn + "running_mean"].mul_(0.9).add_(0.1 * mean.float())
        P[bn + "running_var"].mul_(0.9).add_(0.1 * (var * count / max(count - 1, 1)).float())
        if (bn + "num_batches_tracked") in P:
            P[bn + "num_batches_tracked"] += 1
    return mod


def grad_accumulator(P, grads):
    """-> acc(name, g): adds g to `grads[name]` (the gradients an autograd.Function RETURNS, so that DDP reducer hooks,
    torch.autograd.grad and GradScaler see them), or -- with grads=None, kernel-level tests and tools -- to `P[name].grad`."""
    def acc(name, g):
        p = P[name]
        if not p.requires_grad:
            return
        g = g.to(p.dtype).reshape(p.shape)
        if grads is None:
            p.grad = g if p.grad is None else p.grad + g
        else:
            grads[name] = g if name not in grads else grads[name] + g
    return acc


def synthesis_backward(params, tape, drgb, *, passes=3, grads=None):
    """Gradients of every synthesis parameter in `params` (those that require grad) into `grads` (name -> tensor; `.grad`
    when grads is None) and returns (d fixed_style [B,256], d feat_lr [B,Rh*Rw,256] or None when no half-block is
    pixel-style)."""
    P = params
    cfg, B = tape.cfg, tape.B
    Hg, Wg = cfg["gen_height"], cfg["gen_width"]
    HW = Hg * Wg
    T = (HW + 127) // 128
    dev = drgb.device
    f32 = dict(dtype=torch.float32, device=dev)
    drgb = drgb.reshape(B, 3, HW).float().contiguous()
    H = tape.halves
    n = len(H)
    full = T * C * 128

    acc = grad_accumulator(P, grads)

    # every ToRGB bias sees the full drgb
    drgb_sum = drgb.sum((0, 2))
    small_out, small_grad = [], []          # (tensor with autograd history, its gradient): one autograd.backward at the end
    dout = {}                               # half index -> dL/d(out of that half)   (only the live ones are kept)
    nxt = None                              # (dpre, g1 table [B,2,C], ak [2,C]) of half h+1
    for h in range(n - 1, -1, -1):
        rec = H[h]
        # ---- dL/d(out_h): from half h+1 (dpre*g1 + a + k*x), the skip of the block two halves later, ToRGB
        dskip = None
        if h + 2 < n and H[h + 2]["skip_from"] == h + 1:      # out_h is the input of a block with a residual skip
            dskip = dout[h + 2]
        d = torch.empty(B, T, C, 128, **f32)
        dwrgb = None
        kw = {}
        if rec["rgb"] is not None:
            dwrgb = torch.zeros(3, C, dtype=torch.float64, device=dev)
            kw = dict(drgb=drgb, rgb_w=P[rec["rgb"] + "weight"].detach().reshape(3, C).contiguous(), dwrgb=dwrgb)
        if nxt is not None:
            kw.update(dpre=nxt[0], g1=nxt[1], ak=nxt[2])
        abi.spade_bwd_combine(d, B=B, Hg=Hg, Wg=Wg, x=rec["out"], x_bstride=full, dskip=dskip, **kw)
        if dwrgb is not None:
            acc(rec["rgb"] + "weight", dwrgb.float())
            acc(rec["rgb"] + "bias", drgb_sum)
        dout[h] = d
        dout.pop(h + 3, None)
        # ---- this half-block
        wimg_t = abi.pack_weight(rec["w_sn"].detach().t().contiguous(), Nb=256)[0]
        dpre = torch.empty(B, T, C, 128, **f32)
        sums = torch.zeros(B, 2, C, dtype=torch.float64, device=dev)
        if rec["pixel"]:
            Rh, Rw = cfg["render_height"], cfg["render_width"]
            i = rec["i"]
            p_lr = tape.p["p_lr"]
            # rebuild A1, gamma, beta, pre
            a1 = torch.empty(B, T, 128, 128, **f32)
            abi.spade_a1(_PtrView(p_lr[:, i * 128:]), p_lr.shape[1], rec["p_bias_d"], a1, B=B, Hg=Hg, Wg=Wg, Rh=Rh, Rw=Rw)
            gam = torch.empty(B, T, C, 128, **f32)
            pre = torch.empty(B, T, C, 128, **f32)
            abi.conv1x1_blocked(a1, 128, abi.pack_weight(rec["wg"].contiguous(), Nb=256)[0], rec["bg1"], gam, B=B, Hg=Hg, Wg=Wg, passes=passes)
            abi.conv1x1_blocked(a1, 128, abi.pack_weight(rec["wb"].contiguous(), Nb=256)[0], rec["bb"], pre, B=B, Hg=Hg, Wg=Wg, passes=passes)
            abi.spade_pixel_pre(rec["x"], rec["x_bstride"], rec["mod_d"], gam, pre, B=B, Hg=Hg, Wg=Wg)
            if getattr(tape, "keep_masks", False):      # tests: the LeakyReLU mask this backward differentiates through
                rec["mask"] = pre > 0
                rec["mask_a1"] = a1 > 0
            # conv data / weight gradients on pre (y = lrelu(pre))
            abi.conv1x1_blocked_bwd(d, pre, wimg_t, dpre, sums, B=B, Hg=Hg, Wg=Wg, passes=passes)
            dw, db = abi.spade_bwd_wgrad(d, pre, full, None, B=B, Hg=Hg, Wg=Wg, passes=passes)
            # modulation: dxn (over pre), dgam (over gam), BatchNorm scale/shift sums
            s3 = torch.zeros(3, C, dtype=torch.float64, device=dev)
            abi.spade_pixel_mod_bwd(dpre, rec["x"], rec["x_bstride"], rec["mod_d"], gam, pre, s3, B=B, Hg=Hg, Wg=Wg)
            dxn, dgam = pre, gam
            # gamma/beta MLP: hidden-layer gradient (ReLU mask from A1), weight gradients, bilinear adjoint
            w7 = torch.zeros(256, 512, **f32)
            w7[:128, :256] = rec["wg"].t()
            w7[:128, 256:] = rec["wb"].t()
            da1 = torch.empty(B, HW, 128, **f32)
            s7 = torch.zeros(B, 2, 128, dtype=torch.float64, device=dev)
            abi.conv1x1_blocked_bwd(dgam, a1, abi.pack_weight(w7, Nb=256)[0], da1, s7, g2=dpre, Cout=128, slope=0.0,
                                    pixel_major=True, B=B, Hg=Hg, Wg=Wg, passes=passes)
            dwg, dbg = abi.spade_bwd_wgrad(dgam, a1, T * 128 * 128, None, Cx=128, B=B, Hg=Hg, Wg=Wg, passes=passes)
            dwb, dbb = abi.spade_bwd_wgrad(dpre, a1, T * 128 * 128, None, Cx=128, B=B, Hg=Hg, Wg=Wg, passes=passes)
            sp_ = rec["spade"]
            acc(sp_ + "mlp_gamma.weight", dwg)
            acc(sp_ + "mlp_gamma.bias", dbg)
            acc(sp_ + "mlp_beta.weight", dwb)
            acc(sp_ + "mlp_beta.bias", dbb)
            if "dp" not in tape.p:
                tape.p["dp"] = torch.zeros_like(p_lr)
            dp = tape.p["dp"]
            abi.bilinear_adjoint(da1, _PtrView(dp[:, i * 128:]), dp.shape[1], B=B, Hg=Hg, Wg=Wg, Rh=Rh, Rw=Rw)
            if rec["p_bias"].requires_grad:
                small_out.append(rec["p_bias"])
                small_grad.append(s7[:, 0].float())
            acc(rec["conv"] + "bias", db)
            small_out.append(rec["w_sn"])
            small_grad.append(dw)
            dmod = torch.stack([s3[0], s3[1]]).float()                        # d sc = sum dxn*x, d sh = sum dxn
            dpre = dxn
            g1_tab = rec["mod_d"][0][None, None, :].expand(B, 2, C).contiguous()
            del a1, da1
        else:
            abi.spade_bwd_dgrad(d, rec["x"], rec["x_bstride"], rec["mod_d"], wimg_t, dpre, sums, B=B, Hg=Hg, Wg=Wg, passes=passes)
            dw, db = abi.spade_bwd_wgrad(d, rec["x"], rec["x_bstride"], rec["mod_d"], B=B, Hg=Hg, Wg=Wg, passes=passes)
            acc(rec["conv"] + "bias", db)
            small_out.append(rec["w_sn"])
            small_grad.append(dw)
            dmod = torch.stack([sums[:, 1], sums[:, 0]], dim=1).float()       # d g1 = sum dpre*x, d g0 = sum dpre
            g1_tab = rec["mod_d"]
        ga, gk = torch.autograd.grad(rec["mod"], [rec["ssum"], rec["ssq"]], grad_outputs=dmod, retain_graph=True)
        ak = torch.stack([ga, gk])
        if tape.world > 1:          # every rank's loss depends on the global statistics
            dist.all_reduce(ak, group=tape.process_group)
        ak = torch.stack([ak[0], 2.0 * ak[1]]).float().contiguous()      # d(sum x)/dx = 1, d(sum x^2)/dx = 2x
        small_out.append(rec["mod"])
        small_grad.append(dmod)
        nxt = (dpre, g1_tab, ak)
    # ---- gradient w.r.t. the shared synthesis input x0, then its two parameters
    dx0 = torch.empty(B, T, C, 128, **f32)
    abi.spade_bwd_combine(dx0, B=B, Hg=Hg, Wg=Wg, x=H[0]["x"], x_bstride=0, dpre=nxt[0], g1=nxt[1], ak=nxt[2])
    ip = tape.input["prefix"]
    dw_in, db_in = abi.synth_input_bwd(dx0, tape.input["w"], P[ip + "network.0.bias"].detach(), tape.input["ic"], tape.input["jc"], B)
    acc(ip + "network.0.weight", dw_in)
    acc(ip + "network.0.bias", db_in)
    # ---- all [C]- and [B,C]-sized chains in one autograd pass (accumulates into the Parameters' .grad)
    fs = tape.fixed_style
    leaves = [t for t in small_out if t.requires_grad]
    small = [g for t, g in zip(small_out, small_grad) if t.requires_grad]
    names = [n for n, p in P.items() if isinstance(p, torch.Tensor) and p.requires_grad and p.is_leaf]
    res = torch.autograd.grad(leaves, [P[n] for n in names] + [fs], small, allow_unused=True)
    for n, r in zip(names, res[:-1]):
        if r is not None:
            acc(n, r)
    dfs = res[-1] if res[-1] is not None else torch.zeros_like(fs)
    # ---- render-resolution projection P_lr = X . W_shared^T: feature-map and weight gradients
    dfeat = None
    if tape.px and "dp" in tape.p:
        dp, Ws, X = tape.p["dp"], tape.p["Ws"], tape.p["X"]
        WsT = Ws.t().contiguous()                                                    # [256, n*128]
        dfeat = None
        for c0 in range(0, WsT.shape[1], 256):        # hg_linear takes K <= 256: one product per pair of half-blocks
            img, Nb = abi.pack_weight(WsT[:, c0:c0 + 256].contiguous(), Nb=256)
            part = abi.linear(dp[:, c0:c0 + 256], img, Nb, C, passes=passes)
            dfeat = part if dfeat is None else dfeat.add_(part)
        dfeat = dfeat.reshape(B, -1, C)
        prev = torch.backends.cuda.matmul.allow_tf32
        torch.backends.cuda.matmul.allow_tf32 = False
        dWs = dp.t() @ X                                                             # [n*128, 256]  (plain library GEMM)
        torch.backends.cuda.matmul.allow_tf32 = prev
        for rec in H:
            if rec["pixel"]:
                acc(rec["spade"] + "mlp_shared.0.weight", dWs[rec["i"] * 128:(rec["i"] + 1) * 128])
    return dfs, dfeat
