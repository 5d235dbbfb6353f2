"""Training-mode forward + backward of the SPADE synthesis network on the sm_90a kernels.

Forward: the same 18 fused half-block launches as `synthesis_ops.synthesis_forward`, but every half-block
input is kept (18 activations of B*HW*256 fp32 -- 2.1 GB each at the C2 workload; sized for 180 GB of HBM)
and every [B,C]- / [C]-sized quantity the kernels consume (folded BatchNorm+SPADE tables, spectrally
normalised weights) is built with torch autograd from its leaves.

Backward (`synthesis_backward`, one for every width: autograd through SynthesisNetwork.forward
map3d_generator.py:58-97, SPADEBlock.forward map3d_layers.py:218-238, SPADE2d.forward :176-190, ToRGB :346-352,
SynthesisInput :260-275), walking the half-blocks in reverse over the tape's 256-channel halves (one here, two from
the zero-padded forward of modules/wide_ops.py at hidden_dim 384 / 420; see `SynthesisTape`); per half-block
    hg_spade_bwd_combine  dL/dout   from the next half-block's dpre (+ skip gradient, + ToRGB^T drgb)   per half
    hg_spade_bwd_dgrad    dpre = (W^T dL/dout) * lrelu'(pre), S1 = sum dpre, S2 = sum dpre*x     (wgmma; with two
                          halves hg_conv1x1_blocked_bwd per input half, K = 512)
    hg_spade_bwd_wgrad    dW = dL/dout . y^T, dbias                    (wgmma; per (output half, input half) block)
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
    hg_conv1x1_blocked_bwd dA1 = ([dgam | dpre] . [Wg | Wb]) * relu'(A1)        (wgmma, K = 512 launches, pixel-major out)
    hg_wgrad_blocked   x2  dWg = dgam . A1^T,  dWb = dpre . A1^T                 (wgmma)
    hg_bilinear_adjoint    dP_lr (render resolution)
and once, at the end, d(feature maps) = dP_lr . W_shared (wgmma `hg_linear`, K <= 256 per launch) and dW_shared = dP_lr^T . features
(a plain library GEMM through torch.matmul).

Eval mode (`training=False`: latent inversion, fine-tuning with frozen statistics) is the same schedule with less in it:
the tables come from the running statistics and the stored spectral-norm u / v (no statistics epilogue, no power
iteration, no buffer is written, no collective), so the statistics leaves and with them the a[c] + k[c]*x term do not
exist.  A weight-gradient kernel is launched only for parameters that require grad; with every parameter frozen the
backward is the data-gradient chain to the fixed style and the render features alone.
"""
from __future__ import annotations

import torch
import torch.distributed as dist
import torch.nn.functional as F

from .. import abi
from ..ops.dense import _gemm_nt
from .synthesis_ops import STAT_STRIDE, _PtrView, _gamma_beta_interleaved, _spade, all_reduce_stats, is_pixel_style, sn_weights
from .wide_ops import HALF, _pad2

C = 256


class SynthesisTape:
    """Everything `synthesis_backward` needs from one training forward: `synthesis_forward_train` at hidden_dim 256,
    `wide_ops.synthesis_forward_wide(..., tape=tape)` at the zero-padded widths.

    Every activation is a tuple of nh tile-blocked 256-channel halves [B,T,256,128], nh = 1 at 256 and 2 at the padded
    widths (padded channels hold zeros).  `halves` has one record per half-block:
        x, out          per-half tuples of its input and output
        x_bstride       the batch stride of x: 0 for the batch-shared synthesis input [T,256,128] at 256, T*256*128 otherwise
        mod_d           per-half tuple of the detached folded table: [B,2,256] const style, (sc, sh) [2,256] pixel style
        mod, ssum, ssq  the same table over nh*256 channels, with autograd history from the batch-statistics leaves
                        ssum = sum(x), ssq = sum(x^2)
        w_sn            W / sigma with history; conv, the convolution's parameter prefix
        rgb, rgb_w      the ToRGB parameter prefix and its weight [3,nh*256] (None without ToRGB); skip_from
        pixel           pixel style; then also i (its slice of P_lr), spade, p_bias (with history), p_bias_d and
                        wg, wb [nh*256,128], bg1 = gamma bias + 1, bb [nh*256]
    `input` holds the synthesis input's w [nh*256,2], b [nh*256], ic, jc and parameter prefix."""

    def __init__(self):
        self.halves = []
        self.cfg = None
        self.B = 0
        self.rgb = None


def synthesis_forward_train(params, feat_lr, fixed_style, cfg, *, passes=3, prefix="synthesis_network.",
                            input_prefix="synthesis_input.", process_group=None, training=True):
    """-> (rgb [B,3,Hg,Wg] (no autograd history), tape).  `params`: name -> tensor (Parameters keep their .grad).
    `training=False`: BatchNorm from the running statistics, spectral norm from the stored u / v; no buffer is written."""
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
    world = dist.get_world_size(process_group) if (training and dist.is_available() and dist.is_initialized()) else 1
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
    abi.synth_input(w_in, P[input_prefix + "network.0.bias"].detach(), ic, jc, x0, stats[0] if training else None, B)
    tape.input = dict(w=w_in, b=P[input_prefix + "network.0.bias"].detach(), ic=ic, jc=jc, prefix=input_prefix)

    # spectral normalisation of the 18 convolutions: one launch (power iteration, buffers in place), W / sigma with history
    w_sns = sn_weights(P, [blk(k) + f"conv_{j}." for k, j in halves], training)

    rgb_cur = None
    cur, cur_bstride = x0, 0
    block_in = None
    for idx, (k, j) in enumerate(halves):
        bn = sp(k, j) + "first_norm."
        srow = stats[idx]
        if world > 1:
            all_reduce_stats(srow, process_group)
        count = float(B * HW * world)
        pixel = (k, j) in pxi
        if training:
            # leaves of the batch statistics: their gradients are the a[c], k[c] of dL/dx
            ssum = srow[:C].clone().requires_grad_(True)
            ssq = srow[C:2 * C].clone().requires_grad_(True)
            mod = spade_table(P, bn, ssum, ssq, count, None if pixel else GB[(k, j)])
        else:
            ssum = ssq = None
            mod = spade_table_eval(P, bn, None if pixel else GB[(k, j)])
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
        rec = dict(x=(cur,), x_bstride=cur_bstride, mod=mod, mod_d=(mod_d,), w_sn=w_sn, ssum=ssum, ssq=ssq, conv=conv,
                   skip_from=block_in[2] if use_skip else None, rgb=rgb_name, rgb_w=kw.get("rgb_w"), out=(out,), pixel=pixel)
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
                   bgb=b_il, Rh=Rh, Rw=Rw, skip=block_in[0] if use_skip else None, stats=stats[idx + 1] if training else None, **kw)
        else:
            _spade(cur, cur_bstride, wimg, P[conv + "bias"].detach(), out, B, Hg, Wg, passes, mod=mod_d,
                   skip=block_in[0] if use_skip else None, stats=stats[idx + 1] if training else None, **kw)
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
    mod = _fold(P, bn, mean, var, gb)
    with torch.no_grad():
        P[bn + "running_mean"].mul_(0.9).add_(0.1 * mean.float())
        P[bn + "running_var"].mul_(0.9).add_(0.1 * (var * count / max(count - 1, 1)).float())
        if (bn + "num_batches_tracked") in P:
            P[bn + "num_batches_tracked"] += 1
    return mod


def spade_table_eval(P, bn, gb=None):
    """`spade_table` in eval mode: the table from the running statistics, with autograd history from the BatchNorm weight /
    bias (and gb) only; no buffer is written."""
    return _fold(P, bn, P[bn + "running_mean"].detach().double(), P[bn + "running_var"].detach().double(), gb)


def _fold(P, bn, mean, var, gb):
    sc = P[bn + "weight"].double() * torch.rsqrt(var + 1e-5)
    sh = P[bn + "bias"].double() - mean * sc
    if gb is None:      # BatchNorm scale/shift only; gamma/beta are per pixel
        return torch.stack([sc, sh]).float()
    G, Bt = gb
    return torch.stack([sc[None, :] * G.double(), sh[None, :] * G.double() + Bt.double()], dim=1).float()


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


def _packT(W, ih):
    """Operand image of the transposed input-half `ih` columns of a zero-padded [nh*256, nh*256] weight: the data
    gradient's [256 x K = nh*256] weight."""
    return abi.pack_weight(W[:, ih * HALF:(ih + 1) * HALF].t().contiguous(), Nb=256)[0]


def synthesis_backward(params, tape, drgb, *, passes=3, grads=None):
    """Backward of the training synthesis network at every width (the tape format is `SynthesisTape`'s): gradients of
    every synthesis parameter in `params` that requires grad into `grads` (name -> tensor; `.grad` when grads is None);
    returns (d fixed_style [B,C], d feat_lr [B,Rh*Rw,C] or None when no half-block is pixel-style).  A layer over nh
    halves is a data-gradient launch per input half (K = nh*256 from the output halves' gradients) and a weight-gradient
    launch per (output half, input half) block; padded channels carry zero weights and tables, so their gradients are
    zero up to the trimming to each parameter's shape."""
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
    nh = len(H[0]["x"])
    halves = range(nh)
    W2 = nh * HALF
    sl = lambda c: slice(c * HALF, (c + 1) * HALF)
    full = T * HALF * 128
    new = lambda: torch.empty(B, T, HALF, 128, **f32)
    acc = grad_accumulator(P, grads)
    need = lambda *names: any(P[k].requires_grad for k in names)      # a weight-gradient kernel runs only for these

    def conv_wgrad(d, xs, x_bstride, mods_in):
        """[nh*256, nh*256] weight gradient of a half-block's convolution block by block, [nh*256] bias gradient."""
        dW = torch.empty(W2, W2, **f32)
        dbs = []
        for oh in halves:
            for ih in halves:
                dw, db = abi.spade_bwd_wgrad(d[oh], xs[ih], x_bstride, mods_in[ih], want_bias=ih == 0, **kw)
                dW[sl(oh), sl(ih)] = dw
                if ih == 0:
                    dbs.append(db)
        return dW, torch.cat(dbs)

    # every ToRGB bias sees the full drgb
    drgb_sum = drgb.sum((0, 2))
    small_out, small_grad = [], []          # (tensor with autograd history, its gradient): one autograd pass at the end
    dout = {}                               # half-block index -> dL/d(its out) per half   (only the live ones are kept)
    nxt = None                              # (dpre, g1 table, ak) per half of half-block h+1
    for h in range(n - 1, -1, -1):
        rec = H[h]
        # ---- dL/d(out_h): from half-block h+1 (dpre*g1 + a + k*x), the skip of the block two half-blocks later, ToRGB
        dskip = (None,) * nh
        if h + 2 < n and H[h + 2]["skip_from"] == h + 1:      # out_h is the input of a block with a residual skip
            dskip = dout[h + 2]
        d, dwrgb = [], []
        for c in halves:
            ckw = {}
            if rec["rgb"] is not None:
                dwrgb.append(torch.zeros(3, HALF, dtype=torch.float64, device=dev) if need(rec["rgb"] + "weight") else None)
                ckw = dict(drgb=drgb, rgb_w=rec["rgb_w"][:, sl(c)].contiguous(), dwrgb=dwrgb[c])
            if nxt is not None:
                ckw.update(dpre=nxt[0][c], g1=nxt[1][c], ak=nxt[2][c])
            d.append(abi.spade_bwd_combine(new(), B=B, Hg=Hg, Wg=Wg, x=rec["out"][c], x_bstride=full, dskip=dskip[c], **ckw))
        if rec["rgb"] is not None:
            if dwrgb[0] is not None:
                acc(rec["rgb"] + "weight", torch.cat(dwrgb, -1)[:, :C].float())
            acc(rec["rgb"] + "bias", drgb_sum)
        dout[h] = d
        dout.pop(h + 3, None)
        # ---- this half-block: const style acts on x through its table, pixel style on the rebuilt `pre`
        Wsn = _pad2(rec["w_sn"].detach().reshape(C, C), W2, W2)
        sums = [torch.zeros(B, 2, HALF, dtype=torch.float64, device=dev) for _ in halves]
        want_w = need(rec["conv"] + "weight_orig", rec["conv"] + "bias")
        dW = db = None
        if rec["pixel"]:
            Rh, Rw = cfg["render_height"], cfg["render_width"]
            i = rec["i"]
            p_lr = tape.p["p_lr"]
            # rebuild A1, gamma, beta, pre
            a1 = torch.empty(B, T, 128, 128, **f32)
            abi.spade_a1(_PtrView(p_lr[:, i * 128:]), p_lr.shape[1], rec["p_bias_d"], a1, B=B, Hg=Hg, Wg=Wg, Rh=Rh, Rw=Rw)
            gam, pre = [], []
            for c in halves:
                gam.append(abi.conv1x1_blocked(a1, 128, abi.pack_weight(rec["wg"][sl(c)].contiguous(), Nb=256)[0],
                                               rec["bg1"][sl(c)].contiguous(), new(), **kw))
                pre.append(abi.conv1x1_blocked(a1, 128, abi.pack_weight(rec["wb"][sl(c)].contiguous(), Nb=256)[0],
                                               rec["bb"][sl(c)].contiguous(), new(), **kw))
                abi.spade_pixel_pre(rec["x"][c], rec["x_bstride"], rec["mod_d"][c], gam[c], pre[c], B=B, Hg=Hg, Wg=Wg)
            if getattr(tape, "keep_masks", False):      # tests: the masks this backward differentiates through
                rec["mask"] = [p > 0 for p in pre]
                rec["mask_a1"] = a1 > 0
            # conv data / weight gradients on pre (y = lrelu(pre))
            dpre = [abi.conv1x1_blocked_bwd(d[0], pre[c], _packT(Wsn, c), new(), sums[c], g2=d[1] if nh == 2 else None, **kw)
                    for c in halves]
            if want_w:
                dW, db = conv_wgrad(d, pre, full, (None,) * nh)
            # modulation: dxn (over pre), dgam (over gam), BatchNorm scale/shift sums
            s3 = [torch.zeros(3, HALF, dtype=torch.float64, device=dev) for _ in halves]
            for c in halves:
                abi.spade_pixel_mod_bwd(dpre[c], rec["x"][c], rec["x_bstride"], rec["mod_d"][c], gam[c], pre[c], s3[c], B=B, Hg=Hg, Wg=Wg)
            dxn, dgam = pre, gam
            # gamma/beta MLP: dA1 = ([dgam halves, dpre halves] . [Wg | Wb]) * relu'(A1), K = 2*nh*256 in K = 512 launches
            srcs = dgam + dpre
            wt = torch.cat([rec["wg"], rec["wb"]]).t()                        # [128, 2*nh*256]
            s7 = torch.zeros(B, 2, 128, dtype=torch.float64, device=dev)
            da1 = None
            for k in range(0, len(srcs), 2):
                w7 = torch.zeros(256, 2 * HALF, **f32)
                w7[:128] = wt[:, k * HALF:(k + 2) * HALF]
                part = abi.conv1x1_blocked_bwd(srcs[k], a1, abi.pack_weight(w7, Nb=256)[0], torch.empty(B, HW, 128, **f32), s7,
                                               g2=srcs[k + 1], Cout=128, slope=0.0, pixel_major=True, **kw)
                da1 = part if da1 is None else da1.add_(part)
            sp_ = rec["spade"]
            for gs, nm in ((dgam, "mlp_gamma."), (dpre, "mlp_beta.")):
                if not need(sp_ + nm + "weight", sp_ + nm + "bias"):
                    continue
                dws, dbs = zip(*[abi.spade_bwd_wgrad(gs[c], a1, T * 128 * 128, None, Cx=128, **kw) for c in halves])
                acc(sp_ + nm + "weight", torch.cat(dws)[:C])
                acc(sp_ + nm + "bias", torch.cat(dbs)[:C])
            if "dp" not in tape.p:
                tape.p["dp"] = torch.zeros_like(p_lr)
            dp = tape.p["dp"]
            abi.bilinear_adjoint(da1, _PtrView(dp[:, i * 128:]), dp.shape[1], B=B, Hg=Hg, Wg=Wg, Rh=Rh, Rw=Rw)
            if rec["p_bias"].requires_grad:
                small_out.append(rec["p_bias"])
                small_grad.append(s7[:, 0].float())
            # d sc = sum dxn*x, d sh = sum dxn
            dmod = torch.stack([torch.cat([s[0] for s in s3]), torch.cat([s[1] for s in s3])]).float()
            dpre = dxn
            g1_tab = [m[0][None, None, :].expand(B, 2, HALF).contiguous() for m in rec["mod_d"]]
            del a1, da1, gam
        else:
            if nh == 1:     # the only data-gradient entry point that reads a batch-shared input (block 0 at 256)
                dpre = [abi.spade_bwd_dgrad(d[0], rec["x"][0], rec["x_bstride"], rec["mod_d"][0], _packT(Wsn, 0), new(), sums[0], **kw)]
            else:
                dpre = [abi.conv1x1_blocked_bwd(d[0], rec["x"][c], _packT(Wsn, c), new(), sums[c], g2=d[1], mod=rec["mod_d"][c],
                                                slope=0.2, **kw) for c in halves]
            if want_w:
                dW, db = conv_wgrad(d, rec["x"], rec["x_bstride"], rec["mod_d"])
            # d g1 = sum dpre*x, d g0 = sum dpre
            dmod = torch.stack([torch.cat([s[:, 1] for s in sums], -1), torch.cat([s[:, 0] for s in sums], -1)], dim=1).float()
            g1_tab = rec["mod_d"]
        if want_w:
            acc(rec["conv"] + "bias", db[:C])
            small_out.append(rec["w_sn"])
            small_grad.append(dW[:C, :C].reshape(rec["w_sn"].shape))
        if rec["ssum"] is None:     # eval mode: the statistics are constants, dL/dx has no a + k*x term
            aks = (None,) * nh
        else:
            ga, gk = torch.autograd.grad(rec["mod"], [rec["ssum"], rec["ssq"]], grad_outputs=dmod, retain_graph=True)
            ak = torch.stack([ga, gk])
            if tape.world > 1:          # SyncBatchNorm: every rank's loss depends on the global statistics
                dist.all_reduce(ak, group=tape.process_group)
            ak = torch.stack([ak[0], 2.0 * ak[1]]).float()                     # d(sum x)/dx = 1, d(sum x^2)/dx = 2x
            aks = [ak[:, sl(c)].contiguous() for c in halves]
        small_out.append(rec["mod"])
        small_grad.append(dmod)
        nxt = (dpre, g1_tab, aks)
    # ---- gradient w.r.t. the synthesis input, then its two parameters, per half
    ip = tape.input["prefix"]
    dw_in, db_in = [], []
    for c in halves if need(ip + "network.0.weight", ip + "network.0.bias") else ():
        dx0 = abi.spade_bwd_combine(new(), B=B, Hg=Hg, Wg=Wg, x=H[0]["x"][c], x_bstride=H[0]["x_bstride"], dpre=nxt[0][c], g1=nxt[1][c],
                                    ak=nxt[2][c])
        dw, db = abi.synth_input_bwd(dx0, tape.input["w"][sl(c)].contiguous(), tape.input["b"][sl(c)].contiguous(),
                                     tape.input["ic"], tape.input["jc"], B)
        dw_in.append(dw)
        db_in.append(db)
    if dw_in:
        acc(ip + "network.0.weight", torch.cat(dw_in)[:C])
        acc(ip + "network.0.bias", torch.cat(db_in)[:C])
    # ---- all [C]- and [B,C]-sized chains in one autograd pass
    fs = tape.fixed_style
    leaves = [t for t in small_out if t.requires_grad]
    small = [g for t, g in zip(small_out, small_grad) if t.requires_grad]
    names = [k for k, p in P.items() if isinstance(p, torch.Tensor) and p.requires_grad and p.is_leaf]
    res = torch.autograd.grad(leaves, [P[k] for k in names] + [fs], small, allow_unused=True) if leaves else [None]
    for k, r in zip(names, res[:-1]):
        if r is not None:
            acc(k, r)
    dfs = res[-1] if res[-1] is not None else torch.zeros_like(fs)
    # ---- render-resolution projection P_lr = X . W_shared^T: feature-map and weight gradients
    dfeat = None
    if tape.px and "dp" in tape.p:
        dp, Ws, X = tape.p["dp"], tape.p["Ws"], tape.p["X"]
        dfeat = _gemm_nt(dp, Ws.t().contiguous(), passes=passes).reshape(B, -1, C)
        shared = [rec for rec in H if rec["pixel"] and need(rec["spade"] + "mlp_shared.0.weight")]
        if shared:
            prev = torch.backends.cuda.matmul.allow_tf32
            torch.backends.cuda.matmul.allow_tf32 = False
            dWs = dp.t() @ X                                                             # [n*128, C]  (plain library GEMM)
            torch.backends.cuda.matmul.allow_tf32 = prev
        for rec in shared:
            acc(rec["spade"] + "mlp_shared.0.weight", dWs[rec["i"] * 128:(rec["i"] + 1) * 128])
    return dfs, dfeat
