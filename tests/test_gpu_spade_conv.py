"""The blocked-GEMM engine of csrc/synth.cu launch by launch against fp64: `hg_spade_conv` (const- and pixel-style SPADE
half-blocks), `hg_conv1x1_blocked`, `hg_act_conv1x1_blocked` and `hg_blocked_conv_wide`; then the pixel-style helpers
(`hg_spade_a1`, `hg_bilinear_adjoint`, `hg_spade_pixel_pre`, `hg_spade_pixel_mod_bwd`) and the table producers
(`hg_bn_finalize`, `hg_synth_input`); last, one launch of each class a C2 generator forward runs (512x512, B = 8).

Every engine launch is checked five ways:
  1. valid outputs against the fp64 formula of the kernel's contract, evaluated from the inputs;
  2. the epilogue (next-BatchNorm statistics row, ToRGB) against fp64 evaluated from the kernel's own `out`, so that an
     epilogue error is not hidden under GEMM error;
  3. the padding rows of the inputs hold NaN in one launch and zeros in another: padding adds only zeros to the MMA, so
     valid outputs are bit-identical;
  4. every output lives inside a larger buffer whose guard elements must be untouched;
  5. a repeated launch gives bit-identical outputs (only the statistics use atomics).
Shapes derive from the device's SM count: a one-tile image, last tiles with fewer than / exactly / more than 64 valid
pixels (warpgroup 1 holds only padding in the first two), and a launch whose persistent CTAs each walk tiles of several
samples (per-sample table refresh; backward: per-sample flush of the sums)."""
import importlib
import itertools
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

C = 256
STAT_STRIDE = 520          # modules/synthesis_ops.py: [0:256] sum, [256:512] sumsq, [512] count, pad
U = 2.0 ** -24             # fp32 unit roundoff
G = 64                     # guard elements on each side of an output (keeps 16-byte alignment in fp32 and fp64)
SENTINEL = -1234.5


def _abi():
    return importlib.import_module("3dhumangan_b200.abi")


def _nsm():
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


SHAPES = ["tile1", "lt64", "eq64", "gt64", "multi"]


def _shape(name):
    """(B, Hg, Wg) of a named case."""
    if name == "tile1":
        return 2, 8, 12            # HW 96: one tile per sample
    if name == "lt64":
        return 2, 12, 26           # HW 312: last tile holds 56 valid pixels
    if name == "eq64":
        return 2, 16, 20           # HW 320: last tile holds exactly 64
    if name == "gt64":
        return 2, 40, 25           # HW 1000: last tile holds 104
    n = _nsm()                     # "multi": T < SMs tiles per sample and B*T >= 2 SMs tiles
    Wg = 100
    Hg = (n // 3 + 1) * 128 // Wg
    T = (Hg * Wg + 127) // 128
    B = -(-2 * n // T) + 1
    assert T < n and B * T >= 2 * n and (Hg * Wg) % 128
    return B, Hg, Wg


def _tiles(HW):
    return (HW + 127) // 128


def _tiles_per_cta(B, HW):
    tiles = B * _tiles(HW)
    return -(-tiles // min(tiles, _nsm()))


def _blocked(t, fill=0.0):
    """[B,C,HW] -> tile-blocked [B,T,C,128]; the rows past the image hold `fill`."""
    B, Cc, HW = t.shape
    T = _tiles(HW)
    pad = torch.full((B, Cc, T * 128), fill, dtype=t.dtype, device=t.device)
    pad[:, :, :HW] = t
    return pad.reshape(B, Cc, T, 128).permute(0, 2, 1, 3).contiguous()


def _planar(t, HW):
    B, T, Cc, _ = t.shape
    return t.permute(0, 2, 1, 3).reshape(B, Cc, T * 128)[:, :, :HW]


def _guarded(shape, dtype=torch.float32, fill=float("nan")):
    """(buffer, view): a contiguous view of `shape` inside a buffer with G sentinel elements on each side."""
    n = math.prod(shape)
    buf = torch.full((n + 2 * G,), SENTINEL, dtype=dtype, device="cuda")
    view = buf[G:G + n].view(shape)
    view.fill_(fill)
    return buf, view


def _intact(buf):
    return bool((buf[:G] == SENTINEL).all()) and bool((buf[-G:] == SENTINEL).all())


def _stats_row(count):
    """A guarded statistics row pre-filled with known sums, the count at [512] and markers in the pad [513:520]."""
    buf, row = _guarded((STAT_STRIDE,), torch.float64, 0.0)
    g = torch.Generator(device="cuda").manual_seed(123)
    row[:512] = 100.0 * torch.randn(512, generator=g, device="cuda", dtype=torch.float64)
    row[512] = float(count)
    row[513:] = -1.5 * torch.arange(1, 8, device="cuda", dtype=torch.float64)
    return buf, row, row.clone()


def _rnd(seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return lambda *s: torch.randn(*s, generator=g, device="cuda")


def _rel_max(got, ref):
    return ((got.double() - ref).abs().max() / ref.abs().max()).item()


def _lrelu(v, slope):
    return torch.where(v > 0, v, slope * v)


def _pairwise(levels):
    """Rows of the full product of `levels` (a dict name -> values) chosen greedily until every pair of values of every two
    options appears in some row; deterministic."""
    names = list(levels)
    todo = {(a, va, b, vb) for a, b in itertools.combinations(names, 2) for va in levels[a] for vb in levels[b]}
    rows = []
    while todo:
        best = max(itertools.product(*levels.values()),
                   key=lambda r: sum((a, r[i], b, r[j]) in todo for (i, a), (j, b) in itertools.combinations(enumerate(names), 2)))
        d = dict(zip(names, best))
        todo -= {(a, d[a], b, d[b]) for a, b in itertools.combinations(names, 2)}
        rows.append(d)
    return rows


def _vid(v):
    parts = ["skip" if v["skip"] else "noskip", {0: "norgb", 1: "rgb", 2: "rgbin"}[v["rgb"]], "stats" if v["stats"] else "nostats",
             "xshared" if v["xshared"] else "xfull", f"p{v['passes']}"]
    if "pbias" in v:
        parts += ["pbias" if v["pbias"] else "nopbias", f"pstride{640 if v['pwide'] else 128}", "r" + v["ratio"]]
    return "-".join(parts)


CONST = _pairwise(dict(skip=(0, 1), rgb=(0, 1, 2), stats=(0, 1), xshared=(0, 1), passes=(3, 1)))
PIXEL = _pairwise(dict(skip=(0, 1), rgb=(0, 1, 2), stats=(0, 1), xshared=(0, 1), passes=(3, 1), pbias=(0, 1), pwide=(0, 1),
                       ratio=("1", "int", "40:7", "512:96")))


def _render_size(ratio, Hg, Wg):
    """Render resolution of a pixel-style case: Rh = Rw = 1, an integer ratio, or the nominal non-integer ratios 40/7 and
    C2's 512/96 (exact where the image size allows, otherwise the nearest render size)."""
    if ratio == "1":
        return 1, 1
    if ratio == "int":
        d = lambda n: n // 4 if n % 4 == 0 else n // 2 if n % 2 == 0 else n
        return d(Hg), d(Wg)
    num, den = (40, 7) if ratio == "40:7" else (512, 96)
    return max(1, round(Hg * den / num)), max(1, round(Wg * den / num))


# ----------------------------------------------------------------------------------------------------------------------
# shared checks
# ----------------------------------------------------------------------------------------------------------------------
def _check_stats(row, init, outp, n_t):
    """row = init + (sum, sumsq) over the valid pixels of the kernel's own out, per channel, in fp64.
    Bound: per tile and channel a thread adds its 2 rows (1 fp32 add), three shuffle steps fold the 16 rows of a warp
    (3 adds), and each of the 8 warps adds its total to the CTA's fp32 shared sum, over n_t tiles per CTA: at most
    4 + 8 n_t roundings on any path, each at most u = 2^-24 of a partial sum bounded by sum |v| (sumsq: sum v^2), so
    |err| <= (4 + 8 n_t) u sum|v| (first-order gamma_n bound).  The CTA sums then go to the fp64 row (2^-53 per add)."""
    o = outp.double()
    terms = ((o.sum((0, 2)), o.abs().sum((0, 2))), ((o * o).sum((0, 2)), (o * o).sum((0, 2))))
    for k, (ref, mag) in enumerate(terms):
        err = (row[k * C:(k + 1) * C] - init[k * C:(k + 1) * C] - ref).abs()
        bound = (4 + 8 * n_t) * U * mag + 1e-13 * init[k * C:(k + 1) * C].abs()
        assert (err <= bound).all(), ("sum" if k == 0 else "sumsq", float((err / bound).max()))
    assert torch.equal(row[512:], init[512:]), "the count and pad slots [512:520] must stay untouched"


def _check_rgb(rgb_out, outp, rgb_w, rgb_b, rgb_in):
    """rgb_out = W_rgb out + b (+ rgb_in) in fp64 from the kernel's own out.  Per pixel a lane runs 64 sequential fp32
    fmas (its 64 channels), two shuffle adds fold the 4 lanes of a row, then b and rgb_in are added: at most 68
    roundings, so |err| <= 68 u (sum_c |w_c out_c| + |b| + |rgb_in|)."""
    o = outp.double()
    w = rgb_w.double()
    ref = torch.einsum("kc,bcp->bkp", w, o) + rgb_b.double()[None, :, None]
    mag = torch.einsum("kc,bcp->bkp", w.abs(), o.abs()) + rgb_b.double().abs()[None, :, None]
    if rgb_in is not None:
        ref = ref + rgb_in.double()
        mag = mag + rgb_in.double().abs()
    err = (rgb_out.double() - ref).abs()
    assert (err <= 68 * U * mag).all(), float((err / (68 * U * mag)).max())


def _engine_case(launch, HW, ref, tol, *, n_t=None, rgb=None):
    """Runs `launch(fill)` three times (padding NaN, zeros, zeros again) and applies checks 1-5.  `launch` returns a dict with
    out [B,T,Cout,128], bufs (guarded buffers), and optionally row / init (statistics) and rgb_out."""
    runs = [launch(float("nan")), launch(0.0), launch(0.0)]
    torch.cuda.synchronize()
    for r in runs:
        assert all(_intact(b) for b in r["bufs"]), "a guard element was overwritten"
    a, b, c = runs
    outs = [_planar(r["out"], HW) for r in runs]
    assert torch.equal(outs[0], outs[1]), "NaN in the padding rows changed a valid output"
    assert torch.equal(outs[1], outs[2]), "a repeated launch changed out"
    if "rgb_out" in b:
        assert torch.equal(a["rgb_out"], b["rgb_out"]) and torch.equal(b["rgb_out"], c["rgb_out"])
    err = _rel_max(outs[1], ref)
    assert err < tol, err
    if "row" in b:
        assert torch.isfinite(a["row"]).all(), "NaN padding reached the statistics"
        for r, o in zip(runs, outs):
            _check_stats(r["row"], r["init"], o, n_t)
    if rgb is not None:
        _check_rgb(b["rgb_out"], outs[1], *rgb)
    return err


# ----------------------------------------------------------------------------------------------------------------------
# 1. hg_spade_conv
# ----------------------------------------------------------------------------------------------------------------------
def _spade_case(style, v, shape, seed):
    abi = _abi()
    so = importlib.import_module("3dhumangan_b200.modules.synthesis_ops")
    B, Hg, Wg = _shape(shape)
    HW, T = Hg * Wg, _tiles(Hg * Wg)
    r = _rnd(seed)
    x = r(1 if v["xshared"] else B, C, HW)
    W = r(C, C)
    inv_sigma = (1.0 / torch.linalg.matrix_norm(W.double(), 2)).float().reshape(1)
    wimg = abi.pack_weight(W, Nb=256, scale_dev=inv_sigma)[0]
    bias = 0.1 * r(C)
    skip = r(B, C, HW) if v["skip"] else None
    rgb_w = r(3, C) / 16 if v["rgb"] else None
    rgb_b = r(3) if v["rgb"] else None
    rgb_in = r(B, 3, HW) if v["rgb"] == 2 else None

    xd = x.double().expand(B, C, HW)
    kw = {}
    if style == "const":
        mod = torch.stack([1.0 + 0.5 * r(B, C), 0.5 * r(B, C)], 1).contiguous()         # [B,2,C] (g1, g0)
        pre = xd * mod[:, 0, :, None].double() + mod[:, 1, :, None].double()
        kw.update(mod=mod)
        desc = ""
    else:
        Rh, Rw = _render_size(v["ratio"], Hg, Wg)
        nsl = 5 if v["pwide"] else 1
        i = 2 if v["pwide"] else 0
        p_all = 0.7 * r(B * Rh * Rw, nsl * 128)                                          # [M, n*128] as hg_linear writes it
        p_bias = (0.3 * r(B, 128)).contiguous() if v["pbias"] else None
        scsh = torch.stack([1.0 + 0.3 * r(C), 0.3 * r(C)]).contiguous()                  # [2,C] BatchNorm scale, shift
        wg, wb = r(C, 128) / 16, r(C, 128) / 16
        bg, bb = 0.1 * r(C), 0.1 * r(C)
        w_il, b_il = so._gamma_beta_interleaved(wg, bg, wb, bb)
        kw.update(scsh=scsh, p_lr=so._PtrView(p_all[:, i * 128:]), p_stride=p_all.shape[1], p_bias=p_bias,
                  wgb=abi.pack_weight(w_il, Nb=256)[0], bgb=b_il, Rh=Rh, Rw=Rw)
        P = p_all[:, i * 128:(i + 1) * 128].double().reshape(B, Rh, Rw, 128).permute(0, 3, 1, 2)
        a1 = F.interpolate(P, (Hg, Wg), mode="bilinear", align_corners=False).reshape(B, 128, HW)
        if p_bias is not None:
            a1 = a1 + p_bias.double()[:, :, None]
        a1 = torch.relu(a1)
        gam = 1.0 + torch.einsum("ck,bkp->bcp", wg.double(), a1) + bg.double()[None, :, None]
        bet = torch.einsum("ck,bkp->bcp", wb.double(), a1) + bb.double()[None, :, None]
        pre = (xd * scsh[0, None, :, None].double() + scsh[1, None, :, None].double()) * gam + bet
        desc = f" render {Rh}x{Rw}"
    ref = torch.einsum("oc,bcp->bop", W.double() * inv_sigma.double(), _lrelu(pre, 0.2)) + bias.double()[None, :, None]
    if skip is not None:
        ref = ref + skip.double()

    def launch(fill):
        obuf, out = _guarded((B, T, C, 128))
        bufs, res = [obuf], dict(out=out)
        rk = dict(kw)
        if v["rgb"]:
            rbuf, rgb_out = _guarded((B, 3, HW))
            bufs.append(rbuf)
            rk.update(rgb_w=rgb_w, rgb_b=rgb_b, rgb_in=rgb_in, rgb_out=rgb_out)
            res["rgb_out"] = rgb_out
        if v["stats"]:
            sbuf, row, init = _stats_row(B * HW)
            bufs.append(sbuf)
            rk.update(stats=row)
            res.update(row=row, init=init)
        abi.spade_conv(_blocked(x, fill), 0 if v["xshared"] else T * C * 128, wimg, bias, out, B=B, Hg=Hg, Wg=Wg,
                       skip=None if skip is None else _blocked(skip, fill), passes=v["passes"], **rk)
        res["bufs"] = bufs
        return res

    # passes=3: the bar test_gpu_synthesis_bwd.py::test_dgrad holds this kernel to.  Pixel style chains the [gamma | beta]
    # GEMM (K = 128) into the convolution (K = 256); each bf16x3 GEMM stays near 1e-6 relative, so the same 2e-5 holds.
    # Measured on an H100 80GB HBM3 (700 W): at most 7.2e-6 (const) and 7.0e-6 (pixel) over every case here.
    # passes=1: the suite's bf16 bar, which checks the one-pass stage schedule only (measured at most 3.1e-3).
    tol = 2e-5 if v["passes"] == 3 else 2e-2
    err = _engine_case(launch, HW, ref, tol, n_t=_tiles_per_cta(B, HW), rgb=(rgb_w, rgb_b, rgb_in) if v["rgb"] else None)
    print(f"{style} {_vid(v)} {B}x{Hg}x{Wg}{desc}: max err / max ref {err:.2e}")


@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("v", CONST, ids=_vid)
def test_spade_conv_const(v, shape):
    _spade_case("const", v, shape, 11)


@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("v", PIXEL, ids=_vid)
def test_spade_conv_pixel(v, shape):
    _spade_case("pixel", v, shape, 12)


# ----------------------------------------------------------------------------------------------------------------------
# 2. the engine's other forward entry points
# ----------------------------------------------------------------------------------------------------------------------
def _plain_launch(call, B, T, HW):
    def launch(fill):
        obuf, out = _guarded((B, T, C, 128))
        call(fill, out)
        return dict(out=out, bufs=[obuf])
    return launch


@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("Cin", [64, 128, 256])
def test_conv1x1_blocked(Cin, shape):
    abi = _abi()
    B, Hg, Wg = _shape(shape)
    HW, T = Hg * Wg, _tiles(Hg * Wg)
    r = _rnd(20 + Cin)
    x, W, bias = r(B, Cin, HW), r(C, Cin) / 8, 0.1 * r(C)
    wimg = abi.pack_weight(W, Nb=256)[0]
    ref = torch.einsum("oc,bcp->bop", W.double(), x.double()) + bias.double()[None, :, None]
    call = lambda fill, out: abi.conv1x1_blocked(_blocked(x, fill), Cin, wimg, bias, out, B=B, Hg=Hg, Wg=Wg)
    _engine_case(_plain_launch(call, B, T, HW), HW, ref, 2e-5)


@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("act,K", [(1, 256), (1, 512), (0, 256), (0, 512)], ids=["sine-K256", "sine-K512", "lrelu-K256", "lrelu-K512"])
def test_act_conv1x1_blocked(act, K, shape):
    """out = W [act(x*g1+g0); act(x2*g1+g0)] + b, one [B,2,C] table for both sources.  Sine arguments reach |t| ~ 40 (the
    renderer's FiLM frequencies are 15 f + 30): their fp32 rounding (|t| 2^-24) and the SFU sine (2^-21 absolute after the
    2 pi reduction) perturb each operand by < 4e-6, which the 256- / 512-term sum with |W| ~ 1/16 keeps below 2e-5 of
    max|out|."""
    abi = _abi()
    B, Hg, Wg = _shape(shape)
    HW, T = Hg * Wg, _tiles(Hg * Wg)
    r = _rnd(30 + act + K)
    xs = [r(B, C, HW) for _ in range(K // C)]
    if act == 1:
        mod = torch.stack([15.0 + 5.0 * r(B, C), r(B, C)], 1).contiguous()
    else:
        mod = torch.stack([1.0 + 0.5 * r(B, C), 0.5 * r(B, C)], 1).contiguous()
    W, bias = r(C, K) / 16, 0.1 * r(C)
    wimg = abi.pack_weight(W, Nb=256)[0]
    pre = torch.cat([x.double() * mod[:, 0, :, None].double() + mod[:, 1, :, None].double() for x in xs], 1)
    y = torch.sin(pre) if act == 1 else _lrelu(pre, 0.2)
    ref = torch.einsum("oc,bcp->bop", W.double(), y) + bias.double()[None, :, None]

    def call(fill, out):
        abi.act_conv1x1_blocked(_blocked(xs[0], fill), mod, wimg, bias, out, B=B, Hg=Hg, Wg=Wg,
                                x2=_blocked(xs[1], fill) if K == 512 else None, act=act)
    _engine_case(_plain_launch(call, B, T, HW), HW, ref, 2e-5)


WIDE = {   # name -> (act, slope, tables: 0 none / 1 mod serves both sources / 2 mod + mod2, skip, stats, K)
    "lrelu0.2-mod2-skip-stats": (0, 0.2, 2, True, True, 512),
    "lrelu0.2-mod": (0, 0.2, 1, False, False, 512),
    "slope1-notable-stats": (0, 1.0, 0, False, True, 512),
    "slope1-mod2-skip": (0, 1.0, 2, True, False, 512),
    "sine-mod2-stats": (1, 0.0, 2, False, True, 512),
    "sine-mod-skip": (1, 0.0, 1, True, False, 512),
    "lrelu0.2-K256-mod-skip-stats": (0, 0.2, 1, True, True, 256),
}


@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("variant", list(WIDE))
def test_blocked_conv_wide(variant, shape):
    abi = _abi()
    act, slope, tables, use_skip, use_stats, K = WIDE[variant]
    B, Hg, Wg = _shape(shape)
    HW, T = Hg * Wg, _tiles(Hg * Wg)
    r = _rnd(40 + len(variant))
    xs = [r(B, C, HW) for _ in range(K // C)]
    g1 = (15.0 + 5.0 * r(B, C)) if act == 1 else (1.0 + 0.5 * r(B, C))
    mod = torch.stack([g1, 0.5 * r(B, C)], 1).contiguous() if tables else None
    mod2 = torch.stack([1.0 + 0.5 * r(B, C) + (14.0 if act == 1 else 0.0), 0.5 * r(B, C)], 1).contiguous() if tables == 2 else None
    W, bias = r(C, K) / 16, 0.1 * r(C)
    skip = r(B, C, HW) if use_skip else None
    wimg = abi.pack_weight(W, Nb=256)[0]
    pres = []
    for h, x in enumerate(xs):
        t = mod2 if (h == 1 and mod2 is not None) else mod
        pres.append(x.double() if t is None else x.double() * t[:, 0, :, None].double() + t[:, 1, :, None].double())
    pre = torch.cat(pres, 1)
    y = torch.sin(pre) if act == 1 else _lrelu(pre, slope)
    ref = torch.einsum("oc,bcp->bop", W.double(), y) + bias.double()[None, :, None]
    if skip is not None:
        ref = ref + skip.double()

    def launch(fill):
        obuf, out = _guarded((B, T, C, 128))
        res = dict(out=out, bufs=[obuf])
        row = None
        if use_stats:
            sbuf, row, init = _stats_row(B * HW)
            res.update(row=row, init=init)
            res["bufs"].append(sbuf)
        # the blocked inputs stay referenced until the launch has been issued (abi.ptr keeps only the address)
        xb = [_blocked(x, fill) for x in xs]
        sb = None if skip is None else _blocked(skip, fill)
        abi.call("hg_blocked_conv_wide", abi.ptr(xb[0]), abi.ptr(xb[1] if K == 512 else None), abi.ptr(mod), abi.ptr(mod2), act,
                 float(slope), abi.ptr(wimg), abi.ptr(bias), abi.ptr(sb), abi.ptr(out), abi.ptr(row), None, None, None, None,
                 B, Hg, Wg, 3, abi.stream())
        return res
    # sine operands: the bar argument of test_act_conv1x1_blocked
    _engine_case(launch, HW, ref, 2e-5, n_t=_tiles_per_cta(B, HW))


@pytest.mark.parametrize("shape", ["lt64", "multi"])
def test_blocked_conv_wide_rgb_chain(shape):
    """The two-half ToRGB chain exactly as wide_ops.wide_layer issues it: the first half adds rgb_b and rgb_in, the second
    half accumulates onto the first half's rgb_out with a zero bias."""
    abi = _abi()
    wo = importlib.import_module("3dhumangan_b200.modules.wide_ops")
    B, Hg, Wg = _shape(shape)
    HW = Hg * Wg
    r = _rnd(50)
    xs = [r(B, C, HW) for _ in range(2)]
    mods = [torch.stack([1.0 + 0.5 * r(B, C), 0.5 * r(B, C)], 1).contiguous() for _ in range(2)]
    W512, b512 = r(512, 512) / 22, 0.1 * r(512)
    rgb_w, rgb_b, rgb_in = r(3, 512) / 22, r(3), r(B, 3, HW)
    b0, out0 = _guarded((B, 3, HW))
    b1, out1 = _guarded((B, 3, HW))
    outs = wo.wide_layer(tuple(_blocked(x, float("nan")) for x in xs), W512, b512, mods=mods,
                         rgb=dict(w=rgb_w, b=rgb_b, rgb_in=rgb_in, out0=out0, out1=out1), B=B, Hg=Hg, Wg=Wg, passes=3)
    torch.cuda.synchronize()
    assert _intact(b0) and _intact(b1)
    y = torch.cat([_lrelu(x.double() * m[:, 0, :, None].double() + m[:, 1, :, None].double(), 0.2) for x, m in zip(xs, mods)], 1)
    ref = torch.einsum("oc,bcp->bop", W512.double(), y) + b512.double()[None, :, None]
    for oh in (0, 1):
        assert _rel_max(_planar(outs[oh], HW), ref[:, oh * C:(oh + 1) * C]) < 2e-5
    _check_rgb(out0, _planar(outs[0], HW), rgb_w[:, :C], rgb_b, rgb_in)
    _check_rgb(out1, _planar(outs[1], HW), rgb_w[:, C:], torch.zeros_like(rgb_b), out0)


# ----------------------------------------------------------------------------------------------------------------------
# 3. pixel-style helpers and table producers
# ----------------------------------------------------------------------------------------------------------------------
RATIOS = ["1", "int", "40:7", "512:96"]


def _p_slice(r, B, Rh, Rw):
    """A column slice (the third of five) of a [B*Rh*Rw, 640] projection, as synthesis_ops._spade passes it."""
    p_all = 0.7 * r(B * Rh * Rw, 640)
    return p_all, 256, p_all[:, 256:384]


@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("ratio", RATIOS)
def test_spade_a1(ratio, shape):
    """A1 = relu(bilinear_up(P) + p_bias) in the tile-blocked layout [B,T,128,128], zero in the padding rows.
    Bound: the source index scale (dst + 0.5) - 0.5 is formed in fp32 (scale = R / H rounded too), so each lerp weight is
    off by at most 3 u (R + 1); the lerp itself is 6 roundings and the bias add one more:
    |err| <= u (7 + 12 (R + 1)) (max|P| + max|p_bias|)."""
    abi = _abi()
    so = importlib.import_module("3dhumangan_b200.modules.synthesis_ops")
    B, Hg, Wg = _shape(shape)
    HW, T = Hg * Wg, _tiles(Hg * Wg)
    Rh, Rw = _render_size(ratio, Hg, Wg)
    r = _rnd(60)
    p_all, off, P = _p_slice(r, B, Rh, Rw)
    p_bias = (0.3 * r(B, 128)).contiguous()
    buf, a1 = _guarded((B, T, 128, 128))
    abi.spade_a1(so._PtrView(p_all[:, off:]), p_all.shape[1], p_bias, a1, B=B, Hg=Hg, Wg=Wg, Rh=Rh, Rw=Rw)
    torch.cuda.synchronize()
    assert _intact(buf)
    up = F.interpolate(P.double().reshape(B, Rh, Rw, 128).permute(0, 3, 1, 2), (Hg, Wg), mode="bilinear", align_corners=False)
    ref = torch.relu(up.reshape(B, 128, HW) + p_bias.double()[:, :, None])
    bound = U * (7 + 12 * (max(Rh, Rw) + 1)) * (P.abs().max() + p_bias.abs().max()).item()
    err = (_planar(a1, HW).double() - ref).abs().max().item()
    assert err <= bound, (err, bound)
    assert (a1.permute(0, 2, 1, 3).reshape(B, 128, T * 128)[:, :, HW:] == 0).all()


@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("ratio", RATIOS)
def test_bilinear_adjoint(ratio, shape):
    """dP = adjoint of the bilinear up-sample applied to dA1 [B,HW,128] (pixel-major), written into a column slice of a
    wider buffer: against fp64 autograd of F.interpolate, and the identity <up(P), D> = <P, adj(D)>.
    Bound: a texel sums at most n = (ceil(H/R) + 3) (ceil(W/R) + 3) weighted terms by fp32 fmas, each weight a product of
    two lerp weights off by at most 3 u (R + 1):  |err| <= u ((n + 2) adj(|D|) + 6 (R + 1) n max|D|)."""
    abi = _abi()
    so = importlib.import_module("3dhumangan_b200.modules.synthesis_ops")
    B, Hg, Wg = _shape(shape)
    HW = Hg * Wg
    Rh, Rw = _render_size(ratio, Hg, Wg)
    r = _rnd(70)
    D = r(B, HW, 128)
    buf, dp = _guarded((B * Rh * Rw, 640), fill=7.0)
    abi.bilinear_adjoint(D, so._PtrView(dp[:, 256:]), dp.shape[1], B=B, Hg=Hg, Wg=Wg, Rh=Rh, Rw=Rw)
    torch.cuda.synchronize()
    assert _intact(buf)
    assert (dp[:, :256] == 7.0).all() and (dp[:, 384:] == 7.0).all(), "columns outside the slice were written"
    got = dp[:, 256:384].double().reshape(B, Rh, Rw, 128)

    def adj(d):
        P = torch.zeros(B, 128, Rh, Rw, dtype=torch.float64, device="cuda", requires_grad=True)
        up = F.interpolate(P, (Hg, Wg), mode="bilinear", align_corners=False)
        (up * d.double().permute(0, 2, 1).reshape(B, 128, Hg, Wg)).sum().backward()
        return P.grad.permute(0, 2, 3, 1)
    ref, mag = adj(D), adj(D.abs())
    n = (-(-Hg // Rh) + 3) * (-(-Wg // Rw) + 3)
    bound = U * ((n + 2) * mag + 6 * (max(Rh, Rw) + 1) * n * D.abs().max().item())
    assert ((got - ref).abs() <= bound).all(), float(((got - ref).abs() / bound).max())
    # adjoint identity in fp64 from the kernel's fp32 output
    P = r(B, 128, Rh, Rw).double()
    lhs = (F.interpolate(P, (Hg, Wg), mode="bilinear", align_corners=False).reshape(B, 128, HW) * D.double().permute(0, 2, 1)).sum()
    rhs = (P.permute(0, 2, 3, 1) * got).sum()
    scale = (P.abs().permute(0, 2, 3, 1) * got.abs()).sum()
    assert abs(lhs - rhs) / scale < 1e-6, float(abs(lhs - rhs) / scale)


def _pixel_mod_inputs(shape, xshared, seed):
    B, Hg, Wg = _shape(shape)
    HW = Hg * Wg
    r = _rnd(seed)
    x = r(1 if xshared else B, C, HW)
    scsh = torch.stack([1.0 + 0.3 * r(C), 0.3 * r(C)]).contiguous()
    gam, bet = 1.0 + 0.3 * r(B, C, HW), 0.5 * r(B, C, HW)
    return B, Hg, Wg, HW, x, scsh, gam, bet


@pytest.mark.parametrize("xshared", [False, True], ids=["xfull", "xshared"])
@pytest.mark.parametrize("shape", SHAPES)
def test_spade_pixel_pre(shape, xshared):
    """pre = (x*sc + sh)*gam + bet over bet (synthesis_train.py, rebuilding the pixel-style pre-activation).
    Bound: two fmas, |err| <= 2 u (|x sc + sh| |gam| + |bet|) + u |x sc| |gam|."""
    abi = _abi()
    B, Hg, Wg, HW, x, scsh, gam, bet = _pixel_mod_inputs(shape, xshared, 80)
    T = _tiles(HW)
    xb = _blocked(x, float("nan"))
    buf, pre = _guarded((B, T, C, 128))
    pre.copy_(_blocked(bet, float("nan")))
    abi.spade_pixel_pre(xb, 0 if xshared else T * C * 128, scsh, _blocked(gam, float("nan")), pre, B=B, Hg=Hg, Wg=Wg)
    torch.cuda.synchronize()
    assert _intact(buf)
    xs = x.double().expand(B, C, HW) * scsh[0, None, :, None].double()
    xn = xs + scsh[1, None, :, None].double()
    ref = xn * gam.double() + bet.double()
    bound = 2 * U * (xn.abs() * gam.double().abs() + bet.double().abs()) + U * xs.abs() * gam.double().abs()
    assert ((_planar(pre, HW).double() - ref).abs() <= bound).all()


@pytest.mark.parametrize("xshared", [False, True], ids=["xfull", "xshared"])
@pytest.mark.parametrize("shape", SHAPES)
def test_spade_pixel_mod_bwd(shape, xshared):
    """dxn = dpre*gam (over pre), dgam = dpre*(x*sc + sh) (over gam), and per channel sums[0] += sum dxn*x, sums[1] +=
    sum dxn, sums[2] += sum dgam over the valid pixels (synthesis_train.py: d sc = sum dxn*x, d sh = sum dxn, and the
    gamma-bias gradient).  The padding rows of every input hold NaN, as the unwritten rows of the buffers the backward
    passes here do.  Bound of the sums: each lane adds its 4 pixels (3 adds), 5 shuffle steps fold the warp, the block's
    fp32 shared sum takes one add per tile it walks (n_t), then fp64: |err| <= (9 + n_t) u sum|term|, plus u per product."""
    abi = _abi()
    B, Hg, Wg, HW, x, scsh, gam, bet = _pixel_mod_inputs(shape, xshared, 90)
    T = _tiles(HW)
    dpre = _rnd(91)(B, C, HW)
    bg, gam_dgam = _guarded((B, T, C, 128))
    gam_dgam.copy_(_blocked(gam, float("nan")))
    bd, dxn = _guarded((B, T, C, 128))
    dxn.copy_(_blocked(bet, float("nan")))
    bs, sums = _guarded((3, C), torch.float64, 0.0)
    init = 10.0 * _rnd(92)(3, C).double()
    sums.copy_(init)
    abi.spade_pixel_mod_bwd(_blocked(dpre, float("nan")), _blocked(x, float("nan")), 0 if xshared else T * C * 128, scsh, gam_dgam,
                            dxn, sums, B=B, Hg=Hg, Wg=Wg)
    torch.cuda.synchronize()
    assert _intact(bg) and _intact(bd) and _intact(bs)
    xd = x.double().expand(B, C, HW)
    xn = xd * scsh[0, None, :, None].double() + scsh[1, None, :, None].double()
    r_dxn = dpre.double() * gam.double()
    r_dg = dpre.double() * xn
    assert ((_planar(dxn, HW).double() - r_dxn).abs() <= U * r_dxn.abs()).all()
    xs_abs = (xd * scsh[0, None, :, None].double()).abs()
    assert ((_planar(gam_dgam, HW).double() - r_dg).abs() <= 3 * U * (dpre.double().abs() * xs_abs + r_dg.abs())).all()
    assert torch.isfinite(sums).all(), "padding rows reached the sums"
    for t in (dxn, gam_dgam):
        assert (t.permute(0, 2, 1, 3).reshape(B, C, T * 128)[:, :, HW:] == 0).all(), "dxn / dgam are zero past the image"
    n_t = -(-B * T // min(B * T, 4 * _nsm()))
    k = (10 + n_t) * U
    for i, t in enumerate((r_dxn * xd, r_dxn, r_dg)):
        err = (sums[i] - init[i] - t.sum((0, 2))).abs()
        assert (err <= k * t.abs().sum((0, 2)) + 1e-13 * init[i].abs()).all(), (i, float(err.max()))


@pytest.mark.parametrize("mode,fold", [("train", "scsh"), ("train", "mod"), ("eval", "scsh"), ("eval", "mod")])
def test_bn_finalize(mode, fold):
    """Against fp64 BatchNorm semantics (nn.SyncBatchNorm on one process = F.batch_norm): train mode normalises with the
    batch mean and biased variance and moves the running buffers by momentum 0.1 towards the mean and the UNBIASED
    variance; the count comes from the row's device slot [512] (the host count is 0).  Eval mode normalises with the
    running buffers and leaves them untouched.  Const style folds (1 + gamma, beta) into the per-sample [B,2,C] table.
    Bound: mean / var are rounded to fp32 (u each), rsqrtf is within 2 ulp, then a product and an fma:
    |err| <= 16 u (sum of the magnitudes of the terms)."""
    abi = _abi()
    train = mode == "train"
    r = _rnd(100)
    n = 3000
    data = (0.5 * r(C) + (1.0 + 0.5 * r(C).abs()) * r(n, C)).double()             # per-channel mean and spread
    w, b = 1.0 + 0.2 * r(C), 0.2 * r(C)
    rm, rv = 0.3 * r(C), 1.0 + 0.5 * r(C).abs()
    B = 3
    gb = torch.stack([1.0 + 0.3 * r(B, C), 0.3 * r(B, C)], 1).contiguous() if fold == "mod" else None
    sbuf, row = _guarded((STAT_STRIDE,), torch.float64, 0.0)
    row[:C], row[C:2 * C], row[512] = data.sum(0), (data * data).sum(0), float(n)
    rm_k, rv_k = rm.clone(), rv.clone()
    bo, out = _guarded((B, 2, C) if fold == "mod" else (2, C))
    abi.bn_finalize(row if train else None, w, b, rm_k, rv_k, train, count_dev=row[512:513] if train else None, gb=gb, B=B,
                    scsh=out if fold == "scsh" else None, mod=out if fold == "mod" else None)
    torch.cuda.synchronize()
    assert _intact(sbuf) and _intact(bo)
    rm64, rv64 = rm.double(), rv.double()
    y = F.batch_norm(data, rm64, rv64, w.double(), b.double(), training=train, momentum=0.1, eps=1e-5)
    mean = data.mean(0) if train else rm.double()
    var = data.var(0, unbiased=False) if train else rv.double()
    sc = w.double() / torch.sqrt(var + 1e-5)
    sh = b.double() - mean * sc
    # the folded scale / shift reproduce BatchNorm's output
    assert (y - (data * sc + sh)).abs().max() < 1e-12 * y.abs().max()
    tol = 16 * U
    if fold == "scsh":
        assert ((out[0].double() - sc).abs() <= tol * sc.abs()).all()
        assert ((out[1].double() - sh).abs() <= tol * (b.double().abs() + (mean * sc).abs())).all()
    else:
        Gm, Bt = gb[:, 0].double(), gb[:, 1].double()
        assert ((out[:, 0].double() - sc * Gm).abs() <= tol * (sc * Gm).abs()).all()
        mag = (b.double().abs() + (mean * sc).abs()) * Gm.abs() + Bt.abs()
        assert ((out[:, 1].double() - (sh * Gm + Bt)).abs() <= tol * mag).all()
    if train:
        assert ((rm_k.double() - rm64).abs() <= 4 * U * (rm.double().abs() + mean.abs())).all()
        assert ((rv_k.double() - rv64).abs() <= tol * (rv.double().abs() + var.abs())).all()
    else:
        assert torch.equal(rm_k, rm) and torch.equal(rv_k, rv)


@pytest.mark.parametrize("shape", SHAPES)
def test_synth_input(shape):
    """x0 = sin(w0 i + w1 j + b) on the linspace(-1, 1) grid, tile-blocked [T,C,128] and shared by the batch, and its
    statistics multiplied by the batch size added to a pre-filled row.  Bound of x0: two fmas on |t| <= |w0| + |w1| + |b|
    and sinf (2 ulp): |err| <= 4 u (|w0| + |w1| + |b|) + 2 u.  Bound of the sums: a thread adds ceil(HW / (256 gx))
    values (gx <= 32 blocks per channel), 5 shuffle steps and 8 warp totals follow in fp32, then fp64:
    |err| <= (HW / 256 + 16) u B sum|term|."""
    abi = _abi()
    B, Hg, Wg = _shape(shape)
    HW, T = Hg * Wg, _tiles(Hg * Wg)
    r = _rnd(110)
    w, bias = r(C, 2), 0.5 * r(C)
    ic, jc = torch.linspace(-1, 1, Hg, device="cuda"), torch.linspace(-1, 1, Wg, device="cuda")
    xbuf, x0 = _guarded((T, C, 128))
    sbuf, row, init = _stats_row(B * HW)
    abi.synth_input(w, bias, ic, jc, x0, row, B)
    torch.cuda.synchronize()
    assert _intact(xbuf) and _intact(sbuf)
    t = w[:, 0, None, None].double() * ic.double()[None, :, None] + w[:, 1, None, None].double() * jc.double()[None, None, :]
    ref = torch.sin(t + bias.double()[:, None, None]).reshape(C, HW)
    got = _planar(x0[None], HW)[0].double()
    bound = 4 * U * (w.abs().sum(1) + bias.abs()).double()[:, None] + 2 * U
    assert ((got - ref).abs() <= bound).all()
    k = (HW / 256 + 16) * U * B
    for i, v in enumerate((got, got * got)):
        err = (row[i * C:(i + 1) * C] - init[i * C:(i + 1) * C] - B * v.sum(1)).abs()
        assert (err <= k * v.abs().sum(1) + 1e-13 * init[i * C:(i + 1) * C].abs()).all()
    assert torch.equal(row[512:], init[512:])


# ----------------------------------------------------------------------------------------------------------------------
# 4. the C2 launch: B = 8, 512x512, render 96x96, p_stride 768 ('mixed' mode: six pixel-style half-blocks)
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["pixel-stats-xshared", "const-stats-rgb", "const-skip-rgb-stats"])
def test_c2_launch(kind):
    """One launch of each class tools/spade_bench.py times, at C2 size, where each CTA folds ~124 tiles into fp32 shared
    sums.  Statistics and rgb_out are checked in full against fp64 from the kernel's own out; the variance a BatchNorm
    derives from the row (sumsq/n - mean^2) is held to 1e-4 relative, ten times inside the 1e-3 image contract the
    normalisation feeds; out is checked against fp64 from the inputs at every CTA's first and last tile under the
    grid = min(tiles, SMs) mapping and at a seeded random set of pixels."""
    abi = _abi()
    so = importlib.import_module("3dhumangan_b200.modules.synthesis_ops")
    B, Hg, Wg, Rh, Rw = 8, 512, 512, 96, 96
    HW, T = Hg * Wg, _tiles(Hg * Wg)
    pixel = kind.startswith("pixel")
    xshared = "xshared" in kind
    r = _rnd(120)
    x = r(1 if xshared else B, T, C, 128)                    # tile-blocked; HW is a multiple of 128: no padding
    W = r(C, C)
    inv_sigma = (1.0 / torch.linalg.matrix_norm(W.double(), 2)).float().reshape(1)
    wimg = abi.pack_weight(W, Nb=256, scale_dev=inv_sigma)[0]
    bias = 0.1 * r(C)
    kw = {}
    if pixel:
        p_all = 0.7 * r(B * Rh * Rw, 768)
        p_bias = (0.3 * r(B, 128)).contiguous()
        scsh = torch.stack([1.0 + 0.3 * r(C), 0.3 * r(C)]).contiguous()
        wg, wb, bg, bb = r(C, 128) / 16, r(C, 128) / 16, 0.1 * r(C), 0.1 * r(C)
        w_il, b_il = so._gamma_beta_interleaved(wg, bg, wb, bb)
        kw.update(scsh=scsh, p_lr=so._PtrView(p_all[:, 256:]), p_stride=768, p_bias=p_bias, wgb=abi.pack_weight(w_il, Nb=256)[0],
                  bgb=b_il, Rh=Rh, Rw=Rw)
    else:
        mod = torch.stack([1.0 + 0.5 * r(B, C), 0.5 * r(B, C)], 1).contiguous()
        kw.update(mod=mod)
    skip = r(B, T, C, 128) if "skip" in kind else None
    if "rgb" in kind:
        rgb_w, rgb_b, rgb_in = r(3, C) / 16, r(3), r(B, 3, HW)
        kw.update(rgb_w=rgb_w, rgb_b=rgb_b, rgb_in=rgb_in, rgb_out=torch.empty(B, 3, HW, device="cuda"))
    row = torch.zeros(STAT_STRIDE, dtype=torch.float64, device="cuda")
    row[512] = float(B * HW)
    out = torch.empty(B, T, C, 128, device="cuda")
    abi.spade_conv(x, 0 if xshared else T * C * 128, wimg, bias, out, B=B, Hg=Hg, Wg=Wg, skip=skip, stats=row, **kw)
    torch.cuda.synchronize()

    # statistics and ToRGB from the kernel's own out, in full
    n = B * HW
    n_t = _tiles_per_cta(B, HW)
    s1 = torch.zeros(C, dtype=torch.float64, device="cuda")
    s2, a1 = torch.zeros_like(s1), torch.zeros_like(s1)
    for b in range(B):
        o = out[b].double()
        s1 += o.sum((0, 2))
        s2 += (o * o).sum((0, 2))
        a1 += o.abs().sum((0, 2))
    k = (4 + 8 * n_t) * U
    assert ((row[:C] - s1).abs() <= k * a1).all()
    assert ((row[C:2 * C] - s2).abs() <= k * s2).all()
    mean = s1 / n
    var = torch.zeros_like(s1)
    for b in range(B):
        var += ((out[b].double() - mean[None, :, None]) ** 2).sum((0, 2))
    var /= n
    var_k = row[C:2 * C] / n - (row[:C] / n) ** 2
    verr = ((var_k - var).abs() / var).max().item()
    print(f"C2 {kind}: {n_t} tiles per CTA, derived-variance error {verr:.2e}")
    assert verr < 1e-4, verr
    if "rgb" in kind:
        for b in range(B):
            _check_rgb(kw["rgb_out"][b:b + 1], _planar(out[b:b + 1], HW), rgb_w, rgb_b, rgb_in[b:b + 1])

    # out from the inputs at sampled pixels: every CTA's first and last tile, plus random pixels
    tiles = B * T
    grid = min(tiles, _nsm())
    first = torch.arange(grid)
    last = first + (torch.div(tiles - first + grid - 1, grid, rounding_mode="floor") - 1) * grid
    sel = torch.cat([first, last]).unique()
    pix = (sel[:, None] * 128 + torch.arange(128)[None, :]).reshape(-1)
    pix = torch.cat([pix, torch.randint(0, tiles * 128, (4096,), generator=torch.Generator().manual_seed(121))]).unique().cuda()
    b_i, p_i = pix // HW, pix % HW                              # global pixel -> (sample, pixel)
    t_i, r_i = p_i // 128, p_i % 128
    xv = (x[0, t_i, :, r_i] if xshared else x[b_i, t_i, :, r_i]).double()                              # [n, C]
    if pixel:
        a1s = torch.empty(pix.numel(), 128, dtype=torch.float64, device="cuda")
        for b in range(B):
            m = b_i == b
            P = p_all[b * Rh * Rw:(b + 1) * Rh * Rw, 256:384].double().reshape(1, Rh, Rw, 128).permute(0, 3, 1, 2)
            up = F.interpolate(P, (Hg, Wg), mode="bilinear", align_corners=False).reshape(128, HW)
            a1s[m] = torch.relu(up[:, p_i[m]].t() + p_bias[b].double())
        gam = 1.0 + a1s @ wg.double().t() + bg.double()
        bet = a1s @ wb.double().t() + bb.double()
        pre = (xv * scsh[0].double() + scsh[1].double()) * gam + bet
    else:
        pre = xv * mod[b_i, 0].double() + mod[b_i, 1].double()
    ref = _lrelu(pre, 0.2) @ (W.double() * inv_sigma.double()).t() + bias.double()
    if skip is not None:
        ref = ref + skip[b_i, t_i, :, r_i].double()
    got = out[b_i, t_i, :, r_i].double()
    err = _rel_max(got, ref)
    print(f"C2 {kind}: sampled out max err / max ref {err:.2e} over {pix.numel()} pixels")
    assert err < 2e-5, err
