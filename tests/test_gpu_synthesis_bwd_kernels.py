"""The SPADE half-blocks' backward kernels launch by launch against fp64, in exactly the call forms
`modules/synthesis_train.py::synthesis_backward` issues:

    hg_spade_bwd_dgrad       (csrc/synth.cu, kBwd)   dpre = (W^T dout) * lrelu'(x*g1 + g0); S1 += sum dpre, S2 += sum dpre*x
    hg_conv1x1_blocked_bwd   (csrc/synth.cu, kBwd)   the same over K = 512 (two output halves), on the rebuilt pixel-style
                                                     `pre`, and the gamma/beta MLP's dA1 (Cout 128, pixel-major, ReLU mask)
    hg_wgrad_blocked         (csrc/synth_bwd.cu)     dW = sum dout (x) lrelu(x*g1 + g0), dbias = sum dout
    hg_spade_bwd_combine     (csrc/synth_bwd.cu)     dx = dpre*g1 + a + k*x (+ dskip) (+ W_rgb^T drgb); dW_rgb += drgb . x^T
    hg_synth_input_bwd       (csrc/synth_bwd.cu)     the synthesis input's weight and bias gradients

Every launch is checked five ways, as tests/test_gpu_spade_conv.py checks the forward:
  1. valid outputs against the fp64 formula of the kernel's contract, componentwise: |err| <= bound * sum |a||b| over the
     terms of each output (the LeakyReLU / ReLU masks are reproduced exactly: the kernel forms pre with one fmaf, whose sign
     is the sign of the exact x*g1 + g0, which fp64 evaluates with one rounding that keeps the sign);
  2. the epilogue sums (dgrad's S1 / S2, combine's dW_rgb) against fp64 sums of the kernel's own output;
  3. the padding rows of every input hold NaN in one launch and zeros in another: valid outputs are bit-identical, dx is
     exactly 0 past the image and every sum stays finite;
  4. every output lives inside a larger buffer whose guard elements must be untouched;
  5. a repeated launch gives bit-identical outputs (dgrad's sums, whose CTA totals are fp32 shared-memory atomics, only within
     their bound; dW_rgb, fp64 atomics of fixed per-CTA totals, within fp64 rounding).
Shapes run from one ragged tile to `walk`, where every persistent CTA walks >= 16 tiles across sample boundaries, and one
launch per kernel at the C2 bench size (B = 8, 512x512: 124 tiles per CTA on 132 SMs); the weight gradient also at the
MAP3DBN512 single-GPU batch (B = 32, 512x256: 248 tiles per CTA).  A drift check records the launches of
synthesis_backward on small networks and fails on any call form the matrices below do not hold."""
import importlib
import itertools
import math

import pytest
import torch

from blocked_util import C, SHAPES, U, _blocked, _guarded, _intact, _nsm, _pairwise, _planar, _shape, _sums_bound, _tiles

gpu = pytest.mark.gpu
ALL_SHAPES = SHAPES + ["walk"]

# Componentwise GEMM bound: |err| <= A_p (S_p + sqrt(K) u) sum_k |a_k||b_k|, where S_p is the operand split's relative error
# per product (bf16x3: the dropped lo*lo product and the two lo roundings, ~2^-17; one bf16 pass: 2^-8), K the length of the
# fp32 accumulation and A_p a margin.  The fp32 accumulation error grows like sqrt(K) u on random data (the worst case K u is
# ~100x looser at the weight gradient's K = 8 192).  Measured on an H100 80GB HBM3 (700 W) over every case here, the worst ratio
# of |err| to (S_p + sqrt(K) u) sum|a||b| was 0.44 with bf16x3 operands (weight gradient; data gradients 0.35) and 0.46 with one
# bf16 pass: A_p = 1.5 puts the bound 3.3-4.5x above it.
SPLIT = {3: 2.0 ** -17, 1: 2.0 ** -8}
A_GEMM = {3: 1.5, 1: 1.5}
# csrc/synth_bwd.cu kWgFoldTiles: the weight gradient's register accumulator sums at most this many tiles of 128 pixels before
# it is added to the CTA's fp32 partial
WGRAD_FOLD = 64
# The weight gradient's bar, the one the discriminator's weight gradient holds (tests/test_gpu_discriminator_bwd.py).
WGRAD_L2, WGRAD_MAX = {3: 5e-5, 1: 2e-2}, {3: 2e-4, 1: 5e-2}


def _abi():
    return importlib.import_module("3dhumangan_b200.abi")


def _rnd(seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return lambda *s: torch.randn(*s, generator=g, device="cuda")


def _gemm_bound(mag, K, passes):
    return A_GEMM[passes] * (SPLIT[passes] + math.sqrt(K) * U) * mag


def _check(name, err, bound):
    ratio = (err / bound).max().item()
    print(f"  {name}: {ratio:.3f} of the bound")
    assert ratio <= 1.0, f"{name}: error {ratio:.3f}x the bound"
    return ratio


def _grid(B, HW, per_sm=1):
    tiles = B * _tiles(HW)
    return min(tiles, per_sm * _nsm())


def _n_t(B, HW, per_sm=1):
    """Tiles per CTA of a persistent launch over B * T tiles."""
    tiles = B * _tiles(HW)
    return -(-tiles // _grid(B, HW, per_sm))


def _n_t_sample(B, HW):
    """Tiles a CTA of a grid-min(tiles, SMs) launch walks inside one sample between two flushes of its per-sample sums."""
    return -(-_tiles(HW) // _grid(B, HW))


def _runs(launch):
    """launch(fill) three times: padding NaN, zeros, zeros again."""
    runs = [launch(float("nan")), launch(0.0), launch(0.0)]
    torch.cuda.synchronize()
    for r in runs:
        assert all(_intact(b) for b in r["bufs"]), "a guard element was overwritten"
    return runs


def _same(runs, key, view=lambda t: t):
    a, b, c = (view(r[key]) for r in runs)
    assert torch.equal(a, b), f"NaN in the padding rows changed {key}"
    assert torch.equal(b, c), f"a repeated launch changed {key}"


def _check_sums(runs, key, refs, n_t, what):
    """fp64-atomic per-(sample, channel) sums: each run's increments against fp64 sums of the kernel's own output
    (refs: list over runs of (ref, mag) per sum row), and the runs within fp64 rounding of each other."""
    for r, rr in zip(runs, refs):
        got = r[key] - r["init"]
        assert torch.isfinite(r[key]).all(), f"NaN padding reached {what}"
        for k, (ref, mag) in enumerate(rr):
            err = (got[:, k] - ref).abs()
            _check(f"{what}[{k}]", err, _sums_bound(n_t) * mag + 1e-13 * r["init"][:, k].abs() + 1e-300)


def _lrelu(v, slope):
    return torch.where(v > 0, v, slope * v)


def _mask(pre, slope):
    return torch.where(pre > 0, 1.0, slope)


# ----------------------------------------------------------------------------------------------------------------------
# the matrix: the call forms of synthesis_backward
# ----------------------------------------------------------------------------------------------------------------------
# :394, the only data-gradient entry point that reads a batch-shared input (block 0 at hidden_dim 256)
DGRAD = [dict(xshared=xs, passes=p) for xs in (0, 1) for p in (3, 1)]
# :396 const style over two output halves; :353 pixel style on the rebuilt `pre` (no table, one or two halves); :370 the
# gamma/beta MLP's dA1 (Cout 128, pixel-major, ReLU mask, K = 512 of [dgam | dpre])
CONV_BWD = [dict(form=f, g2=g2, passes=p) for f, g2s in (("const", (1,)), ("pixel", (0, 1)), ("gb", (1,))) for g2 in g2s
            for p in (3, 1)]
CONV_FORMS = {   # form -> (mod table, Cout, slope, pixel-major)
    "const": (True, 256, 0.2, False),
    "pixel": (False, 256, 0.2, False),
    "gb": (False, 128, 0.0, True),
}
# :298 / :377: const (table, Cx 256, x batch-shared or not), the pixel-style conv on `pre` (no table), the gamma/beta MLP
# (Cx 128 on A1, x_bstride = T*128*128); each with and without the bias gradient
WGRAD = [dict(kind=k, xshared=xs, bias=bi, passes=p) for k, xss in (("const", (0, 1)), ("pixel", (0,)), ("gb", (0,)))
         for xs in xss for bi in (1, 0) for p in (3, 1)]
# :323 / :423, pairwise; g1 is a per-sample [B,2,C] table (const style) or the pixel-style BatchNorm scale expanded to one;
# rgb 1: the ToRGB weight gradient is accumulated, 2: the ToRGB weight is frozen (drgb without dwrgb)
COMBINE_LEVELS = dict(dpre=(1, 0), ak=(1, 0), dskip=(1, 0), rgb=(0, 1, 2), xshared=(0, 1), g1=("sample", "pixel"))
COMBINE = _pairwise(COMBINE_LEVELS)


def _vid(v):
    return "-".join(f"{k}{v[k]}" for k in v)


def test_combine_rows_cover_every_option_pair():
    """The combine matrix holds every pair of values of every two options (pure Python)."""
    names = list(COMBINE_LEVELS)
    for a, b in itertools.combinations(names, 2):
        for va in COMBINE_LEVELS[a]:
            for vb in COMBINE_LEVELS[b]:
                assert any(r[a] == va and r[b] == vb for r in COMBINE), (a, va, b, vb)
    assert len(COMBINE) < math.prod(len(v) for v in COMBINE_LEVELS.values())


# ----------------------------------------------------------------------------------------------------------------------
# 1. hg_spade_bwd_dgrad and hg_conv1x1_blocked_bwd
# ----------------------------------------------------------------------------------------------------------------------
def _dgrad_inputs(r, B, HW, K, cout, table, xshared, aux_relu=False):
    """Incoming gradient [B,K,HW], forward input [1 or B,cout,HW], forward weight [K,256] (columns past cout zero), table."""
    dout = r(B, K, HW)
    x = r(1 if xshared else B, cout, HW)
    if aux_relu:
        x = torch.relu(x)                                          # A1 = relu(...): exact zeros where the mask is 0
    W = r(K, 256) / 16
    W[:, cout:] = 0
    mod = torch.stack([1.0 + 0.5 * r(B, cout), 0.5 * r(B, cout)], 1).contiguous() if table else None
    return dout, x, W, mod


def _dgrad_ref(dout, x, W, mod, slope, B, cout):
    xd = x.double().expand(B, -1, -1)
    pre = xd if mod is None else xd * mod[:, 0, :, None].double() + mod[:, 1, :, None].double()
    m = _mask(pre, slope)
    Wd = W[:, :cout].double()
    ref = torch.einsum("oc,bop->bcp", Wd, dout.double()) * m
    mag = torch.einsum("oc,bop->bcp", Wd.abs(), dout.double().abs()) * m
    return ref, mag


def _dgrad_case(kernel, v, B, Hg, Wg, seed):
    abi = _abi()
    HW, T = Hg * Wg, _tiles(Hg * Wg)
    passes = v["passes"]
    if kernel == "dgrad":
        table, cout, slope, pm, K, xshared = True, 256, 0.2, False, 256, v["xshared"]
    else:
        (table, cout, slope, pm), K, xshared = CONV_FORMS[v["form"]], 512 if v["g2"] else 256, 0
    r = _rnd(seed)
    dout, x, W, mod = _dgrad_inputs(r, B, HW, K, cout, table, xshared, aux_relu=kernel != "dgrad" and v["form"] == "gb")
    wimg_t = abi.pack_weight(W.t().contiguous(), Nb=256)[0]
    init = 10.0 * r(B, 2, cout).double()
    ref, mag = _dgrad_ref(dout, x, W, mod, slope, B, cout)

    def launch(fill):
        obuf, out = _guarded((B, HW, cout) if pm else (B, T, cout, 128))
        sbuf, sums = _guarded((B, 2, cout), torch.float64, 0.0)
        sums.copy_(init)
        db = _blocked(dout, fill)
        xb = _blocked(x, fill)
        if kernel == "dgrad":
            abi.spade_bwd_dgrad(db, xb, 0 if xshared else T * C * 128, mod, wimg_t, out, sums, B=B, Hg=Hg, Wg=Wg, passes=passes)
        else:
            abi.conv1x1_blocked_bwd(db[:, :, :256].contiguous(), xb, wimg_t, out, sums, g2=db[:, :, 256:].contiguous() if K == 512 else None,
                                    mod=mod, Cout=cout, slope=slope, pixel_major=pm, B=B, Hg=Hg, Wg=Wg, passes=passes)
        return dict(out=out, sums=sums, init=init, bufs=[obuf, sbuf])

    planar = (lambda t: t.permute(0, 2, 1)) if pm else (lambda t: _planar(t, HW))
    runs = _runs(launch)
    _same(runs, "out", planar)
    got = planar(runs[1]["out"]).double()
    err = _check(f"{kernel} {_vid(v)} {B}x{Hg}x{Wg}: dpre", (got - ref).abs(), _gemm_bound(mag, K, passes) + 1e-300)
    xd = x.double().expand(B, -1, -1)
    refs = []
    for rr in runs:
        o = planar(rr["out"]).double()
        refs.append(((o.sum(2), o.abs().sum(2)), ((o * xd).sum(2), (o * xd).abs().sum(2))))
    _check_sums(runs, "sums", refs, _n_t_sample(B, HW), "S")
    # the CTAs' fp32 shared sums take the 8 warps' totals by shared-memory atomics in any order: a repeated launch moves the
    # sums within twice their bound, not within fp64 rounding
    a, b = runs[1]["sums"], runs[2]["sums"]
    mag_s = torch.stack([m for _, m in refs[1]], 1)
    assert ((a - b).abs() <= 2 * _sums_bound(_n_t_sample(B, HW)) * mag_s + 1e-12 * init.abs()).all(), "repeat moved the sums"
    return err


@gpu
@pytest.mark.parametrize("shape", ALL_SHAPES)
@pytest.mark.parametrize("v", DGRAD, ids=_vid)
def test_dgrad(v, shape):
    _dgrad_case("dgrad", v, *_shape(shape), 200 + v["passes"] + 2 * v["xshared"])


@gpu
@pytest.mark.parametrize("shape", ALL_SHAPES)
@pytest.mark.parametrize("v", CONV_BWD, ids=_vid)
def test_conv1x1_blocked_bwd(v, shape):
    _dgrad_case("conv", v, *_shape(shape), 210 + v["passes"] + 2 * v["g2"] + 4 * list(CONV_FORMS).index(v["form"]))


# ----------------------------------------------------------------------------------------------------------------------
# 2. hg_wgrad_blocked
# ----------------------------------------------------------------------------------------------------------------------
def _wgrad_launch(abi, dout_b, x_b, x_bstride, Cx, mod, want_bias, B, Hg, Wg, passes):
    """hg_wgrad_blocked with guarded outputs and a guarded workspace of the size the binding allocates."""
    wbuf, dw = _guarded((256, Cx))
    bbuf, db = _guarded((256,))
    ws_n = int(abi.lib().hg_spade_bwd_wgrad_workspace_bytes()) // 4
    sbuf, ws = _guarded((ws_n,))
    abi.call("hg_wgrad_blocked", abi.ptr(dout_b), abi.ptr(x_b), int(x_bstride), Cx, abi.ptr(mod), abi.ptr(dw),
             abi.ptr(db if want_bias else None), abi.ptr(ws), B, 256, Hg, Wg, passes, abi.stream())
    return dict(dw=dw, db=db, bufs=[wbuf, bbuf, sbuf])


def _wgrad_bound(mag, ref, n_t, passes):
    """K = the pixels one register accumulator sums; each fold into the partial and the fp32 rounding of the fp64 reduce add
    u |dW| at most (the partial is a sum of fold values bounded by mag)."""
    return _gemm_bound(mag, 128 * min(n_t, WGRAD_FOLD), passes) + (n_t // WGRAD_FOLD) * U * mag + U * ref.abs() + 1e-300


def _wgrad_report(tag, got, ref, passes):
    l2 = ((got - ref).norm() / ref.norm()).item()
    mx = ((got - ref).abs().max() / ref.abs().max()).item()
    print(f"  {tag}: rel-L2 {l2:.2e}, max/max {mx:.2e}")
    assert l2 < WGRAD_L2[passes] and mx < WGRAD_MAX[passes], (l2, mx)


@gpu
@pytest.mark.parametrize("shape", ALL_SHAPES)
@pytest.mark.parametrize("v", WGRAD, ids=_vid)
def test_wgrad(v, shape):
    abi = _abi()
    B, Hg, Wg = _shape(shape)
    HW, T = Hg * Wg, _tiles(Hg * Wg)
    passes = v["passes"]
    Cx = 128 if v["kind"] == "gb" else 256
    r = _rnd(300 + passes + 2 * v["xshared"] + 4 * v["bias"] + 8 * ("const", "pixel", "gb").index(v["kind"]))
    dout = r(B, C, HW)
    x = r(1 if v["xshared"] else B, Cx, HW)
    if v["kind"] == "gb":
        x = torch.relu(x)
    mod = torch.stack([1.0 + 0.5 * r(B, C), 0.5 * r(B, C)], 1).contiguous() if v["kind"] == "const" else None
    xd = x.double().expand(B, -1, -1)
    y = _lrelu(xd if mod is None else xd * mod[:, 0, :, None].double() + mod[:, 1, :, None].double(), 0.2)
    dd = dout.double()
    ref = torch.einsum("bop,bcp->oc", dd, y)
    mag = torch.einsum("bop,bcp->oc", dd.abs(), y.abs())
    db_ref, db_mag = dd.sum((0, 2)), dd.abs().sum((0, 2))
    xbs = 0 if v["xshared"] else T * Cx * 128

    def launch(fill):
        return _wgrad_launch(abi, _blocked(dout, fill), _blocked(x, fill), xbs, Cx, mod, v["bias"], B, Hg, Wg, passes)

    runs = _runs(launch)
    _same(runs, "dw")
    n_t = _n_t(B, HW)
    tag = f"wgrad {_vid(v)} {B}x{Hg}x{Wg} ({n_t} tiles per CTA)"
    got = runs[1]["dw"].double()
    _check(tag + ": dW", (got - ref).abs(), _wgrad_bound(mag, ref, n_t, passes))
    _wgrad_report(tag, got, ref, passes)
    if v["bias"]:
        _same(runs, "db")
        # a thread folds its 8 pixels per chunk (3 levels) into a running sum over 2 n_t chunks, then 3 shuffle steps; fp64
        _check(tag + ": dbias", (runs[1]["db"].double() - db_ref).abs(), (6 + 2 * n_t) * U * db_mag + U * db_ref.abs())
    else:
        assert all(torch.isnan(rr["db"]).all() for rr in runs), "dbias was written although not requested"


# ----------------------------------------------------------------------------------------------------------------------
# 3. hg_spade_bwd_combine
# ----------------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("shape", ALL_SHAPES)
@pytest.mark.parametrize("v", COMBINE, ids=_vid)
def test_combine(v, shape):
    abi = _abi()
    B, Hg, Wg = _shape(shape)
    HW, T = Hg * Wg, _tiles(Hg * Wg)
    r = _rnd(400 + COMBINE.index(v))
    x = r(1 if v["xshared"] else B, C, HW)
    dpre = r(B, C, HW) if v["dpre"] else None
    if v["g1"] == "sample":
        g1 = r(B, 2, C).contiguous()
    else:                                  # the pixel-style BatchNorm scale, expanded to the [B,2,C] table layout
        g1 = (1.0 + 0.3 * r(C))[None, None, :].expand(B, 2, C).contiguous()
    ak = r(2, C).contiguous() if v["ak"] else None
    dskip = r(B, C, HW) if v["dskip"] else None
    drgb = r(B, 3, HW) if v["rgb"] else None
    rgb_w = r(3, C).contiguous() if v["rgb"] else None
    init = 10.0 * r(3, C).double()

    xd = x.double().expand(B, C, HW)
    ref = torch.zeros(B, C, HW, dtype=torch.float64, device="cuda")
    mag = torch.zeros_like(ref)
    if dpre is not None:
        t = dpre.double() * g1[:, 0, :, None].double()
        ref, mag = ref + t, mag + t.abs()
    if ak is not None:
        a, k = ak[0, None, :, None].double(), ak[1, None, :, None].double()
        ref, mag = ref + a + k * xd, mag + a.abs() + (k * xd).abs()
    if dskip is not None:
        ref, mag = ref + dskip.double(), mag + dskip.double().abs()
    if drgb is not None:
        ref = ref + torch.einsum("jc,bjp->bcp", rgb_w.double(), drgb.double())
        mag = mag + torch.einsum("jc,bjp->bcp", rgb_w.double().abs(), drgb.double().abs())

    def launch(fill):
        obuf, dx = _guarded((B, T, C, 128))
        res = dict(dx=dx, bufs=[obuf])
        dwrgb = None
        if v["rgb"] == 1:
            wbuf, dwrgb = _guarded((3, C), torch.float64, 0.0)
            dwrgb.copy_(init)
            res.update(dwrgb=dwrgb, init=init)
            res["bufs"].append(wbuf)
        abi.spade_bwd_combine(dx, B=B, Hg=Hg, Wg=Wg, dpre=None if dpre is None else _blocked(dpre, fill), x=_blocked(x, fill),
                              x_bstride=0 if v["xshared"] else T * C * 128, g1=g1 if dpre is not None else None, ak=ak,
                              dskip=None if dskip is None else _blocked(dskip, fill), drgb=drgb, rgb_w=rgb_w, dwrgb=dwrgb)
        return res

    runs = _runs(launch)
    for rr in runs:
        pad = rr["dx"].permute(0, 2, 1, 3).reshape(B, C, T * 128)[:, :, HW:]
        assert torch.isfinite(pad).all() and (pad == 0).all(), "dx is not exactly 0 past the image"
    _same(runs, "dx")
    got = _planar(runs[1]["dx"], HW).double()
    # dpre*g1 (1 rounding), + fmaf(k, x, a) (2), + dskip (1), three fmaf of the ToRGB term (3): |err| <= 7 u sum |terms|
    _check(f"combine {_vid(v)} {B}x{Hg}x{Wg}: dx", (got - ref).abs(), 7 * U * mag + 1e-300)
    if v["rgb"] == 1:
        dw_ref = torch.einsum("bjp,bcp->jc", drgb.double(), xd)
        dw_mag = torch.einsum("bjp,bcp->jc", drgb.double().abs(), xd.abs())
        # a lane's 4 products and 2 add levels (3), 5 shuffle steps, one fp32 shared add per tile of the CTA, then fp64 atomics
        n_t = _n_t(B, HW, per_sm=4)
        for rr in runs:
            assert torch.isfinite(rr["dwrgb"]).all(), "NaN padding reached dW_rgb"
            _check("dW_rgb", (rr["dwrgb"] - rr["init"] - dw_ref).abs(), (8 + n_t) * U * dw_mag + 1e-13 * init.abs())
        a, b = runs[1]["dwrgb"], runs[2]["dwrgb"]
        assert ((a - b).abs() <= 1e-12 * (dw_mag + init.abs())).all(), "a repeated launch moved dW_rgb beyond fp64 rounding"


# ----------------------------------------------------------------------------------------------------------------------
# 4. hg_synth_input_bwd
# ----------------------------------------------------------------------------------------------------------------------
def _synth_input_ref(dx_planar, w, bias, ic, jc, B, Hg, Wg):
    """(dw, db) in fp64 and their bounds.  Per pixel the kernel sums the batch in fp32 ((B - 1) u sum_b |dx|), forms the
    argument with two fmaf (2 u (|w0 i| + |w1 j| + |b|)), takes cosf (2 ulp: 2 u absolute) and one product (u), then sums
    d*i, d*j, d in fp64 and rounds once to fp32."""
    HW = Hg * Wg
    ii = ic.double()[:, None].expand(Hg, Wg).reshape(HW)
    jj = jc.double()[None, :].expand(Hg, Wg).reshape(HW)
    w0, w1, b0 = w[:, 0, None].double(), w[:, 1, None].double(), bias[:, None].double()
    g = dx_planar.double().sum(0)                                     # [C,HW]
    gabs = dx_planar.double().abs().sum(0)
    arg = w0 * ii + w1 * jj + b0
    d = g * torch.cos(arg)
    e = gabs * (2 * U * ((w0 * ii).abs() + (w1 * jj).abs() + b0.abs()) + 2 * U) + (B - 1) * U * gabs + U * d.abs()
    dw = torch.stack([(d * ii).sum(1), (d * jj).sum(1)], 1)
    dwb = torch.stack([(e * ii.abs()).sum(1) + U * (d * ii).abs().sum(1), (e * jj.abs()).sum(1) + U * (d * jj).abs().sum(1)], 1)
    db = d.sum(1)
    dbb = e.sum(1)
    return dw, dwb + U * dw.abs(), db, dbb + U * db.abs()


@gpu
@pytest.mark.parametrize("shape", ALL_SHAPES)
def test_synth_input_bwd(shape):
    abi = _abi()
    B, Hg, Wg = _shape(shape)
    HW = Hg * Wg
    r = _rnd(500)
    dx = r(B, C, HW)
    w, bias = r(C, 2).contiguous(), 0.5 * r(C)
    ic, jc = torch.linspace(-1, 1, Hg, device="cuda"), torch.linspace(-1, 1, Wg, device="cuda")
    dw_ref, dw_bnd, db_ref, db_bnd = _synth_input_ref(dx, w, bias, ic, jc, B, Hg, Wg)

    def launch(fill):
        wbuf, dw = _guarded((C, 2))
        bbuf, db = _guarded((C,))
        abi.call("hg_synth_input_bwd", abi.ptr(_blocked(dx, fill)), abi.ptr(w), abi.ptr(bias), abi.ptr(ic), abi.ptr(jc), B, C, Hg, Wg,
                 abi.ptr(dw), abi.ptr(db), abi.stream())
        return dict(dw=dw, db=db, bufs=[wbuf, bbuf])

    runs = _runs(launch)
    _same(runs, "dw")
    _same(runs, "db")
    # twice the first-order bound: the second-order terms of the cosine's argument error are not in it
    _check(f"synth_input_bwd {B}x{Hg}x{Wg}: dw", (runs[1]["dw"].double() - dw_ref).abs(), 2 * dw_bnd)
    _check(f"synth_input_bwd {B}x{Hg}x{Wg}: db", (runs[1]["db"].double() - db_ref).abs(), 2 * db_bnd)


# ----------------------------------------------------------------------------------------------------------------------
# 5. training sizes: one launch per kernel at C2 (B = 8, 512x512) and the weight gradient at MAP3DBN512 (B = 32, 512x256)
# ----------------------------------------------------------------------------------------------------------------------
def _chan_major(t, b):
    """[B,T,Cc,128] -> sample b as [Cc, T*128] (HW a multiple of 128)."""
    return t[b].permute(1, 0, 2).reshape(t.shape[2], -1)


@gpu
@pytest.mark.parametrize("kernel", ["dgrad", "conv_const", "wgrad", "combine", "synth_input"])
def test_c2_launch(kernel):
    """One launch at C2 size, where every grid-min(tiles, SMs) CTA walks ~124 tiles (16 per sample).  Outputs against fp64
    built per sample on the device, with the bounds of the small shapes; dgrad's sums from its own output."""
    abi = _abi()
    B, Hg, Wg = 8, 512, 512
    HW, T = Hg * Wg, _tiles(Hg * Wg)
    r = _rnd(600)
    n_t = _n_t(B, HW)
    if kernel in ("dgrad", "conv_const"):
        K = 256 if kernel == "dgrad" else 512
        g = [r(B, T, C, 128) for _ in range(K // 256)]
        x = r(B, T, C, 128)
        W = r(K, 256) / 16
        mod = torch.stack([1.0 + 0.5 * r(B, C), 0.5 * r(B, C)], 1).contiguous()
        wimg_t = abi.pack_weight(W.t().contiguous(), Nb=256)[0]
        out = torch.empty(B, T, C, 128, device="cuda")
        sums = torch.zeros(B, 2, C, dtype=torch.float64, device="cuda")
        if kernel == "dgrad":
            abi.spade_bwd_dgrad(g[0], x, T * C * 128, mod, wimg_t, out, sums, B=B, Hg=Hg, Wg=Wg)
        else:
            abi.conv1x1_blocked_bwd(g[0], x, wimg_t, out, sums, g2=g[1], mod=mod, slope=0.2, B=B, Hg=Hg, Wg=Wg)
        torch.cuda.synchronize()
        worst, n_s = 0.0, _n_t_sample(B, HW)
        Wd = W.double()
        for b in range(B):
            gd = torch.cat([_chan_major(t, b) for t in g]).double()
            xb = _chan_major(x, b).double()
            m = _mask(xb * mod[b, 0, :, None].double() + mod[b, 1, :, None].double(), 0.2)
            ref = (Wd.t() @ gd) * m
            mag = (Wd.abs().t() @ gd.abs()) * m
            o = _chan_major(out, b).double()
            worst = max(worst, _check(f"C2 {kernel} sample {b}: dpre", (o - ref).abs(), _gemm_bound(mag, K, 3)))
            for k, (t, tm) in enumerate(((o.sum(1), o.abs().sum(1)), ((o * xb).sum(1), (o * xb).abs().sum(1)))):
                _check(f"C2 {kernel} sample {b}: S[{k}]", (sums[b, k] - t).abs(), _sums_bound(n_s) * tm + 1e-300)
        print(f"C2 {kernel}: {n_t} tiles per CTA, worst {worst:.3f} of the bound")
    elif kernel == "wgrad":
        _big_wgrad(abi, B, Hg, Wg, r)
    elif kernel == "combine":
        x, dpre, dskip = r(B, T, C, 128), r(B, T, C, 128), r(B, T, C, 128)
        g1, ak = r(B, 2, C).contiguous(), r(2, C).contiguous()
        drgb, rgb_w = r(B, 3, HW), r(3, C).contiguous()
        dx = torch.empty(B, T, C, 128, device="cuda")
        dwrgb = torch.zeros(3, C, dtype=torch.float64, device="cuda")
        abi.spade_bwd_combine(dx, B=B, Hg=Hg, Wg=Wg, dpre=dpre, x=x, x_bstride=T * C * 128, g1=g1, ak=ak, dskip=dskip, drgb=drgb,
                              rgb_w=rgb_w, dwrgb=dwrgb)
        torch.cuda.synchronize()
        dw_ref = torch.zeros(3, C, dtype=torch.float64, device="cuda")
        dw_mag = torch.zeros_like(dw_ref)
        for b in range(B):
            xb = _chan_major(x, b).double()
            rb = drgb[b].double()
            t1 = _chan_major(dpre, b).double() * g1[b, 0, :, None].double()
            t2 = ak[1, :, None].double() * xb
            t3 = rgb_w.double().t() @ rb
            ref = t1 + ak[0, :, None].double() + t2 + _chan_major(dskip, b).double() + t3
            mag = t1.abs() + ak[0, :, None].double().abs() + t2.abs() + _chan_major(dskip, b).double().abs() + rgb_w.double().abs().t() @ rb.abs()
            _check(f"C2 combine sample {b}: dx", (_chan_major(dx, b).double() - ref).abs(), 7 * U * mag)
            dw_ref += rb @ xb.t()
            dw_mag += rb.abs() @ xb.abs().t()
        _check("C2 combine: dW_rgb", (dwrgb - dw_ref).abs(), (8 + _n_t(B, HW, per_sm=4)) * U * dw_mag)
    else:
        dx = r(B, T, C, 128)
        w, bias = r(C, 2).contiguous(), 0.5 * r(C)
        ic, jc = torch.linspace(-1, 1, Hg, device="cuda"), torch.linspace(-1, 1, Wg, device="cuda")
        dw, db = abi.synth_input_bwd(dx, w, bias, ic, jc, B)
        torch.cuda.synchronize()
        planar = dx.permute(0, 2, 1, 3).reshape(B, C, HW)
        dw_ref, dw_bnd, db_ref, db_bnd = _synth_input_ref(planar, w, bias, ic, jc, B, Hg, Wg)
        _check("C2 synth_input_bwd: dw", (dw.double() - dw_ref).abs(), 2 * dw_bnd)
        _check("C2 synth_input_bwd: db", (db.double() - db_ref).abs(), 2 * db_bnd)


def _big_wgrad(abi, B, Hg, Wg, r):
    HW, T = Hg * Wg, _tiles(Hg * Wg)
    dout, x = r(B, T, C, 128), r(B, T, C, 128)
    mod = torch.stack([1.0 + 0.5 * r(B, C), 0.5 * r(B, C)], 1).contiguous()
    dw, db = abi.spade_bwd_wgrad(dout, x, T * C * 128, mod, B=B, Hg=Hg, Wg=Wg)
    torch.cuda.synchronize()
    ref = torch.zeros(C, C, dtype=torch.float64, device="cuda")
    mag = torch.zeros_like(ref)
    db_ref = torch.zeros(C, dtype=torch.float64, device="cuda")
    db_mag = torch.zeros_like(db_ref)
    for b in range(B):
        d = _chan_major(dout, b).double()
        y = _lrelu(_chan_major(x, b).double() * mod[b, 0, :, None].double() + mod[b, 1, :, None].double(), 0.2)
        ref += d @ y.t()
        mag += d.abs() @ y.abs().t()
        db_ref += d.sum(1)
        db_mag += d.abs().sum(1)
        del d, y
    n_t = _n_t(B, HW)
    tag = f"wgrad B={B} {Hg}x{Wg} ({n_t} tiles per CTA)"
    _check(tag + ": dW", (dw.double() - ref).abs(), _wgrad_bound(mag, ref, n_t, 3))
    _wgrad_report(tag, dw.double(), ref, 3)
    _check(tag + ": dbias", (db.double() - db_ref).abs(), (6 + 2 * n_t) * U * db_mag + U * db_ref.abs())


@gpu
def test_wgrad_map3dbn512_batch():
    """hg_wgrad_blocked at the MAP3DBN512 single-GPU batch: B = 32, 512x256, 32 768 tiles, ~248 per CTA on 132 SMs; each fp32
    operand is 4.3 GB, the fp64 reference is accumulated per sample."""
    _big_wgrad(_abi(), 32, 512, 256, _rnd(700))


# ----------------------------------------------------------------------------------------------------------------------
# 6. drift: every launch of synthesis_backward is a call form of the matrices above
# ----------------------------------------------------------------------------------------------------------------------
# entry points synthesis_backward also launches, checked launch by launch in tests/test_gpu_spade_conv.py (and the GEMM of
# ops/dense.py); any other name fails the drift check
OTHER_ENTRY_POINTS = {"hg_pack_weight", "hg_spade_a1", "hg_conv1x1_blocked", "hg_spade_pixel_pre", "hg_spade_pixel_mod_bwd",
                      "hg_bilinear_adjoint", "hg_linear", "hg_dense"}


def _classify(name, a):
    """(kernel, variant dict) of one recorded hg_* call, or None when it is no variant of the matrices."""
    if name == "hg_spade_bwd_dgrad":
        dout, x, xbs, mod, w, dpre, sums, B, Cc, Hg, Wg, passes, _ = a
        return "dgrad", dict(xshared=int(xbs == 0), passes=passes)
    if name == "hg_conv1x1_blocked_bwd":
        g, g2, aux, mod, w, out, sums, cout, slope, pm, act, ascale, rk_w, rk_v, rk_n, B, Hg, Wg, passes, _ = a
        if act != 0 or ascale is not None or rk_v is not None:
            return None
        form = (mod is not None, cout, round(float(slope), 6), bool(pm))
        for f, (table, fc, fs, fpm) in CONV_FORMS.items():
            if form == (table, fc, round(fs, 6), fpm):
                return "conv", dict(form=f, g2=int(g2 is not None), passes=passes)
        return None
    if name == "hg_wgrad_blocked":
        dout, x, xbs, Cx, mod, dw, db, ws, B, Cc, Hg, Wg, passes, _ = a
        T = _tiles(Hg * Wg)
        if mod is not None and Cx == 256:
            kind = "const"
        elif mod is None and Cx == 256 and xbs == T * 256 * 128:
            kind = "pixel"
        elif mod is None and Cx == 128 and xbs == T * 128 * 128:
            kind = "gb"
        else:
            return None
        return "wgrad", dict(kind=kind, xshared=int(xbs == 0), bias=int(db is not None), passes=passes)
    if name == "hg_spade_bwd_combine":
        dpre, x, xbs, g1, ak, dskip, drgb, rgb_w, dx, dwrgb, B, Cc, Hg, Wg, _ = a
        if x is None or (dpre is None) != (g1 is None):
            return None
        return "combine", dict(dpre=int(dpre is not None), ak=int(ak is not None), dskip=int(dskip is not None),
                               rgb=0 if drgb is None else 1 if dwrgb is not None else 2, xshared=int(xbs == 0))
    if name == "hg_synth_input_bwd":
        return "input", {}
    return None


def _in_matrix(kernel, v):
    if kernel == "combine":     # the pairwise rows span the product of these levels (g1's kind is not visible in the call)
        return all(v[k] in COMBINE_LEVELS[k] for k in v)
    return {"dgrad": DGRAD, "conv": CONV_BWD, "wgrad": WGRAD, "input": [{}]}[kernel].count(v) == 1


def _record_backward(port, monkeypatch, C_, mode, training, frozen, mod_blocks=(0, 1, 2)):
    """synthesis_backward on a tiny network; the hg_* calls it makes, as (name, args)."""
    pkg = importlib.import_module("3dhumangan_b200")
    st = importlib.import_module("3dhumangan_b200.modules.synthesis_train")
    wo = importlib.import_module("3dhumangan_b200.modules.wide_ops")
    abi = _abi()
    cfg = pkg.configs.baseline_config("tiny")
    cfg.update(hidden_dim=C_, feature_dim=C_, gen_height=16, gen_width=24, render_height=5, render_width=7, mod_blocks=list(mod_blocks),
               map3d_mode=mode)
    B, Rh, Rw = 2, 5, 7
    params = port.init_generator_params(cfg, seed=9)
    names = [n for n in params if n.startswith(("synthesis_network.", "synthesis_input."))]
    pg = {n: params[n].clone().cuda() for n in names}
    for n in names:
        if n.endswith(("weight_u", "weight_v", "running_mean", "running_var", "num_batches_tracked")):
            continue
        if frozen and (".to_rgbs." in n or ".conv_" in n):
            continue
        pg[n].requires_grad_(True)
    g = torch.Generator().manual_seed(10)
    fixed = (torch.randn(B, 1, C_, generator=g) * 0.5).cuda()
    feat_lr = (torch.randn(B, Rh * Rw, C_, generator=g) * 0.7).cuda()
    if C_ == 256:
        _, tape = st.synthesis_forward_train(pg, feat_lr, fixed, cfg, training=training)
    else:
        tape = st.SynthesisTape()
        wo.synthesis_forward_wide(pg, feat_lr, fixed, cfg, training=training, tape=tape)
    rec = []
    call = abi.call

    def recorder(name, *args, **kw):
        rec.append((name, args))
        return call(name, *args, **kw)
    with monkeypatch.context() as mp:
        mp.setattr(abi, "call", recorder)
        st.synthesis_backward(pg, tape, torch.randn(B, 3, 16, 24, generator=g).cuda())
    torch.cuda.synchronize()
    return rec


@gpu
def test_drift_matrix_holds_every_backward_launch(port, monkeypatch):
    """synthesis_backward at hidden_dim 256 / 384 / 420, 'mixed' / 'isolated', train / eval, all parameters learnable / ToRGB
    and convolution weights frozen, plus an all-const-style network at 256 (block 0 reads the batch-shared synthesis input):
    every launch of the kernels above is a variant of their matrix, and every other launch is an entry point tested
    elsewhere."""
    seen, bad = set(), []
    configs = [(C_, mode, training, frozen, (0, 1, 2)) for C_, mode, training, frozen in
               itertools.product((256, 384, 420), ("mixed", "isolated"), (True, False), (False, True))]
    configs += [(256, "mixed", training, frozen, ()) for training in (True, False) for frozen in (False, True)]
    for C_, mode, training, frozen, mod_blocks in configs:
        for name, args in _record_backward(port, monkeypatch, C_, mode, training, frozen, mod_blocks):
            if name in OTHER_ENTRY_POINTS:
                continue
            got = _classify(name, args)
            if got is None or not _in_matrix(*got):
                bad.append((C_, mode, training, frozen, mod_blocks, name, got))
            else:
                seen.add((got[0], tuple(sorted(got[1].items()))))
    assert not bad, bad[:8]
    print("call forms seen:", sorted(seen))
    assert {k for k, _ in seen} == {"dgrad", "conv", "wgrad", "combine", "input"}
    assert ("dgrad", (("passes", 3), ("xshared", 1))) in seen, "the batch-shared data gradient was not reached"
