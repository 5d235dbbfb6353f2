"""The renderer's data-gradient GEMM launch by launch against fp64, in exactly the call forms
`modules/render_train.py::mlp_backward` issues:

    hg_conv1x1_blocked_bwd (csrc/synth.cu, kBwd, act = 1)
        out[b,c,p] = (sum_k Wt[c,k] ascale[b,k] g[b,k,p] + sum_j rk_w[j,c] rk_v[b,j,p]) * cos(aux[b,c,p] g1[b,c] + g0[b,c])
        S1[b,c] += sum_p out,  S2[b,c] += sum_p out * aux       (d phase / d freq of the FiLM slice the layer reads)

    form     mlp_backward       mod (g1, g0)         ascale          rank-k term
    feat     feature layer      FiLM slice 3         none            rk_n = 3: the rgb head's weight, rk_v = d rgb_pre
    colour   colour layer       FiLM slice 3         [B, nh*256]     rk_n = 1: the sigma head's weight, rk_v = d sigma
    trunk    network.3 .. 1     FiLM slice i-1       [B, nh*256]     none
    first    network.0 halves   m30 = (30, 0)        [B, nh*256]     none

each with K = 256 (hidden_dim 256) and K = 512 (the zero-padded 384 / 420: `g2` holds the second output half and
ascale's columns 256.. scale it), at passes 3 (bf16x3) and 1 (bf16).  Every launch is checked five ways, as
tests/test_gpu_synthesis_bwd_kernels.py checks the SPADE half-blocks:
  1. every valid output against the fp64 formula above, componentwise, with a counted bound: the GEMM term
     A_p (S_p + sqrt(K) u) M |cos| with M = sum |Wt||ascale g| + sum |rk_w||rk_v|, a few u of M for the fp32 operand scale
     and the three-fmaf rank-k chain, and |acc| (|pre| u + COS_ABS) for the mask (the fp32 rounding of pre = fmaf(aux, g1,
     g0) and the reduced SFU cosine);
  2. S1 / S2 against fp64 sums of the kernel's own output, on top of a non-zero init, within `_sums_bound`;
  3. the padding rows of g, g2 and aux hold NaN in one launch and zeros in another: outputs bit-identical, sums finite;
  4. every output and every rk_v lives inside a guarded buffer (rk_n = 1 must not read past [B,1,N]);
  5. a repeated launch gives bit-identical outputs, and sums within twice their bound.
Shapes run from one ragged tile to `walk` (every persistent CTA walks >= 16 tiles across sample boundaries), and each
form once per K at the MAP3DBN512 per-GPU training batch (B = 16, 96x48 rays of 32 samples: 18 432 tiles).  A row per K
whose FiLM arguments are exact in fp32 and reach |pre| ~ 2e3 holds the mask to COS_ABS alone, where an error in the 2 pi
reduction is visible.  Planted reference faults show that the bounds tell a wrong result from a right one.  A replay
checks the launches of mlp_backward on a seeded neural field, and a drift check fails on any call form outside the
matrix.

Measured on an H100 80GB HBM3 (700 W): outputs at most 0.92 of the bound at passes 3 (the tail of the rigorous |pre| u
term: pre's rounding nearly reaches it) and 0.77 at passes 1; the exact-argument rows 0.29; the training batch 0.87; the
replay 0.51; sums at most 0.12.  The reduction fault fails by 57x, every other planted fault by 8.9e3x or more.  The
training-size launches peak at 12.4 GiB of device memory (K = 512)."""
import importlib
import math

import pytest
import torch

import test_gpu_render_kernels as render_kernels
import test_gpu_synthesis_bwd_kernels as synth_bwd
from blocked_util import C, SHAPES, U, _blocked, _guarded, _nsm, _planar, _shape, _sums_bound, _tiles
from test_gpu_synthesis_bwd_kernels import _abi, _check, _check_sums, _gemm_bound, _n_t_sample, _rnd, _runs, _same, _vid

gpu = pytest.mark.gpu
ALL_SHAPES = SHAPES + ["walk"]

# The reduced cosine: Cody-Waite reduction by 2 pi (2 roundings of |r| <= pi) plus the SFU cosine (2^-21.4 on [-pi, pi]);
# the renderer test's SIN_ABS
COS_ABS = render_kernels.SIN_ABS
# oracle/port.py init_generator_params: the sigma / rgb heads and the FiLM layers are uniform(+-sqrt(6/256)/25); the
# standard deviation of that draw
W_STD = math.sqrt(6 / 256) / 25 / math.sqrt(3)
# d sigma and d rgb_pre carry the sigma gain and the compositing weights; drawn at 100x unit scale, the head term is of
# the GEMM term's size, so that a fault in it is visible
RK_SCALE = 100.0
# csrc/synth.cu reduce_2pi: 2 pi = 6.2831854820251465f - 1.7484555314695172e-07f
TWO_PI_LO = 1.7484555314695172e-07

FORMS = {   # form -> (table, ascale, rk_n)
    "feat": ("film", False, 3),
    "colour": ("film", True, 1),
    "trunk": ("film", True, 0),
    "first": ("m30", True, 0),
}
MATRIX = [dict(form=f, K=K, passes=p) for f in FORMS for K in (256, 512) for p in (3, 1)]


# ----------------------------------------------------------------------------------------------------------------------
# the classifier of recorded calls (pure Python; the drift check and the replay use it)
# ----------------------------------------------------------------------------------------------------------------------
def _is_m30(mod):
    return bool((mod[:, 0] == 30).all()) and bool((mod[:, 1] == 0).all())


def _classify(c):
    """Matrix row dict(form, K, passes) of one `abi.conv1x1_blocked_bwd` call (its keyword arguments, with the tensors
    g, aux, g2, mod, ascale, rk_w, rk_v), or None when it is no renderer form.  m30 is recognised by its values, rk_n by
    rk_v's shape and K by g2."""
    if c.get("act", 0) != 1 or c.get("Cout", 256) != 256 or c.get("pixel_major", False) or c.get("mod") is None:
        return None
    K = 512 if c.get("g2") is not None else 256
    asc, rkv, rkw = c.get("ascale"), c.get("rk_v"), c.get("rk_w")
    if asc is not None and tuple(asc.shape) != (c["mod"].shape[0], K):
        return None
    rk_n = 0 if rkv is None else rkv.shape[1]
    if rkv is not None and (rkw is None or tuple(rkw.shape) != (3, 256)):
        return None
    key = ("m30" if _is_m30(c["mod"]) else "film", asc is not None, rk_n)
    form = next((f for f, v in FORMS.items() if v == key), None)
    return None if form is None else dict(form=form, K=K, passes=c.get("passes", 3))


def _wgrad_form(args):
    """(act, Cx, pscale, passes) of one recorded hg_act_wgrad_blocked call (its abi.call arguments)."""
    dout, ps, x, xbs, Cx, mod, act, dw, db, ws, B, Cc, Hg, Wg, passes, _ = args
    return act, Cx, ps is not None, passes


WGRAD_FORMS = {(v[0], v[1], v[2], v[4]) for v in render_kernels.WGRAD.values()}


def _synthetic_call(form, K, passes, B=2, N=256):
    """The keyword arguments mlp_backward passes for a matrix row, on small CPU tensors."""
    table, scaled, rk_n = FORMS[form]
    mod = torch.stack([torch.full((B, C), 30.0), torch.zeros(B, C)], 1) if table == "m30" else torch.randn(B, 2, C) + 30
    c = dict(g=torch.zeros(B, N // 128, C, 128), aux=torch.zeros(B, N // 128, C, 128), g2=torch.zeros(1) if K == 512 else None,
             mod=mod, act=1, ascale=torch.randn(B, K) if scaled else None, rk_w=torch.zeros(3, C) if rk_n else None,
             rk_v=torch.zeros(B, rk_n, N) if rk_n else None, Cout=256, pixel_major=False, passes=passes)
    return c


def test_matrix_is_the_product_of_forms_widths_and_passes():
    """16 rows: every form at K = 256 / 512 and passes 3 / 1 (pure Python)."""
    assert len(MATRIX) == 16 and len({_vid(v) for v in MATRIX}) == 16
    assert {(v["form"], v["K"], v["passes"]) for v in MATRIX} == {(f, K, p) for f in FORMS for K in (256, 512) for p in (3, 1)}


def test_classifier_on_synthetic_calls():
    """Every row's call is classified as that row; calls outside the matrix are not (pure Python)."""
    for v in MATRIX:
        assert _classify(_synthetic_call(v["form"], v["K"], v["passes"])) == v, v
    bad = []
    c = _synthetic_call("trunk", 256, 3)
    bad.append(dict(c, act=0))                                     # a synthesis call
    bad.append(dict(c, Cout=128))
    bad.append(dict(c, pixel_major=True))
    bad.append(dict(c, mod=None))
    bad.append(dict(c, ascale=torch.randn(2, 512)))                # ascale wider than K
    bad.append(dict(_synthetic_call("trunk", 512, 3), ascale=torch.randn(2, 256)))
    bad.append(dict(_synthetic_call("feat", 256, 3), ascale=torch.randn(2, 256)))       # rank 3 with a scale
    bad.append(dict(_synthetic_call("colour", 256, 3), ascale=None))                     # rank 1 without one
    bad.append(dict(_synthetic_call("colour", 256, 3), rk_v=torch.zeros(2, 2, 256)))    # rank 2
    bad.append(dict(_synthetic_call("colour", 256, 3), rk_w=torch.zeros(1, C)))          # a [1,256] head table
    bad.append(dict(_synthetic_call("first", 256, 3), rk_w=torch.zeros(3, C), rk_v=torch.zeros(2, 1, 256)))
    bad.append(dict(_synthetic_call("first", 256, 3), ascale=None))
    for b in bad:
        assert _classify(b) is None
    # a FiLM table equal to m30 except in one entry is a FiLM table
    c = _synthetic_call("first", 256, 1)
    c["mod"][1, 1, 7] = 1e-3
    assert _classify(c) == dict(form="trunk", K=256, passes=1)


def test_wgrad_classifier_on_synthetic_calls():
    """The weight-gradient forms mlp_backward issues are forms of test_gpu_render_kernels.WGRAD (pure Python)."""
    t = object()
    for act, Cx, ps in ((1, 256, True), (1, 256, False), (2, 128, True)):
        for passes in (3, 1):
            args = (t, t if ps else None, t, 0, Cx, t if act == 1 else None, act, t, t, t, 2, 256, 1, 512, passes, None)
            assert _wgrad_form(args) in WGRAD_FORMS, (act, Cx, ps, passes)
    assert (1, 128, True, 3) not in WGRAD_FORMS and (0, 256, False, 3) not in WGRAD_FORMS


# ----------------------------------------------------------------------------------------------------------------------
# inputs, the fp64 reference and the bound
# ----------------------------------------------------------------------------------------------------------------------
def _tables(r, form, B, K, quant=False):
    """(mod [B,2,256], ascale [B,K] or None, rk_w [3,256] or None): FiLM tables f = 30 + 15 randn, phi = randn per sample;
    ascale drawn like f.  Rows of rk_w past rk_n hold finite values the kernel must ignore (the header's contract)."""
    table, scaled, rk_n = FORMS[form]
    if table == "m30":
        mod = torch.stack([torch.full((B, C), 30.0, device="cuda"), torch.zeros(B, C, device="cuda")], 1)
    else:
        f, phi = 30.0 + 15.0 * r(B, C), r(B, C)
        if quant:            # a 2^-4 grid for f and 2^-8 for phi: with aux on a 2^-4 grid, aux*f + phi is exact in fp32
            f, phi = torch.round(f * 16) / 16, torch.round(phi * 256) / 256
        mod = torch.stack([f, phi], 1)
    ascale = (30.0 + 15.0 * r(B, K)).contiguous() if scaled else None
    rk_w = (r(3, C) * W_STD).contiguous() if rk_n else None
    return mod.contiguous(), ascale, rk_w


def _inputs(v, B, HW, seed, quant=False):
    r = _rnd(seed)
    K = v["K"]
    rk_n = FORMS[v["form"]][2]
    mod, ascale, rk_w = _tables(r, v["form"], B, K, quant)
    x = r(B, C, HW)
    if quant:
        x = torch.round(6.0 * x * 16) / 16
    return dict(Wt=(r(C, K) * W_STD).contiguous(), g=r(B, K, HW), x=x, mod=mod, ascale=ascale, rk_w=rk_w,
                rk_v=(RK_SCALE * r(B, rk_n, HW)).contiguous() if rk_n else None, init=10.0 * r(B, 2, C).double())


def _ref(Wt, g, x, mod, ascale, rk_w, rk_v, rk_scale=None, red_fault=False):
    """fp64 out [n,256,P] and its parts, with everything n-major: g [n,K,P], x [n,256,P], mod [n,2,256], ascale [n,K] or
    None, rk_w [3,256], rk_v [n,rk_n,P] or None.  Faults: `rk_scale` [n,256] multiplies the rank-k term per output
    channel; `red_fault` moves the cosine's argument by 2 k 2pi_lo (k = round(pre / 2 pi)), the flipped sign of the low
    term of the reduction."""
    gd = g.double()
    if ascale is not None:
        gd = gd * ascale.double()[:, :, None]
    Wd = Wt.double()
    acc = torch.einsum("ck,nkp->ncp", Wd, gd)
    M = torch.einsum("ck,nkp->ncp", Wd.abs(), gd.abs())
    del gd
    if rk_v is not None:
        kk = rk_v.shape[1]
        rw, rv = rk_w[:kk].double(), rk_v.double()
        t = torch.einsum("jc,njp->ncp", rw, rv)
        tm = torch.einsum("jc,njp->ncp", rw.abs(), rv.abs())
        if rk_scale is not None:
            t, tm = t * rk_scale.double()[:, :, None], tm * rk_scale.double().abs()[:, :, None]
        acc, M = acc + t, M + tm
    pre = x.double() * mod[:, 0, :, None].double() + mod[:, 1, :, None].double()
    arg = pre - 2 * TWO_PI_LO * torch.round(pre / (2 * math.pi)) if red_fault else pre
    cos = torch.cos(arg)
    return dict(out=acc * cos, acc=acc, M=M, cos=cos, pre=pre)


def _bound(R, K, passes, exact_pre=False):
    """|err| of one output.  The accumulator: the GEMM term, plus u M for the fp32 product ascale*g and 3 u M for the
    three fmaf of the rank-k chain.  The mask: COS_ABS, plus u |pre| for the fp32 rounding of pre (absent when aux*g1 + g0
    is exact in fp32).  The output: one rounding of acc * mask."""
    M, acc = R["M"], R["acc"].abs()
    e_acc = _gemm_bound(M, K, passes) + 4 * U * M
    e_mask = COS_ABS if exact_pre else COS_ABS + U * R["pre"].abs()
    return (e_acc + U * (acc + e_acc)) * (R["cos"].abs() + e_mask) + acc * e_mask + 1e-300


def _ref_of(ins, **fault):
    return _ref(ins["Wt"], ins["g"], ins["x"], ins["mod"], ins["ascale"], ins["rk_w"], ins["rk_v"], **fault)


def _tile_ref(ins, b, tile, **over):
    """The reference of sample b's tile `tile` (pixels 128 tile ..), with inputs replaced by `over`."""
    sl = slice(128 * tile, 128 * tile + 128)
    a = dict(Wt=ins["Wt"], g=ins["g"][b:b + 1, :, sl], x=ins["x"][b:b + 1, :, sl], mod=ins["mod"][b:b + 1],
             ascale=None if ins["ascale"] is None else ins["ascale"][b:b + 1], rk_w=ins["rk_w"],
             rk_v=None if ins["rk_v"] is None else ins["rk_v"][b:b + 1, :, sl])
    fault = {k: over.pop(k) for k in ("rk_scale", "red_fault") if k in over}
    a.update(over)
    return _ref(**a, **fault)["out"][0]


# ----------------------------------------------------------------------------------------------------------------------
# 1. the matrix at every shape
# ----------------------------------------------------------------------------------------------------------------------
def _run(ins, v, B, Hg, Wg, tag, exact_pre=False):
    """Three launches (NaN padding, zeros, zeros), the five checks; (kernel output planar fp64, reference, bound, runs,
    fp64 sums of each run's own output)."""
    abi = _abi()
    HW, T = Hg * Wg, _tiles(Hg * Wg)
    K, passes = v["K"], v["passes"]
    wimg_t = abi.pack_weight(ins["Wt"], Nb=256)[0]

    def launch(fill):
        obuf, out = _guarded((B, T, C, 128))
        sbuf, sums = _guarded((B, 2, C), torch.float64, 0.0)
        sums.copy_(ins["init"])
        bufs = [obuf, sbuf]
        rkv = None
        if ins["rk_v"] is not None:
            vbuf, rkv = _guarded(tuple(ins["rk_v"].shape), fill=0.0)
            rkv.copy_(ins["rk_v"])
            bufs.append(vbuf)
        g = ins["g"]
        abi.conv1x1_blocked_bwd(_blocked(g[:, :C], fill), _blocked(ins["x"], fill), wimg_t, out, sums,
                                g2=_blocked(g[:, C:], fill) if K == 512 else None, mod=ins["mod"], act=1, ascale=ins["ascale"],
                                rk_w=ins["rk_w"], rk_v=rkv, B=B, Hg=Hg, Wg=Wg, passes=passes)
        return dict(out=out, sums=sums, init=ins["init"], bufs=bufs)

    planar = lambda t: _planar(t, HW)
    runs = _runs(launch)
    _same(runs, "out", planar)
    R = _ref_of(ins)
    bound = _bound(R, K, passes, exact_pre)
    got = planar(runs[1]["out"]).double()
    _check(f"{tag}: out", (got - R["out"]).abs(), bound)
    xd = ins["x"].double()
    refs = []
    for rr in runs:
        o = planar(rr["out"]).double()
        refs.append(((o.sum(2), o.abs().sum(2)), ((o * xd).sum(2), (o * xd).abs().sum(2))))
    n_s = _n_t_sample(B, HW)
    _check_sums(runs, "sums", refs, n_s, f"{tag}: S")
    # the CTAs' fp32 shared sums take the warps' totals by shared-memory atomics in any order
    a, b = runs[1]["sums"], runs[2]["sums"]
    mag_s = torch.stack([m for _, m in refs[1]], 1)
    assert ((a - b).abs() <= 2 * _sums_bound(n_s) * mag_s + 1e-12 * ins["init"].abs()).all(), "repeat moved the sums"
    return got, R, bound, runs, refs


def _fault(name, got, ref, bound):
    ratio = ((got - ref).abs() / bound).max().item()
    print(f"  fault {name}: {ratio:.0f}x the bound")
    assert ratio > 10, f"fault {name} fails by only {ratio:.1f}x the bound"


@gpu
@pytest.mark.parametrize("shape", ALL_SHAPES)
@pytest.mark.parametrize("v", MATRIX, ids=_vid)
def test_conv1x1_blocked_bwd_render(v, shape):
    B, Hg, Wg = _shape(shape)
    HW, T = Hg * Wg, _tiles(Hg * Wg)
    tiles = B * T
    grid = min(tiles, _nsm())
    tag = f"{_vid(v)} {B}x{Hg}x{Wg} ({-(-tiles // grid)} tiles per CTA, {_n_t_sample(B, HW)} per sample)"
    ins = _inputs(v, B, HW, 800 + MATRIX.index(v))
    got, R, bound, runs, refs = _run(ins, v, B, Hg, Wg, tag)
    if shape != "multi" or v["passes"] != 3:
        return
    # the bounds discriminate: faults built into the reference, against the kernel's output on tile 0 of sample 1
    b, sl = 1, slice(0, 128)
    gt, bt = got[b, :, sl], bound[b, :, sl]
    asc, rkv = ins["ascale"], ins["rk_v"]
    if asc is not None:
        _fault("tile scaled with another sample's ascale row", gt, _tile_ref(ins, b, 0, ascale=asc[0:1]), bt)
    if v["K"] == 512 and asc is not None:
        _fault("K halves' ascale columns swapped", gt, _tile_ref(ins, b, 0, ascale=torch.cat([asc[b:b + 1, C:], asc[b:b + 1, :C]], 1)), bt)
    if rkv is not None:
        _fault("rk_v from another sample", gt, _tile_ref(ins, b, 0, rk_v=rkv[0:1, :, sl]), bt)
    if v["form"] == "colour":
        _fault("rank-k term times ascale", gt, _tile_ref(ins, b, 0, rk_scale=asc[b:b + 1, :C]), bt)
    # a missed flush: one tile's contribution left out of S1 / S2
    o = got[b, :, sl]
    tile_sums = (o.sum(1), (o * ins["x"][b, :, sl].double()).sum(1))
    gs = runs[1]["sums"] - runs[1]["init"]
    for k in (0, 1):
        (ref_s, mag_s) = refs[1][k]
        _fault(f"S{k + 1} without one tile", gs[b, k], ref_s[b] - tile_sums[k], _sums_bound(_n_t_sample(B, HW)) * mag_s[b] + 1e-300)


@gpu
@pytest.mark.parametrize("K", [256, 512])
def test_mask_exact_arguments(K):
    """aux on a 2^-4 grid (|aux| <~ 30), f on a 2^-4 grid and phi on a 2^-8 grid: aux*f + phi is exact in fp32 and |pre|
    reaches ~2e3, so the mask is held to COS_ABS alone.  A flipped sign on the low 2 pi term of the reduction moves the
    cosine by 2 k 2pi_lo, ~1e-4 at k ~ 300: it must fail by more than 10x."""
    v = dict(form="trunk", K=K, passes=3)
    B, Hg, Wg = _shape("multi")
    HW = Hg * Wg
    ins = _inputs(v, B, HW, 850 + K, quant=True)
    pre32 = torch.addcmul(ins["mod"][:, 1, :, None], ins["x"], ins["mod"][:, 0, :, None])
    pre = ins["x"].double() * ins["mod"][:, 0, :, None].double() + ins["mod"][:, 1, :, None].double()
    assert torch.equal(pre32.double(), pre), "the FiLM arguments are not exact in fp32"
    tmax = pre.abs().max().item()
    assert tmax > 1000, tmax
    got, R, bound, _, _ = _run(ins, v, B, Hg, Wg, f"exact-argument {_vid(v)} {B}x{Hg}x{Wg} max|pre| {tmax:.0f}", exact_pre=True)
    _fault("2 pi reduction's low term with the wrong sign", got, _ref_of(ins, red_fault=True)["out"], bound)


# ----------------------------------------------------------------------------------------------------------------------
# 2. the MAP3DBN512 / MAP3DBN512L per-GPU training batch
# ----------------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("K", [256, 512])
@pytest.mark.parametrize("form", list(FORMS))
def test_training_size(form, K):
    """One launch at B = 16, 96x48 rays of 32 samples (N = 147 456 points, 1 152 tiles per sample), where every CTA walks
    ~140 tiles and flushes its sums 16 times.  Every pixel of the first and last sample and 32 seeded tiles of each other
    sample against fp64 (built per sample), the sums of every sample against the kernel's own output."""
    abi = _abi()
    torch.cuda.reset_peak_memory_stats()
    B, N = 16, 96 * 48 * 32
    T = N // 128
    tiles = B * T
    grid = min(tiles, _nsm())
    n_t, n_s = -(-tiles // grid), _n_t_sample(B, N)
    assert tiles == 18432 and n_s == -(-T // grid)
    if _nsm() == 132:
        assert (n_t, n_s) == (140, 9)
    v = dict(form=form, K=K, passes=3)
    r = _rnd(900 + 2 * list(FORMS).index(form) + (K == 512))
    mod, ascale, rk_w = _tables(r, form, B, K)
    rk_n = FORMS[form][2]
    Wt = (r(C, K) * W_STD).contiguous()
    g = [r(B, T, C, 128) for _ in range(K // 256)]
    x = r(B, T, C, 128)
    rk_v = (RK_SCALE * r(B, rk_n, N)).contiguous() if rk_n else None
    out = torch.empty(B, T, C, 128, device="cuda")
    sums = torch.zeros(B, 2, C, dtype=torch.float64, device="cuda")
    abi.conv1x1_blocked_bwd(g[0], x, abi.pack_weight(Wt, Nb=256)[0], out, sums, g2=g[1] if K == 512 else None, mod=mod, act=1,
                            ascale=ascale, rk_w=rk_w, rk_v=rk_v, B=B, Hg=1, Wg=N)
    torch.cuda.synchronize()
    pick = torch.Generator(device="cuda").manual_seed(901)
    worst = 0.0
    for b in range(B):
        idx = torch.arange(T, device="cuda") if b in (0, B - 1) else torch.randperm(T, generator=pick, device="cuda")[:32].sort().values
        n = idx.numel()
        R = _ref(Wt, torch.cat([t[b, idx] for t in g], 1), x[b, idx], mod[b:b + 1].expand(n, 2, C),
                 None if ascale is None else ascale[b:b + 1].expand(n, K), rk_w,
                 None if rk_v is None else rk_v[b].reshape(rk_n, T, 128)[:, idx].permute(1, 0, 2))
        err = (out[b, idx].double() - R["out"]).abs()
        ratio = (err / _bound(R, K, 3)).max().item()
        assert ratio <= 1.0, f"sample {b}: {ratio:.3f}x the bound"
        worst = max(worst, ratio)
        del R, err
        o, xb = out[b].double(), x[b].double()
        for k, (t, tm) in enumerate(((o.sum((0, 2)), o.abs().sum((0, 2))), ((o * xb).sum((0, 2)), (o * xb).abs().sum((0, 2))))):
            _check(f"training {_vid(v)} sample {b}: S{k + 1}", (sums[b, k] - t).abs(), _sums_bound(n_s) * tm + 1e-300)
        del o, xb
    peak = torch.cuda.max_memory_allocated() / 2 ** 30
    print(f"training {_vid(v)} B{B} N{N}: {n_t} tiles per CTA, {n_s} per sample; out worst {worst:.3f} of the bound; "
          f"peak {peak:.1f} GiB")


# ----------------------------------------------------------------------------------------------------------------------
# 3. replay: the launches of mlp_backward on a seeded neural field
# ----------------------------------------------------------------------------------------------------------------------
def _record_convs(monkeypatch, calls):
    """Records every abi.conv1x1_blocked_bwd call with its inputs cloned at call time, its unpacked weight (from
    synthesis_train._packT) and its outputs."""
    abi = _abi()
    st = importlib.import_module("3dhumangan_b200.modules.synthesis_train")
    packs = {}
    pack, conv = st._packT, abi.conv1x1_blocked_bwd

    def pack_rec(W, ih):
        img = pack(W, ih)
        packs[img.data_ptr()] = W[:, ih * 256:(ih + 1) * 256].t().contiguous().clone()
        return img

    def conv_rec(g, aux, wimg_t, out, sums, **kw):
        c = {k: (t.clone() if isinstance(t, torch.Tensor) else t) for k, t in kw.items()}
        c.update(g=g.clone(), aux=aux.clone(), Wt=packs.get(wimg_t.data_ptr()), init=sums.clone())
        res = conv(g, aux, wimg_t, out, sums, **kw)
        c.update(out=out.clone(), sums=sums.clone())
        calls.append(c)
        return res
    monkeypatch.setattr(st, "_packT", pack_rec)
    monkeypatch.setattr(abi, "conv1x1_blocked_bwd", conv_rec)


@gpu
@pytest.mark.parametrize("C_", [256, 420])
def test_replay_mlp_backward(port, monkeypatch, C_):
    """mlp_backward at hidden_dim 256 (mlp_forward_train's tape) and 420 (render_forward_wide's), B = 2, 64 rays of 32
    samples (16 tiles per sample): every data-gradient launch is a matrix row, and its output and sums meet the bounds
    under real activations, FiLM tables, head weights and the zero ascale columns of the 420 padding."""
    import test_gpu_render_train as rtt
    rt = importlib.import_module("3dhumangan_b200.modules.render_train")
    wo = importlib.import_module("3dhumangan_b200.modules.wide_ops")
    cfg, params, names, pts, geo, z, freq, phase, noise, wgt = rtt._setup(port, C_, R=64, S=32)
    B, R_, S = z.shape
    N = R_ * S
    pg = {n: params[n].clone().cuda().requires_grad_(True) for n in names}
    rec = torch.cat([pts, geo], -1).cuda()
    z_vals = z.reshape(B, N).cuda().contiguous()
    if C_ == 256:
        _, tape = rt.mlp_forward_train(pg, freq.cuda(), phase.cuda(), rec, z_vals, None, cfg)
    else:
        monkeypatch.setattr(rt, "geo_records", lambda *a, **k: (rec, z_vals))
        tape = {}
        wo.render_forward_wide(pg, freq.cuda(), phase.cuda(), None, cfg, None, None, tape=tape)
    calls = []
    with monkeypatch.context() as mp:
        _record_convs(mp, calls)
        rt.mlp_backward(tape, wgt[..., 3:].cuda(), wgt[..., :3].cuda())
    torch.cuda.synchronize()
    nh = 1 if C_ == 256 else 2
    assert len(calls) == 7 * nh, len(calls)
    seen = set()
    for i, c in enumerate(calls):
        v = _classify(c)
        assert v is not None and v in MATRIX, (i, v)
        assert c["Wt"] is not None, "the weight image did not come from _packT"
        seen.add(v["form"])
        K, T = v["K"], N // 128
        planar = lambda t: _planar(t, N)
        g = planar(c["g"]) if c["g2"] is None else torch.cat([planar(c["g"]), planar(c["g2"])], 1)
        x = planar(c["aux"])
        Rr = _ref(c["Wt"], g, x, c["mod"], c["ascale"], c["rk_w"], c["rk_v"])
        got = planar(c["out"]).double()
        tag = f"replay {C_} call {i} {_vid(v)}"
        if c["ascale"] is not None and nh == 2:
            tag += f" ({int((c['ascale'] == 0).sum(1)[0])} zero ascale columns)"
        _check(f"{tag}: out", (got - Rr["out"]).abs(), _bound(Rr, K, v["passes"]))
        xd = x.double()
        refs = [((got.sum(2), got.abs().sum(2)), ((got * xd).sum(2), (got * xd).abs().sum(2)))]
        _check_sums([dict(sums=c["sums"], init=c["init"])], "sums", refs, _n_t_sample(B, N), f"{tag}: S")
    assert seen == set(FORMS), seen


# ----------------------------------------------------------------------------------------------------------------------
# 4. drift: every renderer data-gradient launch is a matrix row, every weight-gradient launch a WGRAD form
# ----------------------------------------------------------------------------------------------------------------------
DRIFT = [   # (hidden_dim, training, frozen parameter prefixes, hierarchical_sample, hg_precision)
    (256, True, (), False, "fp32x3"),
    (384, True, (), False, "fp32x3"),
    (420, True, (), False, "fp32x3"),
    (256, False, ("",), False, "fp32x3"),                        # eval, frozen generator: gradients w.r.t. z only
    (420, False, (), False, "fp32x3"),                           # eval, every parameter learnable
    (256, True, ("neural_field.first_layer_",), False, "fp32x3"),
    (420, True, (), True, "fp32x3"),
    (256, True, (), False, "bf16"),
    (420, True, (), False, "bf16"),
]


def _record_generator(pkg, port, monkeypatch, C_, training, frozen, hier, precision):
    """One generator forward + backward; (abi.call records (name, args), classification of every
    abi.conv1x1_blocked_bwd call)."""
    abi = _abi()
    gen = importlib.import_module("3dhumangan_b200.modules.generator")
    cfg = pkg.configs.baseline_config("tiny")
    cfg.update(hidden_dim=C_, feature_dim=C_, gen_height=16, gen_width=16, render_height=4, render_width=4, num_steps=32,
               nerf_noise=0.0, hierarchical_sample=hier)
    G = gen.Map3DGenerator(**cfg).cuda()
    G.load_state_dict(port.init_generator_params(cfg, seed=21, sigma_gain=200.0, sigma_bias=1.0), strict=True)
    G.set_device(torch.device("cuda:0"))
    G.train()
    cg = {k: v.cuda() for k, v in pkg.synthetic.make_conditions(2, seed=22).items()}
    torch.manual_seed(5)
    if not training:      # running statistics from three train-mode forwards, as in tests/test_gpu_eval_backward.py
        with torch.no_grad():
            for _ in range(3):
                G(torch.randn(2, cfg["latent_dim"], device="cuda"), cg, **cfg)
        G.eval()
    for n, p in G.named_parameters():
        p.requires_grad_(not any(n.startswith(f) for f in frozen))
    z = torch.randn(2, cfg["latent_dim"], device="cuda").requires_grad_(True)
    out = G(z, cg, **dict(cfg, hg_precision=precision))
    loss = (out["rgbs"] * torch.randn_like(out["rgbs"])).sum() + (out["rgbs_render"] * torch.randn_like(out["rgbs_render"])).sum()
    rec, forms = [], []
    call, conv = abi.call, abi.conv1x1_blocked_bwd

    def conv_rec(g, aux, wimg_t, out, sums, **kw):
        forms.append(_classify(dict(kw, g=g, aux=aux)) if kw.get("act", 0) == 1 else "act0")
        return conv(g, aux, wimg_t, out, sums, **kw)
    with monkeypatch.context() as mp:
        mp.setattr(abi, "call", lambda name, *a, **k: (rec.append((name, a)), call(name, *a, **k))[1])
        mp.setattr(abi, "conv1x1_blocked_bwd", conv_rec)
        loss.backward()
    torch.cuda.synchronize()
    return rec, forms


@gpu
def test_drift_matrix_holds_every_renderer_backward_launch(pkg, port, monkeypatch):
    """The generator's backward in training at 256 / 384 / 420, in eval mode with a frozen generator and with every
    parameter learnable, with the first layers frozen, with hierarchical_sample at 420 and with hg_precision="bf16":
    every hg_conv1x1_blocked_bwd launch with the cosine mask is a matrix row (the others are SPADE forms of
    tests/test_gpu_synthesis_bwd_kernels.py), every hg_act_wgrad_blocked launch a form of
    tests/test_gpu_render_kernels.py WGRAD, and every matrix row is issued by some configuration."""
    seen, seen_w, bad = set(), set(), []
    for cfg in DRIFT:
        rec, forms = _record_generator(pkg, port, monkeypatch, *cfg)
        convs = [a for n, a in rec if n == "hg_conv1x1_blocked_bwd"]
        assert len(convs) == len(forms), "a data-gradient launch bypassed abi.conv1x1_blocked_bwd"
        assert any(f != "act0" for f in forms), cfg
        for a, f in zip(convs, forms):
            if f == "act0":
                got = synth_bwd._classify("hg_conv1x1_blocked_bwd", a)
                if got is None or not synth_bwd._in_matrix(*got):
                    bad.append((cfg, "synthesis", got))
            elif f is None or f not in MATRIX:
                bad.append((cfg, "renderer", f))
            else:
                seen.add((f["form"], f["K"], f["passes"]))
        for n, a in rec:
            if n == "hg_act_wgrad_blocked":
                w = _wgrad_form(a)
                if w not in WGRAD_FORMS:
                    bad.append((cfg, n, w))
                seen_w.add(w)
    assert not bad, bad[:8]
    print("data-gradient forms seen:", sorted(seen))
    print("weight-gradient forms seen (act, Cx, pscale, passes):", sorted(seen_w))
    missing = [v for v in MATRIX if (v["form"], v["K"], v["passes"]) not in seen]
    assert not missing, missing
