"""The streaming kernels of a training iteration launch by launch against fp64, in the call forms the module code issues and
at the curricula's sizes:

    hg_bias_act / hg_bias_act_grad        (csrc/elementwise.cu)  ops/bias_act.py: the discriminator's LeakyReLU, the VGG16 ReLU
    hg_resample2x                         (csrc/elementwise.cu)  the discriminator's 2x2 pooling / 2x up-sampling and adjoints,
                                                                 and the hg_upfirdn2d fallback of `_pool` / `_up`
    hg_spectral_norm                      (csrc/spectral.cu)     the C2 G's 18 and D's 32 spectral-normed weights, one launch each
    hg_label_histogram -> hg_seg_ce_coef -> hg_seg_ce
                                          (csrc/trainer.cu)      the class-balanced segmentation loss and its gradient
    hg_image_loss                         (csrc/trainer.cu)      L2 / Charbonnier / smooth-L1 reconstruction losses
    hg_mt_grad_norm / hg_mt_adam          (csrc/trainer.cu)      FusedAdam: clip_grad_norm_, Adam and the generator's EMA

Every launch is checked as the GEMM kernels' files check theirs:
  1. componentwise against an fp64 evaluation of the kernel's contract from the same fp32 inputs, with a bound counted from
     the kernel's fp32 arithmetic (k u |terms| for k roundings, u = 2^-24, the CUDA math library's documented ulp errors for
     expf / expm1f / log1pf / tanhf and the intrinsics' documented errors for __expf / __logf), times 2 for the second-order
     terms a first-order count leaves out;
  2. every output sits inside a larger buffer whose guard elements must be untouched;
  3. outputs are pre-filled with NaN, so an element the launch owns and does not write fails the check;
  4. the kernels documented as deterministic (hg_seg_ce, hg_image_loss, hg_mt_grad_norm, hg_spectral_norm) repeat bit for bit;
  5. integer results exactly: the label histogram, and the gradient norm / clip pair, whose fp64 sum the reference forms too.
A drift check records the launches of `Trainer.iteration` in five configurations and fails on a call form the matrices do not
hold.

Not tested: the 64-bit index instances of bias_act (tensors of >= 2^32 elements).  Exercising them needs two 16 GiB tensors
on the device, more than a shared machine should give one test; their arithmetic is the 32-bit instances' with a wider
index type."""
import contextlib
import copy
import importlib
import itertools
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from blocked_util import G, U, _guarded, _intact, _nsm, _pairs, _pairwise

gpu = pytest.mark.gpu
EPS_SN = 1e-12


def _abi():
    return importlib.import_module("3dhumangan_b200.abi")


def _ba():
    return importlib.import_module("3dhumangan_b200.ops.bias_act")


def _rnd(seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return lambda *s: torch.randn(*s, generator=g, device="cuda")


def _check(name, err, bound):
    ratio = (err / bound).max().item()
    print(f"  {name}: {ratio:.3f} of the bound")
    assert ratio <= 1.0, f"{name}: error {ratio:.3f}x the bound"
    return ratio


def _f32(v):
    """The fp32 value a float scalar argument takes, as a Python float."""
    return float(np.float32(v))


def _slices(n, step=1 << 24):
    for a in range(0, n, step):
        yield slice(a, min(n, a + step))


# ----------------------------------------------------------------------------------------------------------------------
# the matrices: the call forms of ops/bias_act.py, discriminator_train._pool / _up, FusedAdam and the losses
# ----------------------------------------------------------------------------------------------------------------------
ACT_NAMES = ["linear", "relu", "lrelu", "tanh", "sigmoid", "elu", "selu", "softplus", "swish"]


def _second(act):
    return _ba_table()[act][4]


def _ba_table():
    # ops/bias_act.ACTIVATIONS without importing the package on a CPU-only run of the coverage tests
    return {
        "linear": (1, 0.0, 1.0, "", False), "relu": (2, 0.0, math.sqrt(2), "y", False),
        "lrelu": (3, 0.2, math.sqrt(2), "y", False), "tanh": (4, 0.0, 1.0, "y", True),
        "sigmoid": (5, 0.0, 1.0, "y", True), "elu": (6, 0.0, 1.0, "y", True), "selu": (7, 0.0, 1.0, "y", True),
        "softplus": (8, 0.0, 1.0, "y", True), "swish": (9, 0.0, math.sqrt(2), "x", True),
    }


# op: fwd = hg_bias_act; grad1 = _BiasActGrad.forward; grad2 = the second-derivative launch of _BiasActGrad.backward.
# bias: the forward's bias (vec: stepB % 4 == 0, the kVecBias instance); tail: n % 4; size: one ragged vector or just past
# one capped trip of the kernel's grid
BA_LEVELS = dict(act=ACT_NAMES, op=("fwd", "grad1", "grad2"), clamp=(0, 1), bias=("none", "vec", "scalar"), tail=(0, 1, 2, 3),
                 size=("ragged", "trip"))


def _ba_valid(v):
    # a bias every 4 elements makes n a multiple of 4; only the smooth activations have a second derivative
    return not (v["bias"] == "vec" and v["tail"] != 0) and not (v["op"] == "grad2" and not _second(v["act"]))


BA = _pairwise(BA_LEVELS, _ba_valid)


def _ba_launch_args(v):
    """The NULL pattern ops/bias_act.py gives a launch: (bias, xref, yref, dy) present.  _BiasAct saves x and b when the
    activation keeps x or has a second derivative, y when it keeps y or clamps; order 2 multiplies by the saved dy."""
    keeps, second = _ba_table()[v["act"]][3], _ba_table()[v["act"]][4]
    if v["op"] == "fwd":
        return (v["bias"] != "none", False, False, False)
    keep_x = keeps == "x" or second
    return (keep_x and v["bias"] != "none", keep_x, keeps == "y" or bool(v["clamp"]), v["op"] == "grad2")


# (up, scale): _Resample2x's forward pool (0.25) / up (1.0) and each one's backward, the other direction at the same scale
RESAMPLE = [(0, 0.25), (1, 1.0), (1, 0.25), (0, 1.0)]
# hg_image_loss: mode x mask x gradient requested
IMAGE_LOSS = [dict(mode=m, mask=mk, grad=gr) for m in (0, 1, 2) for mk in (0, 1) for gr in (1, 0)]
# hg_seg_ce_coef / hg_seg_ce: prior weights x gradient requested
SEG_CE = [dict(prior=p, grad=gr) for p in (0, 1) for gr in (1, 0)]
SN = [dict(training=t) for t in (1, 0)]
# hg_mt_adam: clip coefficient given, write_grad, EMA; a launch without EMA (the discriminator) never passes a decay
ADAM = [dict(clip=1, ema=e) for e in (1, 0)]


def _vid(v):
    return "-".join(f"{k}{v[k]}" for k in v)


def test_bias_act_rows_cover_every_option_pair():
    """The bias_act matrix holds every pair of option values that some valid call form holds (pure Python)."""
    names = list(BA_LEVELS)
    for a, va, b, vb in _pairs(BA_LEVELS, _ba_valid):
        assert any(r[a] == va and r[b] == vb for r in BA), (a, va, b, vb)
    assert all(_ba_valid(r) for r in BA)
    assert len(BA) < math.prod(len(v) for v in BA_LEVELS.values())
    assert len(names) == 6


def test_matrices_reach_every_instance_and_branch():
    """Every template instance and branch of the 32-bit index kernels is some matrix row: kVecBias on / off, all nine act ids,
    order 1 and 2 (the latter for every activation with a second derivative), clamp on / off, the scalar tail at every n % 4 in
    both kernels, the grad kernel with and without xref / yref / dy and bias, pool / up at both scales, the three loss modes with
    and without mask and gradient, the histogram's prior / no-prior coefficients, and Adam chunks with and without a gradient
    (`e.g == nullptr`) and an EMA (`e.ema == nullptr`), which `ADAM_PLAN` holds."""
    fwd = [r for r in BA if r["op"] == "fwd"]
    grad = [r for r in BA if r["op"] != "fwd"]
    assert {r["bias"] for r in fwd} == {"none", "vec", "scalar"}
    assert {r["act"] for r in fwd} == set(ACT_NAMES) and {r["act"] for r in grad if r["op"] == "grad1"} == set(ACT_NAMES)
    assert {r["act"] for r in grad if r["op"] == "grad2"} == {a for a in ACT_NAMES if _second(a)}
    for rows in (fwd, grad):
        assert {r["clamp"] for r in rows} == {0, 1}
        assert {r["tail"] for r in rows} == {0, 1, 2, 3}
        assert {r["size"] for r in rows} == {"ragged", "trip"}
    pats = {_ba_launch_args(r) for r in grad}
    assert any(p[0] for p in pats) and any(not p[0] for p in pats)         # a bias in the grad kernel, and none
    assert {p[1] for p in pats} == {True, False} and {p[2] for p in pats} == {True, False} and {p[3] for p in pats} == {True, False}
    assert {u for u, _ in RESAMPLE} == {0, 1} and {s for _, s in RESAMPLE} == {0.25, 1.0}
    assert {(r["mode"], r["mask"], r["grad"]) for r in IMAGE_LOSS} == set(itertools.product((0, 1, 2), (0, 1), (1, 0)))
    assert {r["prior"] for r in SEG_CE} == {0, 1} and {r["grad"] for r in SEG_CE} == {0, 1}
    assert {r["ema"] for r in ADAM} == {0, 1}
    has_grad = {ADAM_PLAN["grad"](i, k) for i in range(len(ADAM_PLAN["sizes"])) for k in range(ADAM_PLAN["steps"])}
    assert has_grad == {True, False}


# ----------------------------------------------------------------------------------------------------------------------
# 1. hg_bias_act / hg_bias_act_grad
# ----------------------------------------------------------------------------------------------------------------------
# fp32 roundings of act_apply (csrc/elementwise.cu) relative to |act(t)|, from the CUDA math library's maximum ulp errors
# (tanhf 2, expf 2, expm1f 1, log1pf 1; an ulp is at most 2u relative): tanh 2u*2; sigmoid 1/(1+expf(-t)): expf's error scaled
# by e/(1+e) <= 1, the add and the division, 4u+2u; elu 2u; selu expm1f, two products: 2u+2u; softplus log1pf(expf(t)):
# expf's relative error passes through log1p with a factor <= 1, then log1pf, 4u+2u; swish as sigmoid.  lrelu one product.
K_FWD = {"linear": 0, "relu": 0, "lrelu": 1, "tanh": 4, "sigmoid": 6, "elu": 2, "selu": 4, "softplus": 6, "swish": 6}
KS, KSA_A = _f32(1.0507009873554805), _f32(1.6732632423543772)
KSA = _f32(KS * KSA_A)


def _act64(act, t, alpha):
    if act == "linear":
        return t
    if act == "relu":
        return torch.clamp_min(t, 0.0)
    if act == "lrelu":
        return torch.where(t > 0, t, t * alpha)
    if act == "tanh":
        return torch.tanh(t)
    if act == "sigmoid":
        return torch.sigmoid(t)
    if act == "elu":
        return torch.where(t > 0, t, torch.expm1(t))
    if act == "selu":
        return KS * torch.where(t > 0, t, KSA_A * torch.expm1(t))
    if act == "softplus":
        return torch.where(t > 20, t, torch.log1p(torch.exp(t)))
    return t * torch.sigmoid(t)


def _dact64(act, t, alpha):
    """|act'(t)|, for the effect of the rounded x + b."""
    if act in ("linear",):
        return torch.ones_like(t)
    if act == "relu":
        return (t > 0).double()
    if act == "lrelu":
        return torch.where(t > 0, 1.0, abs(alpha))
    if act == "tanh":
        return 1 - torch.tanh(t) ** 2
    if act == "sigmoid":
        s = torch.sigmoid(t)
        return s * (1 - s)
    if act == "elu":
        return torch.where(t > 0, 1.0, torch.exp(t))
    if act == "selu":
        return KS * torch.where(t > 0, 1.0, KSA_A * torch.exp(t))
    if act == "softplus":
        return torch.sigmoid(t)
    s = torch.sigmoid(t)
    return (s * (1 + t * (1 - s))).abs()


def _deriv64(act, order, yy, t, alpha):
    """act_derivative's contract in fp64 (in terms of the saved output yy = y / gain, swish of t) -> (D, M, k, sens): the
    value, the sum of |terms| its fp32 evaluation rounds, the count of roundings on M, and the variable whose rounding
    error perturbs D (yy carries 2u from y * (1/gain); t carries u from x + b)."""
    one = torch.ones_like(yy)
    if act in ("linear", "relu", "lrelu"):
        if order == 2:
            return 0 * one, 0 * one, 0, None
        if act == "linear":
            return one, 0 * one, 0, None
        return torch.where(yy > 0, 1.0, 0.0 if act == "relu" else alpha), 0 * one, 0, None
    if act == "tanh":
        if order == 1:
            return 1 - yy * yy, 1 + yy * yy, 2, "yy"
        return (1 - yy * yy) * (-2 * yy), (1 + yy * yy) * 2 * yy.abs(), 4, "yy"
    if act == "sigmoid":
        a = yy.abs()
        if order == 1:
            return yy * (1 - yy), a * (1 + a), 2, "yy"
        return yy * (1 - yy) * (1 - 2 * yy), a * (1 + a) * (1 + 2 * a), 5, "yy"
    if act in ("elu", "selu"):
        pos = yy >= 0
        c = 1.0 if act == "elu" else KSA
        if order == 1:
            return torch.where(pos, 1.0 if act == "elu" else KS, yy + c), torch.where(pos, 0.0, yy.abs() + c), 1, "yy"
        return torch.where(pos, 0.0, yy + c), torch.where(pos, 0.0, yy.abs() + c), 1, "yy"
    if act == "softplus":
        c = torch.exp(-yy)                 # expf: 2 ulp = 4u on c
        if order == 1:
            return 1 - c, 1 + 4 * c, 3, "yy"
        return c * (1 - c), c * (1 + c) * 4, 4, "yy"
    s = torch.sigmoid(t)                   # 1 / (1 + expf(-t)): 4u + 2u
    if order == 1:
        return s * (1 + t * (1 - s)), s * (1 + t.abs() * (1 + s)) * 6, 3, "t"
    q = s * (1 - s)
    return 2 * q + t * q * (1 - 2 * s), s * (1 + s) * (2 + t.abs() * (1 + 2 * s)) * 6, 6, "t"


def _ba_shape(n_target, bias, tail):
    """(B, C, HW) with B*C*HW >= n_target, the bias along C (stepB = HW), HW % 4 == 0 exactly when the bias is per float4, and
    B*C*HW % 4 == tail."""
    for B, C in ((1, 33), (2, 33), (4, 33), (1, 34), (1, 36)):
        HW = max(1, -(-n_target // (B * C)))
        for h in range(HW, HW + 8):
            if bias == "vec" and h % 4:
                continue
            if bias == "scalar" and h % 4 == 0:
                continue
            if (B * C * h) % 4 == tail:
                return B, C, h
    raise AssertionError((n_target, bias, tail))


def _ba_trip(op):
    """Elements one trip of the capped grid covers: 32 CTAs per SM x 256 threads x 2 float4 (forward) / 1 float4 (gradient)."""
    return _nsm() * 32 * 256 * 4 * (2 if op == "fwd" else 1)


def _ba_fwd_ref(act, x, b, C, HW, alpha, gain, clamp):
    t = x.double()
    mag_t = x.double().abs()
    if b is not None:
        bb = b.double().view(1, C, 1)
        t = t + bb
        mag_t = mag_t + bb.abs()
    a = _act64(act, t, alpha)
    # the rounded x + b moves act by |act'| u |x + b| <= |act'| u (|x| + |b|); act_apply's own roundings and the gain product
    bound = gain * _dact64(act, t, alpha) * U * mag_t + (K_FWD[act] + 1) * U * gain * a.abs()
    y = a * gain
    if clamp >= 0:
        y = y.clamp(-clamp, clamp)
    return y, 2 * bound + 1e-37


def _ba_grad_ref(act, order, g, t, yref, dy, alpha, gain, clamp, y_swish=None):
    gain_inv = 1.0 / gain
    yy = yref.double() * gain_inv if yref is not None else torch.zeros_like(g, dtype=torch.float64)
    D, M, k, sens = _deriv64(act, order, yy, t, alpha)
    errD = k * U * M
    if sens is not None:                   # the rounded input of D: a central difference of D at +-h relative
        h = 2.0 ** -20
        if sens == "yy":
            dp, dm = _deriv64(act, order, yy * (1 + h), t, alpha)[0], _deriv64(act, order, yy * (1 - h), t, alpha)[0]
            errD = errD + 2 * U * (dp - dm).abs() / (2 * h)
        else:
            dp, dm = _deriv64(act, order, yy, t * (1 + h), alpha)[0], _deriv64(act, order, yy, t * (1 - h), alpha)[0]
            errD = errD + U * (dp - dm).abs() / (2 * h)
    scale = g.double() * gain * (dy.double() if dy is not None else 1.0)
    ref = scale * D
    bound = scale.abs() * errD + 3 * U * ref.abs()        # (g * gain) * D * dy: three products
    amb = None
    if clamp >= 0:
        ymask = (y_swish if act == "swish" else yref).double()
        keep = ymask.abs() < clamp
        ref = torch.where(keep, ref, 0.0)
        if act == "swish":                 # the kernel rebuilds y in fp32: near |y| = clamp either side of the mask is right
            amb = (ymask.abs() - clamp).abs() <= 16 * U * clamp
    return ref, 2 * bound + 1e-37, amb


def _ba_case(v, seed):
    abi = _abi()
    act = v["act"]
    aid, alpha, gain = _ba_table()[act][:3]
    alpha, gain = _f32(alpha), _f32(gain)
    clamp = 2.5 if v["clamp"] else -1.0
    n_target = 4 * 331 + 7 if v["size"] == "ragged" else _ba_trip(v["op"]) + 4 * 2048 + 5
    B, C, HW = _ba_shape(n_target, v["bias"], v["tail"])
    n = B * C * HW
    r = _rnd(seed)
    x = 3 * r(B, C, HW)
    b = r(C) if v["bias"] != "none" else None
    step, size = HW, (C if b is not None else 1)
    has_b, has_x, has_y, has_dy = _ba_launch_args(v)
    # the forward output the module saves (yref): this very kernel's
    y = torch.empty_like(x)
    abi.call("hg_bias_act", abi.ptr(x), abi.ptr(b), abi.ptr(y), n, step, size, aid, alpha, gain, clamp, abi.stream())
    if v["op"] == "fwd":
        buf, out = _guarded((B, C, HW))
        abi.call("hg_bias_act", abi.ptr(x), abi.ptr(b), abi.ptr(out), n, step, size, aid, alpha, gain, clamp, abi.stream())
        torch.cuda.synchronize()
        assert _intact(buf), "a guard element was overwritten"
        assert not torch.isnan(out).any(), "an element was not written"
        ref, bound = _ba_fwd_ref(act, x, b, C, HW, alpha, gain, clamp)
        return _check(f"bias_act {_vid(v)} n={n}", (out.double() - ref).abs(), bound)
    g = r(B, C, HW)
    dy = r(B, C, HW) if has_dy else None
    buf, out = _guarded((B, C, HW))
    bb = b if has_b else None
    abi.call("hg_bias_act_grad", abi.ptr(g), abi.ptr(bb), abi.ptr(x if has_x else None), abi.ptr(y if has_y else None), abi.ptr(dy),
             abi.ptr(out), n, step, C if bb is not None else 1, 2 if v["op"] == "grad2" else 1, aid, alpha, gain, clamp, abi.stream())
    torch.cuda.synchronize()
    assert _intact(buf), "a guard element was overwritten"
    assert not torch.isnan(out).any(), "an element was not written"
    t = x.double() + (bb.double().view(1, C, 1) if bb is not None else 0.0)
    if not has_x:
        t = torch.zeros_like(t)
    ref, bound, amb = _ba_grad_ref(act, 2 if v["op"] == "grad2" else 1, g, t, y if has_y else None, dy, alpha, gain, clamp,
                                   y_swish=y if act == "swish" else None)
    err = (out.double() - ref).abs()
    if amb is not None:
        err = torch.where(amb & (out == 0), 0.0, err)
    return _check(f"bias_act_grad {_vid(v)} n={n}", err, bound)


@gpu
@pytest.mark.parametrize("v", BA, ids=_vid)
def test_bias_act(v):
    _ba_case(v, 100 + BA.index(v))


# the real sizes: the discriminator's LeakyReLU (no bias, alpha 0.2, gain 1) at its largest activations, and the VGG16 ReLU
BA_REAL = [("lrelu", (32, 64, 512, 256)), ("lrelu", (8, 64, 512, 512)), ("relu", (8, 64, 224, 224))]


@gpu
@pytest.mark.parametrize("act,shape", BA_REAL, ids=lambda a: "x".join(map(str, a)) if isinstance(a, tuple) else a)
def test_bias_act_real_sizes(act, shape):
    """Forward and first-order gradient (the form the D's backward and its R1 double backward both issue) at the real sizes,
    where every thread of the capped grid takes many trips; the fp64 reference in slices."""
    abi = _abi()
    aid = _ba_table()[act][0]
    alpha, gain = (0.2, 1.0) if act == "lrelu" else (0.0, 1.0)
    alpha = _f32(alpha)
    n = math.prod(shape)
    r = _rnd(150)
    x = r(n)
    ybuf, y = _guarded((n,))
    abi.call("hg_bias_act", abi.ptr(x), None, abi.ptr(y), n, 1, 1, aid, alpha, gain, -1.0, abi.stream())
    torch.cuda.synchronize()
    assert _intact(ybuf) and not torch.isnan(y).any()
    worst = 0.0
    for s in _slices(n):
        ref, bound = _ba_fwd_ref(act, x[s].view(1, 1, -1), None, 1, 1, alpha, gain, -1.0)
        worst = max(worst, (( y[s].double() - ref.view(-1)).abs() / bound.view(-1)).max().item())
    print(f"  {act} {shape} forward: {worst:.3f} of the bound, {-(-n // _ba_trip('fwd'))} trips")
    assert worst <= 1.0
    del x
    g = r(n)
    obuf, out = _guarded((n,))
    abi.call("hg_bias_act_grad", abi.ptr(g), None, None, abi.ptr(y), None, abi.ptr(out), n, 1, 1, 1, aid, alpha, gain, -1.0, abi.stream())
    torch.cuda.synchronize()
    assert _intact(obuf) and not torch.isnan(out).any()
    for s in _slices(n):                  # (g * gain) * mask * 1: exact up to the product by alpha (one rounding)
        ref = g[s].double() * gain * torch.where(y[s] > 0, 1.0, alpha)
        assert ((out[s].double() - ref).abs() <= 2 * U * ref.abs()).all(), "gradient"
    print(f"  {act} {shape} gradient: within 2u, {-(-n // _ba_trip('grad'))} trips")


# ----------------------------------------------------------------------------------------------------------------------
# 2. hg_resample2x and the upfirdn2d fallback
# ----------------------------------------------------------------------------------------------------------------------
def _d_resample_forms(cfg):
    """(up, scale, C, H, W) of every hg_resample2x launch a discriminator forward, backward and R1 double backward issue at the
    config's image size, read off the module's weights as discriminator_forward_train walks them."""
    disc = importlib.import_module("3dhumangan_b200.modules.discriminator")
    P = disc.UNetDiscriminator(**cfg).state_dict()
    H, W = cfg["gen_height"], cfg["gen_width"]
    out_ch = lambda n: P[n + ".weight_orig"].shape[0] if n + ".weight_orig" in P else P[n + ".weight"].shape[0]
    fwd = []
    C = 3
    nb = sum(1 for k in P if k.startswith("body_down.") and k.endswith("conv2.1.weight_orig"))
    for i in range(nb):
        Co = out_ch(f"body_down.{i}.conv2.1")
        fwd.append((0, 0.25, C if i == 0 else Co, H, W))       # the shortcut: pool(x) then conv_s / pool(conv_s(x))
        fwd.append((0, 0.25, Co, H, W))                          # the residual branch
        C, H, W = Co, H // 2, W // 2
    for i in range(nb):
        Cin = P[f"body_up.{i}.conv1.2.weight_orig"].shape[1]
        Co = out_ch(f"body_up.{i}.conv2.1")
        learned = f"body_up.{i}.conv_s.bias" in P
        fwd.append((1, 1.0, Co if learned else Cin, H, W))
        fwd.append((1, 1.0, Cin, H, W))
        C, H, W = Co, 2 * H, 2 * W
    forms = set()
    for up, s, C_, H_, W_ in fwd:
        forms.add((up, s, C_, H_, W_))
        forms.add((1, s, C_, H_ // 2, W_ // 2) if not up else (0, s, C_, 2 * H_, 2 * W_))     # the adjoint, at the same scale
    return sorted(forms)


def _cfg(which):
    pkg = importlib.import_module("3dhumangan_b200")
    if which == "MAP3DBN":
        return pkg.configs.extract_metadata(copy.deepcopy(pkg.configs.MAP3DBN), 0)
    return pkg.configs.baseline_config(which)


def _resample_check(up, scale, planes, H, W, x):
    abi = _abi()
    oshape = (planes, 2 * H, 2 * W) if up else (planes, H // 2, W // 2)
    buf, y = _guarded(oshape)
    abi.call("hg_resample2x", abi.ptr(x), abi.ptr(y), planes, H, W, up, scale, abi.stream())
    torch.cuda.synchronize()
    assert _intact(buf), "a guard element was overwritten"
    worst = 0.0
    step = max(1, (1 << 24) // (4 * H * W))
    for a in range(0, planes, step):
        xs, ys = x[a:a + step], y[a:a + step]
        if up:                             # copies times an exact power of two: bit-exact
            ref = (xs * scale).repeat_interleave(2, 1).repeat_interleave(2, 2)
            assert torch.equal(ys, ref), f"up-sampling planes {a}.. differ"
        else:                              # ((a + b) + (c + d)) * scale, scale a power of two: three roundings, the inner two on
            q = xs.double().view(-1, H // 2, 2, W // 2, 2)            # |a + b| and |c + d|, the outer on their sum: <= (2u + u^2) sum|x|
            ref = q.sum((2, 4)) * scale
            bound = (2 * U + U * U) * q.abs().sum((2, 4)) * scale + 1e-300
            assert not torch.isnan(ys).any(), "an element was not written"
            worst = max(worst, ((ys.double() - ref).abs() / bound).max().item())
    assert worst <= 1.0, worst
    return worst


@gpu
@pytest.mark.parametrize("which", ["MAP3DBN", "C2native"])
def test_resample2x_discriminator_sizes(which):
    """Every pooling / up-sampling form of the discriminator at B = 32 and the config's image size (256x128 / 512x256)."""
    forms = _d_resample_forms(_cfg(which))
    r = _rnd(200)
    worst = 0.0
    for up, scale, C_, H, W in forms:
        assert (W % 2 == 0) if up else (H % 2 == 0 and W % 4 == 0), "a D size would take the upfirdn2d fallback"
        x = r(32 * C_, H, W)
        worst = max(worst, _resample_check(up, scale, 32 * C_, H, W, x))
        del x
        torch.cuda.empty_cache()
    print(f"  {which}: {len(forms)} forms, pooling worst {worst:.3f} of the bound")


@gpu
@pytest.mark.parametrize("up,scale", RESAMPLE)
@pytest.mark.parametrize("hw", [(2, 4), (2, 2), (4, 8), (6, 12), (34, 36)])
def test_resample2x_small(up, scale, hw):
    """The smallest maps `_pool` (H even, W % 4 == 0) and `_up` (W even) still send to this kernel, and a few planes' ragged
    grid."""
    H, W = hw
    if not up and W % 4:
        pytest.skip("pooling needs W % 4 == 0")
    x = _rnd(210)(5, H, W)
    _resample_check(up, scale, 5, H, W, x)


@gpu
@pytest.mark.parametrize("kind,hw", [("pool", (6, 2)), ("pool", (7, 8)), ("pool", (5, 6)), ("up", (3, 5)), ("up", (4, 1))])
def test_resample_fallback_shapes(kind, hw):
    """The shapes `_pool` / `_up` send to hg_upfirdn2d (W = 2 or W % 4 != 0, odd H; odd W), forward and adjoint through
    autograd, against avg_pool2d / nearest up-sampling in fp64."""
    dt = importlib.import_module("3dhumangan_b200.modules.discriminator_train")
    H, W = hw
    r = _rnd(220)
    x = r(2, 3, H, W).requires_grad_(True)
    fn = dt._pool if kind == "pool" else dt._up
    y = fn(x)
    xd = x.detach().double().requires_grad_(True)
    yd = F.avg_pool2d(xd, 2) if kind == "pool" else F.interpolate(xd, scale_factor=2, mode="nearest")
    assert y.shape == yd.shape, (y.shape, yd.shape)
    gy = r(*y.shape)
    (gx,) = torch.autograd.grad(y, x, gy)
    (gxd,) = torch.autograd.grad(yd, xd, gy.double())
    torch.cuda.synchronize()
    # 4 fp32 taps (3 roundings, the filter's 0.25 exact) forward; the adjoint sums at most 4 products of exact 0.25 / 1
    mag = F.avg_pool2d(xd.abs(), 2) if kind == "pool" else F.interpolate(xd.abs(), scale_factor=2, mode="nearest")
    _check(f"fallback {kind} {H}x{W}: y", (y.double() - yd).abs(), 3 * U * mag + 1e-300)
    gmag = (F.interpolate(gy.double().abs(), scale_factor=2, mode="nearest") * 0.25 if kind == "pool" else
            F.avg_pool2d(gy.double().abs(), 2) * 4)
    if kind == "pool" and gmag.shape != gxd.shape:
        gmag = F.pad(gmag, (0, W - gmag.shape[3], 0, H - gmag.shape[2]))
    _check(f"fallback {kind} {H}x{W}: dx", (gx.double() - gxd).abs(), 3 * U * gmag + 1e-300)


# ----------------------------------------------------------------------------------------------------------------------
# 3. hg_spectral_norm
# ----------------------------------------------------------------------------------------------------------------------
def _sn_launch(ws, us, vs, training):
    """hg_spectral_norm on a table built as abi.spectral_norm builds it; inv_sigma guarded and NaN-filled."""
    abi = _abi()
    tab = np.zeros((len(ws), 4), dtype=np.int64)
    for i, (w, u, v) in enumerate(zip(ws, us, vs)):
        N = w.shape[0]
        tab[i] = (w.data_ptr(), u.data_ptr(), v.data_ptr(), N | ((w.numel() // N) << 32))
    table = torch.from_numpy(tab).cuda()
    buf, inv = _guarded((len(ws),))
    abi.call("hg_spectral_norm", abi.ptr(table), len(ws), max(w.shape[0] for w in ws), max(w.numel() // w.shape[0] for w in ws),
             abi.ptr(inv), int(training), EPS_SN, abi.stream())
    torch.cuda.synchronize()
    assert _intact(buf), "a guard element of inv_sigma was overwritten"
    return inv


def _sn_ref_step(W, u, v, training, v_new=None):
    """torch.nn.utils.spectral_norm's hook in fp64 on the same u / v, and componentwise bounds of the kernel's fp32 arithmetic.
    v_new: the kernel's own new v, from which u and sigma are checked (launch by launch within the launch)."""
    N, K = W.shape
    Wd, ud, vd = W.double(), u.double(), v.double()
    out = {}
    if training:
        t = Wd.t() @ ud
        # one fp32 fma chain per column over a group's slice of the N rows, then the <= 32 groups' partials: (N + 32) u sum |W||u|
        e_t = (N + 32) * U * (Wd.abs().t() @ ud.abs())
        nt = t.norm()
        out["v"] = F.normalize(t, dim=0, eps=EPS_SN)
        # the normalisation: the perturbation e_t moves t / |t| by e_t/|t| + |v| (|v|.e_t)/|t|; the norm's own sum (K/1024
        # fma per thread, a 10-level tree), sqrt, reciprocal and product: (K/1024 + 14) u |v|
        vn = out["v"]
        out["v_bound"] = e_t / nt + vn.abs() * (vn.abs() @ e_t) / nt + (K / 1024 + 14) * U * vn.abs()
        vd = v_new.double()
    s = Wd @ vd
    e_s = (K / 32 + 5) * U * (Wd.abs() @ vd.abs())           # a lane's K/32 fmas, a 5-level shuffle tree
    if training:
        ns = s.norm()
        out["u"] = F.normalize(s, dim=0, eps=EPS_SN)
        un = out["u"]
        out["u_bound"] = e_s / ns + un.abs() * (un.abs() @ e_s) / ns + (N / 1024 + 14) * U * un.abs()
        sigma = torch.dot(out["u"], s)                          # = |W v|
        rel = (un.abs() @ e_s) / ns + (N / 1024 + 14) * U
    else:
        sigma = torch.dot(ud, s)
        rel = ((ud.abs() @ e_s) + (N / 1024 + 12) * U * (ud.abs() @ s.abs())) / sigma.abs()
    out["inv"] = 1.0 / sigma
    out["inv_bound"] = (rel + 2 * U) / sigma.abs()
    return out


def _sn_tables():
    """The C2 generator's 18 synthesis convolutions (in synthesis_ops' order) and the C2 discriminator's 32 convolutions (in
    sn_layer_names order), as the modules build their one launch each: weight_orig viewed [N, K], u [N], v [K]."""
    gen = importlib.import_module("3dhumangan_b200.modules.generator")
    disc = importlib.import_module("3dhumangan_b200.modules.discriminator")
    dops = importlib.import_module("3dhumangan_b200.modules.discriminator_ops")
    cfg = _cfg("C2")
    torch.manual_seed(300)
    Gs = gen.Map3DGenerator(**cfg).state_dict()
    nb = cfg["synthesis_blocks"]
    gnames = [f"synthesis_network.network.m3d_{k}.conv_{j}." for k in range(nb) for j in range(2)]
    Ds = disc.UNetDiscriminator(**cfg).state_dict()
    dnames = [n + "." for n in dops.sn_layer_names(Ds)]
    tabs = {}
    for tag, P, names in (("G", Gs, gnames), ("D", Ds, dnames)):
        tabs[tag] = [(P[n + "weight_orig"].cuda().contiguous(), P[n + "weight_u"].cuda().contiguous(), P[n + "weight_v"].cuda().contiguous())
                     for n in names]
    return tabs


def _sn_run(tag, entries, steps=5):
    ws = [w for w, _, _ in entries]
    # u / v live inside guarded buffers: the kernel writes them in place
    ubufs, us, vbufs, vs = [], [], [], []
    for w, u, v in entries:
        b, t = _guarded(tuple(u.shape))
        t.copy_(u)
        ubufs.append(b)
        us.append(t)
        b, t = _guarded(tuple(v.shape))
        t.copy_(v)
        vbufs.append(b)
        vs.append(t)
    worst = {"u": 0.0, "v": 0.0, "inv": 0.0}
    for step in range(steps + 1):
        training = step < steps
        u0, v0 = [u.clone() for u in us], [v.clone() for v in vs]
        inv = _sn_launch(ws, us, vs, training)
        assert all(_intact(b) for b in ubufs + vbufs), "a guard element of u / v was overwritten"
        # repeat identity: the same launch from the same u / v
        u1, v1 = [u.clone() for u in us], [v.clone() for v in vs]
        for a, b in zip(us + vs, u0 + v0):
            a.copy_(b)
        inv2 = _sn_launch(ws, us, vs, training)
        assert torch.equal(inv, inv2), "a repeated launch changed inv_sigma"
        assert all(torch.equal(a, b) for a, b in zip(us + vs, u1 + v1)), "a repeated launch changed u / v"
        for i, w in enumerate(ws):
            Wm = w.reshape(w.shape[0], -1)
            ref = _sn_ref_step(Wm, u0[i], v0[i], training, v_new=vs[i] if training else None)
            if training:
                worst["v"] = max(worst["v"], _ratio(vs[i], ref["v"], ref["v_bound"], f"{tag}[{i}] step {step}: v"))
                worst["u"] = max(worst["u"], _ratio(us[i], ref["u"], ref["u_bound"], f"{tag}[{i}] step {step}: u"))
            else:
                assert torch.equal(us[i], u0[i]) and torch.equal(vs[i], v0[i]), "eval mode changed u / v"
            worst["inv"] = max(worst["inv"], _ratio(inv[i:i + 1], ref["inv"].view(1), ref["inv_bound"].view(1),
                                                   f"{tag}[{i}] step {step}: inv_sigma"))
    print(f"  {tag}: {len(ws)} matrices, {steps} training steps + eval, worst of the bound {worst}")


def _ratio(got, ref, bound, name):
    assert not torch.isnan(got).any(), f"{name}: not written"
    r = ((got.double() - ref).abs() / (2 * bound + 1e-300)).max().item()
    assert r <= 1.0, f"{name}: error {r:.3f}x the bound"
    return r


@gpu
def test_spectral_norm_c2_tables():
    """The C2 G (18 x [256, 256]) and D (32 matrices up to [256, 9216] at 512x512) tables: five training launches in a row,
    each checked from the u / v it started from, then one eval launch; repeat identity on every launch."""
    tabs = _sn_tables()
    assert len(tabs["G"]) == 18 and len(tabs["D"]) == 32
    assert max(w.numel() // w.shape[0] for w, _, _ in tabs["D"]) == 9216          # body_up.1.conv1.2: 3x3 over 1024 channels
    for tag in ("G", "D"):
        _sn_run(tag, tabs[tag])


@gpu
def test_spectral_norm_mixed_groups_table():
    """One launch where the large K (4 608 and the D's largest, 9 216: columns strided over the CTA) share the table with
    K < 1024 matrices (row slices per thread group, summed in shared memory) and an N > K matrix."""
    r = _rnd(310)
    shapes = [(512, 4608), (128, 27), (256, 9216), (64, 576), (3, 64), (1024, 96), (256, 1000)]
    entries = []
    for n, k in shapes:
        entries.append((r(n, k) / k ** 0.5, F.normalize(r(n), dim=0), F.normalize(r(k), dim=0)))
    _sn_run("mixed", entries, steps=2)


# ----------------------------------------------------------------------------------------------------------------------
# 4. hg_label_histogram -> hg_seg_ce_coef -> hg_seg_ce
# ----------------------------------------------------------------------------------------------------------------------
def _labels(kind, B, L, H, W, seed):
    g = torch.Generator().manual_seed(seed)
    if kind == "random":                   # two classes never occur
        lab = torch.randint(0, L, (B, H, W), generator=g)
        lab[(lab == 7) | (lab == 19)] = 0
    elif kind == "background":
        lab = torch.zeros(B, H, W, dtype=torch.int64)
    elif kind == "once":                   # background, one class everywhere else, one class at one pixel
        lab = torch.where(torch.rand(B, H, W, generator=g) < 0.5, 0, 3)
        lab[B - 1, H - 1, W - 1] = 11
    else:                                  # "stripes": the class changes at every pixel
        lab = (torch.arange(B * H * W) % L).view(B, H, W)
    return lab.cuda()


def _seg_case(B, L, H, W, kind, prior_on, seed, grad=True):
    abi = _abi()
    HW = H * W
    total = B * HW
    r = _rnd(seed)
    logits = 3 * r(B, L, H, W)
    labels = _labels(kind, B, L, H, W, seed)
    prior = (1.0 + 0.1 * torch.arange(L, device="cuda", dtype=torch.float32)) if prior_on else None
    # histogram: exact
    hbuf = torch.full((L + 2 * G,), -7, dtype=torch.int32, device="cuda")
    hist = hbuf[G:G + L]
    hist.fill_(-1)
    abi.call("hg_label_histogram", abi.ptr(labels), total, L, abi.ptr(hist), abi.stream())
    torch.cuda.synchronize()
    assert (hbuf[:G] == -7).all() and (hbuf[-G:] == -7).all(), "a guard element of the histogram was overwritten"
    ref_hist = torch.bincount(labels.reshape(-1), minlength=L)[:L]
    assert torch.equal(hist.long(), ref_hist), "label histogram"
    # coefficients: the reference's formula in fp64 from the exact histogram
    cbuf, coef = _guarded((L,))
    abi.call("hg_seg_ce_coef", abi.ptr(hist), abi.ptr(prior), L, float(total), abi.ptr(coef), abi.stream())
    torch.cuda.synchronize()
    assert _intact(cbuf) and not torch.isnan(coef).any()
    occ = ref_hist.double().clone()
    occ[0] = 0
    n_occ = int((occ > 0).sum())
    pw = prior.double() if prior is not None else torch.ones(L, dtype=torch.float64, device="cuda")
    pw = pw / pw.mean()
    if n_occ == 0:
        cref = torch.ones(L, dtype=torch.float64, device="cuda")
    else:
        cref = torch.where(occ > 0, total / (occ * n_occ), 0.0) * pw
    # numel / (occ n_occ) in fp64 rounded to fp32 (u), the prior's fp32 mean (a sequential sum of L terms and a division:
    # (L + 1) u), the quotient and the product (2u)
    _check(f"seg_ce_coef {kind} prior{int(prior_on)}", (coef.double() - cref).abs(), 2 * (L + 4) * U * cref.abs() + 1e-300)
    # loss and dlogits from the kernel's own coefficients
    ld = logits.double().view(B, L, HW)
    lab = labels.view(B, 1, HW)
    cd = coef.double()
    runs = []
    for _ in range(2):
        dbuf, dlog = _guarded((B, L, H, W)) if grad else (None, None)
        lbuf, loss = _guarded((1,))
        ws = torch.empty(2 * 160 * 2, dtype=torch.float64, device="cuda")
        abi.call("hg_seg_ce", abi.ptr(logits), abi.ptr(labels), abi.ptr(coef), abi.ptr(dlog), abi.ptr(loss), abi.ptr(ws), B, L, HW,
                 abi.stream())
        torch.cuda.synchronize()
        assert _intact(lbuf) and (dbuf is None or _intact(dbuf)), "a guard element was overwritten"
        runs.append((loss.clone(), dlog))
    assert torch.equal(runs[0][0], runs[1][0]), "a repeated launch changed the loss"
    if grad:
        assert torch.equal(runs[0][1], runs[1][1]), "a repeated launch changed dlogits"
    loss, dlog = runs[0]
    # per pixel: x_c = fl(v_c - m) (u |x_c|), __expf: 2 + floor(1.173 |x|) ulp (CUDA C Programming Guide, intrinsic functions),
    # an ulp <= 2u relative; s: L - 1 adds; __logf: 2^-21.41 absolute for s in [0.5, 2], 3 ulp otherwise; m + log s - xg: two
    # roundings; w * (): one; the fp32 per-pixel value is summed in fp64 and the mean rounded to fp32 once
    acc = torch.zeros((), dtype=torch.float64, device="cuda")
    acc_b = torch.zeros((), dtype=torch.float64, device="cuda")
    worst_d = 0.0
    scale = 1.0 / total
    for b in range(B):
        x = ld[b]                                                   # [L, HW]
        m = x.max(0).values
        xm = x - m
        e = torch.exp(xm)
        rel_e = U * xm.abs() + 2 * U * (2 + torch.floor(1.173 * xm.abs()))
        s = e.sum(0)
        ds = (e * rel_e).sum(0) + (L - 1) * U * s
        logerr = torch.where((s >= 0.5) & (s <= 2), 2.0 ** -21.41, 6 * U * torch.log(s).abs())
        gt = lab[b, 0]
        xg = x.gather(0, gt[None])[0]
        w = cd[gt]
        ce = m + torch.log(s) - xg
        acc = acc + (w * ce).sum()
        acc_b = acc_b + (w * (ds / s + logerr + 2 * U * (m.abs() + torch.log(s).abs() + xg.abs()) + U * ce.abs())).sum()
        if grad:
            p = e / s
            onehot = torch.zeros_like(x).scatter_(0, gt[None], 1.0)
            dref = w * scale * (p - onehot)
            # k = (w * fl(1/total)) / s: 3 roundings and s's error; v_c's error; the product and the subtraction
            db = w * scale * (p * (3 * U + ds / s + rel_e + U) + U * (p + onehot) + 2 * U * onehot)
            got = dlog[b].view(L, HW).double()
            assert not torch.isnan(got).any(), "an element of dlogits was not written"
            worst_d = max(worst_d, ((got - dref).abs() / (2 * db + 1e-300)).max().item())
    lref = acc / total
    lbound = acc_b / total + U * lref.abs()
    r_loss = _check(f"seg_ce {kind} prior{int(prior_on)} {B}x{L}x{H}x{W}: loss", (loss.double() - lref).abs(), 2 * lbound)
    if grad:
        print(f"  dlogits: {worst_d:.3f} of the bound, {-(-total // (2 * _nsm() * 256))} trips")
        assert worst_d <= 1.0, worst_d
    return r_loss


@gpu
@pytest.mark.parametrize("prior", [0, 1])
@pytest.mark.parametrize("hw", [(256, 128), (512, 256)])
def test_seg_ce_training_sizes(hw, prior):
    """L = 26 at the curricula's [32, 26, 256, 128] and [32, 26, 512, 256] (4.2 M pixels: 63 trips of the 2-CTA/SM grid)."""
    _seg_case(32, 26, hw[0], hw[1], "random", prior, 400 + prior)


@gpu
@pytest.mark.parametrize("kind", ["random", "background", "once", "stripes"])
@pytest.mark.parametrize("prior", [0, 1])
def test_seg_ce_label_maps(kind, prior):
    """A ragged HW (37 x 29, not a multiple of 256), every edge of the coefficient table: no foreground (plain mean CE), a class
    that occurs once, classes that never occur, a class change at every pixel; the launch without dlogits too."""
    _seg_case(3, 26, 37, 29, kind, prior, 410 + prior)
    _seg_case(3, 26, 37, 29, kind, prior, 420 + prior, grad=False)


# ----------------------------------------------------------------------------------------------------------------------
# 5. hg_image_loss
# ----------------------------------------------------------------------------------------------------------------------
def _rho64(mode, d, eps):
    """(rho, rho', bound terms) in fp64; k: the roundings of the kernel's rho on |rho| and of drho on |drho|, sec: |rho''|."""
    z = d.abs()
    if mode == 0:
        return d * d, 2 * d, 1, 0, 2 * torch.ones_like(d)
    if mode == 1:
        rho = torch.sqrt(d * d + eps * eps)
        return rho, d / rho, 4, 5, eps * eps / rho ** 3          # eps*eps, fma, sqrt; + the division
    inside = z < eps
    rho = torch.where(inside, 0.5 * z * z / eps, z - 0.5 * eps)
    drho = torch.where(inside, d / eps, torch.sign(d))
    return rho, drho, 4, 1, torch.full_like(d, 1.0 / eps)       # |rho''| <= 1/beta on both sides of the kink


@gpu
@pytest.mark.parametrize("v", IMAGE_LOSS, ids=_vid)
@pytest.mark.parametrize("hw", [(512, 256), (512, 512)])
def test_image_loss(v, hw):
    abi = _abi()
    mode = v["mode"]
    eps = {0: 0.0, 1: _f32(1e-3), 2: _f32(0.1)}[mode]
    B, H, W = 8, hw[0], hw[1]
    HW = H * W
    total = B * 3 * HW
    r = _rnd(500 + mode)
    pred = r(B, 3, H, W)
    target = pred + 0.15 * r(B, 3, H, W)                      # |d| on both sides of beta = 0.1
    mask = (torch.rand(B, 1, H, W, device="cuda") > 0.3).float() * torch.rand(B, 1, H, W, device="cuda") if v["mask"] else None
    runs = []
    for _ in range(2):
        lbuf, loss = _guarded((1,))
        dbuf, dpred = _guarded((B, 3, H, W)) if v["grad"] else (None, None)
        ws = torch.empty(2 * _nsm(), dtype=torch.float64, device="cuda")
        abi.call("hg_image_loss", abi.ptr(pred), abi.ptr(target), abi.ptr(mask), abi.ptr(dpred), abi.ptr(loss), abi.ptr(ws), B, HW, mode,
                 eps, abi.stream())
        torch.cuda.synchronize()
        assert _intact(lbuf) and (dbuf is None or _intact(dbuf)), "a guard element was overwritten"
        runs.append((loss.clone(), dpred))
    assert torch.equal(runs[0][0], runs[1][0]), "a repeated launch changed the loss"
    loss, dpred = runs[0]
    d = pred.double() - target.double()
    m = mask.double().expand(B, 3, H, W) if mask is not None else torch.ones_like(d)
    rho, drho, k_r, k_d, sec = _rho64(mode, d, eps)
    # d = fl(pred - target) moves rho by |rho'| u |d|; rho's own roundings; m * rho one more; the mean rounded to fp32 once
    lref = (m * rho).sum() / total
    lb = (m * (drho.abs() * U * d.abs() + (k_r + 1) * U * rho)).sum() / total + U * lref.abs()
    _check(f"image_loss {_vid(v)} {H}x{W}: loss", (loss.double() - lref).abs(), 2 * lb)
    if v["grad"]:
        assert torch.equal(runs[0][1], runs[1][1]), "a repeated launch changed dpred"
        assert not torch.isnan(dpred).any(), "an element of dpred was not written"
        scale = 1.0 / total
        dref = m * drho * scale
        # (m * drho) * fl(1/total): three roundings, drho's own, and d's rounding through rho''
        db = m * scale * (sec * U * d.abs() + (k_d + 3) * U * drho.abs())
        _check(f"image_loss {_vid(v)} {H}x{W}: dpred", (dpred.double() - dref).abs(), 2 * db + 1e-300)


# ----------------------------------------------------------------------------------------------------------------------
# 6. hg_mt_grad_norm / hg_mt_adam through FusedAdam
# ----------------------------------------------------------------------------------------------------------------------
# The synthetic schedule for the small table: sizes that put chunk boundaries at 4095 / 4096 / 4097 inside tensors of a group
# whose members lag each other; tensor i gets a gradient at step k when grad(i, k)
ADAM_PLAN = dict(
    sizes=[4095, 4096, 4097, 8191, 8193, 3, 12289, 4096 * 3 + 1],
    groups=[[0, 1, 2], [3, 4, 5], [6, 7]],
    steps=6,
    # tensor 1 skips step 0, tensor 2 skips steps 0-1, tensor 3 every other step, tensor 5 skips 0-2
    grad=lambda i, k: not ((i == 1 and k < 1) or (i == 2 and k < 2) or (i == 3 and k % 2 == 0) or (i == 5 and k < 3)),
)


def _adam_ref(grp, p0, g, m0, v0, st):
    """One torch.optim.Adam step in fp64 from the kernel's own pre-step fp32 state (a slice of one tensor: the update is
    elementwise), with the kernel's clipped fp32 gradient g; st is the step count after the update."""
    q = torch.nn.Parameter(p0.double())
    q.grad = g.double()
    opt = torch.optim.Adam([q], lr=grp["lr"], betas=grp["betas"], eps=grp["eps"], weight_decay=grp["weight_decay"])
    if m0 is not None:
        opt.state[q] = {"step": torch.tensor(float(st - 1)), "exp_avg": m0.double(), "exp_avg_sq": v0.double()}
    opt.step()
    sq = opt.state[q]
    return q.detach(), sq["exp_avg"], sq["exp_avg_sq"]


def _adam_bounds(grp, p0, g, m0, v0, st, m_ref, v_ref, p_ref):
    """Componentwise bounds of mt_adam_kernel's fp32 update (u = 2^-24; the group scalars lr, beta1, beta2, eps,
    1 - beta1^t and sqrt(1 - beta2^t) are rounded to fp32 on the way in, u each)."""
    b1, b2 = grp["betas"]
    wd, eps = grp["weight_decay"], grp["eps"]
    gd, pd = g.double(), p0.double()
    gw = gd + wd * pd
    e_g = U * gw.abs() if wd else torch.zeros_like(gd)
    m_old = m0.double() if m0 is not None else torch.zeros_like(gd)
    v_old = v0.double() if v0 is not None else torch.zeros_like(gd)
    bm = 4 * U * (m_old.abs() + gw.abs()) + e_g
    bv = 6 * U * (b2 * v_old + (1 - b2) * gw * gw) + 2 * (1 - b2) * gw.abs() * e_g
    bc1, bc2s = 1 - b1 ** st, math.sqrt(1 - b2 ** st)
    sv = torch.sqrt(v_ref)
    d = sv / bc2s + eps
    e_d = (sv / bc2s) * (0.5 * torch.where(v_ref > 0, bv / v_ref.clamp_min(1e-300), 0.0) + 3 * U) + 0.5 * torch.sqrt(bv) / bc2s + 2 * U * d
    q = m_ref / d
    e_q = bm / d + q.abs() * e_d / d + U * q.abs()
    step = grp["lr"] / bc1
    e_p = step * e_q + 4 * U * step * q.abs() + U * p_ref.abs()
    return bm, bv, e_p


def _run_fused_adam(named_groups, sizes_for_grad, steps, clip_at, ema_params, seed, scale_for):
    """Step FusedAdam `steps` times with synthetic gradients and check each launch against fp64 from its own pre-step state.
    named_groups: the optimiser's param groups; sizes_for_grad(i, k): tensor i gets a gradient at step k; scale_for(k): gradient
    scale at step k; ema_params: the EMA's parameter list or None."""
    to = importlib.import_module("3dhumangan_b200.ops.trainer_ops")
    ts = importlib.import_module("3dhumangan_b200.train_step")
    opt = to.FusedAdam(named_groups, lr=1e-3, betas=(0.0, 0.9), weight_decay=0.0)
    flat = [p for grp in opt.param_groups for p in grp["params"]]
    ema = ts.ParameterEMA(ema_params, decay=0.999) if ema_params is not None else None
    g = torch.Generator(device="cuda").manual_seed(seed)
    worst = dict(p=0.0, m=0.0, v=0.0, ema=0.0)
    clipped = set()
    for k in range(steps):
        for i, p in enumerate(flat):
            p.grad = torch.randn(p.shape, generator=g, device="cuda") * scale_for(k) if sizes_for_grad(i, k) else None
        pre = {p: (p.detach().clone(), p.grad.clone(), opt.state[p]["exp_avg"].clone() if opt.state[p] else None,
                   opt.state[p]["exp_avg_sq"].clone() if opt.state[p] else None, int(opt.state[p]["step"]) + 1 if opt.state[p] else 1)
               for p in flat if p.grad is not None}
        sh_pre = [s.clone() for s in ema.shadow_params] if ema is not None else None
        # the norm: fp32 squares summed in fp64 by the reference too; the coefficient the kernel's fp32 formula of it
        tot = sum(float((g_.double() ** 2).sum()) for _, g_, _, _, _ in pre.values())
        opt.step(clip_max_norm=clip_at, ema=ema, ema_params=ema_params)
        torch.cuda.synchronize()
        norm32 = np.float32(math.sqrt(tot))
        assert float(opt.last_grad_norm) == float(norm32), (float(opt.last_grad_norm), float(norm32))
        coef = min(np.float32(clip_at) / (norm32 + np.float32(1e-6)), np.float32(1.0))
        if coef < 1:
            clipped.add(k)
        coef = float(np.float32(coef))
        for grp in opt.param_groups:
            for p in grp["params"]:
                if p not in pre:
                    continue
                p0, g0, m0, v0, st = pre[p]
                assert torch.equal(p.grad, g0 * coef), "write_grad: the clipped gradient is not fl(g * coef)"
                assert int(opt.state[p]["step"]) == st
                sm = opt.state[p]
                f = lambda t: None if t is None else t.reshape(-1)
                for sl in _slices(p.numel(), 1 << 22):      # fp64 temporaries of the 56 M-element pool in slices
                    c = lambda t: None if t is None else f(t)[sl]
                    pr, mr, vr = _adam_ref(grp, c(p0), c(p.grad), c(m0), c(v0), st)
                    bm, bv, bp = _adam_bounds(grp, c(p0), c(p.grad), c(m0), c(v0), st, mr, vr, pr)
                    worst["m"] = max(worst["m"], _ratio(c(sm["exp_avg"]), mr, bm + 1e-300, "exp_avg"))
                    worst["v"] = max(worst["v"], _ratio(c(sm["exp_avg_sq"]), vr, bv + 1e-300, "exp_avg_sq"))
                    worst["p"] = max(worst["p"], _ratio(c(p.detach()), pr, bp + 1e-300, "param"))
        if ema is not None:
            # ParameterEMA.update in fp64 on the pre-step shadow, following the kernel's own new parameters
            n = ema.num_updates
            decay = min(ema.decay, (1 + n) / (10 + n))
            omd = _f32(1.0 - decay)
            req = [p for p in ema_params if p.requires_grad]
            for s_, s0, p in zip(ema.shadow_params, sh_pre, req):
                for sl in _slices(p.numel(), 1 << 22):
                    a0, pn = s0.reshape(-1)[sl].double(), p.detach().reshape(-1)[sl].double()
                    ref_s = a0 - (1.0 - decay) * (a0 - pn)
                    # the fp32 decay term (u), sh - p, the product and the subtraction
                    b = U * ref_s.abs() + 3 * U * omd * (a0 - pn).abs() + U * (1 - decay) * (a0 - pn).abs()
                    worst["ema"] = max(worst["ema"], _ratio(s_.reshape(-1)[sl], ref_s, b + 1e-300, "ema"))
        for p in flat:                                      # a parameter without gradient keeps its value
            if p not in pre:
                assert p.grad is None
    return opt, worst, clipped


@gpu
def test_fused_adam_chunks_and_lagging_steps():
    """Chunk boundaries at 4095 / 4096 / 4097 and inside tensors of a group whose members have different `step` counts, a
    parameter without gradient on alternating steps, an EMA over the parameters in reverse order, the clip active on some steps
    and not on others."""
    plan = ADAM_PLAN
    params = [torch.nn.Parameter(torch.randn(n, device="cuda")) for n in plan["sizes"]]
    groups = [{"params": [params[i] for i in gi], "lr": 1e-3 * (1 + j)} for j, gi in enumerate(plan["groups"])]
    order = [i for gi in plan["groups"] for i in gi]
    opt, worst, clipped = _run_fused_adam(groups, lambda i, k: plan["grad"](order[i], k), plan["steps"], 1.0, params[::-1], 600,
                                          lambda k: 1.0 if k % 3 else 1e-4)
    print(f"  small table: worst of the bound {worst}, clip active on steps {sorted(clipped)}")
    assert clipped and len(clipped) < plan["steps"]


@gpu
def test_fused_adam_c2_optimizers():
    """The C2 generator's five groups (with the 219 047 x 256 appearance-code pool) and the discriminator's one, built by
    train_step.make_optimizers; six steps, the clip active and not; within the generator's first group, three parameters lag
    by 1, 2 and 3 steps, which makes exactly 8 (group, step) pairs at step 3; a ninth pair is refused without touching the
    optimiser's state."""
    gen = importlib.import_module("3dhumangan_b200.modules.generator")
    disc = importlib.import_module("3dhumangan_b200.modules.discriminator")
    ts = importlib.import_module("3dhumangan_b200.train_step")
    cfg = _cfg("C2")
    cfg["dataset_length"] = 219047
    torch.manual_seed(610)
    Gm = gen.Map3DGenerator(**cfg).cuda()
    Dm = disc.UNetDiscriminator(**cfg).cuda()
    og, od = ts.make_optimizers(Gm, Dm, cfg)
    gflat = [p for grp in og.param_groups for p in grp["params"]]
    assert len(og.param_groups) == 5 and Gm.latent_pool.latents.shape[0] == 219047
    first = og.param_groups[0]["params"]
    lag = {id(first[0]): 1, id(first[1]): 2, id(first[2]): 3}
    pool = Gm.latent_pool.latents
    ids = [id(p) for p in gflat]
    # the pool has no gradient at step 2 (an unconditional phase between conditional ones): at step 3 the call holds group 0 at
    # steps 4, 3, 2, 1, the pool at 3 and the other three groups at 4, exactly 8 pairs
    has = lambda i, k: k >= lag.get(ids[i], 0) and not (ids[i] == id(pool) and k == 2)
    groups = og.param_groups
    opt, worst, clipped = _run_fused_adam(groups, has, 4, cfg["grad_clip"], list(Gm.parameters()), 620,
                                          lambda k: 1e-6 if k == 2 else 1e-3)
    print(f"  C2 generator: worst of the bound {worst}, clip active on steps {sorted(clipped)}")
    assert clipped and len(clipped) < 4
    steps = {(gi, int(opt.state[p]["step"])) for gi, grp in enumerate(opt.param_groups) for p in grp["params"] if opt.state[p]}
    assert len(steps) == 8, sorted(steps)
    # a ninth (group, step) pair: refused before any state changes
    for p in gflat:
        p.grad = torch.zeros_like(p)
    lagging = [p for p in first[3:] if opt.state[p]][:1]
    opt.state[lagging[0]]["step"] = torch.tensor(0.0)
    before = {p: int(opt.state[p]["step"]) for p in gflat if opt.state[p]}
    with pytest.raises(RuntimeError, match="at most 8"):
        opt.step(clip_max_norm=1.0)
    assert {p: int(opt.state[p]["step"]) for p in gflat if opt.state[p]} == before, "a refused step advanced `step`"
    del opt, og, Gm
    torch.cuda.empty_cache()
    _, worst_d, clipped_d = _run_fused_adam(od.param_groups, lambda i, k: True, 6, cfg["grad_clip"], None, 630,
                                            lambda k: 1e-6 if k == 4 else 1e-2)
    print(f"  C2 discriminator: worst of the bound {worst_d}, clip active on steps {sorted(clipped_d)}")
    assert clipped_d and len(clipped_d) < 6


# ----------------------------------------------------------------------------------------------------------------------
# 7. drift: every launch of these kernels in a Trainer iteration is a call form of the matrices above
# ----------------------------------------------------------------------------------------------------------------------
TAIL_ENTRY_POINTS = {"hg_bias_act", "hg_bias_act_grad", "hg_resample2x", "hg_spectral_norm", "hg_label_histogram", "hg_seg_ce_coef",
                     "hg_seg_ce", "hg_image_loss", "hg_mt_grad_norm", "hg_mt_adam"}
_ID_TO_ACT = {v[0]: k for k, v in _ba_table().items()}


def _classify(name, a):
    """(kernel, variant) of a recorded call, or None when no matrix row holds it."""
    if name == "hg_bias_act":
        x, b, y, n, step, size, aid, alpha, gain, clamp, _ = a
        act = _ID_TO_ACT.get(aid)
        v = dict(act=act, op="fwd", clamp=int(clamp >= 0), bias="none" if b is None else "vec" if step % 4 == 0 else "scalar", tail=n % 4)
        return "bias_act", v, (b is not None, False, False, False)
    if name == "hg_bias_act_grad":
        g, b, xref, yref, dy, out, n, step, size, order, aid, alpha, gain, clamp, _ = a
        act = _ID_TO_ACT.get(aid)
        v = dict(act=act, op=f"grad{order}", clamp=int(clamp >= 0), bias="none" if b is None else "vec" if step % 4 == 0 else "scalar",
                 tail=n % 4)
        return "bias_act", v, (b is not None, xref is not None, yref is not None, dy is not None)
    if name == "hg_resample2x":
        return "resample", (int(a[5]), float(a[6])), None
    if name == "hg_spectral_norm":
        return "sn", dict(training=int(a[5])), float(a[6])
    if name in ("hg_label_histogram",):
        return "hist", {}, None
    if name == "hg_seg_ce_coef":
        return "seg", dict(prior=int(a[1] is not None)), None
    if name == "hg_seg_ce":
        return "seg", dict(grad=int(a[3] is not None)), None
    if name == "hg_image_loss":
        return "image", dict(mode=a[8], mask=int(a[2] is not None), grad=int(a[3] is not None)), None
    if name == "hg_mt_grad_norm":
        return "norm", {}, None
    if name == "hg_mt_adam":
        return "adam", dict(clip=int(a[3] is not None), ema=int(a[6] != 0.0)), int(a[5])
    return None


def _in_matrix(got):
    kernel, v, extra = got
    if kernel == "bias_act":
        # the pairwise rows span the product of the levels; the NULL pattern must be the one ops/bias_act.py gives this form
        if v["act"] is None or any(v[k] not in BA_LEVELS[k] for k in v):
            return False
        if v["op"] == "grad2" and not _second(v["act"]):
            return False
        want = _ba_launch_args(dict(v, size="ragged"))
        if v["op"] == "fwd":
            return extra[0] == want[0]
        # the grad launch carries the forward's bias only when it keeps x: the bias kind of a call without it is not visible
        return extra[1:] == want[1:] and (extra[0] or not want[0])
    if kernel == "resample":
        return v in RESAMPLE
    if kernel == "sn":
        return v in SN and extra == EPS_SN
    if kernel in ("hist", "norm"):
        return True
    if kernel == "seg":
        return all(v[k] in (0, 1) for k in v)
    if kernel == "image":
        return v in IMAGE_LOSS
    if kernel == "adam":
        return v in ADAM and 1 <= extra <= 8
    return False


@contextlib.contextmanager
def _recording(monkeypatch, rec):
    abi = _abi()
    call = abi.call

    def recorder(name, *args, **kw):
        rec.append((name, args))
        return call(name, *args, **kw)
    with monkeypatch.context() as mp:
        mp.setattr(abi, "call", recorder)
        yield


def _drift_configs():
    uncond = lambda r1: [{"name": "uncond", "uncond": True, "rotate": False, "gen_modal": "rgbs", "do_r1": r1}]
    cond = [{"name": "cond", "uncond": False, "rotate": False, "gen_modal": "rgbs", "do_r1": False}]
    return [("uncond-r1", uncond(True), False, None), ("uncond", uncond(False), False, None), ("cond", cond, False, None),
            ("amp", uncond(True), True, None), ("skipped", uncond(False), True, 2.0 ** 120)]


@gpu
def test_drift_matrix_holds_every_trainer_launch(pkg, port, monkeypatch):
    """Trainer(fused=True).iteration at a tiny size: unconditional with and without R1, a conditional phase, fp16 autocast +
    GradScaler, and a step GradScaler skips (an overflowing scale): every launch of the kernels above is a matrix variant."""
    from test_gpu_conditional import _setup
    ts = importlib.import_module("3dhumangan_b200.train_step")
    seen, bad = set(), []
    cfg, pg, pd, G_, D_, batch, _, vgg = _setup(pkg, port, monkeypatch)
    for tag, phases, amp, init_scale in _drift_configs():
        cfg["phases"] = phases
        t = ts.Trainer(G_, D_, cfg, amp=amp, ddp=False, perceptual=vgg)
        if init_scale is not None:
            t.scaler = torch.amp.GradScaler("cuda", init_scale=init_scale)
        rec = []
        with _recording(monkeypatch, rec):
            t.iteration(batch)
        torch.cuda.synchronize()
        if tag == "skipped":
            assert not t.optimizer_G._stepped, "the overflowing scale did not skip the step"
            assert t.ema.num_updates == 1, "the EMA did not follow the skipped step"
        names = {n for n, _ in rec}
        for name, args in rec:
            if name not in TAIL_ENTRY_POINTS:
                continue
            got = _classify(name, args)
            if got is None or not _in_matrix(got):
                bad.append((tag, name, got))
            else:
                k, v, _ = got
                seen.add((k, str(v)))
        assert "hg_bias_act" in names and "hg_resample2x" in names and "hg_seg_ce" in names, (tag, sorted(names))
        del t
    assert not bad, bad[:8]
    print("call forms seen:", sorted(seen))
    assert {k for k, _ in seen} >= {"bias_act", "resample", "sn", "hist", "seg", "norm", "adam", "image"}
