"""The renderer's kernels launch by launch against fp64: `hg_render_mlp` (csrc/render.cu) in compositing and raw mode,
`hg_render_composite` / `_bwd` and `hg_render_heads` / `_bwd` (csrc/render_train.cu), and `hg_act_wgrad_blocked`
(csrc/synth_bwd.cu) as the training renderer calls it.

Inputs are synthetic, as in test_gpu_render_train.py: random points and geometry records, sorted jittered depths, the
seeded neural field of `oracle.port.init_generator_params` with a sigma gain / bias, and FiLM codes that differ per image.
Every output sits inside a buffer with sentinel guards (`_guarded`); unwritten valid outputs start as NaN.  Shapes derive
from the device's SM count, and each case asserts the edge it claims: a ragged last tile (fewer rays than a tile holds),
a single tile, a persistent CTA whose walk crosses an image boundary, or NaN in the padding pixels.

Bounds start from U = 2^-24.  The fp32 rounding of a sine argument, |t| U, is the least error any fp32 evaluation of
sin(t) can have; the heads and the weight gradient are held to first-order bounds built from it, the SFU sine
(2^-21 absolute after the 2 pi reduction) and the fp32 / bf16x3 sums, and the compositing kernels to bounds built from
the roundings of the transmittance products.  The fused MLP chains six sine layers; its bound is AMP U max|t| times the
magnitude of each output, where AMP is the chain's amplification measured on an H100 with a stated margin.  Each group
also checks that its bound discriminates: the kernel's output fails by at least 10x the bound against a reference with
a deliberate small fault (a swapped per-image FiLM table, a finite last delta, a per-image scale from the wrong image)."""
import importlib
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
SIN_ABS = 2.0 ** -20      # Cody-Waite reduction by 2 pi (2 roundings of |r| <= pi) plus the SFU sine (2^-21.4) on [-pi, pi]
GUARD = 128 * 260         # sentinel elements on each side: one whole tile of per-point rows
SENTINEL = -1234.5
C = 256


def _abi():
    return importlib.import_module("3dhumangan_b200.abi")


def _nsm():
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def _guarded(shape, dtype=torch.float32, fill=float("nan")):
    """(buffer, view): a contiguous view of `shape` inside a buffer with GUARD sentinel elements on each side."""
    n = math.prod(shape)
    buf = torch.full((n + 2 * GUARD,), SENTINEL, dtype=dtype, device="cuda")
    view = buf[GUARD:GUARD + n].view(shape)
    view.fill_(fill)
    return buf, view


def _intact(buf):
    return bool((buf[:GUARD] == SENTINEL).all()) and bool((buf[-GUARD:] == SENTINEL).all())


def _walks(tiles, grid, per_img):
    """For each CTA of a persistent launch (tile = blockIdx.x + it * gridDim.x), the set of images its tiles belong to."""
    return [{t // per_img for t in range(i, tiles, grid)} for i in range(grid)]


class _Checks:
    """Collects (name, err, bound) per check, prints the worst ratio of each, then asserts them all."""

    def __init__(self, label):
        self.label, self.rows = label, []

    def add(self, name, err, bound):
        err, bound = err.double(), bound.double()
        ratio = (err / bound).max().item()
        self.rows.append((name, ratio, err.max().item()))
        return ratio

    def done(self):
        print(self.label + ": " + ", ".join(f"{n} {e:.2e} ({r:.3f} of bound)" for n, r, e in self.rows))
        bad = [(n, r) for n, r, _ in self.rows if not r <= 1.0]
        assert not bad, bad


# ----------------------------------------------------------------------------------------------------------------------
# synthetic renderer inputs
# ----------------------------------------------------------------------------------------------------------------------
SIGMA_GAIN, SIGMA_BIAS = 600.0, 5.0    # sigma ~ N(-11, 17^2) at these inputs: rays of every opacity, and with softplus
                                       # a last sample below -21 (its 1e9 delta then leaves the ray partly transparent)


def _field(seed):
    """(fp32 device params, fp64 device params) of the neural field."""
    port = importlib.import_module("oracle.port")
    pkg = importlib.import_module("3dhumangan_b200")
    cfg = pkg.configs.baseline_config("tiny")
    cfg.update(hidden_dim=C, feature_dim=C)
    p = port.init_generator_params(cfg, seed=seed, sigma_gain=SIGMA_GAIN, sigma_bias=SIGMA_BIAS)
    p32 = {k: v.cuda() for k, v in p.items() if k.startswith("neural_field.")}
    return p32, {k: v.double() for k, v in p32.items()}


def _points(B, R, S, seed):
    """rec [B,N,36] (xyz, 31 geometry features, 2 zeros), z [B,N] sorted with jitter (the optical depth of a ray's first
    S-1 samples is about 1 on average), noise [B,N], freq / phase [B,1024] (different per image)."""
    g = torch.Generator().manual_seed(seed)             # drawn on the host: the same inputs on every device
    N = R * S
    rec = torch.zeros(B, N, 36)
    rec[..., :3] = torch.rand(B, N, 3, generator=g) * 2 - 1
    rec[..., 3:34] = torch.rand(B, N, 31, generator=g)
    step = 0.4 / (S + 1)
    z = (8.0 + (step * (0.5 + torch.rand(B, R, S, generator=g))).cumsum(-1)).reshape(B, N)
    noise = torch.randn(B, N, generator=g)
    freq = torch.randn(B, 4 * C, generator=g)
    phase = torch.randn(B, 4 * C, generator=g)
    rec, z, noise, freq, phase = (t.cuda().contiguous() for t in (rec, z, noise, freq, phase))
    return rec, z, noise, freq, phase


def _siren_ref(p64, rec, freq, phase, monkeypatch):
    """port.siren in fp64 on the kernel's own records ([B,N,260] = rgb, feat, sigma) and max |t| over its sine arguments."""
    port = importlib.import_module("oracle.port")
    B, N = rec.shape[:2]
    dirs = torch.zeros(B, N, 3, dtype=torch.float64, device="cuda")
    dirs[..., 2] = -1
    tmax = [0.0]
    sin = torch.sin

    def rec_sin(t):
        tmax[0] = max(tmax[0], t.abs().max().item())
        return sin(t)
    r = rec.double()
    with monkeypatch.context() as mp:
        mp.setattr(port.torch, "sin", rec_sin)
        out = port.siren(p64, r[..., :3], freq.double(), phase.double(), r[..., 3:34], dirs, 1.0, C)
    return out, tmax[0]


def _integrate(raw, z, noise, noise_std, white_back, last_back, clamp, last_delta=None):
    """port.ray_integration in fp64 -> (feat [B,R,256], rgb [B,R,3], depth [B,R], weights [B,R,S], sum of the unabsorbed
    weights [B,R]).  `last_delta` (a fault): the last sample's delta is finite -- the integration runs over one more
    sample at z_last + last_delta whose density is zero (sigma -1e4: relu and softplus give exactly 0 in fp64)."""
    port = importlib.import_module("oracle.port")
    B, R, S, Cc = raw.shape
    z4, n4 = z.double().reshape(B, R, S, 1), noise.double().reshape(B, R, S, 1)
    if last_delta is not None:
        extra = torch.zeros(B, R, 1, Cc, dtype=torch.float64, device=raw.device)
        extra[..., -1] = -1e4
        raw = torch.cat([raw, extra], 2)
        z4 = torch.cat([z4, z4[:, :, -1:] + last_delta], 2)
        n4 = torch.cat([n4, torch.zeros_like(n4[:, :, :1])], 2)
    rgbf, depth, w = port.ray_integration(raw, z4, n4, noise_std, white_back, last_back, clamp)
    w = w[..., 0][..., :S]
    wsum = port.ray_integration(raw, z4, n4, noise_std, False, False, clamp)[2].sum((-2, -1))
    return rgbf[..., 3:], rgbf[..., :3], depth[..., 0], w, wsum


# ----------------------------------------------------------------------------------------------------------------------
# 1. hg_render_mlp, compositing mode
# ----------------------------------------------------------------------------------------------------------------------
# Amplification of the sine-argument rounding through the fused MLP and the compositing, per output: the bound is
# AMP U max|t| times the output's largest magnitude over its image (1 for the weights).  Measured on an H100 80GB HBM3
# (700 W) as max err / (U max|t| magnitude) over the passes=3 cases and two input draws: feat 138, rgb 102, depth 3.5,
# weights 188 (sigma carries the field's gain of 600, so the weights move most); set 3-5x above.
AMP = dict(feat=512.0, rgb=320.0, depth=16.0, weights=768.0)
# passes=1 (bf16 operands, unit roundoff 2^-8 in place of U max|t|): a loose bar that checks the one-pass weight-stage
# schedule only.  Measured: feat 11, rgb 6.4, depth 0.4, weights 13.
AMP1 = dict(feat=48.0, rgb=16.0, depth=2.0, weights=52.0)
# raw mode, per point (no compositing): measured rgb 3.5, feat 43, sigma 35.
AMP_RAW = dict(rgb=16.0, feat=160.0, sigma=128.0)


def _mlp_shape(name):
    """(B, R, S) of a case: `sN-ragged` an image's last tile holds fewer rays than the 128 / S a tile holds; `s128` one
    ray per tile; `tile1` one full tile of one image; `multi` tiles per image < SMs < B * tiles, so some CTA's walk crosses
    an image boundary (and the last tile of each image is ragged)."""
    if name == "multi":
        T = _nsm() // 2 + 1
        return 3, (T - 1) * 4 + 3, 32
    return {"s2-ragged": (2, 145, 2), "s4-ragged": (2, 101, 4), "s8-ragged": (2, 35, 8), "s16-ragged": (2, 39, 16),
            "s16-ragged-p1": (2, 39, 16), "s32-ragged": (2, 21, 32), "s64-ragged": (2, 31, 64), "s128": (2, 25, 128),
            "tile1": (1, 32, 4)}[name]


MLP = {   # name -> (clamp, noise_std, white_back, last_back, want_weights, passes)
    "s2-ragged": ("relu", 0.5, True, False, True, 3),
    "s4-ragged": ("softplus", 0.0, False, True, True, 3),
    "s8-ragged": ("relu", 0.0, True, True, True, 3),
    "s16-ragged": ("softplus", 0.5, True, False, True, 3),
    "s32-ragged": ("relu", 0.5, False, False, False, 3),
    "s64-ragged": ("softplus", 0.5, False, True, True, 3),
    "s128": ("softplus", 0.0, True, True, True, 3),
    "tile1": ("relu", 0.0, False, False, True, 3),
    "multi": ("relu", 0.5, True, False, True, 3),
    "s16-ragged-p1": ("relu", 0.5, False, False, True, 1),
}


def _mlp_inputs(p32, rec, freq, phase):
    ro = importlib.import_module("3dhumangan_b200.modules.render_ops")
    g = lambda n: p32["neural_field." + n]
    heads_b = torch.cat([g("sigma_layer.bias").reshape(1), g("color_layer_linear.bias").reshape(3)]).contiguous()
    return (ro.film_table(p32, freq, phase), ro.pack_render_weights(p32), g("sigma_layer.weight").reshape(-1).contiguous(),
            g("color_layer_linear.weight").contiguous(), g("feature_layer_linear.bias").contiguous(), heads_b)


def _launch_mlp(rec, z, noise, ins, B, R, S, *, noise_std=0.0, white_back=False, last_back=False, clamp="relu",
                want_weights=True, passes=3, raw=False):
    abi = _abi()
    film, wblob, w_sigma, w_rgb, b_feat, heads_b = ins
    N = R * S
    bufs, res = [], {}
    if raw:
        b_, res["raw"] = _guarded((B, N, 260))
        bufs.append(b_)
    else:
        b_, res["ray"] = _guarded((B, R, 260))
        bufs.append(b_)
        if want_weights:
            b_, res["w"] = _guarded((B, N))
            bufs.append(b_)
    abi.call("hg_render_mlp", abi.ptr(rec), abi.ptr(None if raw else z), abi.ptr(noise if noise_std else None), abi.ptr(film),
             abi.ptr(wblob), abi.ptr(w_sigma), abi.ptr(w_rgb), abi.ptr(b_feat), abi.ptr(heads_b), abi.ptr(res.get("ray")),
             abi.ptr(res.get("w")), abi.ptr(res.get("raw")), B, R, S, C, float(noise_std), int(white_back), int(last_back),
             int(clamp == "softplus"), passes, abi.stream())
    res["bufs"] = bufs
    return res


def _per_ray(got, ref):
    """max |got - ref| over every axis after the ray axis ([B,R,...] -> [B,R])."""
    d = (got.double() - ref).abs()
    return d.reshape(d.shape[0], d.shape[1], -1).max(-1).values


@pytest.mark.parametrize("case", list(MLP))
def test_render_mlp_composite(case, monkeypatch):
    clamp, noise_std, white_back, last_back, want_w, passes = MLP[case]
    B, R, S = _mlp_shape(case)
    N, rpt = R * S, 128 // S
    per_img = -(-R // rpt)
    tiles = B * per_img
    grid = min(tiles, _nsm())
    if case == "tile1":
        assert tiles == 1, "single tile"
    elif case == "multi":
        assert per_img < _nsm() < tiles and R % rpt
        assert any(len(w) > 1 for w in _walks(tiles, grid, per_img)), "some CTA's walk must cross an image boundary"
    elif S < 128:
        assert 0 < R % rpt < rpt, "the last tile of each image must be ragged"
    p32, p64 = _field(7)
    rec, z, noise, freq, phase = _points(B, R, S, 100 + S + B)
    ins = _mlp_inputs(p32, rec, freq, phase)
    kw = dict(noise_std=noise_std, white_back=white_back, last_back=last_back, clamp=clamp, want_weights=want_w, passes=passes)
    runs = [_launch_mlp(rec, z, noise, ins, B, R, S, **kw) for _ in range(2)]
    torch.cuda.synchronize()
    for r in runs:
        assert all(_intact(b) for b in r["bufs"]), "a write landed outside [B,R,260] / [B,N]"
    assert torch.equal(runs[0]["ray"], runs[1]["ray"]), "a repeated launch changed ray_out"
    if want_w:
        assert torch.equal(runs[0]["w"], runs[1]["w"]), "a repeated launch changed the weights"
    ray = runs[0]["ray"]
    assert torch.isfinite(ray).all(), "every ray is written"

    raw, tmax = _siren_ref(p64, rec, freq, phase, monkeypatch)
    raw = raw.reshape(B, R, S, 260)
    feat, rgb, depth, w, wsum = _integrate(raw, z, noise, noise_std, white_back, last_back, clamp)
    partial = ((wsum > 0.05) & (wsum < 0.95)).double().mean().item()
    assert partial > 0.1, f"only {partial:.3f} of the rays are partly opaque"

    if passes == 3:
        scale, amp = U * tmax, AMP
    else:
        scale, amp = 2.0 ** -8, AMP1
    mags = dict(feat=feat.abs().amax((1, 2)), rgb=rgb.abs().amax((1, 2)), depth=depth.abs().amax(1), weights=torch.ones(B, device="cuda"))
    gots = dict(feat=ray[..., :256], rgb=ray[..., 256:259], depth=ray[..., 259:260])
    refs = dict(feat=feat, rgb=rgb, depth=depth[..., None])
    if want_w:
        gots["weights"], refs["weights"] = runs[0]["w"].reshape(B, R, S), w
    chk = _Checks(f"render_mlp {case} B{B} R{R} S{S} max|t| {tmax:.1f} partly-opaque {partial:.2f}")
    bounds = {}
    for q in gots:
        bounds[q] = amp[q] * scale * mags[q][:, None].expand(B, R)
        chk.add(q, _per_ray(gots[q], refs[q]), bounds[q])
    chk.done()

    # the bounds discriminate
    if case == "multi":
        # image 0's FiLM table swapped with image 1's: the table refresh of a walk that crosses into image 1
        sw = torch.tensor([1, 0] + list(range(2, B)), device="cuda")
        raw_f, _ = _siren_ref(p64, rec, freq[sw], phase[sw], monkeypatch)
        feat_f = _integrate(raw_f.reshape(B, R, S, 260), z, noise, noise_std, white_back, last_back, clamp)[0]
        ratio = (_per_ray(ray[..., :256], feat_f) / bounds["feat"]).max().item()
        print(f"  fault: {ratio:.0f}x the bound")
        assert ratio > 10, f"a swapped FiLM table fails by only {ratio:.1f}x the bound"
    if want_w and passes == 3 and not last_back:
        # the last sample's delta taken as one sample spacing instead of 1e9
        w_f = _integrate(raw, z, noise, noise_std, white_back, last_back, clamp, last_delta=0.4 / (S + 1))[3]
        ratio = (_per_ray(gots["weights"], w_f) / bounds["weights"]).max().item()
        print(f"  fault: {ratio:.0f}x the bound")
        assert ratio > 10, f"a finite last delta fails by only {ratio:.1f}x the bound"


# ----------------------------------------------------------------------------------------------------------------------
# 2. hg_render_mlp, raw mode
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("S", [8, 32])
def test_render_mlp_raw(S, monkeypatch):
    """Per point [rgb, feat, sigma] against port.siren at a ragged ray count (the last tile of each image holds fewer rays
    than 128 / S): every existing point is written, and no row past the last ray is (the guard spans a whole tile of
    rows).  Bound: AMP's chain amplification, per point, with the magnitude of each output over its image."""
    rpt = 128 // S
    B, R = 2, 3 * rpt + rpt // 2 + 1
    assert 0 < R % rpt < rpt
    N = R * S
    p32, p64 = _field(8)
    rec, z, noise, freq, phase = _points(B, R, S, 200 + S)
    ins = _mlp_inputs(p32, rec, freq, phase)
    runs = [_launch_mlp(rec, None, None, ins, B, R, S, raw=True) for _ in range(2)]
    torch.cuda.synchronize()
    for r in runs:
        assert all(_intact(b) for b in r["bufs"]), "a row past the last ray was written"
    got = runs[0]["raw"]
    assert torch.equal(got, runs[1]["raw"]), "a repeated launch changed raw_out"
    assert torch.isfinite(got).all(), "every existing point is written"
    ref, tmax = _siren_ref(p64, rec, freq, phase, monkeypatch)
    chk = _Checks(f"render_mlp raw S{S} B{B} R{R} max|t| {tmax:.1f}")
    bounds = {}
    for q, sl in (("rgb", slice(0, 3)), ("feat", slice(3, 259)), ("sigma", slice(259, 260))):
        amp = AMP_RAW[q]
        mag = ref[..., sl].abs().amax((1, 2))
        bounds[q] = amp * U * tmax * mag[:, None].expand(B, N)
        chk.add(q, (got[..., sl].double() - ref[..., sl]).abs().amax(-1), bounds[q])
    chk.done()
    # image 0's FiLM table swapped with image 1's
    ref_f, _ = _siren_ref(p64, rec, freq[[1, 0]], phase[[1, 0]], monkeypatch)
    ratio = ((got[..., 3:259].double() - ref_f[..., 3:259]).abs().amax(-1) / bounds["feat"]).max().item()
    print(f"  fault: {ratio:.0f}x the bound")
    assert ratio > 10, ratio


# ----------------------------------------------------------------------------------------------------------------------
# 3. hg_render_composite and hg_render_composite_bwd
# ----------------------------------------------------------------------------------------------------------------------
COMP = [dict(S=S, last_back=lb, softplus=sp, white_back=(i + sp) % 2 == 1, noise=(i + lb) % 2 == 1)
        for i, S in enumerate((8, 16, 32, 64, 128)) for lb in (0, 1) for sp in (0, 1)]


def _cid(v):
    return f"S{v['S']}-{'lastback' if v['last_back'] else 'nolastback'}-{'softplus' if v['softplus'] else 'relu'}-" \
           f"{'white' if v['white_back'] else 'black'}-{'noise' if v['noise'] else 'nonoise'}"


def _blocked(t):
    """[B,C,N] -> tile-blocked [B,T,C,128]."""
    B, Cc, N = t.shape
    return t.reshape(B, Cc, N // 128, 128).permute(0, 2, 1, 3).contiguous()


def _planar(t):
    B, T, Cc, _ = t.shape
    return t.permute(0, 2, 1, 3).reshape(B, Cc, T * 128)


@pytest.mark.parametrize("v", COMP, ids=_cid)
def test_render_composite(v, port):
    """ray_out, the weights (absorbed by the last sample with last_back, as port.ray_integration returns them), and d feat,
    d rgb_pre, d sigma against port.ray_integration with fp64 autograd; B = 2 images of 3 tiles each.  With relu and noise
    the reference uses the kernel's own clamp mask (the gradient is discontinuous there).
    Bounds: each alpha is within 4 U (expf, 1 - e, the fp32 delta), each transmittance within the sum of its factors'
    errors, so |d w_s| <= 5 (s + 1) U; the forward sums add S + 2 roundings of sum w |v|, and white_back adds the error of
    sum w.  The backward: d feat and d rgb_pre carry the weight's error times |d ray_out| and a few roundings of their own;
    d sigma is held per ray to (16 S + 259) U of the ray's largest reference gradient (q T - suffix / tr cancels).
    Measured on an H100 80GB HBM3 (700 W): at most 0.65 of the bound (d rgb_pre), 0.25 for the weights; a finite last
    delta fails the weights by 1.2e4x the bound or more."""
    abi = _abi()
    S, lb, sp, wb = v["S"], bool(v["last_back"]), bool(v["softplus"]), bool(v["white_back"])
    nstd = 0.5 if v["noise"] else 0.0
    B, T = 2, 3
    N = T * 128
    R = N // S
    g = torch.Generator(device="cuda").manual_seed(S * 4 + 2 * lb + sp)
    sig = torch.randn(B, N, generator=g, device="cuda") * 40 + 10     # dense: samples absorb, yet many rays stay partly clear
    if sp:
        sig = sig - 20                                                 # softplus: last samples below -21 keep rays partly clear
    step = 0.4 / (S - 1) / 10
    z = (8.0 + (step * (0.5 + torch.rand(B, R, S, generator=g, device="cuda"))).cumsum(-1)).reshape(B, N).contiguous()
    noise = torch.randn(B, N, generator=g, device="cuda")
    rgbp = torch.randn(B, 3, N, generator=g, device="cuda")
    feat = torch.randn(B, C, N, generator=g, device="cuda")
    dray = torch.randn(B, R, 260, generator=g, device="cuda")
    dray[..., 259] = 0                                                 # depth carries no gradient
    featb = _blocked(feat)
    nz = noise if nstd else None

    def fwd():
        b1, ray = _guarded((B, R, 260))
        b2, w = _guarded((B, N))
        abi.call("hg_render_composite", abi.ptr(sig), abi.ptr(z), abi.ptr(nz), abi.ptr(rgbp), abi.ptr(featb), abi.ptr(ray),
                 abi.ptr(w), B, R, S, float(nstd), int(wb), int(sp), int(lb), abi.stream())
        return ray, w, (b1, b2)

    def bwd(last_back):
        b1, df = _guarded((B, T, C, 128))
        b2, dp = _guarded((B, 3, N))
        b3, ds = _guarded((B, N))
        abi.call("hg_render_composite_bwd", abi.ptr(sig), abi.ptr(z), abi.ptr(nz), abi.ptr(rgbp), abi.ptr(featb), abi.ptr(dray),
                 abi.ptr(df), abi.ptr(dp), abi.ptr(ds), B, R, S, float(nstd), int(wb), int(sp), int(last_back), abi.stream())
        return df, dp, ds, (b1, b2, b3)

    f1, f2 = fwd(), fwd()
    k1, k2 = bwd(lb), bwd(lb)
    k0 = bwd(not lb)
    torch.cuda.synchronize()
    assert all(_intact(b) for r in (f1, f2, k1, k2, k0) for b in r[-1]), "a guard element was overwritten"
    for a, b in zip(f1[:2] + k1[:3], f2[:2] + k2[:3]):
        assert torch.equal(a, b), "a repeated launch changed an output"
    ray, w = f1[0], f1[1]
    df, dp, ds = _planar(k1[0]), k1[1], k1[2]

    # fp64 reference: port.ray_integration on [feat | sigmoid(rgb_pre) | sigma]
    sd, fd, rd = (t.double().requires_grad_(True) for t in (sig, feat, rgbp))
    vals = torch.cat([fd.permute(0, 2, 1), torch.sigmoid(rd).permute(0, 2, 1), sd[..., None]], -1).reshape(B, R, S, 260)
    n64 = noise.double().reshape(B, R, S, 1)
    relu = port.F.relu
    if not sp and nstd:
        mask = ((sig + noise * nstd) > 0).double().reshape(B, R, S, 1)
        port.F.relu = lambda t: t * mask
    try:
        out, depth, wr = port.ray_integration(vals, z.double().reshape(B, R, S, 1), n64, nstd, wb, lb, "softplus" if sp else "relu")
        (out * dray[..., :259].double()).sum().backward()
    finally:
        port.F.relu = relu
    out, depth, wr = out.detach(), depth.detach()[..., 0], wr.detach()[..., 0]
    wsum_ref = _integrate(vals.detach(), z, noise, nstd, wb, lb, "softplus" if sp else "relu")[4]
    partial = ((wsum_ref > 0.05) & (wsum_ref < 0.95)).double().mean().item()
    assert partial > 0.1, f"only {partial:.3f} of the rays are partly opaque"

    chk = _Checks(f"composite {_cid(v)} partly-opaque {partial:.2f}")
    vabs = vals.detach()[..., :259].abs()                                       # [B,R,S,259]: feat | rgb
    s_idx = torch.arange(S, device="cuda", dtype=torch.float64)
    dw = 5 * (s_idx + 1) * U                                                    # |d w_s|
    fbound = (dw[None, None, :, None] * vabs).sum(2) + (S + 2) * U * (wr[..., None] * vabs).sum(2)
    if wb:
        fbound = fbound + dw.sum() + S * U
    chk.add("ray feat|rgb", (ray[..., :259].double() - out).abs(), fbound)
    zb = z.double().reshape(B, R, S)
    dbound = (dw * zb).sum(-1) + dw.sum() * zb[..., -1] + (S + 2) * U * (wr * zb).sum(-1)
    chk.add("depth", (ray[..., 259].double() - depth).abs(), dbound)
    wbound = (dw + (lb * (dw.sum() + S * U) * (s_idx == S - 1)))[None, None].expand(B, R, S)
    werr = (w.double().reshape(B, R, S) - wr).abs()
    chk.add("weights", werr, wbound)

    # backward: d feat = wv dr and d rgb_pre = wv dr s (1 - s) with |d wv| the weight's bound; d sigma per ray within
    # (16 S + 259) U of the ray's largest reference gradient (q T - suffix / tr cancels)
    wvb = wbound.reshape(B, R, S, 1)
    g_f = fd.grad.reshape(B, C, R, S).permute(0, 2, 3, 1)
    g_p = rd.grad.reshape(B, 3, R, S).permute(0, 2, 3, 1)
    g_s = sd.grad.reshape(B, R, S)
    drd = dray.double()
    sg = torch.sigmoid(rgbp.double()).reshape(B, 3, R, S).permute(0, 2, 3, 1)
    chk.add("dfeat", (df.reshape(B, C, R, S).permute(0, 2, 3, 1).double() - g_f).abs(),
            wvb * drd[:, :, None, :C].abs() + 2 * U * g_f.abs())
    chk.add("drgbp", (dp.reshape(B, 3, R, S).permute(0, 2, 3, 1).double() - g_p).abs(),
            wvb * drd[:, :, None, C:C + 3].abs() * sg * (1 - sg) + 16 * U * g_p.abs())
    chk.add("dsig", _per_ray(ds.reshape(B, R, S), g_s), (16 * S + 259) * U * g_s.abs().amax(-1) + 1e-30)
    chk.done()
    # the flag changes the gradient: without it the last sample's feature gradient differs
    assert not torch.equal(_planar(k0[0]), df)
    # the weights bound discriminates: a finite last delta
    if not lb:
        wf = _integrate(vals.detach(), z, noise, nstd, wb, lb, "softplus" if sp else "relu", last_delta=step)[3]
        ratio = ((w.double().reshape(B, R, S) - wf).abs() / wbound).max().item()
        print(f"  fault: {ratio:.0f}x the bound")
        assert ratio > 10, ratio


# ----------------------------------------------------------------------------------------------------------------------
# 4. hg_render_heads and hg_render_heads_bwd
# ----------------------------------------------------------------------------------------------------------------------
def _heads_shape(name):
    """(B, T): `tile1` one image of one tile; `multi` B*T >= 2 * 4 SMs tiles with T <= 4 SMs, so every block of
    heads_bwd (grid min(4 SMs, B*T)) walks tiles of at least two images."""
    if name == "tile1":
        return 1, 1
    grid = 4 * _nsm()
    B = 3
    T = -(-2 * grid // B)
    return B, T


def _heads_inputs(B, T, seed):
    """out3 / linc tile-blocked [B,T,256,128]; channels 0..15 reach |t| ~ 10^3 (large Cody-Waite k), the rest |t| <~ 60."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    rn = lambda *s: torch.randn(*s, generator=g, device="cuda")
    spread = torch.ones(C, device="cuda")
    spread[:16] = 4.0
    mod3 = torch.stack([30.0 + 15.0 * rn(B, C).clamp(-1.9, 1.9), rn(B, C)], 1).contiguous()
    out3 = (rn(B, T, C, 128) * spread[None, None, :, None]).contiguous()
    linc = (rn(B, T, C, 128) * spread[None, None, :, None]).contiguous()
    w_sigma = 0.1 * rn(C)
    w_rgb = 0.1 * rn(3, C)
    heads_b = rn(4)
    return out3, linc, mod3, w_sigma, w_rgb, heads_b


def _heads_ref(out3, linc, mod3):
    """h4, c [B,C,N] in fp64, and the per-element error of each (|t| U + SIN_ABS)."""
    f, ph = mod3[:, 0].double()[:, :, None], mod3[:, 1].double()[:, :, None]
    t_h = f * _planar(out3).double() + ph
    t_c = f * _planar(linc).double() + ph
    return torch.sin(t_h), torch.sin(t_c), U * t_h.abs() + SIN_ABS, U * t_c.abs() + SIN_ABS, max(t_h.abs().max().item(), t_c.abs().max().item())


@pytest.mark.parametrize("shape", ["tile1", "multi"])
def test_render_heads(shape):
    """sig = w_sigma . sin(f out3 + phi) + b_sigma, rgb_pre_j = W_rgb[j] . sin(f linc + phi) + b_j per point.
    Bound: each sine within |t| U + SIN_ABS, then 256 sequential fmas and the bias add:
    |err| <= sum |w| (|t| U + SIN_ABS) + 257 U (sum |w h| + |b|).  Measured on an H100 80GB HBM3 (700 W) at |t| up to
    1.1e3: at most 0.045 of the bound; a swapped FiLM table fails by 2.7e4x."""
    abi = _abi()
    B, T = _heads_shape(shape)
    N = T * 128
    if shape == "tile1":
        assert B * T == 1
    else:
        assert B * T > 4 * _nsm()
    out3, linc, mod3, w_sigma, w_rgb, heads_b = _heads_inputs(B, T, 300 + B)

    def launch():
        b1, sig = _guarded((B, N))
        b2, rgbp = _guarded((B, 3, N))
        abi.call("hg_render_heads", abi.ptr(out3), abi.ptr(linc), abi.ptr(mod3), abi.ptr(w_sigma), abi.ptr(w_rgb), abi.ptr(heads_b),
                 abi.ptr(sig), abi.ptr(rgbp), B, N, abi.stream())
        return sig, rgbp, (b1, b2)
    r1, r2 = launch(), launch()
    torch.cuda.synchronize()
    assert all(_intact(b) for r in (r1, r2) for b in r[2])
    assert torch.equal(r1[0], r2[0]) and torch.equal(r1[1], r2[1]), "a repeated launch changed an output"
    h4, cc, eh, ec, tmax = _heads_ref(out3, linc, mod3)
    assert shape == "tile1" or tmax > 500, tmax
    ws, wr, hb = w_sigma.double(), w_rgb.double(), heads_b.double()
    ref_s = torch.einsum("c,bcn->bn", ws, h4) + hb[0]
    ref_r = torch.einsum("jc,bcn->bjn", wr, cc) + hb[1:, None]
    bnd_s = torch.einsum("c,bcn->bn", ws.abs(), eh) + 257 * U * (torch.einsum("c,bcn->bn", ws.abs(), h4.abs()) + hb[0].abs())
    bnd_r = torch.einsum("jc,bcn->bjn", wr.abs(), ec) + 257 * U * (torch.einsum("jc,bcn->bjn", wr.abs(), cc.abs()) + hb[1:, None].abs())
    chk = _Checks(f"heads {shape} B{B} T{T} max|t| {tmax:.0f}")
    chk.add("sig", (r1[0].double() - ref_s).abs(), bnd_s)
    chk.add("rgbp", (r1[1].double() - ref_r).abs(), bnd_r)
    chk.done()
    if B > 1:        # image 0's FiLM table swapped with image 1's
        h4f = _heads_ref(out3, linc, mod3[[1, 0] + list(range(2, B))])[0]
        ref_f = torch.einsum("c,bcn->bn", ws, h4f) + hb[0]
        ratio = ((r1[0].double() - ref_f).abs() / bnd_s).max().item()
        print(f"  fault: {ratio:.0f}x the bound")
        assert ratio > 10, ratio


@pytest.mark.parametrize("shape", ["tile1", "multi"])
def test_render_heads_bwd(shape):
    """acc += [sum dsig h4, sum drgbp_j c, sum dsig, sum drgbp_j] over every point of every image, onto a pre-filled fp64
    accumulator.  Bound: a product with the sine's error, 3 adds of a lane's 4 points, 5 shuffle steps and one fp32 add per
    tile the block walks (n_t), then exact fp64 atomics: |err| <= sum |g| (|t| U + SIN_ABS) + (n_t + 10) U sum |g h|.
    Not repeated bit for bit: the fp64 atomics add the blocks in any order.  Measured on an H100 80GB HBM3 (700 W): at
    most 0.086 of the bound; a swapped FiLM table fails by 4.7e3x."""
    abi = _abi()
    B, T = _heads_shape(shape)
    N = T * 128
    grid = min(4 * _nsm(), B * T)
    n_t = -(-B * T // grid)
    if shape == "tile1":
        assert B * T == 1
    else:
        assert B * T > 4 * _nsm() and all(len(w) > 1 for w in _walks(B * T, grid, T)), "every block walks several images"
    out3, linc, mod3, *_ = _heads_inputs(B, T, 400 + B)
    g = torch.Generator(device="cuda").manual_seed(401)
    dsig = torch.randn(B, N, generator=g, device="cuda")
    drgbp = torch.randn(B, 3, N, generator=g, device="cuda")
    bufa, acc = _guarded((4 * C + 4,), torch.float64, 0.0)
    init = 10.0 * torch.randn(4 * C + 4, generator=g, device="cuda", dtype=torch.float64)
    acc.copy_(init)
    abi.call("hg_render_heads_bwd", abi.ptr(out3), abi.ptr(linc), abi.ptr(mod3), abi.ptr(dsig), abi.ptr(drgbp), abi.ptr(acc), B, N,
             abi.stream())
    torch.cuda.synchronize()
    assert _intact(bufa)

    def ref_of(m3):
        h4, cc, eh, ec, tmax = _heads_ref(out3, linc, m3)
        gs, gr = dsig.double(), drgbp.double()
        ref = torch.cat([torch.einsum("bn,bcn->c", gs, h4), torch.einsum("bjn,bcn->jc", gr, cc).reshape(-1), gs.sum().reshape(1),
                         gr.sum((0, 2))])
        bnd = torch.cat([torch.einsum("bn,bcn->c", gs.abs(), eh) + (n_t + 10) * U * torch.einsum("bn,bcn->c", gs.abs(), h4.abs()),
                         (torch.einsum("bjn,bcn->jc", gr.abs(), ec) + (n_t + 10) * U * torch.einsum("bjn,bcn->jc", gr.abs(), cc.abs())).reshape(-1),
                         (n_t + 10) * U * gs.abs().sum().reshape(1), (n_t + 10) * U * gr.abs().sum((0, 2))])
        return ref, bnd, tmax
    ref, bnd, tmax = ref_of(mod3)
    chk = _Checks(f"heads_bwd {shape} B{B} T{T} n_t {n_t} max|t| {tmax:.0f}")
    got = acc - init
    bnd = bnd + 1e-15 * init.abs()
    chk.add("dw_sigma", (got[:C] - ref[:C]).abs(), bnd[:C])
    chk.add("dW_rgb", (got[C:4 * C] - ref[C:4 * C]).abs(), bnd[C:4 * C])
    chk.add("db", (got[4 * C:] - ref[4 * C:]).abs(), bnd[4 * C:])
    chk.done()
    if B > 1:        # image 0's FiLM table swapped with image 1's
        ref_f, _, _ = ref_of(mod3[[1, 0] + list(range(2, B))])
        ratio = ((got[:4 * C] - ref_f[:4 * C]).abs() / bnd[:4 * C]).max().item()
        print(f"  fault: {ratio:.0f}x the bound")
        assert ratio > 10, ratio


# ----------------------------------------------------------------------------------------------------------------------
# 5. hg_act_wgrad_blocked
# ----------------------------------------------------------------------------------------------------------------------
WGRAD = {   # name -> (act, Cx, pscale, shape, passes); passes 1 is the bf16 training leg (hg_precision="bf16")
    "sine-pscale-few": (1, 256, True, "few", 3),
    "sine-pscale-multi": (1, 256, True, "multi", 3),
    "sine-nopscale-multi": (1, 256, False, "multi", 3),
    "identity-cx128-few": (2, 128, True, "few", 3),
    "identity-cx128-multi": (2, 128, True, "multi", 3),
    "sine-pscale-multi-p1": (1, 256, True, "multi", 1),
    "sine-nopscale-multi-p1": (1, 256, False, "multi", 1),
    "identity-cx128-multi-p1": (2, 128, True, "multi", 1),
}


def _wgrad_shape(name):
    """(B, Hg, Wg): `few` B * T < SMs tiles with a ragged last tile; `multi` T < SMs <= B * T / 2 with a ragged last tile,
    so every CTA (grid = SMs) walks tiles of at least two images."""
    if name == "few":
        return 2, 12, 26                     # HW 312: 3 tiles, the last holds 56 pixels
    n = _nsm()
    T = n // 3 + 1
    Wg = 100
    Hg = (T * 128 - 60) // Wg
    B = -(-2 * n // T)
    return B, Hg, Wg


@pytest.mark.parametrize("case", list(WGRAD))
def test_act_wgrad_blocked(case):
    """dW[o,i] = sum_b sum_p (ps[b,o] dout[b,o,p]) act(x[b,i,p] g1[b,i] + g0[b,i]), db[o] = sum ps dout, over the valid
    pixels; act 1 = sine with the per-image FiLM table (the colour and network layers), act 2 = identity with no table,
    Cx = 128 and the x_bstride T*128*128 of the first layers' weight gradient (render_train.mlp_backward).  The padding
    pixels of dout and x hold NaN in one launch and zeros in another, and the outputs are bit-identical.
    Bound: bf16x3 operands drop at most 3 * 2^-18 of each product (48 U), one rounding of ps*dout, fp32 accumulation of
    64-term chunks and of the 6 n_t chunk products a CTA adds, then a fixed-order fp64 reduction:
    |err| <= (116 + 6 n_t) U sum |terms| + sum |ps dout| (|t| U + SIN_ABS for the sine; |t| U for the affine).
    One bf16 pass (passes 1) rounds each operand once to 8 significant bits, so a product carries up to 2^-8 + 2^-18
    (64 U) in place of the 48 U of bf16x3: |err| <= 2^-8 sum |terms| + (132 + 6 n_t) U sum |terms| + the same sine term.
    That worst-case bound is ~500x the bf16x3 one and cannot see a one-tile fault, so the fault runs at passes 3 only.
    Measured on an H100 80GB HBM3 (700 W): at most 0.18 of the bound (0.025 at passes 1); one tile scaled with another
    image's pscale row fails by 277x or more."""
    abi = _abi()
    act, Cx, use_ps, shape, passes = WGRAD[case]
    B, Hg, Wg = _wgrad_shape(shape)
    HW = Hg * Wg
    T = -(-HW // 128)
    tiles = B * T
    grid = min(tiles, _nsm())
    n_t = -(-tiles // grid)
    assert HW % 128, "ragged last tile"
    if shape == "few":
        assert tiles < _nsm()
    else:
        assert all(len(w) > 1 for w in _walks(tiles, grid, T)), "every CTA walks tiles of several images"
    g = torch.Generator(device="cuda").manual_seed(500 + len(case) + B)
    rn = lambda *s: torch.randn(*s, generator=g, device="cuda")
    dout = rn(B, C, HW)
    x = rn(B, Cx, HW)
    mod = torch.stack([30.0 + 15.0 * rn(B, C), rn(B, C)], 1).contiguous() if act == 1 else None
    ps = (30.0 + 15.0 * rn(B, C)).contiguous() if use_ps else None
    ws = torch.empty(int(abi.lib().hg_spade_bwd_wgrad_workspace_bytes()) // 4, device="cuda")

    def blocked(t, fill):
        Bc, Cc, _ = t.shape
        pad = torch.full((Bc, Cc, T * 128), fill, device="cuda")
        pad[:, :, :HW] = t
        return pad.reshape(Bc, Cc, T, 128).permute(0, 2, 1, 3).contiguous()

    def launch(fill):
        b1, dw = _guarded((C, Cx))
        b2, db = _guarded((C,))
        db_, xb = blocked(dout, fill), blocked(x, fill)
        abi.call("hg_act_wgrad_blocked", abi.ptr(db_), abi.ptr(ps), abi.ptr(xb), T * Cx * 128, Cx, abi.ptr(mod), act, abi.ptr(dw),
                 abi.ptr(db), abi.ptr(ws), B, C, Hg, Wg, passes, abi.stream())
        torch.cuda.synchronize()      # the workspace is shared by the launches
        return dw.clone(), db.clone(), (b1, b2)
    runs = [launch(float("nan")), launch(0.0), launch(0.0)]
    assert all(_intact(b) for r in runs for b in r[2])
    for i in (0, 1):
        assert torch.equal(runs[i][0], runs[i + 1][0]) and torch.equal(runs[i][1], runs[i + 1][1]), \
            "NaN padding or a repeated launch changed dW / db"
    dw, db = runs[1][0], runs[1][1]

    def ref_of(psd):
        xd = x.double()
        if act == 1:
            t = xd * mod[:, 0, :, None].double() + mod[:, 1, :, None].double()
            y, ey = torch.sin(t), U * t.abs() + SIN_ABS
        else:
            y, ey = xd, torch.zeros_like(xd)
        gd = dout.double() * (psd[:, :, None] if psd is not None else 1.0)
        ref_w = torch.einsum("bop,bip->oi", gd, y)
        ref_b = gd.sum((0, 2))
        coef = (116 + 6 * n_t) * U if passes == 3 else 2.0 ** -8 + (132 + 6 * n_t) * U
        bw = coef * torch.einsum("bop,bip->oi", gd.abs(), y.abs()) + torch.einsum("bop,bip->oi", gd.abs(), ey)
        bb = (116 + 6 * n_t) * U * gd.abs().sum((0, 2))
        return ref_w, ref_b, bw, bb
    psd = ps.double() if ps is not None else None
    ref_w, ref_b, bw, bb = ref_of(psd)
    chk = _Checks(f"act_wgrad {case} B{B} {Hg}x{Wg} T{T} n_t {n_t}")
    chk.add("dW", (dw.double() - ref_w).abs(), bw)
    chk.add("db", (db.double() - ref_b).abs(), bb)
    chk.done()
    if ps is not None and B > 1 and passes == 3:
        # one tile's pscale row belonging to the wrong image: tile 0 of image 1 scaled with image 0's row
        x_t = x[1:2, :, :128]
        gd_t = dout[1:2, :, :128].double()
        y_t = torch.sin(x_t.double() * mod[1:2, 0, :, None].double() + mod[1:2, 1, :, None].double()) if act == 1 else x_t.double()
        dpsd = (psd[0] - psd[1])[None, :, None]
        ref_f = ref_w + torch.einsum("bop,bip->oi", gd_t * dpsd, y_t)
        ratio = ((dw.double() - ref_f).abs() / bw).max().item()
        print(f"  fault: {ratio:.0f}x the bound")
        assert ratio > 10, ratio
