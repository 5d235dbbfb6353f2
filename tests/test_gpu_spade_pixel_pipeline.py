"""The pixel-style `hg_spade_conv` kernel across tile boundaries, against fp64.

Each persistent CTA of `spade_pixel_kernel` carries state from one tile to the next: the position and phase of its
16 KB weight-ring units (24 fills per fp32x3 tile, 12 per bf16 tile, over 4 units), the activation and residual rings, and
the per-sample A1 gather.  A CTA that mixed up two tiles' samples, or one ring unit's phase, would read another tile's
operands.  These launches are built so that such a mix-up cannot pass:
  - `smp1`:  SMs + 1 tiles of one sample: every CTA takes one tile, CTA 0 takes two (the only walk with a next tile),
             and the last tile is ragged;
  - `walk`:  at least 3 x SMs tiles over several samples of fewer than SMs tiles each, so every step of every CTA's walk
             lands in another sample; the last tile of each sample is ragged.
Each shape runs at passes 3 (fp32x3) and 1 (bf16), with ToRGB (rgb_w + rgb_in), with the next-BatchNorm statistics, with
a residual, and with all three.  Every output sits between sentinel guards, and a repeated launch gives a bit-identical
out and rgb_out (the statistics use float atomics in shared memory and are checked against their bound instead)."""
import importlib
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

C = 256
STAT_STRIDE = 520          # modules/synthesis_ops.py: [0:256] sum, [256:512] sumsq, [512] count, pad
U = 2.0 ** -24
G = 64                     # guard elements on each side of an output
SENTINEL = -1234.5


def _nsm():
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def _shape(name):
    """(B, Hg, Wg) of a named case."""
    n = _nsm()
    if name == "smp1":                       # T = n + 1, last tile holds 88 pixels
        HW = n * 128 + 88
        return 1, HW // 8, 8
    T = n // 2 + 3                           # fewer than n tiles per sample, last tile holds 72 pixels
    HW = (T - 1) * 128 + 72
    B = -(-3 * n // T) + 1
    return B, HW // 8, 8


def _tiles(HW):
    return (HW + 127) // 128


def _blocked(t):
    B, Cc, HW = t.shape
    T = _tiles(HW)
    pad = torch.zeros((B, Cc, T * 128), dtype=t.dtype, device=t.device)
    pad[:, :, :HW] = t
    return pad.reshape(B, Cc, T, 128).permute(0, 2, 1, 3).contiguous()


def _planar(t, HW):
    B, T, Cc, _ = t.shape
    return t.permute(0, 2, 1, 3).reshape(B, Cc, T * 128)[:, :, :HW]


def _guarded(shape, dtype=torch.float32, fill=float("nan")):
    n = math.prod(shape)
    buf = torch.full((n + 2 * G,), SENTINEL, dtype=dtype, device="cuda")
    view = buf[G:G + n].view(shape)
    view.fill_(fill)
    return buf, view


def _intact(buf):
    return bool((buf[:G] == SENTINEL).all()) and bool((buf[-G:] == SENTINEL).all())


@pytest.mark.parametrize("flags", ["rgb", "stats", "skip", "rgb-stats-skip"])
@pytest.mark.parametrize("passes", [3, 1])
@pytest.mark.parametrize("shape", ["smp1", "walk"])
def test_pixel_pipeline(shape, passes, flags):
    abi = importlib.import_module("3dhumangan_b200.abi")
    so = importlib.import_module("3dhumangan_b200.modules.synthesis_ops")
    B, Hg, Wg = _shape(shape)
    HW, T = Hg * Wg, _tiles(Hg * Wg)
    tiles, n = B * T, _nsm()
    assert tiles == n + 1 if shape == "smp1" else (tiles >= 3 * n and T < n)
    grid = min(tiles, n)
    n_t = -(-tiles // grid)
    Rh, Rw = max(1, round(Hg * 96 / 512)), max(1, round(Wg * 96 / 512))
    g = torch.Generator(device="cuda").manual_seed(140 + passes)
    r = lambda *s: torch.randn(*s, generator=g, device="cuda")
    x = r(B, C, HW)
    W = r(C, C)
    inv_sigma = (1.0 / torch.linalg.matrix_norm(W.double(), 2)).float().reshape(1)
    wimg = abi.pack_weight(W, Nb=256, scale_dev=inv_sigma)[0]
    bias = 0.1 * r(C)
    p_all = 0.7 * r(B * Rh * Rw, 384)                          # the slice at columns 128:256 is P_lr (p_stride 384)
    p_bias = (0.3 * r(B, 128)).contiguous()
    scsh = torch.stack([1.0 + 0.3 * r(C), 0.3 * r(C)]).contiguous()
    wg, wb, bg, bb = r(C, 128) / 16, r(C, 128) / 16, 0.1 * r(C), 0.1 * r(C)
    w_il, b_il = so._gamma_beta_interleaved(wg, bg, wb, bb)
    skip = r(B, C, HW) if "skip" in flags else None
    rgb = "rgb" in flags
    rgb_w, rgb_b, rgb_in = (r(3, C) / 16, r(3), r(B, 3, HW)) if rgb else (None, None, None)
    xb, skipb = _blocked(x), None if skip is None else _blocked(skip)
    kw = dict(scsh=scsh, p_lr=so._PtrView(p_all[:, 128:]), p_stride=384, p_bias=p_bias, wgb=abi.pack_weight(w_il, Nb=256)[0],
              bgb=b_il, Rh=Rh, Rw=Rw)

    # fp64 reference from the inputs, per sample
    P = p_all[:, 128:256].double().reshape(B, Rh, Rw, 128).permute(0, 3, 1, 2)
    a1 = torch.relu(F.interpolate(P, (Hg, Wg), mode="bilinear", align_corners=False).reshape(B, 128, HW) + p_bias.double()[:, :, None])
    gam = 1.0 + torch.einsum("ck,bkp->bcp", wg.double(), a1) + bg.double()[None, :, None]
    bet = torch.einsum("ck,bkp->bcp", wb.double(), a1) + bb.double()[None, :, None]
    pre = (x.double() * scsh[0, None, :, None].double() + scsh[1, None, :, None].double()) * gam + bet
    ref = torch.einsum("oc,bcp->bop", W.double() * inv_sigma.double(), torch.where(pre > 0, pre, 0.2 * pre)) + bias.double()[None, :, None]
    if skip is not None:
        ref = ref + skip.double()
    del a1, gam, bet, pre

    def launch():
        obuf, out = _guarded((B, T, C, 128))
        res, bufs, rk = dict(out=out), [obuf], dict(kw)
        if rgb:
            rbuf, rgb_out = _guarded((B, 3, HW))
            bufs.append(rbuf)
            rk.update(rgb_w=rgb_w, rgb_b=rgb_b, rgb_in=rgb_in, rgb_out=rgb_out)
            res["rgb_out"] = rgb_out
        if "stats" in flags:
            sbuf, row = _guarded((STAT_STRIDE,), torch.float64, 0.0)
            row[512] = float(B * HW)
            bufs.append(sbuf)
            rk.update(stats=row)
            res["row"] = row
        abi.spade_conv(xb, T * C * 128, wimg, bias, out, B=B, Hg=Hg, Wg=Wg, skip=skipb, passes=passes, **rk)
        res["bufs"] = bufs
        return res

    runs = [launch(), launch()]
    torch.cuda.synchronize()
    for res in runs:
        assert all(_intact(b) for b in res["bufs"]), "a guard element was overwritten"
    outs = [_planar(res["out"], HW) for res in runs]
    assert torch.equal(outs[0], outs[1]), "a repeated launch changed out"
    assert torch.isfinite(outs[0]).all(), "a valid output is not finite"
    # passes 3: the 2e-5 bar of test_gpu_spade_conv.py's pixel-style cases; passes 1: its bf16 bar
    tol = 2e-5 if passes == 3 else 2e-2
    err_s = [((outs[0][b].double() - ref[b]).abs().max() / ref[b].abs().max()).item() for b in range(B)]
    print(f"{shape} p{passes} {flags}: B {B} T {T} grid {grid}, max err / max ref per sample {max(err_s):.2e}")
    assert max(err_s) < tol, err_s
    o = outs[0].double()
    if rgb:
        assert torch.equal(runs[0]["rgb_out"], runs[1]["rgb_out"]), "a repeated launch changed rgb_out"
        w = rgb_w.double()
        rref = torch.einsum("kc,bcp->bkp", w, o) + rgb_b.double()[None, :, None] + rgb_in.double()
        mag = torch.einsum("kc,bcp->bkp", w.abs(), o.abs()) + rgb_b.double().abs()[None, :, None] + rgb_in.double().abs()
        assert ((runs[0]["rgb_out"].double() - rref).abs() <= 68 * U * mag).all(), "rgb_out"   # bound of test_gpu_spade_conv
    if "stats" in flags:
        for res in runs:
            row = res["row"]
            for k, (s, mag) in enumerate(((o.sum((0, 2)), o.abs().sum((0, 2))), ((o * o).sum((0, 2)), (o * o).sum((0, 2))))):
                assert ((row[k * C:(k + 1) * C] - s).abs() <= (4 + 8 * n_t) * U * mag).all(), ("sum", "sumsq")[k]
            assert row[512] == float(B * HW) and (row[513:] == 0).all(), "the count and pad slots must stay untouched"
