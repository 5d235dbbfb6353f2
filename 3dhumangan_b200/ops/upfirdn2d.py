"""upfirdn2d: pad / zero-insert up-sample / FIR / decimate  (reference: lib/components/ops/upfirdn2d.py:117-161,
upfirdn2d.cu:29-375).  Same Python signatures (`upfirdn2d`, `setup_filter`, `filter2d`, `upsample2d`,
`downsample2d`); one implementation, the sm_90a kernel behind `hg_upfirdn2d`.

Differentiable to any order in x: the adjoint of an up/FIR/down pass is the same kind of pass with up and
down exchanged, the filter flipped and the padding mirrored (upfirdn2d.py:213-231 does the same), so the
backward of the autograd op below is another application of itself.
"""
import numpy as np
import torch

from .. import abi


def _pair(v):
    if isinstance(v, int):
        return v, v
    v = list(v)
    assert len(v) == 2
    return int(v[0]), int(v[1])


def _padding(p):
    if isinstance(p, int):
        p = [p, p]
    p = [int(v) for v in p]
    if len(p) == 2:
        p = [p[0], p[0], p[1], p[1]]
    assert len(p) == 4
    return p


def setup_filter(f, device=torch.device("cpu"), normalize=True, flip_filter=False, gain=1, separable=None):
    """upfirdn2d.py:66-113."""
    if f is None:
        f = 1
    f = torch.as_tensor(f, dtype=torch.float32)
    assert f.ndim in (0, 1, 2) and f.numel() > 0
    if f.ndim == 0:
        f = f[np.newaxis]
    if separable is None:
        separable = f.ndim == 1 and f.numel() >= 8
    if f.ndim == 1 and not separable:
        f = f.ger(f)
    assert f.ndim == (1 if separable else 2)
    if normalize:
        f = f / f.sum()
    if flip_filter:
        f = f.flip(list(range(f.ndim)))
    f = f * (gain ** (f.ndim / 2))
    return f.to(device=device)


def _run(x, f2d, upx, upy, downx, downy, px0, px1, py0, py1, flip, gain):
    B, C, H, W = x.shape
    fH, fW = f2d.shape
    outH = (H * upy + py0 + py1 - fH) // downy + 1
    outW = (W * upx + px0 + px1 - fW) // downx + 1
    y = torch.empty(B, C, max(outH, 0), max(outW, 0), dtype=torch.float32, device=x.device)
    if y.numel() == 0:
        return y
    with torch.cuda.device_of(x):
        abi.call("hg_upfirdn2d", abi.ptr(x), abi.ptr(f2d), abi.ptr(y), B * C, H, W, outH, outW, fH, fW, upx, upy,
                                         downx, downy, px0, py0, int(bool(flip)), float(gain), abi.stream())
    return y


class _Pass(torch.autograd.Function):
    """One 2-D up/FIR/down pass.  geom = (upx, upy, downx, downy, px0, px1, py0, py1, flip, gain)."""

    @staticmethod
    def forward(ctx, x, f2d, geom):
        ctx.geom, ctx.in_hw = geom, (x.shape[2], x.shape[3])
        ctx.save_for_backward(f2d)
        return _run(x.contiguous(), f2d, *geom)

    @staticmethod
    def backward(ctx, dy):
        (f2d,) = ctx.saved_tensors
        upx, upy, downx, downy, px0, px1, py0, py1, flip, gain = ctx.geom
        ih, iw = ctx.in_hw
        oh, ow = dy.shape[2], dy.shape[3]
        fh, fw = f2d.shape
        # dx[i] = sum_o dy[o] * g[i*up - o*down + pad0]: a pass over dy with up<->down, the filter mirrored
        # (pad0' = taps - 1 - pad0) and pad1' whatever makes the output the input's size again
        back = (downx, downy, upx, upy, fw - px0 - 1, iw * upx - ow * downx + px0 - upx + 1, fh - py0 - 1,
                ih * upy - oh * downy + py0 - upy + 1, not flip, gain)
        dx = _Pass.apply(dy, f2d, back) if ctx.needs_input_grad[0] else None
        return dx, None, None


_SEP_TAPS = (4, 6, 8, 12, 16)


class _SepPass(torch.autograd.Function):
    """Both 1-D passes of a separable 2x up- or down-sampling FIR in ONE kernel (`hg_upfirdn2d_sep2`, the intermediate stays
    in shared memory).  geom = (up, down, px0, px1, py0, py1, flip, gain) with (up, down) in {(2, 1), (1, 2)}.  Its adjoint
    is the other direction with the filter mirrored, so the backward is another `_SepPass` (any order)."""

    @staticmethod
    def forward(ctx, x, f1d, geom):
        up, down, px0, px1, py0, py1, flip, gain = geom
        x = x.contiguous()
        B, C, H, W = x.shape
        T = f1d.numel()
        outH = (H * up + py0 + py1 - T) // down + 1
        outW = (W * up + px0 + px1 - T) // down + 1
        ctx.geom, ctx.in_hw = geom, (H, W)
        ctx.save_for_backward(f1d)
        y = torch.empty(B, C, max(outH, 0), max(outW, 0), dtype=torch.float32, device=x.device)
        if y.numel():
            with torch.cuda.device_of(x):
                abi.call("hg_upfirdn2d_sep2", abi.ptr(x), abi.ptr(f1d), abi.ptr(y), B * C, H, W, outH, outW, T, int(up == 2),
                         px0, py0, int(bool(flip)), float(gain), abi.stream())
        return y

    @staticmethod
    def backward(ctx, dy):
        (f1d,) = ctx.saved_tensors
        up, down, px0, px1, py0, py1, flip, gain = ctx.geom
        ih, iw = ctx.in_hw
        oh, ow = dy.shape[2], dy.shape[3]
        T = f1d.numel()
        back = (down, up, T - px0 - 1, iw * up - ow * down + px0 - up + 1, T - py0 - 1, ih * up - oh * down + py0 - up + 1,
                not flip, gain)
        dx = _SepPass.apply(dy, f1d, back) if ctx.needs_input_grad[0] else None
        return dx, None, None


def upfirdn2d(x, f, up=1, down=1, padding=0, flip_filter=False, gain=1, impl="cuda"):
    assert x.ndim == 4
    upx, upy = _pair(up)
    downx, downy = _pair(down)
    px0, px1, py0, py1 = _padding(padding)
    xin = x.float()
    if f is None:
        f = torch.ones(1, 1, dtype=torch.float32, device=x.device)
    f = f.detach().to(device=x.device, dtype=torch.float32).contiguous()
    flip = bool(flip_filter)
    fused = (f.ndim == 1 and f.numel() in _SEP_TAPS and upx == upy and downx == downy and (upx, downx) in ((2, 1), (1, 2))
             and float(gain) >= 0)
    if fused:       # the reference's call shapes (augment.py:314,325): one kernel, no HBM round trip of the intermediate
        y = _SepPass.apply(xin, f, (upx, downx, px0, px1, py0, py1, flip, float(gain)))
    elif f.ndim == 2:
        y = _Pass.apply(xin, f, (upx, upy, downx, downy, px0, px1, py0, py1, flip, float(gain)))
    else:  # separable: a [1,fw] pass then a [fh,1] pass, gain split as in upfirdn2d.py:243-244
        g = float(gain) ** 0.5
        y = _Pass.apply(xin, f[None, :].contiguous(), (upx, 1, downx, 1, px0, px1, 0, 0, flip, g))
        y = _Pass.apply(y, f[:, None].contiguous(), (1, upy, 1, downy, 0, 0, py0, py1, flip, g))
    return y.to(x.dtype)


def _filter_size(f):
    if f is None:
        return 1, 1
    return (int(f.shape[-1]), int(f.shape[0]))


def filter2d(x, f, padding=0, flip_filter=False, gain=1, impl="cuda"):
    px0, px1, py0, py1 = _padding(padding)
    fw, fh = _filter_size(f)
    p = [px0 + fw // 2, px1 + (fw - 1) // 2, py0 + fh // 2, py1 + (fh - 1) // 2]
    return upfirdn2d(x, f, padding=p, flip_filter=flip_filter, gain=gain)


def upsample2d(x, f, up=2, padding=0, flip_filter=False, gain=1, impl="cuda"):
    upx, upy = _pair(up)
    px0, px1, py0, py1 = _padding(padding)
    fw, fh = _filter_size(f)
    p = [px0 + (fw + upx - 1) // 2, px1 + (fw - upx) // 2, py0 + (fh + upy - 1) // 2, py1 + (fh - upy) // 2]
    return upfirdn2d(x, f, up=up, padding=p, flip_filter=flip_filter, gain=gain * upx * upy)


def downsample2d(x, f, down=2, padding=0, flip_filter=False, gain=1, impl="cuda"):
    downx, downy = _pair(down)
    px0, px1, py0, py1 = _padding(padding)
    fw, fh = _filter_size(f)
    p = [px0 + (fw - downx + 1) // 2, px1 + (fw - downx) // 2, py0 + (fh - downy + 1) // 2, py1 + (fh - downy) // 2]
    return upfirdn2d(x, f, down=down, padding=p, flip_filter=flip_filter, gain=gain)
