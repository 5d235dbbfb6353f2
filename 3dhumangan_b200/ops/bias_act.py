"""bias_act: y = clamp(act(x + b) * gain)  (reference: lib/components/ops/bias_act.py:52-86, bias_act.cu:24-165).

Same Python signature as the reference op.  The reference defaults to `impl='ref'` (plain torch
ops) and its CUDA plugin cannot even be built (SURVEY.md fact 2); here there is exactly one
implementation, the sm_90a kernels behind `hg_bias_act` / `hg_bias_act_grad`.

Differentiable to second order like the reference's cached autograd classes (bias_act.py:124-207):
the forward op saves y (or x for swish), its backward is itself an autograd op whose backward
re-applies the first derivative to the incoming gradient and, for the smooth activations, adds the
second-derivative term towards x and b.
"""
import math

import torch

from .. import abi

# name -> (id, default alpha, default gain, keeps 'x'|'y'|'', has a second derivative)   (bias_act.py:22-32)
ACTIVATIONS = {
    "linear": (1, 0.0, 1.0, "", False), "relu": (2, 0.0, math.sqrt(2), "y", False),
    "lrelu": (3, 0.2, math.sqrt(2), "y", False), "tanh": (4, 0.0, 1.0, "y", True),
    "sigmoid": (5, 0.0, 1.0, "y", True), "elu": (6, 0.0, 1.0, "y", True), "selu": (7, 0.0, 1.0, "y", True),
    "softplus": (8, 0.0, 1.0, "y", True), "swish": (9, 0.0, math.sqrt(2), "x", True),
}


def _geometry(x, dim, b):
    step = 1
    for s in x.shape[dim + 1:]:
        step *= s
    return step, (x.shape[dim] if b is not None else 1)


def _launch_fwd(x, b, dim, spec):
    aid, alpha, gain, clamp = spec
    y = torch.empty_like(x)
    step, size = _geometry(x, dim, b)
    with torch.cuda.device_of(x):
        abi.call("hg_bias_act", abi.ptr(x), abi.ptr(b), abi.ptr(y), x.numel(), step, size, aid, alpha, gain, clamp,
                 abi.stream())
    return y


def _launch_grad(g, b, xref, yref, dy, dim, order, spec):
    aid, alpha, gain, clamp = spec
    g = g.contiguous()
    dy = dy.contiguous() if dy is not None else None
    out = torch.empty_like(g)
    step, size = _geometry(g, dim, b)
    with torch.cuda.device_of(g):
        abi.call("hg_bias_act_grad", abi.ptr(g), abi.ptr(b), abi.ptr(xref), abi.ptr(yref),
                 abi.ptr(dy), abi.ptr(out), g.numel(), step, size, order, aid,
                 alpha, gain, clamp, abi.stream())
    return out


def _sum_to_bias(t, dim):
    return t.sum([i for i in range(t.ndim) if i != dim])


class _BiasAct(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, b, dim, act, spec):
        y = _launch_fwd(x, b, dim, spec)
        keeps, second = ACTIVATIONS[act][3], ACTIVATIONS[act][4]
        ctx.dim, ctx.act, ctx.spec = dim, act, spec
        keep_x = keeps == "x" or second
        ctx.save_for_backward(x if keep_x else None, b if keep_x else None, y if keeps == "y" or spec[3] >= 0 else None)
        return y

    @staticmethod
    def backward(ctx, dy):
        x, b, y = ctx.saved_tensors
        dx = db = None
        if ctx.needs_input_grad[0] or ctx.needs_input_grad[1]:
            dx = _BiasActGrad.apply(dy, x, b, y, ctx.dim, ctx.act, ctx.spec)
        if ctx.needs_input_grad[1]:
            db = _sum_to_bias(dx, ctx.dim)
        return dx, db, None, None, None


class _BiasActGrad(torch.autograd.Function):
    @staticmethod
    def forward(ctx, dy, x, b, y, dim, act, spec):
        dx = _launch_grad(dy, b, x, y, None, dim, 1, spec)
        ctx.dim, ctx.act, ctx.spec = dim, act, spec
        ctx.save_for_backward(dy if ACTIVATIONS[act][4] else None, x, b, y)
        return dx

    @staticmethod
    def backward(ctx, d_dx):
        dy, x, b, y = ctx.saved_tensors
        second = ACTIVATIONS[ctx.act][4]
        d_dy = d_x = d_b = None
        if ctx.needs_input_grad[0]:
            d_dy = _BiasActGrad.apply(d_dx, x, b, y, ctx.dim, ctx.act, ctx.spec)
        if second and (ctx.needs_input_grad[1] or ctx.needs_input_grad[2]):
            d_x = _launch_grad(d_dx, b, x, y, dy, ctx.dim, 2, ctx.spec)
        if second and ctx.needs_input_grad[2]:
            d_b = _sum_to_bias(d_x, ctx.dim)
        return d_dy, d_x, d_b, None, None, None, None


def bias_act(x, b=None, dim=1, act="linear", alpha=None, gain=None, clamp=None, impl="cuda"):
    if act not in ACTIVATIONS:
        raise RuntimeError(f"bias_act: unknown activation {act!r}")
    aid, dalpha, dgain = ACTIVATIONS[act][:3]
    if clamp is not None and clamp < 0:
        raise RuntimeError("bias_act: clamp must be None or >= 0")
    spec = (aid, float(dalpha if alpha is None else alpha), float(dgain if gain is None else gain),
            float(-1 if clamp is None else clamp))
    if b is not None:
        if b.ndim != 1 or not (0 <= dim < x.ndim) or b.shape[0] != x.shape[dim]:
            raise RuntimeError("bias_act: bias must be 1-D and match x.shape[dim]")
        b = b.float().contiguous()
    y = _BiasAct.apply(x.float().contiguous(), b, dim, act, spec)
    return y.to(x.dtype)
