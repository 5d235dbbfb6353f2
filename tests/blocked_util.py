"""Shapes, layouts and checks shared by the launch-by-launch tests of the blocked-GEMM engine (tests/test_gpu_spade_conv.py,
forward) and of the SPADE half-blocks' backward kernels (tests/test_gpu_synthesis_bwd_kernels.py)."""
import itertools
import math

import torch

C = 256
U = 2.0 ** -24             # fp32 unit roundoff
G = 64                     # guard elements on each side of an output (keeps 16-byte alignment in fp32 and fp64)
SENTINEL = -1234.5


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
    n = _nsm()
    if name == "walk":             # T > SMs tiles per sample and >= 16 tiles per CTA: each persistent CTA walks several
        Wg = 100                   # tiles of one sample, then crosses into the next; the last tile holds 60 valid pixels
        Hg = (5 * n // 2) * 128 // Wg + 1
        T = (Hg * Wg + 127) // 128
        B = -(-16 * n // T)
        assert T > n and B * T >= 16 * n and (Hg * Wg) % 128 and (Hg * Wg) % 4 == 0
        return B, Hg, Wg
    # "multi": T < SMs tiles per sample and B*T >= 2 SMs tiles
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


def _pairs(levels, valid=None):
    """Every (option, value, option, value) pair that some row of the product of `levels` allowed by `valid` contains."""
    names = list(levels)
    rows = [dict(zip(names, r)) for r in itertools.product(*levels.values())]
    return {(a, d[a], b, d[b]) for d in rows if valid is None or valid(d) for a, b in itertools.combinations(names, 2)}


def _pairwise(levels, valid=None):
    """Rows of the full product of `levels` (a dict name -> values), restricted to the rows `valid` accepts (all when None),
    chosen greedily until every pair of values of every two options that some allowed row holds appears in a row;
    deterministic."""
    names = list(levels)
    todo = _pairs(levels, valid)
    cands = [r for r in itertools.product(*levels.values()) if valid is None or valid(dict(zip(names, r)))]
    rows = []
    while todo:
        best = max(cands,
                   key=lambda r: sum((a, r[i], b, r[j]) in todo for (i, a), (j, b) in itertools.combinations(enumerate(names), 2)))
        d = dict(zip(names, best))
        todo -= {(a, d[a], b, d[b]) for a, b in itertools.combinations(names, 2)}
        rows.append(d)
    return rows


def _sums_bound(n_t):
    """Relative bound of the engine's epilogue column sums: per tile and channel a thread adds its 2 rows (1 fp32 add),
    three shuffle steps fold the 16 rows of a warp (3 adds), and each of the 8 warps adds its total to the CTA's fp32
    shared sum, over n_t tiles per CTA between flushes: at most 4 + 8 n_t roundings on any path, each at most u = 2^-24
    of a partial sum bounded by sum |v|, so |err| <= (4 + 8 n_t) u sum|v| (first-order gamma_n bound).  The flushes go to
    fp64 (2^-53 per add)."""
    return (4 + 8 * n_t) * U


def _check_stats(row, init, outp, n_t):
    """row = init + (sum, sumsq) over the valid pixels of the kernel's own out, per channel, in fp64, within `_sums_bound`."""
    o = outp.double()
    terms = ((o.sum((0, 2)), o.abs().sum((0, 2))), ((o * o).sum((0, 2)), (o * o).sum((0, 2))))
    for k, (ref, mag) in enumerate(terms):
        err = (row[k * C:(k + 1) * C] - init[k * C:(k + 1) * C] - ref).abs()
        bound = _sums_bound(n_t) * mag + 1e-13 * init[k * C:(k + 1) * C].abs()
        assert (err <= bound).all(), ("sum" if k == 0 else "sumsq", float((err / bound).max()))
    assert torch.equal(row[512:], init[512:]), "the count and pad slots [512:520] must stay untouched"
