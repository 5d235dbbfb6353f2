"""The renderer's input stage launch by launch against fp64: `hg_vertex_ik`, `hg_knn_prep` and `hg_geo_features`
(csrc/geo.cu), `hg_sample_fine` and `hg_merge_samples` (csrc/sample.cu).

Every launch goes through `abi.call` with buffers the test owns, so that each output can be pre-filled with NaN (an
element the kernel does not write fails) and sits between guard elements that must stay untouched.  Each launch is
repeated and must repeat bit for bit (every kernel here is deterministic).

Bounds start from U = 2^-24 and count the roundings of the kernel's fp32 arithmetic, componentwise; each check prints
its worst error and the fraction of its bound that error uses.  Where the kernel is specified as exact -- the nearest
index and squared distance (the fp32 restatement of `oracle.port.knn1`), the Morton sort and its cluster boxes, the
merge (`torch.sort(stable=True)` + gather) -- the comparison is bit for bit.  The fp64 references use the fp32 values
of the kernels' constants (2.4f, 1.3f, 0.2f, 1e-5f): those are the operations the kernels and the fp32 oracle perform.

A drift check records the calls of the module code in the forwards that reach these kernels and fails on any call
form the matrices below do not hold.  Non-finite inputs (NaN and overflowing points, NaN depths, a NaN FiLM code)
close the file: a NaN point has nearest index 0 and d2 NaN, as `knn1` gives, and NaN depths sort last."""
import importlib
import math
from ctypes import c_void_p

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
GUARD = 1024
SENTINEL = -1234.5
ISENTINEL = -77
F32 = lambda v: float(np.float32(v))          # noqa: E731  the fp32 value of a kernel constant
SUB = 65536                                   # fp64 checks: at least this many points per launch (all when fewer)


def _abi():
    return importlib.import_module("3dhumangan_b200.abi")


def _pkg():
    return importlib.import_module("3dhumangan_b200")


def _port():
    return importlib.import_module("oracle.port")


def _nsm():
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def _guarded(shape, dtype=torch.float32, fill=float("nan")):
    """(buffer, view): a contiguous view of `shape` inside a buffer with GUARD sentinel elements on each side."""
    n = math.prod(shape)
    sent = ISENTINEL if dtype == torch.int32 else SENTINEL
    buf = torch.full((n + 2 * GUARD,), sent, dtype=dtype, device="cuda")
    view = buf[GUARD:GUARD + n].view(shape)
    view.fill_(ISENTINEL if dtype == torch.int32 else fill)
    return buf, view


def _intact(*bufs):
    for buf in bufs:
        if buf is None:
            continue
        sent = ISENTINEL if buf.dtype == torch.int32 else SENTINEL
        assert bool((buf[:GUARD] == sent).all()) and bool((buf[-GUARD:] == sent).all()), "guard elements overwritten"


def _written(*views):
    for v in views:
        if v is None:
            continue
        if v.dtype == torch.int32:
            assert not bool((v == ISENTINEL).any()), "unwritten integer output"
        else:
            assert not bool(v.isnan().any()), "unwritten (NaN) output"


def _same(a, b):
    """Bit-identical, NaN payloads included."""
    if a is None:
        return b is None
    if a.dtype == torch.float32:
        return torch.equal(a.view(torch.int32), b.view(torch.int32))
    return torch.equal(a, b)


class _Checks:
    """Collects (name, err, bound) per check, prints the worst ratio of each, then asserts them all."""

    def __init__(self, label):
        self.label, self.rows = label, []

    def add(self, name, err, bound):
        err, bound = err.double(), bound.double()
        assert err.shape == bound.shape
        ratio = (err / bound.clamp_min(1e-300)).max().item() if err.numel() else 0.0
        ratio = ratio if not math.isnan(ratio) else math.inf
        self.rows.append((name, ratio, err.max().item() if err.numel() else 0.0))
        return ratio

    def done(self):
        print(self.label + ": " + ", ".join(f"{n} {e:.2e} ({r:.3f} of bound)" for n, r, e in self.rows))
        bad = [(n, r) for n, r, _ in self.rows if not r <= 1.0]
        assert not bad, bad


def _sub(total):
    """Strided subsample of [0, total) with at least SUB entries (all when fewer), the last index included."""
    step = max(1, total // SUB)
    idx = torch.arange(0, total, step, device="cuda")
    if int(idx[-1]) != total - 1:
        idx = torch.cat([idx, torch.tensor([total - 1], device="cuda")])
    return idx


_COND = {}


def _cond(B, seed=5):
    """Synthetic posed bodies (V = 6890) on the device, cached per (B, seed)."""
    key = (B, seed)
    if key not in _COND:
        _COND[key] = {k: v.cuda() for k, v in _pkg().synthetic.make_conditions(B, seed=seed).items()}
    return _COND[key]


# ======================================================================================================================
# hg_vertex_ik
# ======================================================================================================================
def _rot(g, n):
    """n random rotations (fp64) from QR of Gaussian matrices."""
    q, r = torch.linalg.qr(torch.randn(n, 3, 3, generator=g, dtype=torch.float64))
    q = q * torch.sign(torch.diagonal(r, dim1=-2, dim2=-1))[:, None, :]
    return q


def _fk(kind, B, g):
    fk = torch.zeros(B, 24, 4, 4, dtype=torch.float64)
    fk[:, :, 3, 3] = 1
    n = B * 24
    if kind == "swap":            # 90-degree rotations with zero diagonals: every column needs a row swap
        perms = [(1, 2, 0), (2, 0, 1)]
        R = torch.zeros(n, 3, 3, dtype=torch.float64)
        for i in range(n):
            p = perms[i % 2]
            for r in range(3):
                R[i, r, p[r]] = 1.0 if (i + r) % 3 else -1.0
    elif kind == "scale":         # rotations times per-axis scales in 1e-2..1e2
        s = 10.0 ** (torch.rand(n, 3, generator=g, dtype=torch.float64) * 4 - 2)
        R = _rot(g, n) * s[:, None, :]
    else:                         # the posed synthetic skeleton's kind: rigid
        R = _rot(g, n)
    fk[:, :, :3, :3] = R.reshape(B, 24, 3, 3)
    fk[:, :, :3, 3] = torch.randn(B, 24, 3, generator=g, dtype=torch.float64)
    return fk.float()


def _lbs(kind, B, V, g):
    if kind == "convex":
        w = torch.softmax(torch.randn(B, V, 24, generator=g) * 3, -1)
    elif kind == "sparse":       # up to 4 joints, as SMPL's skinning weights
        w = torch.rand(B, V, 24, generator=g)
        keep = torch.rand(B, V, 24, generator=g).argsort(-1) < 4
        w = w * keep
        w = w / w.sum(-1, keepdim=True)
    else:                        # single joint
        j = torch.randint(0, 24, (B, V), generator=g)
        w = torch.nn.functional.one_hot(j, 24).float()
    return w.float().contiguous()


def _run_vertex_ik(fk, lbs):
    abi = _abi()
    B, V = lbs.shape[:2]
    buf, out = _guarded((B, V, 16))
    abi.call("hg_vertex_ik", abi.ptr(fk), abi.ptr(lbs), B, V, abi.ptr(out), abi.stream())
    return buf, out


VIK_V = [1, 127, 128, 129, 6890]
VIK_CASES = [(fk, w) for fk in ("rigid", "swap", "scale") for w in ("convex", "sparse", "single")]


@pytest.mark.parametrize("V", VIK_V)
@pytest.mark.parametrize("fk_kind,w_kind", VIK_CASES)
def test_vertex_ik(V, fk_kind, w_kind):
    """vertex_ik[b,v] = sum_j w_j inverse(fk_j) against fp64.  The bound per element is gamma_25 sum_j |w_j||ik_j| (the
    24 fused multiply-adds) plus sum_j |w_j| 32 kappa_j U max|ik_j| (Gauss-Jordan with partial pivoting on a 4x4,
    kappa_j the fp64 2-norm condition number of fk_j)."""
    _abi().require_device()
    g = torch.Generator().manual_seed(V * 7 + len(fk_kind) + 3 * len(w_kind))
    B = 3
    fk, lbs = _fk(fk_kind, B, g).cuda(), _lbs(w_kind, B, V, g).cuda()
    buf, out = _run_vertex_ik(fk, lbs)
    buf2, out2 = _run_vertex_ik(fk, lbs)
    torch.cuda.synchronize()
    _intact(buf, buf2)
    _written(out)
    assert _same(out, out2), "not repeatable"
    ik = torch.linalg.inv(fk.double())                                   # [B,24,4,4]
    kappa = torch.linalg.cond(fk.double())                               # [B,24]
    w = lbs.double()
    ref = torch.einsum("bvj,bjk->bvk", w, ik.reshape(B, 24, 16))
    gam = 25 * U / (1 - 25 * U)
    inv_err = 32 * kappa * U * ik.abs().flatten(2).amax(-1)               # [B,24]
    bound = gam * torch.einsum("bvj,bjk->bvk", w.abs(), ik.abs().reshape(B, 24, 16)) \
        + torch.einsum("bvj,bj->bv", w.abs(), inv_err)[..., None]
    c = _Checks(f"vertex_ik V={V} {fk_kind}/{w_kind}")
    c.add("vertex_ik", (out.double() - ref).abs(), bound)
    c.done()


# ======================================================================================================================
# hg_knn_prep
# ======================================================================================================================
def _body(kind, V, g):
    """[V,3] fp32 vertex set of a given shape."""
    if kind == "blob":
        v = torch.randn(V, 3, generator=g) * torch.tensor([0.3, 0.8, 0.15])
    elif kind == "flat":
        v = torch.randn(V, 3, generator=g)
        v[:, 2] = 0.25
    elif kind == "line":
        v = torch.randn(V, 3, generator=g)
        v[:, 1] = -0.5
        v[:, 2] = 0.125
    elif kind == "point":
        v = torch.full((V, 3), 0.375)
    elif kind == "dup":          # every vertex twice (or more), at scattered indices
        base = torch.randn((V + 1) // 2, 3, generator=g)
        v = base[torch.randint(0, base.shape[0], (V,), generator=g)]
    elif kind == "lattice":      # integer lattice (exact fp32 distances), vertex indices shuffled
        n = math.ceil(V ** (1 / 3))
        c = torch.arange(n, dtype=torch.float32)
        grid = torch.stack(torch.meshgrid(c, c, c, indexing="ij"), -1).reshape(-1, 3)
        v = grid[torch.randperm(grid.shape[0], generator=g)[:V]]
    else:
        raise ValueError(kind)
    return v.float().contiguous()


def _spread10(q):
    q = q.astype(np.uint32) & 1023
    q = (q | (q << 16)) & 0x030000FF
    q = (q | (q << 8)) & 0x0300F00F
    q = (q | (q << 4)) & 0x030C30C3
    q = (q | (q << 2)) & 0x09249249
    return q


def _morton(verts):
    """The kernel's Morton codes, restated on the host in fp32 (every operation is a single IEEE rounding)."""
    v = verts.astype(np.float32)
    lo, hi = v.min(0), v.max(0)
    ext = np.maximum(hi - lo, np.float32(1e-20)).astype(np.float32)
    with np.errstate(invalid="ignore", over="ignore"):
        q = (((v - lo).astype(np.float32) / ext).astype(np.float32) * np.float32(1023.0)).astype(np.float32)
    q = np.clip(np.trunc(q), 0, 1023).astype(np.int64)
    code = np.zeros(v.shape[0], dtype=np.int64)
    for d in range(3):
        code |= _spread10(q[:, d]).astype(np.int64) << d
    return code


def _run_knn_prep(verts):
    abi = _abi()
    B, V = verts.shape[:2]
    Vp = int(abi.lib().hg_knn_padded(V))
    sbuf, srt = _guarded((B, Vp, 4))
    bbuf, box = _guarded((B, Vp // 32, 2, 4))
    abi.call("hg_knn_prep", abi.ptr(verts), B, V, abi.ptr(srt), abi.ptr(box), abi.stream())
    return Vp, (sbuf, srt), (bbuf, box)


KNN_V = [1, 31, 32, 33, 6890, 8192]
KNN_BODIES = ["blob", "flat", "line", "point", "dup"]


@pytest.mark.parametrize("V", KNN_V)
@pytest.mark.parametrize("kind", KNN_BODIES)
def test_knn_prep(V, kind):
    """Exact: the first V entries are a permutation of the vertex indices carrying their exact coordinates, the pads
    repeat the last entry, the Morton codes are non-decreasing with equal codes in index order, and every box is the
    exact min / max of its 32 members."""
    _abi().require_device()
    g = torch.Generator().manual_seed(V + 11 * len(kind))
    B = 2
    verts = torch.stack([_body(kind, V, g) for _ in range(B)]).cuda()
    if V == 6890 and kind == "blob":
        verts = _cond(B)["vertices"].contiguous()
    Vp, (sb, srt), (bb, box) = _run_knn_prep(verts)
    _, (sb2, srt2), (bb2, box2) = _run_knn_prep(verts)
    torch.cuda.synchronize()
    _intact(sb, bb, sb2, bb2)
    _written(srt, box)
    assert _same(srt, srt2) and _same(box, box2), "not repeatable"
    s = srt.cpu().numpy()
    bx = box.cpu().numpy()
    vv = verts.cpu().numpy()
    for b in range(B):
        idx = s[b, :, 3].view(np.int32)
        assert np.array_equal(np.sort(idx[:V]), np.arange(V)), "not a permutation"
        assert np.array_equal(s[b, V:].view(np.int32), np.broadcast_to(s[b, V - 1].view(np.int32), (Vp - V, 4)))
        assert np.array_equal(s[b, :, :3], vv[b, idx]), "coordinates do not follow their index"
        code = _morton(vv[b])[idx[:V]]
        key = code * 8192 + idx[:V]
        assert (np.diff(key) > 0).all(), "Morton order (ties by index) broken"
        mem = s[b, :, :3].reshape(Vp // 32, 32, 3)
        assert np.array_equal(bx[b, :, 0, :3], mem.min(1)) and np.array_equal(bx[b, :, 1, :3], mem.max(1)), "box"
        assert (bx[b, :, :, 3] == 0).all()
    if kind == "point":
        assert (np.diff(s[0, :V, 3].view(np.int32)) > 0).all()      # every code 0: index order


# ======================================================================================================================
# hg_geo_features
# ======================================================================================================================
def _geo_call(body, *, points_in=None, rays=None, legacy=False, scaler=1.0, brute=False, outputs=("nearest", "points"),
              z_out=True):
    """One hg_geo_features launch with guarded, NaN-filled outputs.  body: dict(vertices, tpose, skel, vik) [B,...];
    rays: dict(xs, ys, zs, focals, scales, c2w, jitter).  Returns dict of views, and the list of guard buffers."""
    abi = _abi()
    verts = body["vertices"]
    B, V = verts.shape[:2]
    if points_in is not None:
        N, Rw, Rh, S = points_in.shape[1], 0, 0, 0
        r = dict(xs=None, ys=None, zs=None, focals=None, scales=None, c2w=None, jitter=None)
    else:
        r = rays
        Rw, Rh, S = r["xs"].numel(), r["ys"].numel(), r["zs"].numel()
        N = Rw * Rh * S
    bufs, out = [], {}

    def mk(name, shape, dtype=torch.float32):
        b, v = _guarded(shape, dtype)
        bufs.append(b)
        out[name] = v
        return v

    rec = mk("rec", (B, N, 36))
    zv = mk("z_vals", (B, N)) if points_in is None and z_out else None
    pts = mk("points", (B, N, 3)) if "points" in outputs else None
    near = mk("nearest", (B, N), torch.int32) if "nearest" in outputs else None
    d2 = mk("nearest_d2", (B, N)) if "nearest" in outputs else None
    ksort = kbox = None
    if not brute:
        Vp = int(abi.lib().hg_knn_padded(V))
        ksort = torch.empty(B, Vp, 4, device="cuda")
        kbox = torch.empty(B, Vp // 32, 2, 4, device="cuda")
        abi.call("hg_knn_prep", abi.ptr(verts), B, V, abi.ptr(ksort), abi.ptr(kbox), abi.stream())
    args = [r["xs"], r["ys"], r["zs"], r["focals"], r["scales"], r["c2w"], r["jitter"], points_in, body["skel"], verts,
            body["tpose"], body["vik"], ksort, kbox]
    abi.call("hg_geo_features", *[abi.ptr(t) for t in args], B, Rw, Rh, S, V, N, float(scaler), int(bool(legacy)),
             abi.ptr(rec), abi.ptr(zv), abi.ptr(pts), abi.ptr(near), abi.ptr(d2), abi.stream())
    out["sorted"], out["boxes"] = ksort, kbox
    return out, bufs


def _random_body(V, B, g, kind="blob"):
    verts = torch.stack([_body(kind, V, g) for _ in range(B)])
    return {"vertices": verts.cuda(), "tpose": torch.randn(B, V, 3, generator=g).cuda(),
            "skel": torch.randn(B, 24, 3, generator=g).cuda(),
            "vik": (torch.randn(B, V, 16, generator=g) * 0.5).cuda()}


def _synthetic_body(B, seed=5):
    c = _cond(B, seed)
    return {"vertices": c["vertices"].contiguous(), "tpose": c["tpose_vertices"].contiguous(),
            "skel": c["skeletons_xyz"].contiguous(), "vik": _abi().vertex_ik(c["fk_matrices"], c["lbs_weights"])}


def _knn_exact(points, verts):
    """port.knn1 on the device (its fp32 operations, in its order) -> (d2, idx int32)."""
    d2, idx = _port().knn1(points, verts, chunk=2048)
    return d2, idx.int()


def _check_nearest(c, pts_flat, bidx, verts, near, d2):
    """fp64: the chosen vertex is within 11 U of the true minimum distance (each fp32 d2 is within 5 U of its exact
    value), and the reported d2 within 5 U of the chosen vertex's exact distance."""
    dmin, dch = [], []
    for s in range(0, pts_flat.shape[0], 2048):
        p = pts_flat[s:s + 2048].double()
        vb = verts[bidx[s:s + 2048]].double()                              # [n,V,3]
        dd = ((p[:, None, :] - vb) ** 2).sum(-1)
        dmin.append(dd.min(1).values)
        dch.append(dd.gather(1, near[s:s + 2048].long()[:, None])[:, 0])
    dmin, dch = torch.cat(dmin), torch.cat(dch)
    c.add("nearest (fp64 distance)", dch - dmin, 11 * U * dmin + 1e-300)
    c.add("nearest_d2", (d2.double() - dch).abs(), 5 * U * dch + 1e-300)
    return dch


def _features_ref(pts, skel, tpose, vik, near, dch, legacy, scaler):
    """fp64 record of points pts [n,3] (fp32 values), with the kernel's nearest index and its vertex_ik; and its bound."""
    p = pts.double()
    ref = torch.zeros(p.shape[0], 36, dtype=torch.float64, device=p.device)
    bnd = torch.zeros_like(ref)
    sc = F32(scaler)
    ref[:, :3] = p * sc
    bnd[:, :3] = U * ref[:, :3].abs()
    e = p[:, None, :] - skel.double()                                          # [n,24,3]
    jd = e.norm(dim=-1) / F32(2.4)
    o_jd, o_ca = (3, 27) if legacy else (6, 3)
    ref[:, o_jd:o_jd + 24] = jd
    bnd[:, o_jd:o_jd + 24] = 6 * U * jd + 1e-30
    ik = vik.double().reshape(-1, 4, 4)
    hom = torch.cat([p, torch.ones_like(p[:, :1])], -1)
    terms = ik[:, :3, :] * hom[:, None, :]                                     # [n,3,4]
    cano = terms.sum(-1)
    T = terms.abs().sum(-1)
    g4 = 5 * U
    ref[:, o_ca + 0] = cano[:, 0] / 2
    bnd[:, o_ca + 0] = g4 * T[:, 0] / 2
    ref[:, o_ca + 1] = (cano[:, 1] + F32(0.2)) / 2
    bnd[:, o_ca + 1] = (g4 * (T[:, 1] + F32(0.2))) / 2
    ref[:, o_ca + 2] = cano[:, 2] / F32(1.3)
    bnd[:, o_ca + 2] = g4 * T[:, 2] / F32(1.3) + U * ref[:, o_ca + 2].abs()
    tv = tpose.double()
    ref[:, 30], ref[:, 31], ref[:, 32] = tv[:, 0], tv[:, 1], tv[:, 2] / F32(0.2)
    bnd[:, 32] = U * ref[:, 32].abs()
    ref[:, 33] = dch.sqrt() / F32(1.3)
    bnd[:, 33] = 5 * U * ref[:, 33]
    return ref, bnd + 1e-300


def _check_records(c, rec, pts, bidx, body, near, dch, legacy, scaler, tag=""):
    V = body["vertices"].shape[1]
    flat = bidx.long() * V + near.long()
    ref, bnd = _features_ref(pts, body["skel"][bidx], body["tpose"].reshape(-1, 3)[flat], body["vik"].reshape(-1, 16)[flat],
                             near, dch, legacy, scaler)
    err = (rec.double() - ref).abs()
    c.add(f"rec xyz{tag}", err[:, :3], bnd[:, :3])
    o_jd, o_ca = (3, 27) if legacy else (6, 3)
    c.add(f"rec joint distances{tag}", err[:, o_jd:o_jd + 24], bnd[:, o_jd:o_jd + 24])
    c.add(f"rec canonical point{tag}", err[:, o_ca:o_ca + 3], bnd[:, o_ca:o_ca + 3])
    c.add(f"rec T-pose vertex{tag}", err[:, 30:33], bnd[:, 30:33])
    c.add(f"rec nearest distance{tag}", err[:, 33:34], bnd[:, 33:34])
    assert bool((rec[:, 34:36] == 0).all()) and not bool(rec[:, 34:36].signbit().any()), "pad columns must be +0"


def _points_check(label, body, pts_in, *, legacy=False, scaler=2 / 2.85, outputs_off=False, brute_equal=True):
    """points_in launch: bit-exact nearest / d2 against port.knn1 (subsample) and against the kernel's brute force (every
    point), fp64 nearest and record bounds (subsample), guards, NaN prefill and a bit-identical repeat."""
    B, N = pts_in.shape[:2]
    V = body["vertices"].shape[1]
    brute_ok = V <= 8192
    a, bufs = _geo_call(body, points_in=pts_in, legacy=legacy, scaler=scaler, brute=not brute_ok)
    a2, bufs2 = _geo_call(body, points_in=pts_in, legacy=legacy, scaler=scaler, brute=not brute_ok)
    torch.cuda.synchronize()
    _intact(*bufs, *bufs2)
    _written(a["rec"], a["points"], a["nearest"], a["nearest_d2"])
    for k in ("rec", "points", "nearest", "nearest_d2"):
        assert _same(a[k], a2[k]), f"{k} not repeatable"
    del a2, bufs2
    if brute_ok and brute_equal:
        bf, bbufs = _geo_call(body, points_in=pts_in, legacy=legacy, scaler=scaler, brute=True)
        torch.cuda.synchronize()
        _intact(*bbufs)
        for k in ("nearest", "nearest_d2", "rec"):
            assert _same(a[k], bf[k]), f"pruned and brute-force {k} differ"
        del bf, bbufs
    if outputs_off:
        o, obufs = _geo_call(body, points_in=pts_in, legacy=legacy, scaler=scaler, brute=not brute_ok, outputs=())
        torch.cuda.synchronize()
        _intact(*obufs)
        assert _same(o["rec"], a["rec"]), "records depend on the optional outputs"
        del o, obufs
    assert torch.equal(a["points"], pts_in), "points output"
    sel = _sub(B * N)
    bidx = sel // N
    p = pts_in.reshape(-1, 3)[sel]
    near, d2 = a["nearest"].reshape(-1)[sel], a["nearest_d2"].reshape(-1)[sel]
    assert bool((near >= 0).all()) and bool((near < V).all())
    for b in range(B):
        m = bidx == b
        if bool(m.any()):
            rd2, ridx = _knn_exact(p[m][None], body["vertices"][b:b + 1])
            assert torch.equal(near[m], ridx[0]), "nearest index differs from port.knn1"
            assert _same(d2[m], rd2[0]), "nearest d2 differs from port.knn1"
    c = _Checks(label)
    dch = _check_nearest(c, p, bidx, body["vertices"], near, d2)
    _check_records(c, a["rec"].reshape(-1, 36)[sel], p, bidx, body, near, dch, legacy, scaler)
    c.done()
    return a


NN_V = [1, 31, 33, 6890, 8192, 8193, 12047]


@pytest.mark.parametrize("V", NN_V)
@pytest.mark.parametrize("legacy", [False, True])
def test_geo_points_bodies(V, legacy):
    """Random and on-vertex points, points on box faces and far points up to |p| ~ 1e3 on bodies of every size: the
    pruned path (V <= 8192, against the kernel's own brute force too) and the brute-force path (V > 8192)."""
    _abi().require_device()
    g = torch.Generator().manual_seed(V + legacy)
    B = 2
    body = _synthetic_body(B) if V == 6890 else _random_body(V, B, g)
    verts = body["vertices"].cpu()
    N = 3000
    pts = (torch.rand(B, N, 3, generator=g) - 0.5) * torch.tensor([2.0, 3.0, 1.5])
    k = min(V, 400)
    pts[:, :k] = verts[:, torch.randperm(V, generator=g)[:k]]                      # exactly on vertices
    face = verts[:, torch.randint(0, V, (500,), generator=g)]                      # on a vertex's coordinate plane
    pts[:, 400:900] = torch.where(torch.rand(B, 500, 3, generator=g) < 0.5, face, pts[:, 400:900])
    far = torch.randn(B, 400, 3, generator=g)
    pts[:, 900:1300] = far / far.norm(dim=-1, keepdim=True) * (10.0 ** torch.empty(B, 400, 1).uniform_(0, 3, generator=g))
    _points_check(f"geo points V={V} legacy={legacy}", body, pts.cuda().contiguous(), legacy=legacy, outputs_off=True)


def _pruned_sim(pts, srt, box, strict):
    """numpy restatement of the kernel's two-pass pruned search (fp32, one rounding per operation) for one body.
    strict=True prunes a cluster whose lower bound equals the running best."""
    p = pts.astype(np.float32)
    xyz, vid = srt[:, :3].astype(np.float32), srt[:, 3].view(np.int32)
    M = srt.shape[0] // 32

    def d2(q):
        e = (p[:, None, :] - q[None, :, :]).astype(np.float32)
        sq = (e * e).astype(np.float32)
        return ((sq[..., 0] + sq[..., 1]).astype(np.float32) + sq[..., 2]).astype(np.float32)

    best = np.full(p.shape[0], np.inf, dtype=np.float32)
    bi = np.full(p.shape[0], 0x7fffffff, dtype=np.int64)

    def take(dd, ii):
        upd = (dd < best) | ((dd == best) & (ii < bi))
        best[upd], bi[upd] = dd[upd], ii[upd]

    for m in range(M):
        take(d2(xyz[m * 32:m * 32 + 1])[:, 0], np.full(p.shape[0], vid[m * 32]))
    hit = np.zeros(p.shape[0], dtype=bool)
    for m in range(M):
        lo, hi = box[m, 0, :3].astype(np.float32), box[m, 1, :3].astype(np.float32)
        bxyz = np.maximum(np.maximum((lo - p).astype(np.float32), (p - hi).astype(np.float32)), np.float32(0))
        sq = (bxyz * bxyz).astype(np.float32)
        lb = ((sq[:, 0] + sq[:, 1]).astype(np.float32) + sq[:, 2]).astype(np.float32)
        scan = lb < best if strict else lb <= best
        hit |= (lb == best)
        dd = d2(xyz[m * 32:(m + 1) * 32])
        for i in range(32):
            di, ii = np.where(scan, dd[:, i], np.inf).astype(np.float32), np.full(p.shape[0], vid[m * 32 + i])
            upd = scan & ((di < best) | ((di == best) & (ii < bi)))
            best[upd], bi[upd] = di[upd], ii[upd]
    return bi, hit


def test_geo_cross_cluster_ties():
    """A lattice body (integer coordinates, indices shuffled) and points halfway between lattice neighbours: two vertices
    at exactly the same fp32 distance, often in different clusters, where a later cluster's box lower bound equals the
    running best.  The lowest index must win; the case asserts that pruning on `lb < best` would answer differently."""
    _abi().require_device()
    g = torch.Generator().manual_seed(77)
    B, V = 2, 6859
    body = _random_body(V, B, g, kind="lattice")
    verts = body["vertices"].cpu()
    N = 4000
    base = verts[:, torch.randint(0, V, (N,), generator=g)]
    axis = torch.randint(0, 3, (B, N), generator=g)
    step = torch.nn.functional.one_hot(axis, 3).float() * 0.5
    pts = (base + step).contiguous()
    a = _points_check("geo cross-cluster ties", body, pts.cuda(), legacy=False)
    srt, box = a["sorted"].cpu().numpy(), a["boxes"].cpu().numpy()
    differs = 0
    for b in range(B):
        loose, hit = _pruned_sim(pts[b].numpy(), srt[b], box[b], strict=False)
        strict, _ = _pruned_sim(pts[b].numpy(), srt[b], box[b], strict=True)
        assert np.array_equal(loose, a["nearest"][b].cpu().numpy().astype(np.int64)), "host restatement differs"
        differs += int((loose != strict).sum())
    print(f"cross-cluster ties: {differs} points where pruning on lb < best would return another vertex")
    assert differs > 0, "the case no longer exercises a tie across clusters"


def test_geo_lattice_points_as_surface_makes_them():
    """Chunks of 2^17 lattice points `origin + h * (i, j, k)` in fp32, as `surface.density_lattice` makes them."""
    _abi().require_device()
    surface = importlib.import_module("3dhumangan_b200.surface")
    body = _synthetic_body(1)
    origin, h, (nz, ny, nx) = surface.lattice_box(body["vertices"][0], 96, 0.1, None)
    o = torch.tensor(origin, dtype=torch.float32, device="cuda")
    i = torch.arange(0, 1 << 17, device="cuda") + 3 * (1 << 17)
    idx = torch.stack([i % nx, i // nx % ny, i // (nx * ny)], 1).float()
    pts = (o + h * idx)[None].contiguous()
    _points_check("geo lattice chunk 2^17", body, pts, legacy=False, scaler=2 / 2.85)


def test_geo_points_chunk_2_24():
    """One chunk of 2^24 points on one body (about 248 grid-stride trips per CTA): pruned equals brute force on every
    point, fp64 checks on a strided subsample."""
    _abi().require_device()
    body = _synthetic_body(1)
    g = torch.Generator(device="cuda").manual_seed(3)
    pts = ((torch.rand(1, 1 << 24, 3, device="cuda", generator=g) - 0.5) * torch.tensor([1.6, 3.0, 1.2], device="cuda"))
    _points_check("geo points 2^24", body, pts.contiguous(), legacy=True)


# ---------------------------------------------------------------------------------------------------------- ray path
def _ray_tables(Rw, Rh, S, start=0.88, end=1.12):
    f = dict(dtype=torch.float32, device="cuda")
    return torch.linspace(-Rw / Rh, Rw / Rh, Rw, **f), torch.linspace(-1, 1, Rh, **f), torch.linspace(start, end, S, **f)


def _rays_ref(r, B, Rw, Rh, S, sel):
    """fp64 restatement of port.initial_rays + jitter_and_transform at flat point indices `sel` (over B*N), from the
    same fp32 tables, and componentwise bounds of the kernel's fp32 arithmetic: (points, z, bound points, bound z)."""
    N = Rw * Rh * S
    b, p = sel // N, sel % N
    s, ray = p % S, p // S
    w, h = ray % Rw, ray // Rw
    xs, ys, zs = r["xs"].double(), r["ys"].double(), r["zs"].double()
    foc, scl = r["focals"].double()[b], r["scales"].double()[b]
    v = torch.stack([xs[w], ys[h], foc], -1)
    d = v / (v.norm(dim=-1, keepdim=True) + 1e-12)
    zc = foc / scl
    z0 = zs[s] + zc
    Z = zs[s].abs() + zc.abs()
    ez = 3 * U * Z
    if r["jitter"] is not None:
        j = r["jitter"].double().reshape(-1)[sel]
        delta = zs[1] - zs[0]
        off = (j - 0.5) * delta
        Zd = zs[0].abs() + zs[1].abs() + 2 * zc.abs()
        eoff = (j - 0.5).abs() * (2 * U * Zd + 2 * U * delta.abs()) + U * off.abs()
        z = z0 + off
        ez = ez + eoff + U * z.abs()
    else:
        off = torch.zeros_like(z0)
        z = z0
    c = d * z[:, None]
    ec = d.abs() * ez[:, None] + 8 * U * d.abs() * (z0.abs() + off.abs())[:, None]
    M = r["c2w"].double()[b]
    world = torch.einsum("nij,nj->ni", M[:, :3, :3], c) + M[:, :3, 3]
    ew = torch.einsum("nij,nj->ni", M[:, :3, :3].abs(), ec) \
        + 5 * U * (torch.einsum("nij,nj->ni", M[:, :3, :3].abs(), c.abs()) + M[:, :3, 3].abs())
    return world, z, ew + 1e-300, ez + 1e-300


# (name, B, Rw, Rh, S): the shapes the module code issues
RAY_SIZES = [("tiny", 2, 16, 16, 32), ("MAP3DBN", 32, 64, 32, 32), ("MAP3DBN512", 32, 96, 48, 32), ("C2", 8, 96, 96, 32),
             ("C5", 1, 192, 192, 128), ("B133", 133, 4, 4, 8)]
RAY_FORMS = [(True, False, ("nearest", "points")), (False, True, ())]       # (jitter, legacy, optional outputs)


@pytest.mark.parametrize("size", RAY_SIZES, ids=[s[0] for s in RAY_SIZES])
@pytest.mark.parametrize("form", RAY_FORMS, ids=["jitter-outputs", "nojitter-legacy-bare"])
def test_geo_rays(size, form):
    """Ray path at the module's sizes: points and z against fp64 (subsample), the nearest index against port.knn1 on the
    kernel's own points (subsample), pruned equal to brute force on every point, and the records against fp64."""
    abi = _abi()
    abi.require_device()
    name, B, Rw, Rh, S = size
    jit, legacy, outs = form
    N = Rw * Rh * S
    cfg = _pkg().configs.baseline_config("C2")
    xs, ys, zs = _ray_tables(Rw, Rh, S, cfg["ray_start"], cfg["ray_end"])
    cond = _cond(B, seed=9)
    body = _synthetic_body(B, seed=9)
    g = torch.Generator(device="cuda").manual_seed(B * 31 + S)
    r = dict(xs=xs, ys=ys, zs=zs, focals=cond["intrinsics"][:, 0, 0].contiguous(), scales=cond["scales"].contiguous(),
             c2w=cond["cam2world_matrices"].contiguous(),
             jitter=torch.rand(B, N, device="cuda", generator=g) if jit else None)
    grid = min((N + 511) // 512, max(1, _nsm() // B))
    trips = math.ceil(N / (grid * 512))
    print(f"{name}: B={B} N={N} CTAs per body {grid}, trips per CTA {trips}")
    a, bufs = _geo_call(body, rays=r, legacy=legacy, scaler=2 / 2.85, outputs=("nearest", "points"))
    torch.cuda.synchronize()
    _intact(*bufs)
    _written(a["rec"], a["z_vals"], a["points"], a["nearest"], a["nearest_d2"])
    a2, bufs2 = _geo_call(body, rays=r, legacy=legacy, scaler=2 / 2.85, outputs=outs)
    torch.cuda.synchronize()
    _intact(*bufs2)
    assert _same(a["rec"], a2["rec"]) and _same(a["z_vals"], a2["z_vals"]), "not repeatable / depends on optional outputs"
    del a2, bufs2
    bf, bbufs = _geo_call(body, rays=r, legacy=legacy, scaler=2 / 2.85, brute=True, outputs=("nearest",), z_out=False)
    torch.cuda.synchronize()
    _intact(*bbufs)
    assert _same(a["nearest"], bf["nearest"]) and _same(a["nearest_d2"], bf["nearest_d2"]) and _same(a["rec"], bf["rec"])
    del bf, bbufs
    sel = _sub(B * N)
    bidx = sel // N
    c = _Checks(f"geo rays {name} jitter={jit} legacy={legacy}")
    world, z, ew, ez = _rays_ref(r, B, Rw, Rh, S, sel)
    p = a["points"].reshape(-1, 3)[sel]
    c.add("points", (p.double() - world).abs(), ew)
    c.add("z_vals", (a["z_vals"].reshape(-1)[sel].double() - z).abs(), ez)
    near, d2 = a["nearest"].reshape(-1)[sel], a["nearest_d2"].reshape(-1)[sel]
    for b in range(B):
        m = bidx == b
        rd2, ridx = _knn_exact(p[m][None], body["vertices"][b:b + 1])
        assert torch.equal(near[m], ridx[0]) and _same(d2[m], rd2[0]), "nearest differs from port.knn1"
    dch = _check_nearest(c, p, bidx, body["vertices"], near, d2)
    _check_records(c, a["rec"].reshape(-1, 36)[sel], p, bidx, body, near, dch, legacy, 2 / 2.85)
    c.done()


# ======================================================================================================================
# hg_sample_fine
# ======================================================================================================================
SF_S = [3, 4, 8, 16, 32, 33, 63, 64]
SF_STRIDES = [260, 1]
SF_CLAMPS = ["relu", "softplus"]
SF_NOISE = [0.0, 0.5]


def _sf_inputs(B, Rw, Rh, S, seed):
    """Rays of four kinds, one after another: a miss (every density zero), one dominant opaque sample, a dense shell
    (transmittance 0 behind it), and pre-activations at exactly 20 and on both sides of it (softplus' threshold)."""
    g = torch.Generator().manual_seed(seed)
    R = Rw * Rh
    n = B * R
    zs = torch.linspace(0.88, 1.12, S)
    z = zs + (torch.rand(n, S, generator=g) - 0.5) * (zs[1] - zs[0]) * 0.9 + 10.0
    kind = torch.arange(n) % 4
    sig = torch.empty(n, S)
    sig[kind == 0] = -torch.rand(int((kind == 0).sum()), S, generator=g) - 1.0
    dom = torch.full((n, S), -5.0)
    hit = torch.randint(0, S, (n,), generator=g)
    dom.scatter_(1, hit[:, None], 1e4)
    sig[kind == 1] = dom[kind == 1]
    sig[kind == 2] = (torch.randn(n, S, generator=g) * 50 + 200)[kind == 2]
    edge = torch.tensor([20.0, F32(np.nextafter(np.float32(20), np.float32(30))),
                         F32(np.nextafter(np.float32(20), np.float32(0))), 19.5, 20.5, 0.0, -20.0, 5.0])
    sig[kind == 3] = edge[torch.randint(0, 8, (int((kind == 3).sum()), S), generator=g)]
    noise = torch.randn(n, S, generator=g)
    u = torch.rand(n, S, generator=g)
    c2w = torch.eye(4).repeat(B, 1, 1)
    c2w[:, :3, :3] = _rot(g, B).float()
    c2w[:, :3, 3] = torch.randn(B, 3, generator=g) * 3
    focals = 8 + torch.rand(B, generator=g) * 4
    return z, sig, noise, u, c2w, focals


def _run_sample_fine(sig, stride, z, noise, u, noise_std, clamp, xs, ys, focals, c2w, B, Rw, Rh, S):
    abi = _abi()
    n = B * Rw * Rh
    sbuf = torch.full((n * S * stride,), float("nan"), device="cuda")
    sview = sbuf[stride - 1::stride] if stride > 1 else sbuf
    sview.copy_(sig.reshape(-1))
    zb, fz = _guarded((B, Rw * Rh * S))
    pb, fp = _guarded((B, Rw * Rh * S, 3))
    abi.call("hg_sample_fine", c_void_p(sview.data_ptr()), int(stride), abi.ptr(z), abi.ptr(noise), abi.ptr(u),
             float(noise_std), int(clamp == "softplus"), abi.ptr(xs), abi.ptr(ys), abi.ptr(focals), abi.ptr(c2w), B, Rw, Rh, S,
             abi.ptr(fz), abi.ptr(fp), abi.stream())
    return (zb, fz), (pb, fp)


def _sf_ref(z, sig, noise, u, noise_std, clamp, S):
    """fp64 hierarchical_oracle.sample_pdf pipeline with componentwise bounds on the kernel's cdf knots, bins and z.
    Returns the candidates (z_ref, bound) [n,S] and their masks -- one per cdf bin u may fall in given the knots'
    bounds, and per denom branch where denom lies within its bound of 1e-5 -- and the mask of ambiguous samples."""
    zd, sg = z.double(), sig.double()
    n = zd.shape[0]
    pre = sg + noise.double() * noise_std
    epre = 2 * U * (pre.abs() + (noise.double() * noise_std).abs()) if noise_std else torch.zeros_like(pre)
    if clamp == "relu":                    # a pre-activation surely below 0 gives exactly 0: alpha 0, T unchanged
        dens, eden = pre.clamp_min(0), torch.where(pre + epre < 0, 0 * epre, epre)
    else:
        sp = torch.where(pre > 20, pre, torch.log1p(torch.exp(pre.clamp_max(20))))
        dens = sp
        eden = epre + torch.where(pre > 20, 0 * pre, 4 * U * torch.sigmoid(pre) + 2 * U * sp) + 3e-9
    delta = torch.cat([zd[:, 1:] - zd[:, :-1], torch.full((n, 1), 1e9, dtype=torch.float64, device=zd.device)], 1)
    x = delta * dens
    ex = delta * eden + 2 * U * x
    e = torch.exp(-x)
    ee = torch.where((x == 0) & (ex == 0), 0 * e, e * ex + 4 * U * e)   # expf: 2 ulp; expf(-0) = 1 exactly
    alpha = 1 - e
    ea = ee + U * alpha
    tr = (1 - alpha) + F32(1e-12)
    etr = ea + U * (1 - alpha) + U * tr + 1e-19
    T = torch.cat([torch.ones(n, 1, dtype=torch.float64, device=zd.device), torch.cumprod(tr, 1)[:, :-1]], 1)
    eT = torch.cat([torch.zeros(n, 1, dtype=torch.float64, device=zd.device), torch.cumsum(T * etr, 1)[:, :-1]], 1) \
        + (U + S * 1e-16) * T
    w = alpha * T
    ew = alpha * eT + T * ea + 2 * U * w
    wt = (w + 1e-5 + 1e-5)[:, 1:S - 1]
    ewt = (ew + U * (w + 1e-5) + U * (w + 2e-5))[:, 1:S - 1] + 2 * abs(F32(1e-5) - 1e-5)
    tot = wt.sum(1, keepdim=True)
    etot = ewt.sum(1, keepdim=True) + U * tot
    q = wt / tot
    eq = ewt / tot + wt * etot / tot ** 2 + U * q
    zero = torch.zeros(n, 1, dtype=torch.float64, device=zd.device)
    cdf = torch.cat([zero, torch.cumsum(q, 1)], 1)                                     # [n, S-1]
    ecdf = torch.cat([zero, torch.cumsum(eq, 1)], 1) + U * cdf + 1e-15
    mid = 0.5 * (zd[:, :-1] + zd[:, 1:])
    emid = U * mid.abs()
    ud = u.double()
    nk = S - 1
    lo_min = ((cdf + ecdf)[:, None, :] < ud[:, :, None]).sum(-1)                       # [n,S]
    lo_max = ((cdf - ecdf)[:, None, :] < ud[:, :, None]).sum(-1)
    thr = F32(1e-5)
    cands, oks = [], []
    for dl in range(int((lo_max - lo_min).max()) + 1):
        lo = (lo_min + dl).clamp_max(nk)
        valid = (lo_min + dl) <= lo_max
        below, above = (lo - 1).clamp_min(0), lo.clamp_max(S - 2)
        c0, c1 = cdf.gather(1, below), cdf.gather(1, above)
        e0, e1 = ecdf.gather(1, below), ecdf.gather(1, above)
        b0, b1 = mid.gather(1, below), mid.gather(1, above)
        eb0, eb1 = emid.gather(1, below), emid.gather(1, above)
        den = c1 - c0
        eden_ = e0 + e1 + U * den.abs()
        for branch in (0, 1):        # 0: den as computed, 1: den < eps -> 1
            if branch == 0:
                ok = valid & (den + eden_ >= thr) & (den > 0)
                dd, ed = den, eden_
            else:
                ok = valid & (den - eden_ < thr)
                dd, ed = torch.ones_like(den), torch.zeros_like(den)
            num = ud - c0
            enum = e0 + U * num.abs()
            t = num / dd
            et = (enum + t.abs() * ed) / dd + U * t.abs()
            dz = b1 - b0
            edz = eb0 + eb1 + U * dz.abs()
            zr = b0 + t * dz
            ez = eb0 + t.abs() * edz + dz.abs() * et + U * (t * dz).abs() + U * zr.abs()
            cands.append((zr, ez + 1e-300))
            oks.append(ok)
    amb = torch.stack(oks, -1).sum(-1) > 1
    return cands, oks, amb


def _check_sample_fine(label, z, sig, noise, u, noise_std, clamp, xs, ys, focals, c2w, B, Rw, Rh, S, fz, fp, amb_cap=0.05):
    n = B * Rw * Rh
    cands, oks, amb = _sf_ref(z, sig, noise, u, noise_std, clamp, S)
    kz = fz.reshape(n, S).double()
    ratio = torch.full_like(kz, math.inf)
    err = torch.full_like(kz, math.inf)
    for (zr, ez), ok in zip(cands, oks):            # the closest admissible candidate, relative to its own bound
        r = (kz - zr).abs() / ez
        better = ok & (r < ratio)
        ratio, err = torch.where(better, r, ratio), torch.where(better, (kz - zr).abs(), err)
    c = _Checks(label)
    worst = ratio.max().item()
    c.rows.append(("fine z", worst if not math.isnan(worst) else math.inf, err.max().item()))
    # fine points from the kernel's own z: origin + (M d) z with d = normalize(x, y, focal)
    R = Rw * Rh
    ray = torch.arange(n, device="cuda")
    b, r_ = ray // R, ray % R
    v = torch.stack([xs.double()[r_ % Rw], ys.double()[r_ // Rw], focals.double()[b]], -1)
    d = v / (v.norm(dim=-1, keepdim=True) + 1e-12)
    M = c2w.double()[b]
    wv = torch.einsum("nij,nj->ni", M[:, :3, :3], d)
    ewv = 9 * U * torch.einsum("nij,nj->ni", M[:, :3, :3].abs(), d.abs())
    want = M[:, None, :3, 3] + wv[:, None, :] * kz[..., None]
    ep = ewv[:, None, :] * kz.abs()[..., None] + U * (wv[:, None, :] * kz[..., None]).abs() + U * want.abs() + 1e-300
    c.add("fine points", (fp.reshape(n, S, 3).double() - want).abs(), ep)
    frac = amb.double().mean().item()
    print(f"{label}: ambiguous fraction {frac:.2e}")
    c.done()
    assert frac <= amb_cap, f"ambiguous fraction {frac:.3e}"


@pytest.mark.parametrize("S", SF_S)
@pytest.mark.parametrize("stride", SF_STRIDES)
@pytest.mark.parametrize("clamp", SF_CLAMPS)
@pytest.mark.parametrize("noise_std", SF_NOISE)
def test_sample_fine(S, stride, clamp, noise_std):
    """hg_sample_fine against fp64 sample_pdf on 70 rays (not a multiple of the 4-warp block) of the four kinds; the
    sigma entries sit in a NaN-filled buffer at the given element stride."""
    _abi().require_device()
    B, Rw, Rh = 2, 7, 5
    z, sig, noise, u, c2w, focals = (t.cuda().contiguous() for t in _sf_inputs(B, Rw, Rh, S, seed=S * 13 + stride))
    xs, ys, _ = _ray_tables(Rw, Rh, S)
    zf, nf, uf = z.reshape(B, -1), noise.reshape(B, -1), u
    (zb, fz), (pb, fp) = _run_sample_fine(sig, stride, zf, nf, uf, noise_std, clamp, xs, ys, focals, c2w, B, Rw, Rh, S)
    (zb2, fz2), (pb2, fp2) = _run_sample_fine(sig, stride, zf, nf, uf, noise_std, clamp, xs, ys, focals, c2w, B, Rw, Rh, S)
    torch.cuda.synchronize()
    _intact(zb, pb, zb2, pb2)
    _written(fz, fp)
    assert _same(fz, fz2) and _same(fp, fp2), "not repeatable"
    _check_sample_fine(f"sample_fine S={S} stride={stride} {clamp} noise={noise_std}", z, sig, noise, u, noise_std, clamp,
                       xs, ys, focals, c2w, B, Rw, Rh, S, fz, fp)


def test_sample_fine_c2():
    """C2 size: B = 8, 96 x 96 rays, S = 32, the fused raw output's stride."""
    _abi().require_device()
    B, Rw, Rh, S = 8, 96, 96, 32
    z, sig, noise, u, c2w, focals = (t.cuda().contiguous() for t in _sf_inputs(B, Rw, Rh, S, seed=5))
    xs, ys, _ = _ray_tables(Rw, Rh, S)
    (zb, fz), (pb, fp) = _run_sample_fine(sig, 260, z.reshape(B, -1), noise.reshape(B, -1), u, 0.5, "softplus", xs, ys,
                                          focals, c2w, B, Rw, Rh, S)
    torch.cuda.synchronize()
    _intact(zb, pb)
    _written(fz, fp)
    _check_sample_fine("sample_fine C2", z, sig, noise, u, 0.5, "softplus", xs, ys, focals, c2w, B, Rw, Rh, S, fz, fp)


# ======================================================================================================================
# hg_merge_samples
# ======================================================================================================================
MS_S = [1, 4, 8, 16, 32, 64]


def _merge_inputs(B, R, S, seed):
    """Per ray group: random depths, ties inside the fine set, fine-coarse ties, and all 2S depths equal."""
    g = torch.Generator().manual_seed(seed)
    cz = (torch.rand(B, R, S, generator=g) * 0.01 + 0.005).cumsum(-1)
    fz = torch.rand(B, R, S, generator=g) * cz[..., -1:]
    kind = torch.arange(R) % 4
    k1, k2, k3 = kind == 1, kind == 2, kind == 3
    fz[:, k1] = fz[:, k1][..., torch.randint(0, S, (S,), generator=g)]                 # ties inside the fine set
    take = torch.randint(0, S, (S,), generator=g)
    fz[:, k2] = torch.where(torch.rand(S, generator=g) < 0.5, cz[:, k2][..., take], fz[:, k2])   # fine == coarse
    fz[:, k3] = 0.25
    cz[:, k3] = 0.25
    frec, crec = torch.randn(B, R * S, 36, generator=g), torch.randn(B, R * S, 36, generator=g)
    return fz.reshape(B, R * S), cz.reshape(B, R * S), frec, crec


def _run_merge(frec, fz, crec, cz, B, R, S, perm=True):
    abi = _abi()
    rb, rec = _guarded((B, R * 2 * S, 36))
    zb, z = _guarded((B, R * 2 * S))
    pb, pm = _guarded((B, R * 2 * S), torch.int32) if perm else (None, None)
    abi.call("hg_merge_samples", abi.ptr(frec), abi.ptr(fz), abi.ptr(crec), abi.ptr(cz), B, R, S, abi.ptr(rec), abi.ptr(z),
             abi.ptr(pm), abi.stream())
    return (rb, rec), (zb, z), (pb, pm)


def _merge_ref(frec, fz, crec, cz, B, R, S):
    all_z = torch.cat([fz.reshape(B, R, S), cz.reshape(B, R, S)], -1)
    _, order = torch.sort(all_z, dim=-1, stable=True)
    all_rec = torch.cat([frec.reshape(B, R, S, 36), crec.reshape(B, R, S, 36)], 2)
    return order.int(), torch.gather(all_z, -1, order), torch.gather(all_rec, 2, order[..., None].expand(-1, -1, -1, 36))


def _check_merge(frec, fz, crec, cz, B, R, S):
    (rb, rec), (zb, z), (pb, pm) = _run_merge(frec, fz, crec, cz, B, R, S)
    (rb2, rec2), (zb2, z2), _ = _run_merge(frec, fz, crec, cz, B, R, S, perm=False)
    torch.cuda.synchronize()
    _intact(rb, zb, pb, rb2, zb2)
    _written(pm)
    order, zr, rr = _merge_ref(frec, fz, crec, cz, B, R, S)
    assert torch.equal(pm.reshape(B, R, 2 * S), order), "permutation differs from torch.sort(stable=True)"
    assert _same(z.reshape(B, R, 2 * S), zr), "merged depths"
    assert _same(rec.reshape(B, R, 2 * S, 36), rr), "merged records"
    assert _same(rec, rec2) and _same(z, z2), "not repeatable / depends on perm_out"


@pytest.mark.parametrize("S", MS_S)
def test_merge_samples(S):
    """Exact against torch.sort(stable=True) + gather on 3 x 37 rays (ragged against the 4-warp block)."""
    _abi().require_device()
    B, R = 3, 37
    fz, cz, frec, crec = (t.cuda().contiguous() for t in _merge_inputs(B, R, S, seed=S))
    _check_merge(frec, fz, crec, cz, B, R, S)


def test_merge_samples_c2():
    _abi().require_device()
    B, R, S = 8, 96 * 96, 32
    fz, cz, frec, crec = (t.cuda().contiguous() for t in _merge_inputs(B, R, S, seed=99))
    _check_merge(frec, fz, crec, cz, B, R, S)


# ======================================================================================================================
# non-finite inputs
# ======================================================================================================================
def test_geo_non_finite_points():
    """NaN, +-inf and overflowing points: nearest index and d2 equal port.knn1's (index 0 and d2 NaN for a NaN point,
    the lowest index at d2 = inf where every distance overflows), on the pruned and the brute-force path; finite points
    in the same launch are unaffected."""
    _abi().require_device()
    inf, nan = float("inf"), float("nan")
    B = 2
    for V in (6890, 8193):
        g = torch.Generator().manual_seed(V)
        body = _synthetic_body(B) if V == 6890 else _random_body(V, B, g)
        pts = (torch.rand(B, 600, 3, generator=g) - 0.5) * 2
        special = torch.tensor([[nan, 0, 0], [0, nan, 0], [nan, nan, nan], [inf, 0, 0], [-inf, 0, 0], [0, 0, inf],
                                [inf, -inf, 0], [1e20, 0, 0], [0, -3e19, 0], [1e19, 0, 0], [2e19, 2e19, 2e19],
                                [1.8e19, 0.5, 0.5], [nan, inf, 0]])
        pts[:, 100:100 + special.shape[0]] = special
        pts = pts.cuda().contiguous()
        outs = [_geo_call(body, points_in=pts, brute=brute) for brute in ((False, True) if V <= 8192 else (True,))]
        torch.cuda.synchronize()
        for o, bufs in outs:
            _intact(*bufs)
            _written(o["nearest"])
            assert _same(o["nearest"], outs[0][0]["nearest"]) and _same(o["nearest_d2"], outs[0][0]["nearest_d2"])
            for b in range(B):
                rd2, ridx = _knn_exact(pts[b:b + 1], body["vertices"][b:b + 1])
                assert torch.equal(o["nearest"][b], ridx[0]), "nearest differs from port.knn1"
                kd = o["nearest_d2"][b]
                assert bool(((kd == rd2[0]) | (kd.isnan() & rd2[0].isnan())).all()), "d2 differs from port.knn1"
            nanpt = pts[..., :].isnan().any(-1)
            assert bool((o["nearest"][nanpt] == 0).all()) and bool(o["nearest_d2"][nanpt].isnan().all())


def test_merge_samples_nan_depths():
    """NaN depths sort after every number, NaN ties by position, exactly as torch.sort(stable=True)."""
    _abi().require_device()
    for S in (4, 32, 64):
        B, R = 2, 37
        fz, cz, frec, crec = _merge_inputs(B, R, S, seed=S + 1000)
        g = torch.Generator().manual_seed(S)
        fz[torch.rand(fz.shape, generator=g) < 0.2] = float("nan")
        cz[torch.rand(cz.shape, generator=g) < 0.1] = float("nan")
        fz.reshape(B, R, S)[:, 5] = float("nan")                       # whole fine set NaN
        cz.reshape(B, R, S)[:, 6] = float("nan")
        fz.reshape(B, R, S)[:, 6] = float("nan")                       # all 2S NaN
        cz.reshape(B, R, S)[:, 7, 0] = float("inf")
        fz.reshape(B, R, S)[:, 7, -1] = -float("inf")
        _check_merge(*(t.cuda().contiguous() for t in (frec, fz, crec, cz)), B, R, S)


def test_hierarchical_forward_with_nan_code(pkg, port):
    """A NaN in one body's FiLM frequencies makes its coarse sigma NaN; under softplus (relu's fmaxf maps NaN to 0) its
    weights, cdf and fine points are NaN too.  The forward returns NaN colours and features for that body, every nearest
    index stays in [0, V), and the other body is bit-identical to a clean run."""
    from test_oracle_pin_hierarchical import hierarchical_case
    ren = importlib.import_module("3dhumangan_b200.modules.render_ops")
    hier = importlib.import_module("3dhumangan_b200.modules.hierarchical")
    cfg, params, cond, z, (u, noise), _ = hierarchical_case("softplus_n5")
    assert cfg["clamp_mode"] == "softplus"
    with torch.no_grad():
        freq, phase = port.mapping_network(params, z)
    gp = {k: v.cuda() for k, v in params.items()}
    cg = {k: v.cuda() for k, v in cond.items()}
    nd = pkg.rng.HierarchicalNoise(noise.coarse.cuda(), noise.u_pdf.cuda(), noise.final.cuda())
    fq = freq.cuda()
    bad = fq.clone()
    bad[0, 7] = float("nan")
    V = cond["vertices"].shape[1]
    h = hier.merged_records(gp, bad, phase.cuda(), cg, cfg, u.cuda(), nd, want_nearest=True, want_fine=True)
    outs = [ren.render_forward(gp, f, phase.cuda(), cg, cfg, u.cuda(), nd, want_nearest=True) for f in (fq, bad)]
    torch.cuda.synchronize()
    assert bool(h["fine_z"][0].isnan().all()), "the NaN body's fine depths must be NaN"
    assert bool(h["z_vals"][0].isnan().any()) and not bool(h["fine_z"][1].isnan().any())
    clean, o = outs
    near = o["nearest"]
    assert bool((near >= 0).all()) and bool((near < V).all())
    ro = o["ray_out"]
    assert bool(ro[0, ..., :259].isnan().all()), "the NaN body's colours and features must be NaN"
    assert _same(ro[1:], clean["ray_out"][1:]), "the other body changed"
    assert _same(near[1:], clean["nearest"][1:])


# ======================================================================================================================
# drift: every call of these kernels in the module code is a form of the matrices above
# ======================================================================================================================
GEO_FORMS = {(("rays", j, l, p, n, False)) for j in (True, False) for l in (False, True) for p in (False, True)
             for n in (False, True)} | {("points", False, l, p, n, b) for l in (False, True) for p in (False, True)
                                        for n in (False, True) for b in (False, True)}
SF_FORMS = {(st, cl, ns, s) for st in SF_STRIDES for cl in SF_CLAMPS for ns in SF_NOISE for s in SF_S}
MS_FORMS = set(MS_S)


def _forms_outside(calls):
    bad = []
    for kind, form in calls:
        if kind == "geo" and form not in GEO_FORMS:
            bad.append((kind, form))
        if kind == "sample_fine" and form not in SF_FORMS:
            bad.append((kind, form))
        if kind == "merge" and form not in MS_FORMS:
            bad.append((kind, form))
        if kind == "vertex_ik" and form > 8192:
            bad.append((kind, form))
    return bad


def test_drift_matrix_holds_every_module_call(pkg, port, monkeypatch):
    abi = _abi()
    gen = importlib.import_module("3dhumangan_b200.modules.generator")
    surface = importlib.import_module("3dhumangan_b200.surface")
    calls = []
    orig = {n: getattr(abi, n) for n in ("vertex_ik", "geo_features", "sample_fine", "merge_samples")}

    def vik(fk, lbs):
        calls.append(("vertex_ik", lbs.shape[1]))
        return orig["vertex_ik"](fk, lbs)

    def geo(*a, **k):
        calls.append(("geo", ("points" if k.get("points_in") is not None else "rays", k.get("jitter") is not None,
                              bool(k.get("legacy_mode", False)), bool(k.get("want_points", False)),
                              bool(k.get("want_nearest", False)), bool(k.get("brute_force", False)))))
        return orig["geo_features"](*a, **k)

    def sf(sigma, stride, *a, **k):
        calls.append(("sample_fine", (int(stride), k["clamp_mode"], float(k["noise_std"]), int(k["S"]))))
        return orig["sample_fine"](sigma, stride, *a, **k)

    def ms(*a, **k):
        calls.append(("merge", int(k["S"])))
        return orig["merge_samples"](*a, **k)

    for n, f in (("vertex_ik", vik), ("geo_features", geo), ("sample_fine", sf), ("merge_samples", ms)):
        monkeypatch.setattr(abi, n, f)

    def tiny(C=256, **over):
        cfg = pkg.configs.baseline_config("tiny")
        cfg.update(gen_height=64, gen_width=64, render_height=8, render_width=8, num_steps=32, nerf_noise=0.5,
                   hidden_dim=C, feature_dim=C, latent_dim=C, legacy_mode=C == 420, **over)
        G = gen.Map3DGenerator(**cfg).cuda()
        G.load_state_dict({k: v.cuda() for k, v in port.init_generator_params(cfg, seed=5, sigma_gain=200.0,
                                                                               sigma_bias=1.0).items()})
        G.set_device(torch.device("cuda:0"))
        return G, cfg

    B = 2
    cond = {k: v.cuda() for k, v in pkg.synthetic.make_conditions(B, seed=3).items()}
    runs = []
    for tag, C, hier, train in (("fused 256", 256, False, False), ("training 256", 256, False, True),
                                ("legacy 420", 420, False, False), ("hierarchical 256", 256, True, False),
                                ("hierarchical 420", 420, True, False)):
        G, cfg = tiny(C, hierarchical_sample=hier)
        G.train(train)
        zl = torch.randn(B, cfg["latent_dim"], generator=torch.Generator().manual_seed(4)).cuda()
        n0 = len(calls)
        with torch.set_grad_enabled(train):
            G(zl, cond, **cfg)
        runs.append((tag, len(calls) - n0))
    G, cfg = tiny(256)
    g = torch.Generator().manual_seed(5)
    n0 = len(calls)
    surface.density_lattice(G, cond, freq=torch.randn(1, 1024, generator=g).cuda(),
                            phase=torch.randn(1, 1024, generator=g).cuda(), resolution=14)
    runs.append(("density_lattice", len(calls) - n0))
    torch.cuda.synchronize()
    print("drift: calls per run", runs, "forms", sorted(set(calls), key=str))
    assert all(k > 0 for _, k in runs), runs
    assert not _forms_outside(calls), _forms_outside(calls)
    # the check refuses a form it has not seen
    assert _forms_outside([("sample_fine", (260, "relu", 1.0, 32)), ("merge", 128), ("geo", ("rays", True, False, False,
                                                                                              False, True))])
