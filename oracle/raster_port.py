"""CPU oracle for the SMPL label-map rasteriser (SURVEY.md 8f-2): `SHHQPreprocessor._forward_rasterize`
(lib/data/preprocessor.py:138-176) with the pytorch3d 0.6.2 pieces it calls restated for exactly the settings it uses.

TEST INFRASTRUCTURE ONLY (imported by tests/ and tests/golden/make_golden_raster.py).

Restated contract of `MeshRasterizer(RasterizationSettings(image_size=(H, W), blur_radius=0.0, faces_per_pixel=1))` with
`PerspectiveCameras(focal_length=f, R, T, in_ndc=True)`; each convention is named where it is used below:
  * world -> view, row vectors: X_view = X @ R + T                                (Transform3d.rotate(R).translate(T))
  * projection: x = f X / Z, y = f Y / Z, principal point 0; the view-space Z is kept as z   (MeshRasterizer.transform)
  * pixel centres in non-square NDC: +X points left, +Y points up, the shorter side spans [-1, 1] and the longer side
    +-(long / short); pixel (yi, xi) samples (ndc(W-1-xi, W, H), ndc(H-1-yi, H, W))   (PixToNonSquareNdc)
  * a face is skipped when its largest z is < 0, when |edge(v0, v1, v2)| <= 1e-8 (zero area), or when the pixel centre lies
    outside its x/y bounding box; no back-face culling
  * barycentrics: edge functions in pytorch3d's operand order over area + 1e-8, then perspective correction
    (`perspective_correct=None` resolves to `cameras.is_perspective()` = True) with the denominator clamped at 1e-8
  * inside = all three corrected barycentrics > 0 (strict; blur_radius = 0 admits nothing outside); a pixel is skipped
    when pz = b0 z0 + b1 z1 + b2 z2 < 0
  * faces_per_pixel = 1: the smallest pz wins; on equal pz the lowest face index wins (pytorch3d's CUDA kernel leaves the
    order of equal depths to its binning -- unpinned; this is the rule the device kernel implements)
  * outputs: pix_to_face = b*F + face (packed Meshes), zbuf = pz, bary = corrected barycentrics; -1 on background
Every arithmetic step is one fp32 operation with one rounding, in the order written (pytorch3d's own build lets the compiler
contract some of them into FMAs: that last-bit difference is unpinned).  The device kernel reproduces these roundings, so it
is compared bit for bit.  Bounding boxes and faces that can have no pixel are found by exact fp32 comparisons, so looping over
the faces' boxes gives what a loop over every (face, pixel) pair gives.

PINNING: tests/golden/make_golden_raster.py runs the reference's own `forward_with_rotation` / `_forward_rasterize` with
`Meshes`, `PerspectiveCameras` and the rasteriser below injected; tests/test_oracle_pin_raster.py checks `preprocess` against
that fixture, which pins the camera construction, the `% F` of packed face ids, the barycentric argmax and the label offsets."""
import json
import math

import numpy as np
import torch

EPS = np.float32(1e-8)
F32 = np.float32


def pix_ndc(i, S1, S2):
    """PixToNonSquareNdc: centre of pixel index i along a side of S1 pixels (other side S2)."""
    rng = F32(2.0)
    if S1 > S2:
        rng = F32(S1) * rng / F32(S2)
    off = rng / F32(2.0)
    return -off + (rng * np.asarray(i, dtype=np.float32) + off) / F32(S1)


def edge(px, py, ax, ay, bx, by):
    """EdgeFunctionForward(p, a, b) = (p - a).x * (b - a).y - (p - a).y * (b - a).x."""
    return (px - ax) * (by - ay) - (py - ay) * (bx - ax)


def bary_persp(px, py, x, y, z):
    """BarycentricCoordsForward + BarycentricPerspectiveCorrectionForward -> (w0, w1, w2, pz)."""
    area = edge(x[2], y[2], x[0], y[0], x[1], y[1]) + EPS
    b0 = edge(px, py, x[1], y[1], x[2], y[2]) / area
    b1 = edge(px, py, x[2], y[2], x[0], y[0]) / area
    b2 = edge(px, py, x[0], y[0], x[1], y[1]) / area
    t0 = (b0 * z[1]) * z[2]
    t1 = (z[0] * b1) * z[2]
    t2 = (z[0] * z[1]) * b2
    denom = np.maximum((t0 + t1) + t2, EPS)
    w0, w1, w2 = t0 / denom, t1 / denom, t2 / denom
    return w0, w1, w2, (w0 * z[0] + w1 * z[1]) + w2 * z[2]


def project(verts, R, T, focal):
    """verts [B,V,3], R [B,3,3], T [B,3] -> [B,V,3] = (f X/Z, f Y/Z, Z) of X_view = X @ R + T (numpy fp32)."""
    X = np.asarray(verts, dtype=np.float32)
    R = np.asarray(R, dtype=np.float32)
    T = np.asarray(T, dtype=np.float32)
    f = F32(focal)
    xv = [((X[..., 0] * R[:, None, 0, j] + X[..., 1] * R[:, None, 1, j]) + X[..., 2] * R[:, None, 2, j]) + T[:, None, j] for j in range(3)]
    return np.stack([(f * xv[0]) / xv[2], (f * xv[1]) / xv[2], xv[2]], -1)


def rasterize(proj, faces, H, W):
    """proj [B,V,3] (NDC x, y, view z), faces [F,3] -> pix_to_face [B,H,W] int64, zbuf [B,H,W], bary [B,H,W,3]."""
    proj = np.asarray(proj, dtype=np.float32)
    faces = np.asarray(faces, dtype=np.int64)
    B, F = proj.shape[0], faces.shape[0]
    xs_asc = pix_ndc(np.arange(W), W, H)          # NDC index i; pixel column = W-1-i
    ys_asc = pix_ndc(np.arange(H), H, W)
    p2f = np.full((B, H, W), -1, dtype=np.int64)
    zbuf = np.full((B, H, W), -1, dtype=np.float32)
    bary = np.full((B, H, W, 3), -1, dtype=np.float32)
    for b in range(B):
        tri = proj[b][faces]                      # [F,3,3]
        x, y, z = tri[..., 0].T, tri[..., 1].T, tri[..., 2].T       # each [3,F]
        with np.errstate(invalid="ignore", over="ignore"):
            area = edge(x[0], y[0], x[1], y[1], x[2], y[2])
            xmin, xmax, ymin, ymax = x.min(0), x.max(0), y.min(0), y.max(0)
            ok = ~(z.max(0) < 0) & ~((area <= EPS) & (area >= -EPS))
            ok &= np.isfinite(xmin) & np.isfinite(xmax) & np.isfinite(ymin) & np.isfinite(ymax) & np.isfinite(area)
        # exact bounding-box test: NDC indices whose centre lies in [min, max]
        i0 = np.searchsorted(xs_asc, xmin, "left")
        i1 = np.searchsorted(xs_asc, xmax, "right")
        j0 = np.searchsorted(ys_asc, ymin, "left")
        j1 = np.searchsorted(ys_asc, ymax, "right")
        nx, ny = np.maximum(i1 - i0, 0), np.maximum(j1 - j0, 0)
        cnt = np.where(ok, nx * ny, 0)
        fid = np.repeat(np.arange(F), cnt)
        if fid.size == 0:
            continue
        k = np.arange(fid.size) - np.repeat(np.cumsum(cnt) - cnt, cnt)
        ii = i0[fid] + k % nx[fid]
        jj = j0[fid] + k // nx[fid]
        px, py = xs_asc[ii], ys_asc[jj]
        with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
            w0, w1, w2, pz = bary_persp(px, py, x[:, fid], y[:, fid], z[:, fid])
            keep = ~(pz < 0) & (w0 > 0) & (w1 > 0) & (w2 > 0)
        fid, ii, jj, pz, w = fid[keep], ii[keep], jj[keep], pz[keep], np.stack([w0, w1, w2], -1)[keep]
        pix = (H - 1 - jj) * W + (W - 1 - ii)
        order = np.lexsort((fid, pz, pix))          # by pixel, then depth, then face
        first = np.ones(order.size, dtype=bool)
        first[1:] = pix[order][1:] != pix[order][:-1]
        sel = order[first]
        p = pix[sel]
        p2f[b].reshape(-1)[p] = b * F + fid[sel]
        zbuf[b].reshape(-1)[p] = pz[sel] + F32(0.0)           # -0 -> +0
        bary[b].reshape(-1, 3)[p] = w[sel]
    return p2f, zbuf, bary


def resolve(p2f, bary, faces, faces_to_labels, tpose0):
    """preprocessor.py:156-174 on the rasteriser's outputs -> (segments [B,H,W] int64, semantics [B,3,H,W])."""
    p2f = torch.as_tensor(p2f)
    bary = torch.as_tensor(bary)
    faces = torch.as_tensor(faces, dtype=torch.int64)
    labels = torch.as_tensor(faces_to_labels, dtype=torch.int64)
    bg = p2f < 0
    f = p2f % faces.shape[0]
    vert = torch.gather(faces[f], -1, torch.argmax(bary, -1, keepdim=True))[..., 0]
    vert[bg] = -1
    sem = torch.as_tensor(tpose0)[vert]
    sem[bg] = 0
    seg = labels[f] + 2
    seg[bg] = 1
    return seg, sem.permute(0, 3, 1, 2).contiguous()


def camera(cond, h_rotation, v_rotation, r_rotation):
    """preprocessor.py:72-98 + :145-148 -> (R_raster [B,3,3], T_raster [B,3], focal) of the rasterising camera."""
    from oracle import smpl_port as sp
    _, R_raster = sp.cam2world_fix_body(cond["full_pose"].float(), cond["R"].float(), cond["T"].float(), h_rotation, v_rotation, r_rotation)
    focal = 1.0 / math.tan(math.pi * 1 / 180 / 2)
    T = cond["T"][:, :3, -1].clone().float()
    T[:, -1] = focal / cond["scales"].float() * 0.5
    return R_raster, T, -focal


def preprocess(cond, faces, faces_to_labels, H, W, h_rotation, v_rotation, r_rotation):
    """The whole `forward_with_rotation` raster path -> dict(proj, pix_to_face, zbuf, bary, rasterized_segments,
    rasterized_semantics)."""
    R, T, focal = camera(cond, h_rotation, v_rotation, r_rotation)
    proj = project(cond["vertices"].float().numpy(), R.numpy(), T.numpy(), focal)
    p2f, zbuf, bary = rasterize(proj, faces, H, W)
    seg, sem = resolve(p2f, bary, faces, faces_to_labels, cond["tpose_vertices"][0].float())
    return {"proj": proj, "pix_to_face": p2f, "zbuf": zbuf, "bary": bary, "rasterized_segments": seg, "rasterized_semantics": sem}


# ---- stand-ins for the pytorch3d objects `_forward_rasterize` constructs (fixture generation) ------------------------------
class Meshes:
    def __init__(self, verts, faces):
        self.verts, self.faces = verts, faces

    def to(self, device):
        return self


class PerspectiveCameras:
    def __init__(self, focal_length, R, T, in_ndc=True, device="cpu"):
        if not in_ndc:
            raise ValueError("only in_ndc=True is restated")
        self.focal, self.R, self.T = float(np.float32(focal_length)), R, T


class MeshRasterizer:
    def __init__(self, H, W):
        self.H, self.W = H, W

    def __call__(self, meshes, cameras):
        faces = meshes.faces[0].numpy()
        if any(not torch.equal(meshes.faces[0], fb) for fb in meshes.faces):
            raise ValueError("one face list for the batch is restated")
        proj = project(meshes.verts.float().numpy(), cameras.R.float().numpy(), cameras.T.float().numpy(), cameras.focal)
        p2f, zbuf, bary = rasterize(proj, faces, self.H, self.W)
        t = torch.from_numpy
        return t(p2f)[..., None], t(zbuf)[..., None], t(bary)[..., None, :], torch.full_like(t(zbuf)[..., None], -1.0)


def faces_to_labels(path, n_faces=13776):
    """lib/data/preprocessor.py:187-192."""
    d = json.load(open(path))
    idx = list(range(n_faces))
    lab = torch.tensor(d["smpl_faces_to_densepose_faces"], dtype=torch.long)[idx]
    return torch.tensor(d["densepose_faces_to_labels"], dtype=torch.long)[lab]
