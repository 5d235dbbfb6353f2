"""numpy restatement of the iso-surface rule of `hg_iso_count` / `hg_iso_emit` (include/hg3d.h, csrc/surface.cu).

Written from the rule, not from the kernel: the winding of every (tet, inside-code) case is fixed here by a geometric test
on the edge midpoints (the triangle's normal must point from the tet's inside corners to its outside ones), where the
kernel derives it from permutation parities.  Vertex positions and normals follow the rule's fp32 arithmetic one rounded
operation at a time, so they agree with the kernel to the last bits; faces must agree exactly.
"""
from __future__ import annotations

import numpy as np

SLOTS = ((1, 0, 0), (0, 1, 0), (0, 0, 1), (1, 1, 0), (1, 0, 1), (0, 1, 1), (1, 1, 1))     # (dx, dy, dz) per edge slot
PERMS = ((0, 1, 2), (0, 2, 1), (1, 0, 2), (1, 2, 0), (2, 0, 1), (2, 1, 0))                 # Kuhn tets, in face order
f32 = np.float32


def tet_corners(t):
    """The 4 corners (dx, dy, dz) of tet t: c, c+e_a, c+e_a+e_b, c+(1,1,1)."""
    a, b, _ = PERMS[t]
    u1 = [0, 0, 0]
    u1[a] = 1
    u2 = list(u1)
    u2[b] = 1
    return [(0, 0, 0), tuple(u1), tuple(u2), (1, 1, 1)]


def _edge(t, i, j):
    """Tet edge (i, j) -> (owner corner (dx,dy,dz), slot)."""
    c = tet_corners(t)
    i, j = min(i, j), max(i, j)
    d = tuple(c[j][k] - c[i][k] for k in range(3))
    return c[i], SLOTS.index(d)


def _tables():
    """TAB[t, code] -> up to 2 triangles of 3 (owner dx, dy, dz, slot); NTRI[t, code]."""
    tab = np.zeros((6, 16, 2, 3, 4), dtype=np.int64)
    ntri = np.zeros((6, 16), dtype=np.int64)
    for t in range(6):
        pos = np.array(tet_corners(t), dtype=np.float64)
        for code in range(16):
            ins = [v for v in range(4) if code >> v & 1]
            out = [v for v in range(4) if not code >> v & 1]
            if len(ins) in (0, 4):
                continue
            if len(ins) == 2:
                a, b = ins
                c, d = out
                q = [(a, c), (a, d), (b, d), (b, c)]
                tris = [(q[0], q[1], q[2]), (q[0], q[2], q[3])]
            else:
                lone = ins[0] if len(ins) == 1 else out[0]
                rest = [v for v in range(4) if v != lone]
                tris = [tuple((lone, r) for r in rest)]
            toward = pos[out].mean(0) - pos[ins].mean(0)
            for k, tri in enumerate(tris):
                m = [0.5 * (pos[i] + pos[j]) for i, j in tri]
                if np.dot(np.cross(m[1] - m[0], m[2] - m[0]), toward) < 0:
                    tri = (tri[0], tri[2], tri[1])
                for v, (i, j) in enumerate(tri):
                    owner, slot = _edge(t, i, j)
                    tab[t, code, k, v] = (*owner, slot)
            ntri[t, code] = len(tris)
    return tab, ntri


TAB, NTRI = _tables()


def _popcount(x):
    x = x.astype(np.int64)
    return sum((x >> s) & 1 for s in range(7))


def _gradient(v):
    """Central differences in index units, one-sided at the border, per axis (z, y, x) in fp32."""
    out = []
    for ax in range(3):
        g = np.empty_like(v)
        n = v.shape[ax]
        sl = lambda a, b: tuple(slice(a, b) if k == ax else slice(None) for k in range(3))
        g[sl(1, n - 1)] = (v[sl(2, n)] - v[sl(0, n - 2)]) * f32(0.5)
        g[sl(0, 1)] = v[sl(1, 2)] - v[sl(0, 1)]
        g[sl(n - 1, n)] = v[sl(n - 1, n)] - v[sl(n - 2, n - 1)]
        out.append(g)
    return out[2], out[1], out[0]          # gx, gy, gz


def iso_surface(lattice, level, origin=(0.0, 0.0, 0.0), spacing=1.0, cell_chunk=1 << 21):
    """lattice [Nz,Ny,Nx] -> (vertices [V,3] fp32, normals [V,3] fp32, faces [F,3] int64) by the rule of include/hg3d.h."""
    v = np.ascontiguousarray(lattice, dtype=f32)
    nz, ny, nx = v.shape
    assert min(v.shape) >= 2
    level = f32(level)
    inside = v > level
    flat_in = inside.reshape(-1)
    n = v.size
    zz, yy, xx = np.meshgrid(np.arange(nz), np.arange(ny), np.arange(nx), indexing="ij")
    xx, yy, zz = xx.reshape(-1), yy.reshape(-1), zz.reshape(-1)
    mask = np.zeros(n, dtype=np.int64)
    for s, (dx, dy, dz) in enumerate(SLOTS):
        ok = (xx + dx < nx) & (yy + dy < ny) & (zz + dz < nz)
        p = np.nonzero(ok)[0]
        q = p + dx + dy * nx + dz * nx * ny
        mask[p] |= (flat_in[p] != flat_in[q]).astype(np.int64) << s
    cnt = _popcount(mask)
    voff = np.concatenate([[0], np.cumsum(cnt)[:-1]]).astype(np.int64)

    # ---- vertices in (point, slot) order
    gx, gy, gz = (g.reshape(-1) for g in _gradient(v))
    vf = v.reshape(-1)
    pts, slots = [], []
    for s in range(7):
        p = np.nonzero(mask >> s & 1)[0]
        pts.append(p)
        slots.append(np.full(p.shape, s))
    p = np.concatenate(pts)
    s = np.concatenate(slots)
    order = np.lexsort((s, p))
    p, s = p[order], s[order]
    d = np.array(SLOTS, dtype=np.int64)[s]
    q = p + d[:, 0] + d[:, 1] * nx + d[:, 2] * nx * ny
    va, vb = vf[p], vf[q]
    t = (level - va) / (vb - va)
    o = [f32(c) for c in origin]
    h = f32(spacing)
    pos = []
    for k, coord in enumerate((xx, yy, zz)):
        c = coord[p].astype(f32)
        c = np.where(d[:, k] == 1, c + t, c)
        pos.append(o[k] + h * c)
    verts = np.stack(pos, 1).astype(f32)
    nrm = [g[p] + t * (g[q] - g[p]) for g in (gx, gy, gz)]
    ln = np.sqrt((nrm[0] * nrm[0] + nrm[1] * nrm[1]) + nrm[2] * nrm[2])
    safe = np.where(ln > 0, ln, f32(1))
    normals = np.stack([np.where(ln > 0, -(c / safe), f32(0)) for c in nrm], 1).astype(f32)

    # ---- faces in (cell, tet, triangle) order
    cz, cy, cx = np.meshgrid(np.arange(nz - 1), np.arange(ny - 1), np.arange(nx - 1), indexing="ij")
    cells = (cx + cy * nx + cz * nx * ny).reshape(-1)
    faces = []
    for c0 in range(0, cells.size, cell_chunk):
        c = cells[c0:c0 + cell_chunk]
        codes = np.zeros((c.size, 6), dtype=np.int64)
        for ti in range(6):
            for vi, (dx, dy, dz) in enumerate(tet_corners(ti)):
                codes[:, ti] |= flat_in[c + dx + dy * nx + dz * nx * ny].astype(np.int64) << vi
        e = TAB[np.arange(6)[None, :], codes]                        # [c, 6, 2, 3, 4]
        owner = c[:, None, None, None] + e[..., 0] + e[..., 1] * nx + e[..., 2] * nx * ny
        idx = voff[owner] + _popcount(mask[owner] & ((1 << e[..., 3]) - 1))
        valid = np.arange(2)[None, None, :] < NTRI[np.arange(6)[None, :], codes][..., None]
        faces.append(idx[valid])
    faces = np.concatenate(faces) if faces else np.zeros((0, 3), dtype=np.int64)
    return verts, normals, faces.reshape(-1, 3)


# ---------------------------------------------------------------------------------------------------------------- mesh facts
def directed_edges(faces):
    f = np.asarray(faces, dtype=np.int64)
    return np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]])


def closed_and_oriented(faces):
    """Every undirected edge lies in exactly 2 faces and is used once in each direction."""
    e = directed_edges(faces)
    key = e[:, 0] * (1 << 32) + e[:, 1]
    rev = e[:, 1] * (1 << 32) + e[:, 0]
    uniq, counts = np.unique(key, return_counts=True)
    if (counts != 1).any():
        return False
    return bool(np.isin(rev, uniq).all())


def euler_characteristic(faces):
    f = np.asarray(faces, dtype=np.int64)
    V = np.unique(f).size
    e = np.sort(directed_edges(f), 1)
    E = np.unique(e[:, 0] * (1 << 32) + e[:, 1]).size
    return V - E + f.shape[0]


def components(faces):
    """Number of edge-connected face components (union-find over the vertex ids)."""
    f = np.asarray(faces, dtype=np.int64)
    ids = np.unique(f)
    parent = {int(i): int(i) for i in ids}

    def find(a):
        while parent[a] != a:
            parent[a] = parent[parent[a]]
            a = parent[a]
        return a

    for a, b, c in f:
        ra = find(int(a))
        for o in (int(b), int(c)):
            ro = find(o)
            if ro != ra:
                parent[ro] = ra
    return len({find(int(i)) for i in ids})


def signed_volume(verts, faces):
    v = np.asarray(verts, dtype=np.float64)[np.asarray(faces, dtype=np.int64)]
    return float(np.einsum("ij,ij->i", v[:, 0], np.cross(v[:, 1], v[:, 2])).sum() / 6.0)


def face_normals(verts, faces):
    v = np.asarray(verts, dtype=np.float64)[np.asarray(faces, dtype=np.int64)]
    return np.cross(v[:, 1] - v[:, 0], v[:, 2] - v[:, 0])


def area(verts, faces):
    return float(np.linalg.norm(face_normals(verts, faces), axis=1).sum() / 2.0)
