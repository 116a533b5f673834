"""Marching tetrahedra of csrc/avc_mesh.cu (``k_march_tets``) and the welding of ``NeuSRenderer.extract_geometry``,
restated in float64 numpy, vectorised over cubes.

Every cube of the [nx][ny][nz] field u is cut into the six tetrahedra around its 0 -> 7 diagonal (corner c sits at
(c & 1, c >> 1 & 1, c >> 2 & 1)).  A corner is inside when u > iso, compared on the float32 values the kernel reads.  A
tetrahedron with 1 or 3 inside corners gives one triangle and one with 2 gives a quad split in two; its vertices lie on
the (inside, outside) corner pairs, linearly interpolated, and each triangle is turned so that its normal points away
from the inside corners.  Every vertex carries the key the welding merges on: the grid edge {p, q} as
(lower point's linear index) * 8 + (direction bits of q - p), or, when the outside corner's value equals iso so that
the crossing IS that grid point, the point's own linear index * 8 + 0.  Welding keeps one vertex per key, drops the
triangles that two welded corners made degenerate, removes the vertices no triangle references any more, and rescales
index coordinates to the bounding box like models/renderer.py:33-35.
"""
from __future__ import annotations

import numpy as np

TETS = np.array([[0, 1, 3, 7], [0, 1, 5, 7], [0, 2, 3, 7], [0, 2, 6, 7], [0, 4, 5, 7], [0, 4, 6, 7]])
CORNERS = np.array([[c & 1, (c >> 1) & 1, (c >> 2) & 1] for c in range(8)])


def _tables():
    """Per (tetrahedron, inside mask over its 4 corners): the triangles as [q][3][(inside corner, outside corner)] in the
    kernel's order, and the direction from the outside corners' centroid to the inside corners'."""
    tris, dirs = {}, {}
    for t in range(6):
        for m in range(1, 15):
            ins = [int(TETS[t][k]) for k in range(4) if m >> k & 1]
            outs = [int(TETS[t][k]) for k in range(4) if not m >> k & 1]
            pairs = [(a, b) for a in ins for b in outs]
            order = [(0, 1, 2)] if len(ins) != 2 else [(0, 1, 3), (0, 3, 2)]
            tris[t, m] = np.array([[pairs[i] for i in o] for o in order])
            dirs[t, m] = CORNERS[ins].mean(0) - CORNERS[outs].mean(0)
    return tris, dirs


_TRIS, _DIRS = _tables()


def _linear(p, shape):
    return (p[..., 0].astype(np.int64) * shape[1] + p[..., 1]) * shape[2] + p[..., 2]


def _corner_values(u, x0, x1):
    """[x1 - x0, ny - 1, nz - 1, 8] float32 corner values of the cubes whose x index is in [x0, x1)."""
    _, ny, nz = u.shape
    return np.stack([u[x0 + dx:x1 + dx, dy:ny - 1 + dy, dz:nz - 1 + dz] for dx, dy, dz in CORNERS], -1)


def cube_counts(u, iso, x0=0, x1=None):
    """Triangles per cube, [x1 - x0, ny - 1, nz - 1] int32, for the cubes whose x index is in [x0, x1) (avc_march_count
    writes the whole grid, x-major)."""
    u = np.asarray(u, dtype=np.float32)
    x1 = u.shape[0] - 1 if x1 is None else x1
    ins = _corner_values(u, x0, x1) > np.float32(iso)
    n = np.zeros(ins.shape[:3], dtype=np.int32)
    for t in TETS:
        ni = ins[..., t].sum(-1)
        n += np.where(ni == 2, 2, np.where((ni == 1) | (ni == 3), 1, 0)).astype(np.int32)
    return n


def march(u, iso):
    """The triangles avc_march_emit writes, in its order (cube, tetrahedron, then the two halves of a quad).
    -> dict: counts [ncubes] int32; pos [T, 3, 3] float64 index coordinates; key [T, 3] int64; normal [T, 3] float64
    (the cross product of the triangle's edges, so its norm is twice the area)."""
    u = np.ascontiguousarray(u, dtype=np.float32)
    shape = u.shape
    iso32 = np.float32(iso)
    counts = cube_counts(u, iso32).reshape(-1)
    cid = np.flatnonzero(counts)
    base = np.stack(np.unravel_index(cid, tuple(s - 1 for s in shape)), 1)             # [M, 3]
    cpos = base[:, None, :] + CORNERS[None]                                              # [M, 8, 3]
    vals = u[cpos[..., 0], cpos[..., 1], cpos[..., 2]]                                   # [M, 8] float32
    ins = vals > iso32
    order, pos, key, nrm = [], [], [], []
    for t in range(6):
        mask = (ins[:, TETS[t]] * np.array([1, 2, 4, 8])).sum(1)
        for m in range(1, 15):
            sel = np.flatnonzero(mask == m)
            if sel.size == 0:
                continue
            for q, tri in enumerate(_TRIS[t, m]):                                        # tri [3, 2] corner pairs
                ci, co = tri[:, 0], tri[:, 1]
                vi, vo = vals[sel][:, ci].astype(np.float64), vals[sel][:, co].astype(np.float64)
                tt = (np.float64(iso32) - vi) / (vo - vi)                                # [S, 3]
                p = cpos[sel][:, ci] + tt[..., None] * (CORNERS[co] - CORNERS[ci])[None]  # [S, 3, 3]
                lo, hi = np.minimum(ci, co), np.maximum(ci, co)
                k = _linear(cpos[sel][:, lo], shape) * 8 + (hi - lo)
                k = np.where(vals[sel][:, co] == iso32, _linear(cpos[sel][:, co], shape) * 8, k)
                n = np.cross(p[:, 1] - p[:, 0], p[:, 2] - p[:, 0])
                flip = n @ _DIRS[t, m] > 0                                               # normal must leave the body
                p[flip] = p[flip][:, [0, 2, 1]]
                k[flip] = k[flip][:, [0, 2, 1]]
                n[flip] = -n[flip]
                order.append(sel * 12 + t * 2 + q)
                pos.append(p)
                key.append(k)
                nrm.append(n)
    if not order:
        return dict(counts=counts, pos=np.zeros((0, 3, 3)), key=np.zeros((0, 3), np.int64), normal=np.zeros((0, 3)))
    s = np.argsort(np.concatenate(order), kind="stable")
    return dict(counts=counts, pos=np.concatenate(pos)[s], key=np.concatenate(key)[s], normal=np.concatenate(nrm)[s])


def weld(pos, key):
    """extract_geometry's welding: one vertex per key (in ascending key order), triangles with two equal corners
    dropped, unreferenced vertices removed.  -> (vertices [V, 3], triangles [T', 3] int64, keys [V])"""
    uniq, inv = np.unique(key.reshape(-1), return_inverse=True)
    verts = np.zeros((uniq.size, 3))
    verts[inv] = pos.reshape(-1, 3)
    tri = inv.reshape(-1, 3)
    tri = tri[(tri[:, 0] != tri[:, 1]) & (tri[:, 1] != tri[:, 2]) & (tri[:, 0] != tri[:, 2])]
    used = np.zeros(uniq.size, dtype=bool)
    used[tri.reshape(-1)] = True
    remap = np.cumsum(used) - 1
    return verts[used], remap[tri].astype(np.int64), uniq[used]


def rescale(verts, shape, bound_min, bound_max):
    """Index coordinates -> the bounding box (models/renderer.py:33-35)."""
    lo, hi = np.asarray(bound_min, np.float64), np.asarray(bound_max, np.float64)
    return verts / (np.asarray(shape, np.float64) - 1.0) * (hi - lo) + lo


def extract_geometry(u, iso, bound_min, bound_max):
    """NeuSRenderer.extract_geometry on a given field: (vertices [V, 3] float64 world, triangles [T, 3] int64)."""
    r = march(u, iso)
    v, f, _ = weld(r["pos"], r["key"])
    return rescale(v, np.shape(u), bound_min, bound_max), f


def grid_point_fields():
    """fp64 fields on a 9^3 grid centred at (4, 4, 4).  At threshold 0 the first, a sphere of non-integer radius^2, has
    no crossing on a grid point; the other four take integer values, and many of their crossings are grid points."""
    X, Y, Z = np.mgrid[0:9, 0:9, 0:9].astype(np.float64) - 4.0
    r2 = X * X + Y * Y + Z * Z
    return {"sphere 6.3 - r^2": 6.3 - r2, "sphere 9 - r^2": 9 - r2, "sphere 4 - r^2": 4 - r2,
            "cube 2 - max|x|": 2 - np.maximum(np.maximum(np.abs(X), np.abs(Y)), np.abs(Z)),
            "octahedron 3 - sum|x|": 3 - (np.abs(X) + np.abs(Y) + np.abs(Z))}


def topology(verts, tris):
    """Invariants of a triangle mesh: counts of undirected edges not shared by exactly two triangles, of directed
    edges used more than once (inconsistent winding), of zero-area triangles, of vertices at a position another vertex
    also has, of unreferenced vertices; and the Euler characteristic V - E + F."""
    verts, tris = np.asarray(verts), np.asarray(tris, np.int64)
    V = verts.shape[0]
    d = np.concatenate([tris[:, [0, 1]], tris[:, [1, 2]], tris[:, [2, 0]]])
    _, dcount = np.unique(d[:, 0] * V + d[:, 1], return_counts=True)
    e = np.sort(d, 1)
    _, ecount = np.unique(e[:, 0] * V + e[:, 1], return_counts=True)
    a, b, c = verts[tris[:, 0]], verts[tris[:, 1]], verts[tris[:, 2]]
    area2 = np.linalg.norm(np.cross(b - a, c - a), axis=1)
    _, pcount = np.unique(verts, axis=0, return_counts=True)
    used = np.zeros(V, dtype=bool)
    used[tris.reshape(-1)] = True
    return dict(edges_not_two=int((ecount != 2).sum()), directed_repeated=int((dcount > 1).sum()),
                zero_area=int((area2 == 0).sum()), coincident=int((pcount - 1).sum()), orphans=int((~used).sum()),
                euler=int(V - ecount.size + tris.shape[0]))
