"""The texture atlas of avatarclip_b200.bake in float64 numpy: the cell grid, each texel's owning face and surface point,
the corner UVs, and smooth vertex normals.  Layout as avc_bake_texel_points in include/avc_b200.h."""
from __future__ import annotations

import math

import numpy as np

MIN_CELL = 8


def grid(F: int, T: int):
    """(m, c): the m x m grid of cells c texels wide; c < MIN_CELL means the atlas does not fit."""
    m = math.isqrt((F + 1) // 2 - 1) + 1
    return m, T // m


def corners(c: int, side: int) -> np.ndarray:
    """[3, 2] cell-local (x, y) of the UV corners of face 2k + side."""
    p = np.array([[3.0, 1.0], [c - 1.0, 1.0], [c - 1.0, c - 3.0]])
    return p[:, ::-1].copy() if side else p


def texel_owner(F: int, T: int) -> np.ndarray:
    """[T, T] int64 owning face of every texel (row y, column x), -1 where unused."""
    m, c = grid(F, T)
    y, x = np.mgrid[0:T, 0:T]
    q, r = x // c, y // c
    i, j = x - q * c, y - r * c
    f = 2 * (r * m + q) + (i < j)
    return np.where((q < m) & (r < m) & (f < F), f, -1)


def uv(F: int, T: int) -> np.ndarray:
    """[F, 3, 2] corner UVs, v = 0 at the top row."""
    m, c = grid(F, T)
    f = np.arange(F)
    k = f // 2
    org = np.stack([k % m, k // m], 1).astype(np.float64) * c
    loc = np.where((f % 2 == 1)[:, None, None], corners(c, 1)[None], corners(c, 0)[None])
    return (org[:, None, :] + loc) / T


def barycentric(px, py, c: int, side):
    """Clamped barycentrics of cell-local points in the UV triangle of their face (side 0: face 2k, 1: face 2k + 1)."""
    px, py = np.where(side, py, px), np.where(side, px, py)
    L = c - 4.0
    be = (py - 1.0) / L
    al = (px - py - 2.0) / L
    b = np.maximum(np.stack([1.0 - al - be, al, be], -1), 0.0)
    return b / b.sum(-1, keepdims=True)


def texel_points(verts, faces, T: int):
    """(owner [T*T] int64, points [T*T, 3] float64): what avc_bake_texel_points writes."""
    verts = np.asarray(verts, np.float64)
    faces = np.asarray(faces, np.int64)
    F = faces.shape[0]
    m, c = grid(F, T)
    own = texel_owner(F, T).reshape(-1)
    y, x = np.divmod(np.arange(T * T), T)
    i, j = x % c, y % c
    b = barycentric(i + 0.5, j + 0.5, c, i < j)
    used = own >= 0
    pts = np.zeros((T * T, 3))
    tri = verts[faces[own[used]]]                                       # [n, 3 corners, 3]
    pts[used] = (b[used][:, :, None] * tri).sum(1)
    return own, pts


def footprint_owners(F: int, T: int, p) -> np.ndarray:
    """[..., 4] owners of the 2 x 2 texel centres a bilinear sample at texel-space points p [..., 2] reads (-2 for a
    texel outside the texture)."""
    own = texel_owner(F, T)
    p = np.asarray(p, np.float64)
    x0 = np.floor(p[..., 0] - 0.5).astype(np.int64)
    y0 = np.floor(p[..., 1] - 0.5).astype(np.int64)
    out = []
    for dy in (0, 1):
        for dx in (0, 1):
            x, y = x0 + dx, y0 + dy
            ok = (x >= 0) & (x < T) & (y >= 0) & (y < T)
            out.append(np.where(ok, own[np.clip(y, 0, T - 1), np.clip(x, 0, T - 1)], -2))
    return np.stack(out, -1)


def vertex_normals(verts, faces) -> np.ndarray:
    """[V, 3] per vertex the normalised sum of its faces' (v1 - v0) x (v2 - v0); (0, 1, 0) where the sum is zero."""
    verts = np.asarray(verts, np.float64)
    faces = np.asarray(faces, np.int64)
    n = np.cross(verts[faces[:, 1]] - verts[faces[:, 0]], verts[faces[:, 2]] - verts[faces[:, 0]])
    acc = np.zeros_like(verts)
    for k in range(3):
        np.add.at(acc, faces[:, k], n)
    length = np.linalg.norm(acc, axis=1, keepdims=True)
    return np.where(length > 0, acc / np.where(length > 0, length, 1.0), np.array([0.0, 1.0, 0.0]))
