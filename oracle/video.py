"""CPU oracle (test infrastructure, never on the product path): the video renderer of avc_video.cu (semantics in
include/avc_b200.h, avc_video_*) restated in fp64 with numpy: the CSR adjacency, projection, the per-frame vertex
normals, the z-buffer and the resolve.

It also flags the samples fp32 rasterisation may decide either way: a face's edge within ``EDGE_EPS_PX`` pixels of
the sample centre (the sample may fall on either side of it), or two faces, or a face and such an edge-near face,
within a relative depth of ``DEPTH_EPS``.

PARITY UNPINNED: there is no third-party renderer to pin this against (the reference renders none of its results;
AvatarAnimate's visualize.py draws through pyrender, absent here); the oracle checks the kernels against their own
stated semantics only.
"""
from __future__ import annotations

import numpy as np

NEAR = 1e-2
AMBIENT, DIFFUSE = 0.25, 0.75
GREY = 200.0
EDGE_EPS_PX = 1e-3
DEPTH_EPS = 1e-6


def adjacency(faces, V: int):
    """(offsets [V+1], vf): each vertex's faces in ascending face order; indices outside [0, V) skipped."""
    f = np.asarray(faces, dtype=np.int64).reshape(-1)
    ids = np.arange(f.size) // 3
    ok = (f >= 0) & (f < V)
    f, ids = f[ok], ids[ok]
    order = np.argsort(f, kind="stable")
    offsets = np.zeros(V + 1, dtype=np.int64)
    np.add.at(offsets, f + 1, 1)
    return np.cumsum(offsets), ids[order]


def vertex_normals(verts, faces):
    """Per vertex the sum of (v1 - v0) x (v2 - v0) over its faces, fp64."""
    v = np.asarray(verts, dtype=np.float64)
    f = np.asarray(faces, dtype=np.int64).reshape(-1, 3)
    cr = np.cross(v[f[:, 1]] - v[f[:, 0]], v[f[:, 2]] - v[f[:, 0]])
    n = np.zeros_like(v)
    for k in range(3):
        np.add.at(n, f[:, k], cr)
    return n


def project(verts, cam, image_size: int, supersample: int):
    """(u, v, z) [V,3]: supersampled pixel coordinates (pixel xi covers [xi, xi + 1)) and camera depth."""
    v = np.asarray(verts, dtype=np.float64)
    k = np.asarray(cam, dtype=np.float32).astype(np.float64)
    R, t, focal = k[:12].reshape(3, 4)[:, :3], k[:12].reshape(3, 4)[:, 3], k[12]
    p = v @ R.T + t
    fs, h = focal * supersample, 0.5 * image_size * supersample
    return np.stack([fs * p[:, 0] / p[:, 2] + h, fs * p[:, 1] / p[:, 2] + h, p[:, 2]], 1)


def raster(proj, faces, is_: int):
    """Per sample of the is x is grid: the winning face (-1: none), its depth, and the ambiguity flag."""
    f = np.asarray(faces, dtype=np.int64).reshape(-1, 3)
    best = np.full((is_, is_), np.inf)
    second = np.full((is_, is_), np.inf)
    edge_z = np.full((is_, is_), np.inf)
    face = np.full((is_, is_), -1, dtype=np.int64)
    for fi in range(f.shape[0]):
        a, b, c = proj[f[fi, 0]], proj[f[fi, 1]], proj[f[fi, 2]]
        if min(a[2], b[2], c[2]) <= NEAR:
            continue
        det = (b[1] - c[1]) * (a[0] - c[0]) + (c[0] - b[0]) * (a[1] - c[1])
        if det == 0:
            continue
        xs, ys = [a[0], b[0], c[0]], [a[1], b[1], c[1]]
        x0, x1 = max(0, int(np.ceil(min(xs) - 0.5 - EDGE_EPS_PX))), min(is_ - 1, int(np.floor(max(xs) - 0.5 + EDGE_EPS_PX)))
        y0, y1 = max(0, int(np.ceil(min(ys) - 0.5 - EDGE_EPS_PX))), min(is_ - 1, int(np.floor(max(ys) - 0.5 + EDGE_EPS_PX)))
        if x0 > x1 or y0 > y1:
            continue
        yy, xx = np.meshgrid(np.arange(y0, y1 + 1) + 0.5, np.arange(x0, x1 + 1) + 0.5, indexing="ij")
        w0 = ((b[1] - c[1]) * (xx - c[0]) + (c[0] - b[0]) * (yy - c[1])) / det
        w1 = ((c[1] - a[1]) * (xx - c[0]) + (a[0] - c[0]) * (yy - c[1])) / det
        w2 = 1 - w0 - w1
        # signed distance (pixels) of the sample to each edge: w_k |det| / |edge opposite k|
        lens = [np.hypot(b[0] - c[0], b[1] - c[1]), np.hypot(c[0] - a[0], c[1] - a[1]), np.hypot(a[0] - b[0], a[1] - b[1])]
        dist = np.minimum(np.minimum(w0 * abs(det) / lens[0], w1 * abs(det) / lens[1]), w2 * abs(det) / lens[2])
        inside = (w0 >= 0) & (w1 >= 0) & (w2 >= 0)
        near_edge = np.abs(dist) < EDGE_EPS_PX
        z = 1 / (w0 / a[2] + w1 / b[2] + w2 / c[2])
        sl = (slice(y0, y1 + 1), slice(x0, x1 + 1))
        B, S, FC, E = best[sl], second[sl], face[sl], edge_z[sl]
        nearer = inside & (z < B)
        S[nearer] = B[nearer]
        S[inside & ~nearer] = np.minimum(S[inside & ~nearer], z[inside & ~nearer])
        B[nearer], FC[nearer] = z[nearer], fi
        E[near_edge] = np.minimum(E[near_edge], z[near_edge])
    lim = best * (1 + DEPTH_EPS)
    covered = np.isfinite(best)
    ambiguous = np.where(covered, (second <= lim) | (edge_z <= lim), np.isfinite(edge_z))
    return face, best, ambiguous


def shade(proj, nrm, faces, colors, cam, face, image_size: int, supersample: int, background=(255, 255, 255)):
    """The resolve for a given winning face per sample (-1: background): the sample values [is,is,3] in fp64 and
    their supersample means [n,n,3]."""
    n, ss = image_size, supersample
    f = np.asarray(faces, dtype=np.int64).reshape(-1, 3)
    cov = face >= 0
    val = np.empty(face.shape + (3,))
    val[:] = np.asarray(background, dtype=np.float64)
    fc = face[cov]
    ys, xs = np.nonzero(cov)
    a, b, c = proj[f[fc, 0]], proj[f[fc, 1]], proj[f[fc, 2]]
    xp, yp = xs + 0.5, ys + 0.5
    det = (b[:, 1] - c[:, 1]) * (a[:, 0] - c[:, 0]) + (c[:, 0] - b[:, 0]) * (a[:, 1] - c[:, 1])
    w0 = ((b[:, 1] - c[:, 1]) * (xp - c[:, 0]) + (c[:, 0] - b[:, 0]) * (yp - c[:, 1])) / det
    w1 = ((c[:, 1] - a[:, 1]) * (xp - c[:, 0]) + (a[:, 0] - c[:, 0]) * (yp - c[:, 1])) / det
    w2 = 1 - w0 - w1
    z = 1 / (w0 / a[:, 2] + w1 / b[:, 2] + w2 / c[:, 2])
    bw = np.stack([w0 * z / a[:, 2], w1 * z / b[:, 2], w2 * z / c[:, 2]], 1)          # perspective-correct
    if colors is None:
        col = np.full((fc.size, 3), GREY)
    else:
        cv = np.asarray(colors, dtype=np.float64)
        col = sum(bw[:, k:k + 1] * cv[f[fc, k]] for k in range(3))
    nv = sum(bw[:, k:k + 1] * nrm[f[fc, k]] for k in range(3))
    zc = np.asarray(cam, dtype=np.float32).astype(np.float64)[8:11]
    ln = np.linalg.norm(nv, axis=1)
    ndotv = np.where(ln > 0, np.abs(nv @ zc) / np.where(ln > 0, ln, 1), 0.0)
    val[cov] = col * (AMBIENT + DIFFUSE * np.minimum(ndotv, 1.0))[:, None]
    return val, val.reshape(n, ss, n, ss, 3).mean((1, 3)), np.stack([w0, w1, w2], 1)


def render_frame(verts, faces, colors, cam, image_size: int, supersample: int, background=(255, 255, 255)):
    """One frame -> dict(rgb [n,n,3] uint8, value [n,n,3] fp64 before rounding, face [is,is], ambiguous [is,is],
    pixel_ambiguous [n,n])."""
    n, ss = image_size, supersample
    f = np.asarray(faces, dtype=np.int64).reshape(-1, 3)
    proj = project(verts, cam, n, ss)
    face, _, amb = raster(proj, f, n * ss)
    _, value, _ = shade(proj, vertex_normals(verts, f), f, colors, cam, face, n, ss, background)
    return dict(rgb=np.clip(np.rint(value), 0, 255).astype(np.uint8), value=value, face=face, ambiguous=amb,
                pixel_ambiguous=amb.reshape(n, ss, n, ss).any((1, 3)))


# ---------------------------------------------------------------- hand-built cases (shared by the CPU and GPU tests)
def axis_camera(focal: float) -> np.ndarray:
    """Identity rotation, camera at the origin looking along +z."""
    return np.array([1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0, focal], dtype=np.float32)


def case_quad():
    """A camera-facing quad at depth 2 spanning output pixels [10, 51) x [20, 44) of a 64 px image (focal 100): two
    triangles whose shared diagonal passes through no sample centre at supersample 1 or 2.  Returns (verts, faces,
    colors, camera, image_size, covered output pixels)."""
    u = np.array([10.0, 51.0, 51.0, 10.0])
    v = np.array([20.0, 20.0, 44.0, 44.0])
    z = 2.0
    verts = np.stack([(u - 32) / 100 * z, (v - 32) / 100 * z, np.full(4, z)], 1).astype(np.float32)
    faces = np.array([[0, 1, 2], [0, 2, 3]], dtype=np.int32)
    colors = np.full((4, 3), 90, dtype=np.uint8)
    return verts, faces, colors, axis_camera(100.0), 64, 41 * 24


def case_overlap():
    """A red triangle at depth 2 in front of a larger green one at depth 3 (listed first); the red one wins where both
    cover.  Returns (verts, faces, colors, camera, image_size, a pixel inside both)."""
    verts = np.array([[-0.3, -0.3, 2], [0.3, -0.3, 2], [0, 0.3, 2],
                      [-0.9, -0.9, 3], [0.9, -0.9, 3], [0, 0.9, 3]], dtype=np.float32)
    faces = np.array([[3, 4, 5], [0, 1, 2]], dtype=np.int32)
    colors = np.array([[255, 0, 0]] * 3 + [[0, 255, 0]] * 3, dtype=np.uint8)
    return verts, faces, colors, axis_camera(100.0), 64, (32, 32)


def case_tilted(colors: bool = True):
    """A quad whose normal is 60 degrees off the camera axis (plane z = 3 + y tan 60), constant colour (200, 120, 40)
    or the grey 200: every covered pixel is colour * (0.25 + 0.75 cos 60) = (125, 75, 25) or 125.  Returns (verts,
    faces, colors, camera, image_size, the pixel value, an interior pixel)."""
    t = np.tan(np.radians(60.0))
    xy = np.array([[-0.4, -0.2], [0.4, -0.2], [0.4, 0.2], [-0.4, 0.2]])
    verts = np.stack([xy[:, 0], xy[:, 1], 3 + xy[:, 1] * t], 1).astype(np.float32)
    faces = np.array([[0, 1, 2], [0, 2, 3]], dtype=np.int32)
    col = np.tile(np.array([[200, 120, 40]], dtype=np.uint8), (4, 1)) if colors else None
    want = (125, 75, 25) if colors else (125, 125, 125)
    return verts, faces, col, axis_camera(100.0), 64, want, (31, 32)
