"""avc_mesh_decimate (quadric-error edge collapse, include/avc_b200.h) restated in float64 numpy, round by round:
quadrics, flags, candidates, keys, selection, cap and collapse.  Every array operation is elementwise and in the order
the header states (no np.linalg, no pairwise sums), so the result equals the kernel's bit for bit.  Plus metrics for
judging a simplified mesh: a topology summary and a two-sided surface distance."""
from __future__ import annotations

import numpy as np
from scipy.spatial import cKDTree

MAX_DEG = 32
BOUNDARY_WEIGHT = 10.0
DET_EPS = 1e-9
FLIP_COS = 0.25
NO_KEY = np.uint64(0xFFFFFFFFFFFFFFFF)
_PAIRS = [(i, j) for i in range(4) for j in range(i, 4)]      # the ten quadric entries 00 01 02 03 11 12 13 22 23 33


def _cross(e, f):
    return np.stack([e[:, 1] * f[:, 2] - e[:, 2] * f[:, 1], e[:, 2] * f[:, 0] - e[:, 0] * f[:, 2],
                     e[:, 0] * f[:, 1] - e[:, 1] * f[:, 0]], 1)


def _dot(e, f):
    return (e[:, 0] * f[:, 0] + e[:, 1] * f[:, 1]) + e[:, 2] * f[:, 2]


def _plane(n, o, w):
    """[N,10] plane quadrics of normal n through o; w None: 0.5 |n| (the face area)."""
    ln = np.sqrt(_dot(n, n))
    nz = ln != 0
    with np.errstate(invalid="ignore", divide="ignore"):
        u = n / ln[:, None]
        p = np.concatenate([u, -_dot(u, o)[:, None]], 1)
    p = np.where(nz[:, None], p, 0.0)
    w = np.where(nz, 0.5 * ln if w is None else w, 0.0)
    return np.stack([w * (p[:, i] * p[:, j]) for i, j in _PAIRS], 1)


def _cost(q, v):
    x, y, z = v[:, 0], v[:, 1], v[:, 2]
    s0 = ((q[:, 0] * x + q[:, 1] * y) + q[:, 2] * z) + q[:, 3]
    s1 = ((q[:, 1] * x + q[:, 4] * y) + q[:, 5] * z) + q[:, 6]
    s2 = ((q[:, 2] * x + q[:, 5] * y) + q[:, 7] * z) + q[:, 8]
    s3 = ((q[:, 3] * x + q[:, 6] * y) + q[:, 8] * z) + q[:, 9]
    return ((x * s0 + y * s1) + z * s2) + s3


def optimal_point(q, pa, pb):
    """(v [N,3] float64, cost [N] clamped at 0) of edges with summed quadrics q [N,10] and ends pa, pb."""
    c00 = q[:, 4] * q[:, 7] - q[:, 5] * q[:, 5]
    c01 = q[:, 5] * q[:, 2] - q[:, 1] * q[:, 7]
    c02 = q[:, 1] * q[:, 5] - q[:, 4] * q[:, 2]
    c11 = q[:, 0] * q[:, 7] - q[:, 2] * q[:, 2]
    c12 = q[:, 1] * q[:, 2] - q[:, 0] * q[:, 5]
    c22 = q[:, 0] * q[:, 4] - q[:, 1] * q[:, 1]
    det = (q[:, 0] * c00 + q[:, 1] * c01) + q[:, 2] * c02
    tr = (q[:, 0] + q[:, 4]) + q[:, 7]
    m = (pa + pb) * 0.5
    e = pb - pa
    r0, r1, r2 = -q[:, 3], -q[:, 6], -q[:, 8]
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        vs = np.stack([((r0 * c00 + r1 * c01) + r2 * c02) / det, ((r0 * c01 + r1 * c11) + r2 * c12) / det,
                       ((r0 * c02 + r1 * c12) + r2 * c22) / det], 1)
        dv = vs - m
        use = (det > DET_EPS * ((tr * tr) * tr)) & (_dot(dv, dv) <= _dot(e, e))
        cs = _cost(q, vs)
    ca, cb, cm = _cost(q, pa), _cost(q, pb), _cost(q, m)
    pick_a = (ca <= cb) & (ca <= cm)
    pick_b = ~pick_a & (cb <= cm)
    v = np.where(pick_a[:, None], pa, np.where(pick_b[:, None], pb, m))
    c = np.where(pick_a, ca, np.where(pick_b, cb, cm))
    v = np.where(use[:, None], vs, v)
    c = np.where(use, cs, c)
    return v, np.fmax(c, 0.0)                    # fmax as the kernel's: a NaN cost (non-finite input) becomes 0


def _edges(T, ids):
    """Half-edges of faces T [n,3] with face ids ``ids``: (lo, hi, edge id 3 f + k, opposite vertex) per h = 3 i + k."""
    ha, hb, hc = T.reshape(-1), T[:, [1, 2, 0]].reshape(-1), T[:, [2, 0, 1]].reshape(-1)
    hid = (3 * ids[:, None] + np.arange(3)).reshape(-1)
    return np.minimum(ha, hb), np.maximum(ha, hb), hid, hc


def quadrics(pos, tri, valid):
    """[V,10] initial vertex quadrics: per vertex, in ascending face order, the face quadric then its boundary edges'."""
    V = pos.shape[0]
    ids = np.flatnonzero(valid)
    T = tri[ids]
    p = pos.astype(np.float64)
    p0, p1, p2 = p[T[:, 0]], p[T[:, 1]], p[T[:, 2]]
    n = _cross(p1 - p0, p2 - p0)
    Kf = _plane(n, p0, None)
    lo, hi, _, _ = _edges(T, ids)
    _, inv, cnt = np.unique(lo * V + hi, return_inverse=True, return_counts=True)
    bnd = (cnt[inv.reshape(-1)] == 1).reshape(-1, 3)
    items_v, items_f, items_s, terms = [], [], [], []
    for j in range(3):
        items_v.append(T[:, j]); items_f.append(ids); items_s.append(np.zeros_like(ids)); terms.append(Kf)
    for k in range(3):
        sel = np.flatnonzero(bnd[:, k])
        a, b = T[sel, k], T[sel, (k + 1) % 3]
        e = p[b] - p[a]
        Ke = _plane(_cross(e, n[sel]), p[a], BOUNDARY_WEIGHT * _dot(e, e))
        for end in (a, b):
            items_v.append(end); items_f.append(ids[sel]); items_s.append(np.full(sel.size, 1 + k)); terms.append(Ke)
    iv, jf, ks = np.concatenate(items_v), np.concatenate(items_f), np.concatenate(items_s)
    K = np.concatenate(terms)
    order = np.lexsort((ks, jf, iv))
    iv, K = iv[order], K[order]
    first = np.searchsorted(iv, iv)
    rank = np.arange(iv.size) - first
    Q = np.zeros((V, 10))
    for r in range(int(rank.max(initial=-1)) + 1):
        s = rank == r
        Q[iv[s]] = Q[iv[s]] + K[s]
    return Q


def _rows(t):
    """[n,3] int64 rows as one structured value each, so that rows compare whole (no packed key to overflow)."""
    return np.ascontiguousarray(t, np.int64).view([("a", np.int64), ("b", np.int64), ("c", np.int64)]).reshape(-1)


def _expand(off, verts):
    """For each entry of ``verts``: (entry index, position in the CSR) over its range off[v]:off[v+1]."""
    start, n = off[verts], off[verts + 1] - off[verts]
    owner = np.repeat(np.arange(verts.size), n)
    pos = np.arange(owner.size) - np.repeat(np.cumsum(n) - n, n) + np.repeat(start, n)
    return owner, pos


def _flip_ok(p, T, vf, off, mover, other, vr, m):
    owner, j = _expand(off, mover)
    face = T[vf[j]]
    keep = ~(face == other[owner, None]).any(1)
    owner, face = owner[keep], face[keep]
    old = p[face]                                                  # [k,3,3]
    new = np.where((face == mover[owner, None])[:, :, None], vr[owner][:, None, :], old)
    n = _cross(old[:, 1] - old[:, 0], old[:, 2] - old[:, 0])
    mm = _cross(new[:, 1] - new[:, 0], new[:, 2] - new[:, 0])
    good = _dot(n, mm) > FLIP_COS * (np.sqrt(_dot(n, n)) * np.sqrt(_dot(mm, mm)))
    return np.bincount(owner[~good], minlength=m) == 0


def decimate(verts, faces, target: int, colors=None) -> dict:
    """avc_mesh_decimate: {vertices [K,3] float32, faces [T,3] int64, colors [K,3] float32 or None, rounds}."""
    pos = np.array(verts, dtype=np.float32).reshape(-1, 3)
    tri = np.array(faces, dtype=np.int64).reshape(-1, 3)
    col = None if colors is None else np.array(colors, dtype=np.float32).reshape(-1, 3)
    V, F = pos.shape[0], tri.shape[0]
    if F <= target:
        return dict(vertices=pos, faces=tri, colors=col, rounds=0)
    alive = ((tri >= 0) & (tri < V)).all(1) & (tri[:, 0] != tri[:, 1]) & (tri[:, 1] != tri[:, 2]) & \
        (tri[:, 0] != tri[:, 2])
    Q = quadrics(pos, tri, alive)
    lock = np.zeros(V, bool)
    remap = np.arange(V)
    rounds = 0
    while True:
        ids = np.flatnonzero(alive)
        if ids.size <= target:
            break
        T = tri[ids]
        lo, hi, hid, opp = _edges(T, ids)
        _, inv, cnt = np.unique(lo * V + hi, return_inverse=True, return_counts=True)
        inv = inv.reshape(-1)
        nf = cnt[inv]
        minid = np.full(cnt.size, np.iinfo(np.int64).max)
        np.minimum.at(minid, inv, hid)
        omin = np.full(cnt.size, np.iinfo(np.int64).max)
        omax = np.full(cnt.size, -1)
        np.minimum.at(omin, inv, opp)
        np.maximum.at(omax, inv, opp)
        canon = hid == minid[inv]
        lock[lo[canon & (nf > 2)]] = True
        lock[hi[canon & (nf > 2)]] = True
        bnd = np.zeros(V, bool)
        bnd[lo[nf == 1]] = True
        bnd[hi[nf == 1]] = True
        deg = np.bincount(T.reshape(-1), minlength=V)
        E = np.flatnonzero(canon & (nf <= 2))
        a, b, nfe, eid = lo[E], hi[E], nf[E], hid[E]
        c, d = omin[inv[E]], omax[inv[E]]
        ok = ~lock[a] & ~lock[b] & (deg[a] <= MAX_DEG) & (deg[b] <= MAX_DEG) & ~((nfe == 2) & bnd[a] & bnd[b])
        # link condition over the neighbour lists of the live edges
        ulo, uhi = lo[canon], hi[canon]
        src, dst = np.concatenate([ulo, uhi]), np.concatenate([uhi, ulo])
        o = np.argsort(src, kind="stable")
        nbr, noff = dst[o], np.concatenate([[0], np.cumsum(np.bincount(src, minlength=V))])
        ekeys = np.sort(ulo * V + uhi)
        owner, j = _expand(noff, a)
        w, bb = nbr[j], b[owner]
        k = np.minimum(w, bb) * V + np.maximum(w, bb)
        hit = (w != bb) & (ekeys[np.minimum(np.searchsorted(ekeys, k), ekeys.size - 1)] == k)
        common = np.bincount(owner[hit], minlength=E.size)
        ok &= common == nfe
        fkeys = _rows(np.sort(T, 1))

        def has_face(x):
            return np.isin(_rows(np.sort(np.stack([x, c, d], 1), 1)), fkeys)
        ok &= ~((nfe == 2) & ((c == d) | (has_face(a) & has_face(b))))
        E, a, b, nfe, eid = E[ok], a[ok], b[ok], nfe[ok], eid[ok]
        p = pos.astype(np.float64)
        q = Q[a] + Q[b]
        v, cost = optimal_point(q, p[a], p[b])
        vr = v.astype(np.float32).astype(np.float64)
        fo = np.argsort(T.reshape(-1), kind="stable")
        vf = fo // 3
        foff = np.concatenate([[0], np.cumsum(deg)])
        ok = _flip_ok(p, T, vf, foff, a, b, vr, a.size) & _flip_ok(p, T, vf, foff, b, a, vr, a.size)
        a, b, nfe, eid, q, v, cost = a[ok], b[ok], nfe[ok], eid[ok], q[ok], v[ok], cost[ok]
        key = (cost.astype(np.float32).view(np.uint32).astype(np.uint64) << np.uint64(32)) | eid.astype(np.uint64)
        vmin = np.full(V, NO_KEY, dtype=np.uint64)
        np.minimum.at(vmin, a, key)
        np.minimum.at(vmin, b, key)
        ring = np.full(a.size, NO_KEY, dtype=np.uint64)
        for x in (a, b):
            owner, j = _expand(foff, x)
            vm = vmin[T[vf[j]]].min(1)
            np.minimum.at(ring, owner, vm)
        s = np.flatnonzero(ring >= key)
        if s.size == 0:
            break
        s = s[np.argsort(key[s])]
        keep = np.cumsum(nfe[s]) <= ids.size - target
        keep[0] = True
        s = s[keep]
        rounds += 1
        a, b = a[s], b[s]
        if col is not None:
            pa, pb = p[a], p[b]
            e = pb - pa
            ee = _dot(e, e)
            with np.errstate(invalid="ignore", divide="ignore"):
                t = np.where(ee > 0, _dot(v[s] - pa, e) / ee, 0.0)
            t = np.minimum(np.maximum(t, 0.0), 1.0)
            ca, cb = col[a].astype(np.float64), col[b].astype(np.float64)
            col[a] = (ca + t[:, None] * (cb - ca)).astype(np.float32)
        pos[a] = v[s].astype(np.float32)
        Q[a] = q[s]
        remap[b] = a
        t2 = remap[tri[ids]]
        tri[ids] = t2
        alive[ids] = (t2[:, 0] != t2[:, 1]) & (t2[:, 1] != t2[:, 2]) & (t2[:, 0] != t2[:, 2])
    keep_v = remap == np.arange(V)
    new = np.cumsum(keep_v) - 1
    return dict(vertices=pos[keep_v], faces=new[tri[alive]], colors=None if col is None else col[keep_v],
                rounds=rounds)


# ---------------------------------------------------------------- metrics
def topology(verts, faces) -> dict:
    """Undirected edges on one face (boundary) and on more than two (non-manifold), directed edges used twice or more
    (inconsistent orientation), and the Euler characteristic V - E + F over the referenced vertices."""
    f = np.asarray(faces, np.int64).reshape(-1, 3)
    d = np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]])
    n = int(max(np.asarray(verts).shape[0], 1))
    _, dcount = np.unique(d[:, 0] * n + d[:, 1], return_counts=True)
    e = np.sort(d, 1)
    _, ecount = np.unique(e[:, 0] * n + e[:, 1], return_counts=True)
    used = np.unique(f)
    return dict(boundary_edges=int((ecount == 1).sum()), nonmanifold_edges=int((ecount > 2).sum()),
                misoriented_edges=int((dcount > 1).sum()), euler=int(used.size - ecount.size + f.shape[0]))


def area(verts, faces) -> float:
    v = np.asarray(verts, np.float64)
    f = np.asarray(faces, np.int64).reshape(-1, 3)
    return float(0.5 * np.linalg.norm(np.cross(v[f[:, 1]] - v[f[:, 0]], v[f[:, 2]] - v[f[:, 0]]), axis=1).sum())


def spacing_for(verts, faces, samples: int = 2_000_000) -> float:
    """The sample spacing that puts ``samples`` points on the mesh."""
    return (area(verts, faces) / samples) ** 0.5


def sample_surface(verts, faces, spacing: float, seed: int = 0) -> np.ndarray:
    """Points uniform by area on the mesh, one per spacing^2 of area (at least one per mesh): [N,3] float64."""
    v = np.asarray(verts, np.float64)
    f = np.asarray(faces, np.int64).reshape(-1, 3)
    p0, p1, p2 = v[f[:, 0]], v[f[:, 1]], v[f[:, 2]]
    area = 0.5 * np.linalg.norm(np.cross(p1 - p0, p2 - p0), axis=1)
    n = max(1, int(np.ceil(area.sum() / spacing ** 2)))
    rng = np.random.default_rng(seed)
    fi = rng.choice(f.shape[0], n, p=area / area.sum())
    r1, r2 = rng.random(n), rng.random(n)
    s = np.sqrt(r1)
    return (1 - s)[:, None] * p0[fi] + (s * (1 - r2))[:, None] * p1[fi] + (s * r2)[:, None] * p2[fi]


def surface_distance(va, fa, vb, fb, spacing: float) -> dict:
    """Two-sided distance between meshes A and B: each one's area-uniform samples (``spacing`` apart on average) to the
    nearest sample of the other, both directions pooled.  The samples resolve distances down to about spacing / 2."""
    sa, sb = sample_surface(va, fa, spacing, 1), sample_surface(vb, fb, spacing, 2)
    d = np.concatenate([cKDTree(sb).query(sa)[0], cKDTree(sa).query(sb)[0]])
    return dict(mean=float(d.mean()), p99=float(np.percentile(d, 99)), max=float(d.max()), samples=int(d.size))


# ---------------------------------------------------------------- small test meshes
def grid(n: int):
    """A flat n x n grid of squares over [0, 1]^2 at z = 0, two triangles each, counter-clockwise seen from +z."""
    x = np.linspace(0.0, 1.0, n + 1, dtype=np.float32)
    X, Y = np.meshgrid(x, x, indexing="ij")
    v = np.stack([X.reshape(-1), Y.reshape(-1), np.zeros(X.size, np.float32)], 1)
    i, j = np.mgrid[0:n, 0:n]
    p = (i * (n + 1) + j).reshape(-1)
    f = np.concatenate([np.stack([p, p + n + 1, p + n + 2], 1), np.stack([p, p + n + 2, p + 1], 1)])
    return v, f.astype(np.int64)


def sphere(res: int = 24, radius: float = 0.8):
    """A closed sphere from oracle/mesh.py's marching tetrahedra on the analytic field radius^2 - |x|^2 over [-1, 1]^3."""
    from . import mesh
    g = np.linspace(-1.0, 1.0, res)
    X, Y, Z = np.meshgrid(g, g, g, indexing="ij")
    v, f = mesh.extract_geometry(radius * radius - (X * X + Y * Y + Z * Z), 0.0, [-1, -1, -1], [1, 1, 1])
    return v.astype(np.float32), f


def tetrahedron():
    v = np.array([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 1]], np.float32)
    return v, np.array([[0, 2, 1], [0, 1, 3], [0, 3, 2], [1, 2, 3]], np.int64)


def fan(n: int = 8):
    """``grid(n)`` with two extra triangles on its boundary edge (0, 1): that edge has three faces (a non-manifold fan).
    Returns (vertices, faces, the fan's vertices)."""
    v, f = grid(n)
    V = v.shape[0]
    pages = np.array([[0.0, 0.5 / n, 0.3], [0.0, 0.5 / n, -0.3]], np.float32)
    f = np.concatenate([f, [[0, 1, V], [1, 0, V + 1]]])
    return np.concatenate([v, pages]), f, np.array([0, 1, V, V + 1])
