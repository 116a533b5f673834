"""The marching-tetrahedra oracle (oracle/mesh.py) on analytic fields, without a GPU: vertices on the surface, the
topology of closed and open surfaces, outward normals, and the fields whose crossings land exactly on grid points."""
import numpy as np
import pytest

from oracle import mesh as M


def _grid(shape):
    return np.meshgrid(*[np.arange(n, dtype=np.float64) for n in shape], indexing="ij")


def _mesh(u64, iso=0.0):
    """fp32 field from an fp64 one -> (welded index-space vertices, triangles, keys, march record)."""
    r = M.march(u64.astype(np.float32), iso)
    v, f, k = M.weld(r["pos"], r["key"])
    return v, f, k, r


def _normals(v, f):
    return np.cross(v[f[:, 1]] - v[f[:, 0]], v[f[:, 2]] - v[f[:, 0]])


def _closed(v, f, euler):
    t = M.topology(v, f)
    assert t == dict(edges_not_two=0, directed_repeated=0, zero_area=0, coincident=0, orphans=0, euler=euler), t


def _sphere(shape, c, R):
    X, Y, Z = _grid(shape)
    return R - np.sqrt((X - c[0]) ** 2 + (Y - c[1]) ** 2 + (Z - c[2]) ** 2)


def _outward(v, f, grad):
    """Every triangle's normal within 90 degrees of -grad u (towards decreasing u) at its centroid."""
    n = _normals(v, f)
    g = grad(v[f].mean(1))
    assert ((n * -g).sum(1) > 0).all()


def test_oblique_plane():
    n = 12
    X, Y, Z = _grid((n, n, n))
    u = 0.3137 * X - 0.4519 * Y + 7.3311 - Z         # z = 0.31 x - 0.45 y + 7.33: inside (0, 11) over the square, no grid point on it
    v, f, _, r = _mesh(u)
    assert r["counts"].sum() == f.shape[0] > 0
    plane = 0.3137 * v[:, 0] - 0.4519 * v[:, 1] + 7.3311 - v[:, 2]
    assert np.abs(plane).max() < 1e-5                 # the field is the plane rounded to fp32
    nz = _normals(v, f)
    assert (nz[:, 2] > 0).all()                       # decreasing u is +z
    assert abs(nz[:, 2].sum() / 2 - (n - 1) ** 2) < 1e-9   # a graph over the whole x-y square
    t = M.topology(v, f)
    assert t["directed_repeated"] == t["zero_area"] == t["coincident"] == t["orphans"] == 0 and t["euler"] == 1
    d = np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]])
    e, cnt = np.unique(np.sort(d, 1), axis=0, return_counts=True)
    border = e[cnt == 1]
    assert set(np.unique(cnt)) == {1, 2} and border.shape[0] > 0
    on_side = lambda p: (np.isin(p[:, 0], [0, n - 1]) | np.isin(p[:, 1], [0, n - 1]))
    assert on_side(v[border[:, 0]]).all() and on_side(v[border[:, 1]]).all()
    _outward(v, f, lambda p: np.broadcast_to(np.array([0.3137, -0.4519, -1.0]), p.shape))


def test_sphere_on_surface_and_closed():
    c, R = np.array([15.3, 14.7, 15.1]), 11.2
    v, f, _, _ = _mesh(_sphere((32, 32, 32), c, R))
    r = np.linalg.norm(v - c, axis=1)
    # linear interpolation of R - |x| along an edge of length h <= sqrt(3) cuts inside the sphere by at most about
    # h^2 / (8 R); the fp32 rounding of the field adds ~1e-6
    err = np.abs(r - R).max()
    assert err < 3.0 / (8 * R) and (r <= R + 1e-5).all(), err
    _closed(v, f, 2)
    _outward(v, f, lambda p: -(p - c) / np.linalg.norm(p - c, axis=1, keepdims=True))


def test_torus_has_euler_characteristic_zero():
    c, Rt, rt = np.array([16.2, 15.7, 9.9]), 9.0, 3.5
    X, Y, Z = _grid((34, 33, 20))
    q = np.sqrt((X - c[0]) ** 2 + (Y - c[1]) ** 2) - Rt
    v, f, _, _ = _mesh(rt - np.sqrt(q ** 2 + (Z - c[2]) ** 2))
    _closed(v, f, 0)

    def grad(p):
        d = p - c
        s = np.sqrt(d[:, 0] ** 2 + d[:, 1] ** 2)
        w = np.stack([d[:, 0] / s * (s - Rt), d[:, 1] / s * (s - Rt), d[:, 2]], 1)
        return -w / np.linalg.norm(w, axis=1, keepdims=True)
    _outward(v, f, grad)


def test_two_disjoint_balls():
    c1, c2 = np.array([7.2, 8.1, 8.4]), np.array([19.7, 8.6, 7.9])
    shape = (28, 17, 17)
    u = np.maximum(_sphere(shape, c1, 5.3), _sphere(shape, c2, 4.6))
    v, f, _, _ = _mesh(u)
    _closed(v, f, 4)

    def grad(p):
        d1, d2 = p - c1, p - c2
        n1, n2 = np.linalg.norm(d1, axis=1, keepdims=True), np.linalg.norm(d2, axis=1, keepdims=True)
        return np.where(5.3 - n1 > 4.6 - n2, -d1 / n1, -d2 / n2)
    _outward(v, f, grad)


GRID_POINT_FIELDS = M.grid_point_fields()


def _cube_grad(p):
    x = p - 4.0
    a = np.abs(x)
    return -np.sign(x) * (a == a.max(1, keepdims=True))


GRID_POINT_GRADS = {"sphere": lambda p: -2 * (p - 4.0), "cube": _cube_grad, "octahedron": lambda p: -np.sign(p - 4.0)}


@pytest.mark.parametrize("name", list(GRID_POINT_FIELDS))
def test_crossings_on_grid_points_are_welded(name):
    """Integer fields at threshold 0: crossings land exactly on grid points (except on the generic sphere).  Each such
    point is one vertex, the triangles it collapses are dropped, and what remains is a closed, consistently wound
    sphere without zero-area triangles or coincident vertices."""
    u = GRID_POINT_FIELDS[name]
    v, f, k, r = _mesh(u)
    _closed(v, f, 2)
    on_point = (k % 8) == 0
    assert on_point.any() == (name != "sphere 6.3 - r^2")
    assert np.array_equal(v[on_point], np.round(v[on_point])) and np.all(u[tuple(v[on_point].astype(int).T)] == 0)
    _outward(v, f, GRID_POINT_GRADS[name.split()[0]])


def test_keys_name_the_edge_or_point_each_vertex_lies_on():
    rng = np.random.default_rng(3)
    shape = (7, 5, 9)
    u = rng.integers(-2, 3, size=shape).astype(np.float32) + rng.choice([0.0, 0.5], size=shape).astype(np.float32)
    r = M.march(u, 0.0)
    k, p = r["key"].reshape(-1), r["pos"].reshape(-1, 3)
    code, lin = k % 8, k // 8
    lo = np.stack(np.unravel_index(lin, shape), 1)
    step = np.stack([code & 1, code >> 1 & 1, code >> 2 & 1], 1)
    assert set(np.unique(code)) <= {0, 1, 2, 3, 4, 5, 6, 7} and (code == 0).any() and (code == 7).any()
    off = p - lo                                                   # on the segment lo -> lo + step
    assert (off[step == 0] == 0).all()
    s = np.where(step.sum(1) > 0, off.sum(1) / np.maximum(step.sum(1), 1), 0)
    assert np.allclose(off, s[:, None] * step, atol=1e-12) and (s >= 0).all() and (s <= 1).all()
    assert (s[code == 0] == 0).all() and (s[code != 0] < 1).all()  # a crossing that IS a grid point carries its key
    # one position per key: the welding loses nothing
    order = np.argsort(k, kind="stable")
    ks, ps = k[order], p[order]
    same = ks[1:] == ks[:-1]
    assert np.array_equal(ps[1:][same], ps[:-1][same])


def test_counts_per_cube_and_per_slab():
    rng = np.random.default_rng(5)
    u = rng.standard_normal((6, 11, 8)).astype(np.float32)
    r = M.march(u, 0.37)
    assert r["counts"].sum() == r["key"].shape[0] and r["counts"].max() <= 12
    full = M.cube_counts(u, 0.37)
    assert np.array_equal(full.reshape(-1), r["counts"])
    assert np.array_equal(M.cube_counts(u, 0.37, 2, 4), full[2:4])


def test_inside_is_strictly_above_the_fp32_threshold():
    """The field is compared with the threshold as fp32, and a value equal to it is outside: a field of 0.1f at
    threshold 0.1 is empty, although 0.1f > 0.1 in fp64."""
    u = np.full((3, 4, 5), 0.1, dtype=np.float32)
    assert M.march(u, 0.1)["key"].shape == (0, 3)
    u[1, 2, 2] = np.nextafter(np.float32(0.1), np.float32(1))
    r = M.march(u, 0.1)
    assert r["counts"].sum() > 0
    v, f, k = M.weld(r["pos"], r["key"])
    assert (k % 8 == 0).all()                         # every crossing is one of the neighbours, which equal the threshold
    assert np.array_equal(v, np.round(v)) and np.abs(v - [1, 2, 2]).max() == 1
    _closed(v, f, 2)                                  # the closed surface of the one inside point's neighbourhood


@pytest.mark.parametrize("fill", [-1.0, 1.0])
def test_uniform_fields_have_no_surface(fill):
    u = np.full((4, 3, 5), fill, dtype=np.float32)
    v, f = M.extract_geometry(u, 0.0, [-1, -1, -1], [1, 1, 1])
    assert v.shape == (0, 3) and f.shape == (0, 3)


def test_rescale_to_the_bounding_box():
    v = np.array([[0.0, 0.0, 0.0], [6.0, 4.0, 2.0], [3.0, 1.0, 0.5]])
    w = M.rescale(v, (7, 5, 3), [-1.0, 0.0, 2.0], [1.0, 2.0, 3.0])
    assert np.allclose(w, [[-1.0, 0.0, 2.0], [1.0, 2.0, 3.0], [0.0, 0.5, 2.25]], atol=0, rtol=0)
