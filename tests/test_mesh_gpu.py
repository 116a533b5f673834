"""Marching tetrahedra on the GPU (csrc/avc_mesh.cu through avc_march_count / avc_march_emit, and
NeuSRenderer.extract_geometry's welding) against the float64 oracle of oracle/mesh.py: per-cube counts, the edge and
point keys, vertex positions, triangles and their orientation, on non-cubic and minimal grids, thresholds off zero,
empty results, crossings exactly on grid points, the shipped small checkpoint's field, and resolution 512."""
import os
import time
import zlib
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import util_neus as U
from oracle import mesh as M
from oracle import neus

pytestmark = pytest.mark.gpu

# fp32 vertex error in index units: tt = (iso - v_in) / (v_out - v_in) carries <= 3 roundings (<= 1.5 * 2^-23 as
# tt <= 1), and adding it to the integer corner one more (2^-24 |p|)
POS_BAR = lambda p: 2.0 ** -23 * (np.abs(p) + 4.0)


def _march_gpu(u, iso):
    """avc_march_count + the exclusive scan + avc_march_emit on a float32 field -> (counts, verts [T,3,3], keys [T,3])."""
    from avatarclip_b200 import _lib
    L = _lib.lib()
    nx, ny, nz = u.shape
    ut = torch.from_numpy(np.ascontiguousarray(u, dtype=np.float32)).cuda()
    counts = torch.full(((nx - 1) * (ny - 1) * (nz - 1),), -1, dtype=torch.int32, device="cuda")
    _lib.check(L.avc_march_count(_lib.ptr(ut), nx, ny, nz, float(iso), _lib.ptr(counts), _lib.stream_ptr()), "count")
    incl = torch.cumsum(counts, 0, dtype=torch.int64)
    T = int(incl[-1])
    verts = torch.full((T * 3, 3), float("nan"), dtype=torch.float32, device="cuda")
    keys = torch.full((T * 3,), -1, dtype=torch.int64, device="cuda")
    if T:
        offsets = (incl - counts).to(torch.int32)
        _lib.check(L.avc_march_emit(_lib.ptr(ut), nx, ny, nz, float(iso), _lib.ptr(offsets), _lib.ptr(verts),
                                    _lib.ptr(keys), _lib.stream_ptr()), "emit")
    return counts.cpu().numpy(), verts.cpu().numpy().reshape(T, 3, 3), keys.cpu().numpy().reshape(T, 3)


def _same_cycle(a, b):
    """Row-wise: the triples are the same cyclic sequence."""
    return np.stack([(a == np.roll(b, s, axis=1)).all(1) for s in range(3)]).any(0)


def _check_abi(u, iso):
    """The kernel against the oracle on one field; returns what was measured."""
    u = np.ascontiguousarray(u, dtype=np.float32)
    counts, verts, keys = _march_gpu(u, iso)
    want = M.march(u, iso)
    assert np.array_equal(counts, want["counts"])
    T = keys.shape[0]
    assert T == want["key"].shape[0]
    if T == 0:
        return dict(T=0)
    # the triangles, as key triples, row for row (the emit order is fixed by the counts)
    assert np.array_equal(np.sort(keys, 1), np.sort(want["key"], 1))
    # the kernel orients exactly (integer midpoints), so only a triangle degenerate in fp64 may differ
    area = np.linalg.norm(want["normal"], axis=1) / 2
    flipped = ~_same_cycle(keys, want["key"])
    assert (area[flipped] == 0).all(), area[flipped].max()
    # every copy of a key's vertex is bitwise the same
    k, p = keys.reshape(-1), verts.reshape(-1, 3)
    order = np.argsort(k, kind="stable")
    ks, ps = k[order], p[order].view(np.uint32)
    same = ks[1:] == ks[:-1]
    assert np.array_equal(ps[1:][same], ps[:-1][same])
    # positions per key against fp64
    _, first = np.unique(k, return_index=True)
    _, wfirst = np.unique(want["key"].reshape(-1), return_index=True)
    got, ref = p[first].astype(np.float64), want["pos"].reshape(-1, 3)[wfirst]
    err = np.abs(got - ref)
    assert (err <= POS_BAR(ref)).all(), err.max()
    return dict(T=T, pos_err=float(err.max()), flipped=int(flipped.sum()), degenerate=int((area == 0).sum()))


def _smooth(shape, seed):
    """A smooth field with several closed and open sheets across the grid, off the grid points."""
    rng = np.random.default_rng(seed)
    X, Y, Z = np.meshgrid(*[np.arange(n, dtype=np.float64) for n in shape], indexing="ij")
    a = rng.uniform(0.3, 0.9, 3)
    ph = rng.uniform(0, 2 * np.pi, 3)
    return np.sin(a[0] * X + ph[0]) * np.cos(a[1] * Y + ph[1]) + 0.6 * np.sin(a[2] * Z + ph[2] + 0.2 * X)


SHAPES = [(2, 3, 70), (33, 17, 5), (70, 2, 9), (2, 2, 2), (3, 2, 2), (2, 2, 3), (41, 37, 29)]


@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("kind", ["smooth", "normal", "integers"])
@pytest.mark.parametrize("iso", [0.0, 0.37, -0.37])
def test_march_equals_oracle(shape, kind, iso):
    """Counts, keys, orientation and positions on non-cubic grids (an x/y/z mix-up changes the counts and the keys),
    the 2x2x2 minimum, thresholds off zero; 'integers' is a field of {-1, -0.37, 0, 0.37, 1}, so crossings land on
    grid points at every threshold tested."""
    rng = np.random.default_rng(zlib.crc32(repr((shape, kind, iso)).encode()))
    if kind == "smooth":
        u = _smooth(shape, 1)
    elif kind == "normal":
        u = rng.standard_normal(shape)
    else:
        u = rng.choice([-1.0, -0.37, 0.0, 0.37, 1.0], size=shape)
    rec = _check_abi(u, iso)
    U.log_parity("march_abi", dict(shape=list(shape), kind=kind, iso=iso, **rec))


def test_march_every_cube_pattern():
    """All 3^8 assignments of {below, equal to, above} the threshold to the 8 corners of a cube: pattern j is the cube
    at z = 2j of a 2 x 2 x 13122 grid (the cubes between two patterns mix their neighbours' corners)."""
    iso = 0.25
    digits = (np.arange(3 ** 8)[:, None] // 3 ** np.arange(8)[None]) % 3          # [6561, 8]
    c = np.arange(8)[None]
    vals = np.where(digits == 0, -0.5 - 0.125 * c, np.where(digits == 1, iso, 1.0 + 0.125 * c))
    u = np.empty((2, 2, 2 * 3 ** 8), np.float32)
    for k in range(8):
        u[k & 1, k >> 1 & 1, (k >> 2 & 1)::2] = vals[:, k]
    rec = _check_abi(u, iso)
    counts = M.cube_counts(u, iso).reshape(-1)[::2]
    assert set(np.unique(counts)) == set(range(0, 13, 2))          # six tetrahedra: the total is always even
    U.log_parity("march_abi_patterns", rec)


# ---------------------------------------------------------------- extract_geometry on a given field
BOX = ([-1.01, -0.7, -1.2], [1.01, 1.3, 0.9])


def _extract(u, iso=0.0, box=BOX):
    """NeuSRenderer.extract_geometry with extract_fields replaced by the given cubic field."""
    from avatarclip_b200.renderer import NeuSRenderer
    ut = torch.from_numpy(np.ascontiguousarray(u, dtype=np.float32)).cuda()
    stub = SimpleNamespace(extract_fields=lambda bmin, bmax, res: ut)
    return NeuSRenderer.extract_geometry(stub, box[0], box[1], u.shape[0], threshold=iso)


def _check_extract(u, iso=0.0, box=BOX):
    """extract_geometry against the oracle: the same vertices (in the same order, welded by key) within the fp32 bar,
    the same triangles in the same orientation."""
    v, f = _extract(u, iso, box)
    r = M.march(np.asarray(u, np.float32), iso)
    wv, wf, _ = M.weld(r["pos"], r["key"])
    assert v.shape == wv.shape and f.shape == wf.shape and v.dtype == np.float64 and f.dtype == np.int64
    scale = (np.asarray(box[1]) - np.asarray(box[0])) / (u.shape[0] - 1)
    world = M.rescale(wv, u.shape, *box)
    bar = POS_BAR(wv) * scale + 4 * 2.0 ** -24 * (np.abs(world) + np.abs(box).max())     # + the fp32 rescale
    assert (np.abs(v - world) <= bar).all()
    assert np.array_equal(np.sort(f, 1), np.sort(wf, 1))
    assert _same_cycle(f, wf).all()
    return v, f


@pytest.mark.parametrize("name", list(M.grid_point_fields()))
def test_extract_geometry_welds_crossings_on_grid_points(name):
    """The fields of oracle.mesh.grid_point_fields: one vertex per grid point the surface passes through, the collapsed
    triangles dropped, no vertex left unreferenced; the mesh is a closed, consistently wound sphere."""
    u = M.grid_point_fields()[name]
    _check_abi(u, 0.0)
    v, f = _check_extract(u)
    t = M.topology(v, f)
    assert t == dict(edges_not_two=0, directed_repeated=0, zero_area=0, coincident=0, orphans=0, euler=2), t


@pytest.mark.parametrize("n,iso", [(2, 0.0), (17, 0.37), (40, -0.37)])
def test_extract_geometry_equals_oracle(n, iso):
    _check_extract(_smooth((n, n, n), 2), iso)
    _check_extract(np.random.default_rng(n).choice([-1.0, -0.37, 0.0, 0.37, 1.0], size=(n, n, n)), iso)


@pytest.mark.parametrize("fill", [-2.0, 0.0, 3.0])
def test_empty_result(fill):
    """All outside (a value equal to the threshold is outside) or all inside: zero triangles, nothing emitted."""
    u = np.full((9, 9, 9), fill, np.float32)
    counts, verts, keys = _march_gpu(u, 0.0)
    assert (counts == 0).all() and keys.shape == (0, 3)
    v, f = _extract(u)
    assert v.shape == (0, 3) and f.shape == (0, 3) and v.dtype == np.float64 and f.dtype == np.int64


def test_extract_geometry_refuses_more_triangles_than_int32_offsets_hold():
    """A 565^3 checkerboard has 12 triangles in each of its 564^3 cubes, 2 153 046 528 > 2^31 - 1 in all: the call
    raises before anything is emitted instead of wrapping the offsets."""
    from avatarclip_b200._lib import AvcError
    n = 565
    i = torch.arange(n, device="cuda")
    u = torch.where((i[:, None, None] + i[None, :, None] + i[None, None, :]) % 2 == 1, 1.0, -1.0).float()
    assert M.cube_counts(u[:3, :3, :3].cpu().numpy(), 0.0).min() == 12
    from avatarclip_b200.renderer import NeuSRenderer
    stub = SimpleNamespace(extract_fields=lambda bmin, bmax, res: u)
    with pytest.raises(AvcError, match="int32"):
        NeuSRenderer.extract_geometry(stub, [-1.0] * 3, [1.0] * 3, n)
    del u
    torch.cuda.empty_cache()


# ---------------------------------------------------------------- the shipped small checkpoint
@pytest.fixture(scope="module")
def shipped(tmp_path_factory):
    """confs/examples_small/example.conf with the small stand-pose checkpoint; the SDF network's parameters in fp64 for
    the oracle."""
    from avatarclip_b200.runner import Runner
    tmp = tmp_path_factory.mktemp("mesh_run")
    ag = U.reference_tree(tmp / "ref")
    text = open(os.path.join(ag, "confs/examples_small/example.conf")).read()
    for old, new in (("./exp/", str(tmp / "exp") + "/"), ("./data/", ag + "/data/"),
                     ("./pretrained_models/", ag + "/pretrained_models/")):
        text = text.replace(old, new)
    (tmp / "example.conf").write_text(text.replace("        extra_color = True\n", ""))
    r = Runner(str(tmp / "example.conf"), "validate_mesh", "smpl", device="cuda")
    assert r.renderer.cfg.engine == 1
    box = tuple([float(x) for x in b] for b in (r.dataset.object_bbox_min, r.dataset.object_bbox_max))   # validate_mesh's
    c = dict(r.conf["model.sdf_network"])
    sconf = neus.SDFConf(**{k: (tuple(v) if k == "skip_in" else v) for k, v in c.items()})
    p64 = {k: v.detach().double().cpu() for k, v in r.sdf_network.state_dict().items()}
    return r, sconf, p64, box


FIELD_REL = 5e-5          # engine 1's value chain against fp64, relative to max |u| (test_neus_gpu's bar)


def _axes(box, n):
    """The grid coordinates extract_fields evaluates (float32 linspace on the device)."""
    return [torch.linspace(box[0][i], box[1][i], n, device="cuda").cpu().double() for i in range(3)]


def _u64(p64, sconf, pts):
    with torch.no_grad():
        return torch.cat([-neus.sdf_value(p64, sconf, pts[i:i + 65536]).reshape(-1)
                          for i in range(0, pts.shape[0], 65536)]).numpy()


def _check_field(u, u64, bar, iso=0.0):
    """The fp32 field within the bar of fp64, and inside / outside the same wherever fp64 is farther than the bar from
    the threshold."""
    err = np.abs(u.astype(np.float64) - u64)
    assert err.max() <= bar, (err.max(), bar)
    differ = (u > np.float32(iso)) != (u64 > iso)
    assert (np.abs(u64[differ] - iso) <= bar).all()
    return float(err.max()), int(differ.sum())


def _check_network_mesh(v, f, p64, sconf, box, n):
    t = M.topology(v, f)
    assert t["edges_not_two"] == t["directed_repeated"] == t["coincident"] == t["zero_area"] == t["orphans"] == 0, t
    with torch.no_grad():
        s = np.abs(neus.sdf_value(p64, sconf, torch.from_numpy(v)).numpy().reshape(-1))
    h = max(hi - lo for lo, hi in zip(*box)) / (n - 1)
    # linear interpolation of a network field: measured on the fp64 field at 64 / 128, max 0.76 h / 1.15 h,
    # 99th percentile 0.26 h / 0.21 h
    assert s.max() <= 2 * h and np.quantile(s, 0.99) <= 0.5 * h, (s.max() / h, np.quantile(s, 0.99) / h)
    return t, float(s.max() / h)


def test_shipped_checkpoint_whole_grid(shipped):
    """extract_fields at 64 on engine 1 against fp64 everywhere, the kernel against the oracle on that field, and the
    mesh: closed, edge-manifold, consistently wound, its vertices near the zero set."""
    r, sconf, p64, box = shipped
    n = 64
    u = r.renderer.extract_fields(*box, n).cpu().numpy()
    X = torch.stack(torch.meshgrid(*_axes(box, n), indexing="ij"), -1).reshape(-1, 3)
    u64 = _u64(p64, sconf, X).reshape(n, n, n)
    bar = FIELD_REL * np.abs(u64).max()
    field_err, differ = _check_field(u, u64, bar)
    rec = _check_abi(u, 0.0)
    v, f = r.renderer.extract_geometry(*box, n)
    wv, wf = M.extract_geometry(u, 0.0, *box)
    assert v.shape == wv.shape and np.array_equal(np.sort(f, 1), np.sort(wf, 1))
    t, smax = _check_network_mesh(v, f, p64, sconf, box, n)
    U.log_parity("march_shipped_64", dict(field_err=field_err, bar=bar, classified_differently=differ, euler=t["euler"],
                                          vertex_sdf_max_over_h=smax, **rec))


def test_shipped_checkpoint_crossing_cubes_at_128(shipped):
    """At 128 the fp64 field is evaluated on the corners of the cubes the kernel found crossing only."""
    r, sconf, p64, box = shipped
    n = 128
    u = r.renderer.extract_fields(*box, n).cpu().numpy()
    rec = _check_abi(u, 0.0)
    cube = np.flatnonzero(M.cube_counts(u, 0.0).reshape(-1))
    base = np.stack(np.unravel_index(cube, (n - 1,) * 3), 1)
    pts = np.unique((base[:, None, :] + M.CORNERS[None]).reshape(-1, 3), axis=0)
    ax = _axes(box, n)
    X = torch.stack([ax[i][torch.from_numpy(pts[:, i])] for i in range(3)], 1)
    u64 = _u64(p64, sconf, X)
    bar = FIELD_REL * float(max(np.abs(u64).max(), np.abs(u).max()))
    field_err, differ = _check_field(u[tuple(pts.T)], u64, bar)
    v, f = r.renderer.extract_geometry(*box, n)
    t, smax = _check_network_mesh(v, f, p64, sconf, box, n)
    U.log_parity("march_shipped_128", dict(corners=int(pts.shape[0]), field_err=field_err, bar=bar,
                                           classified_differently=differ, euler=t["euler"],
                                           vertex_sdf_max_over_h=smax, **rec))


def test_shipped_checkpoint_at_512(shipped):
    """--mode validate_mesh's resolution: counts against the oracle on a slab of x-planes through the body, the whole
    mesh closed and consistently wound, two calls bitwise equal.  Prints the time and the peak of torch's allocator for
    one extract_geometry call.  fp32 index coordinates are 2^-15 apart near 512, so a crossing closer than that to a
    grid point rounds onto it: a few vertices of different edges may share a position there, and their triangles have
    zero area in fp32; their count is logged and bounded."""
    from avatarclip_b200 import _lib
    r, sconf, p64, box = shipped
    n = 512
    u = r.renderer.extract_fields(*box, n)
    counts = torch.empty((n - 1) ** 3, dtype=torch.int32, device="cuda")
    _lib.check(_lib.lib().avc_march_count(_lib.ptr(u), n, n, n, 0.0, _lib.ptr(counts), _lib.stream_ptr()), "count")
    x0, x1 = 248, 264
    got = counts.reshape(n - 1, n - 1, n - 1)[x0:x1].cpu().numpy()
    want = M.cube_counts(u[x0:x1 + 1].cpu().numpy(), 0.0)
    assert np.array_equal(got, want) and want.sum() > 0
    del u, counts
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    t0 = time.perf_counter()
    v, f = r.renderer.extract_geometry(*box, n)
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    peak = torch.cuda.max_memory_allocated() - base
    v2, f2 = r.renderer.extract_geometry(*box, n)
    assert np.array_equal(v, v2) and np.array_equal(f, f2)
    t = M.topology(v, f)
    assert t["edges_not_two"] == t["directed_repeated"] == t["orphans"] == 0, t
    assert t["coincident"] + t["zero_area"] <= 1e-5 * f.shape[0], t
    name = torch.cuda.get_device_name()
    print(f"[mesh] extract_geometry at 512^3 on {name}: {dt:.2f} s, peak allocated {peak / 2 ** 30:.2f} GiB, "
          f"{v.shape[0]} vertices, {f.shape[0]} triangles, Euler characteristic {t['euler']}")
    U.log_parity("march_shipped_512", dict(device=name, seconds=dt, peak_bytes=int(peak), V=int(v.shape[0]),
                                           T=int(f.shape[0]), euler=t["euler"], coincident=t["coincident"],
                                           zero_area=t["zero_area"]))
