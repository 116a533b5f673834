"""The tangent-space normal map of avatarclip_b200.bake in float64 (oracle/normal_map.py): corner tangents and their
handedness on the atlas, texel frames and glTF's decode, the 8-bit encode, the search's bracket rule, the .glb layout
that export.write_glb writes with a normal map, and the export CLI's --normal_map flag."""
import numpy as np
import pytest

from oracle import bake as B
from oracle import drive as D
from oracle import export as E
from oracle import normal_map as NM


def _deg(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    c = (a * b).sum(-1) / (np.linalg.norm(a, axis=-1) * np.linalg.norm(b, axis=-1))
    return np.degrees(np.arccos(np.clip(c, -1, 1)))


def _flat_faces(rng, F):
    """F separate planar triangles in random orientations, each with its own three vertices and the face normal on
    them (counter-clockwise seen from the normal)."""
    v = rng.normal(0, 1, (F, 3, 3))
    n = np.cross(v[:, 1] - v[:, 0], v[:, 2] - v[:, 0])
    n /= np.linalg.norm(n, axis=1, keepdims=True)
    return v.reshape(-1, 3), np.arange(3 * F).reshape(F, 3), np.repeat(n, 3, 0)


def _uv_jacobian(verts, faces, uv):
    """[F, 3] dP/du and dP/dv of the affine map from each face's UV triangle to its positions."""
    p = np.asarray(verts)[faces]
    e = np.stack([p[:, 1] - p[:, 0], p[:, 2] - p[:, 0]], 2)                  # [F, 3, 2]
    d = np.stack([uv[:, 1] - uv[:, 0], uv[:, 2] - uv[:, 0]], 2)              # [F, 2, 2]: columns (du, dv)
    J = e @ np.linalg.inv(d)                                                 # [F, 3, 2]
    return J[..., 0], J[..., 1]


@pytest.mark.parametrize("F,T", [(2, 16), (9, 48), (40, 256)])
def test_tangents_flip_on_mirrored_faces_and_bitangent_points_up(F, T):
    rng = np.random.default_rng(F)
    v, f, n = _flat_faces(rng, F)
    uv = B.uv(F, T)
    tg = NM.corner_tangents(v, f, n, uv)
    assert np.allclose(np.linalg.norm(tg[..., :3], axis=-1), 1) and np.abs((tg[..., :3] * n[f]).sum(-1)).max() < 1e-12
    w = tg[..., 3]
    assert (w[0::2] == -1).all() and (w[1::2] == 1).all()                    # the atlas mirrors faces 2k + 1
    dpdu, dpdv = _uv_jacobian(v, f, uv)
    Bt = w[..., None] * np.cross(n[f], tg[..., :3])
    assert (np.einsum("fkd,fd->fk", tg[..., :3], dpdu) > 0).all()            # T along increasing u
    assert (np.einsum("fkd,fd->fk", Bt, dpdv) < 0).all()                     # B along decreasing v: the image's top
    # on a flat face T, B are the unit dP/du, -dP/dv when those are orthogonal; always in the face's plane
    assert np.abs(np.einsum("fkd,fd->fk", Bt, np.cross(dpdu, dpdv))).max() < 1e-9


def test_degenerate_faces_take_the_pinned_fallback():
    v = np.array([[0, 0, 0], [1, 0, 0], [2, 0, 0], [0, 0, 0], [0, 0, 0], [0, 0, 0]], np.float64)
    f = np.array([[0, 1, 2], [3, 4, 5]])                                     # collinear; a point
    n = np.tile([0.0, 0.6, 0.8], (6, 1))
    tg = NM.corner_tangents(v, f, n, B.uv(2, 16))
    assert np.allclose(tg[0, :, :3], [1, 0, 0])                              # collinear along x: still a tangent
    e = np.array([1.0, 0, 0])                                                # the axis of n's smallest |component|
    assert np.allclose(tg[1, :, :3], e) and (tg[1, :, 3] == 1).all()


def _quad_frames(T=32):
    """A unit quad in the z = 0 plane (normals +z) on a T x T atlas: (verts, faces, normals, texels, frames)."""
    v = np.array([[0, 0, 0], [1, 0, 0], [1, 1, 0], [0, 1, 0]], np.float64)
    f = np.array([[0, 1, 2], [0, 2, 3]])
    n = np.tile([0.0, 0.0, 1.0], (4, 1))
    tg = NM.corner_tangents(v, f, n, B.uv(2, T))
    texels = np.flatnonzero(B.texel_owner(2, T).reshape(-1) >= 0)
    return v, f, n, texels, NM.texel_frames(f, n, tg, T, texels)


def test_flat_map_decodes_to_the_interpolated_normal():
    _, _, n, texels, fr = _quad_frames()
    dec = NM.decode(np.tile([128, 128, 255], (texels.size, 1)), fr[:, 0], fr[:, 1], fr[:, 2])
    assert _deg(dec, fr[:, 2]).max() < 0.5 and np.allclose(fr[:, 2], [0, 0, 1])
    # frames are orthonormal and right- or left-handed by w
    G = np.einsum("nij,nkj->nik", fr, fr)
    assert np.abs(G - np.eye(3)).max() < 1e-12


def test_map_tilted_towards_green_tilts_towards_decreasing_v():
    T = 32
    v, f, n, texels, fr = _quad_frames(T)
    own, _ = NM.texel_bary(texels, 2, T)
    dpdu, dpdv = _uv_jacobian(v, f, B.uv(2, T))
    dec = NM.decode(np.tile([128, 230, 200], (texels.size, 1)), fr[:, 0], fr[:, 1], fr[:, 2])
    up = -dpdv[own] / np.linalg.norm(dpdv[own], axis=1, keepdims=True)       # decreasing v, in the surface
    right = dpdu[own] / np.linalg.norm(dpdu[own], axis=1, keepdims=True)
    assert ((dec * up).sum(1) > 0.5).all() and (np.abs((dec * right).sum(1)) < 0.05).all()
    dec = NM.decode(np.tile([230, 128, 200], (texels.size, 1)), fr[:, 0], fr[:, 1], fr[:, 2])
    assert ((dec * right).sum(1) > 0.5).all()


def test_encode_decode_round_trip_within_quantisation():
    rng = np.random.default_rng(3)
    m = 20000
    q, _ = np.linalg.qr(rng.normal(size=(m, 3, 3)))
    fr = np.transpose(q, (0, 2, 1)).copy()                                   # rows orthonormal, either handedness
    g = rng.normal(size=(m, 3)) * rng.uniform(0.01, 100, (m, 1))
    rgb, flat, back = NM.encode(fr, g, np.ones(m, np.int32))
    assert not flat.any()
    n = g / np.linalg.norm(g, axis=1, keepdims=True)
    assert np.array_equal(back, (fr[:, 2] * n).sum(1) <= 0)
    err = _deg(NM.decode(rgb, fr[:, 0], fr[:, 1], fr[:, 2]), n)
    assert err.max() < 0.4, err.max()
    # flat texels: no bracket, or a vanishing gradient
    rgb, flat, back = NM.encode(fr[:3], np.array([[0, 0, 1.0], [1e-7, 0, 0], [0, 1, 0]]), np.array([0, 1, 1]))
    assert flat.tolist() == [True, True, False] and (rgb[:2] == [128, 128, 255]).all() and not back[:2].any()


def test_bracket_picks_the_sign_change_nearest_zero_outside_on_a_tie():
    D = 1.5
    t = NM.offsets(D)
    assert np.isclose(t[0], -D) and np.isclose(t[-1], D) and np.allclose(np.diff(t), 2 * D / 15)
    s = np.ones((5, NM.K))
    s[0, :3] = -1                                 # one crossing at [t2, t3]
    s[1, :5] = -1; s[1, 11:] = -1                 # [t4, t5] and [t10, t11]: equidistant, the outside wins
    s[2, 6] = 0.0                                 # an exact zero is the root; no interval on either side
    s[3] = -s[3]                                  # no crossing
    s[4, :7] = -1; s[4, 9:] = -1                  # [t6, t7] (distance 1.5 steps) and [t8, t9] (1.5): outside
    lo, hi, st = NM.bracket(s, D)
    assert (lo[0], hi[0], st[0]) == (t[2], t[3], 1)
    assert (lo[1], hi[1], st[1]) == (t[10], t[11], 2)
    assert (lo[2], hi[2], st[2]) == (t[6], t[6], 1)
    assert (lo[3], hi[3], st[3]) == (0.0, 0.0, 0)
    assert (lo[4], hi[4], st[4]) == (t[8], t[9], 2)
    assert NM.ties(s, 1e-3).tolist() == [False, True, True, False, True]


def test_snap_finds_a_plane_within_the_bisection_bound():
    rng = np.random.default_rng(4)
    p = rng.normal(size=(500, 3))
    N = rng.normal(size=(500, 3))
    N /= np.linalg.norm(N, axis=1, keepdims=True)
    nrm = np.array([0.3, -0.5, 0.8]) / np.linalg.norm([0.3, -0.5, 0.8])
    D = 4.0
    lo, hi, st, x, _ = NM.snap(p, N, D, lambda q: q @ nrm - 0.25)
    hit = st != 0
    assert hit.mean() > 0.5
    assert (np.abs(x[hit] @ nrm - 0.25) <= (2 * D / 15) / 2 ** NM.STEPS).all()
    assert (hi - lo)[hit].max() <= (2 * D / 15) / 2 ** NM.STEPS * (1 + 1e-9)


# ---------------------------------------------------------------- .glb
def _textured_rig(rng, N=40, F=30):
    W = np.zeros((30, 24), np.float32)
    for r in range(30):
        W[r, rng.choice(24, 3, replace=False)] = rng.random(3) + 0.1
    W /= W.sum(1, keepdims=True)
    n = rng.normal(0, 1, (N, 3))
    return dict(name="toy", vertices=rng.normal(0, 0.5, (N, 3)).astype(np.float32),
                triangles=rng.integers(0, N, (F, 3)).astype(np.int32), joints=rng.normal(0, 0.3, (24, 3)).astype(np.float32),
                nearest=rng.integers(0, 30, N), colors=rng.random((N, 3)).astype(np.float32), lbs_weights=W,
                parents=np.asarray(D.olbs.SMPL_PARENTS, dtype=np.int64),
                normals=(n / np.linalg.norm(n, axis=1, keepdims=True)).astype(np.float32))


def test_glb_with_normal_map_round_trip(tmp_path):
    import cv2 as cv
    from avatarclip_b200 import export as X
    rng = np.random.default_rng(8)
    rig = _textured_rig(rng)
    F, T = rig["triangles"].shape[0], 64
    uv = B.uv(F, T).reshape(-1, 2).astype(np.float32)
    image = rng.integers(0, 256, (T, T, 3), dtype=np.uint8)
    nmap = rng.integers(0, 256, (T, T, 3), dtype=np.uint8)
    tg = NM.corner_tangents(rig["vertices"], rig["triangles"], rig["normals"], uv).reshape(-1, 4).astype(np.float32)
    plain = X.write_glb(rig, str(tmp_path / "a.glb"), texture=(uv, image))
    none = X.write_glb(rig, str(tmp_path / "b.glb"), texture=(uv, image), normal_map=None)
    assert open(plain, "rb").read() == open(none, "rb").read()
    j0 = E.read_glb(plain)["json"]
    assert "TANGENT" not in j0["meshes"][0]["primitives"][0]["attributes"] and len(j0["images"]) == 1
    assert "normalTexture" not in j0["materials"][0]
    path = X.write_glb(rig, str(tmp_path / "n.glb"), texture=(uv, image), normal_map=(tg, nmap))
    glb = E.read_glb(path)
    j = glb["json"]
    prim = j["meshes"][0]["primitives"][0]
    at = prim["attributes"]
    acc = j["accessors"][at["TANGENT"]]
    assert acc["count"] == 3 * F and acc["type"] == "VEC4" and acc["componentType"] == 5126
    got = E.accessor(glb, at["TANGENT"])
    assert np.array_equal(got, tg)
    assert np.abs(np.linalg.norm(got[:, :3], axis=1) - 1).max() < 1e-6 and set(np.unique(got[:, 3])) <= {-1.0, 1.0}
    mat = j["materials"][prim["material"]]
    assert mat["normalTexture"] == {"index": 1, "texCoord": 0}
    assert mat["pbrMetallicRoughness"]["baseColorTexture"] == {"index": 0}
    src = j["textures"][1]["source"]
    assert src == 1 and j["textures"][0]["source"] == 0 and j["textures"][1]["sampler"] == 0

    def png(i):
        bv = j["bufferViews"][j["images"][i]["bufferView"]]
        return cv.imdecode(np.frombuffer(glb["bin"][bv["byteOffset"]:bv["byteOffset"] + bv["byteLength"]], np.uint8),
                           cv.IMREAD_UNCHANGED)[..., ::-1]
    assert np.array_equal(png(0), image) and np.array_equal(png(1), nmap)
    # everything else is as without the map
    for k in ("POSITION", "NORMAL", "TEXCOORD_0", "JOINTS_0", "WEIGHTS_0"):
        assert np.array_equal(E.accessor(glb, at[k]), E.accessor(E.read_glb(plain), j0["meshes"][0]["primitives"][0]
                                                                  ["attributes"][k])), k


def test_glb_normal_map_needs_texture_and_matching_tangents(tmp_path):
    from avatarclip_b200 import export as X
    rig = _textured_rig(np.random.default_rng(9))
    F = rig["triangles"].shape[0]
    tex = (B.uv(F, 64).reshape(-1, 2), np.zeros((64, 64, 3), np.uint8))
    nm = (np.tile([1.0, 0, 0, 1], (3 * F, 1)), np.zeros((64, 64, 3), np.uint8))
    with pytest.raises(ValueError, match="colour texture"):
        X.write_glb(rig, str(tmp_path / "a.glb"), normal_map=nm)
    with pytest.raises(ValueError, match="tangents"):
        X.write_glb(rig, str(tmp_path / "b.glb"), texture=tex, normal_map=(nm[0][:-1], nm[1]))
    assert not (tmp_path / "a.glb").exists() and not (tmp_path / "b.glb").exists()


# ---------------------------------------------------------------- CLI
def test_cli_normal_map_needs_conf(tmp_path, capsys):
    from avatarclip_b200 import export as X
    base = ["--mesh", str(tmp_path / "nope.ply"), "--smpl", str(tmp_path / "nope.npz"), "--stand_pose",
            str(tmp_path / "nope.npy"), "--out", str(tmp_path / "o.glb")]
    with pytest.raises(SystemExit) as e:
        X.main(base + ["--normal_map"])
    err = capsys.readouterr().err
    assert e.value.code == 2 and "--normal_map needs --conf" in err and "no such file" not in err
    a = X.build_parser().parse_args(base + ["--conf", "c.conf", "--normal_map"])
    assert a.normal_map and not X.build_parser().parse_args(base).normal_map
    with pytest.raises(ValueError, match="need conf"):
        X.export_avatar(str(tmp_path / "nope.ply"), str(tmp_path / "o.glb"), {}, str(tmp_path / "p.npy"),
                        normal_map=True)
    assert not (tmp_path / "o.glb").exists()
