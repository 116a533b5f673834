"""The texture atlas of avatarclip_b200.bake (oracle/bake.py in float64): ownership, the bilinear-footprint invariant
and the refusal threshold; the textured .glb that export.write_glb writes, parsed back; the export CLI's texture flags."""
import os

import numpy as np
import pytest

from oracle import bake as B
from oracle import drive as D
from oracle import export as E

SIZES = [(1, 8), (2, 8), (3, 16), (7, 24), (8, 23), (100, 80), (101, 97), (1000, 256), (4097, 512), (20001, 1024)]


def _inside_points(F, T, rng, n_random=6):
    """Texel-space points inside every face's UV triangle: the corners, the edge midpoints, the centroid and random
    barycentric combinations.  -> [F, P, 2]"""
    uv = B.uv(F, T) * T                                                          # [F, 3, 2]
    w = [np.eye(3), np.array([[0.5, 0.5, 0], [0, 0.5, 0.5], [0.5, 0, 0.5], [1 / 3, 1 / 3, 1 / 3]])]
    w.append(rng.dirichlet(np.ones(3), n_random))
    w = np.concatenate(w)                                                        # [P, 3]
    return np.einsum("pk,fkd->fpd", w, uv)


@pytest.mark.parametrize("F,T", SIZES)
def test_every_footprint_stays_on_its_own_face(F, T):
    rng = np.random.default_rng(F * 7919 + T)
    m, c = B.grid(F, T)
    assert c >= B.MIN_CELL and m * m >= (F + 1) // 2 > (m - 1) * (m - 1)
    own = B.texel_owner(F, T)
    # one owner per texel; cell k holds only faces 2k and 2k + 1; every face owns texels; nothing past the last face
    y, x = np.mgrid[0:T, 0:T]
    used = own >= 0
    k = (y // c) * m + x // c
    assert np.array_equal(own[used] // 2, k[used])
    assert np.array_equal(np.unique(own[used]), np.arange(F))
    assert not used[(x >= m * c) | (y >= m * c) | (2 * k >= F)].any()
    uv = B.uv(F, T)
    assert uv.min() > 0 and uv.max() < 1
    fp = B.footprint_owners(F, T, _inside_points(F, T, rng))                     # [F, P, 4]
    assert (fp == np.arange(F)[:, None, None]).all()


@pytest.mark.parametrize("F,T", [(1, 8), (9, 40), (1000, 256)])
def test_texel_points_are_in_their_triangles(F, T):
    rng = np.random.default_rng(F)
    verts = rng.normal(0, 1, (F + 2, 3))
    faces = np.stack([np.arange(F), np.arange(F) + 1, np.arange(F) + 2], 1)
    own, pts = B.texel_points(verts, faces, T)
    used = own >= 0
    _, c = B.grid(F, T)
    y, x = np.divmod(np.arange(T * T), T)
    b = B.barycentric(x % c + 0.5, y % c + 0.5, c, x % c < y % c)
    assert (b >= 0).all() and np.allclose(b.sum(1), 1)
    tri = verts[faces[own[used]]]
    assert np.allclose(pts[used], (b[used][:, :, None] * tri).sum(1))
    assert (pts[~used] == 0).all()
    # texels whose centre lies inside the UV triangle keep their barycentrics unclamped: the map is affine there
    cen = np.stack([x + 0.5, y + 0.5], 1)[used]
    corner = B.uv(F, T)[own[used]] * T
    e1, e2, d = corner[:, 1] - corner[:, 0], corner[:, 2] - corner[:, 0], cen - corner[:, 0]
    det = e1[:, 0] * e2[:, 1] - e1[:, 1] * e2[:, 0]
    al = (d[:, 0] * e2[:, 1] - d[:, 1] * e2[:, 0]) / det
    be = (e1[:, 0] * d[:, 1] - e1[:, 1] * d[:, 0]) / det
    inside = (al >= 0) & (be >= 0) & (al + be <= 1)
    assert inside.mean() > 0.2
    assert np.allclose(b[used][inside], np.stack([1 - al - be, al, be], 1)[inside])


def test_refusal_threshold_names_the_smallest_texture():
    from avatarclip_b200 import bake
    for F in (1, 2, 3, 50, 803006, 1 << 30):
        m, _ = B.grid(F, 1)
        smallest = 8 * m
        if smallest <= bake.MAX_TEXTURE_SIZE:
            assert bake.atlas_grid(F, smallest) == (m, 8) == B.grid(F, smallest)
        if smallest - 1 >= 1:
            with pytest.raises(bake.AtlasTooSmall) as e:
                bake.atlas_grid(F, min(smallest - 1, bake.MAX_TEXTURE_SIZE))
            msg = str(e.value)
            assert f"{F} faces" in msg and f"smallest texture size that fits is {smallest}" in msg
            assert "--resolution" in msg
    # the 803 006 triangles of the default clustering need 8 * 634 texels; at 2048 the cells are 3 wide
    assert B.grid(803006, 2048) == (634, 3)
    with pytest.raises(Exception):
        bake.atlas_grid(0, 64)
    with pytest.raises(Exception):
        bake.atlas_grid(10, bake.MAX_TEXTURE_SIZE + 1)


# ---------------------------------------------------------------- textured .glb
def _textured_rig(rng, N=40, F=30):
    W = np.zeros((30, 24), np.float32)
    for r in range(30):
        idx = rng.choice(24, 3, replace=False)
        W[r, idx] = rng.random(3) + 0.1
    W /= W.sum(1, keepdims=True)
    n = rng.normal(0, 1, (N, 3)).astype(np.float32)
    return dict(name="toy", vertices=rng.normal(0, 0.5, (N, 3)).astype(np.float32),
                triangles=rng.integers(0, N, (F, 3)).astype(np.int32), joints=rng.normal(0, 0.3, (24, 3)).astype(np.float32),
                nearest=rng.integers(0, 30, N), colors=rng.random((N, 3)).astype(np.float32), lbs_weights=W,
                parents=np.asarray(D.olbs.SMPL_PARENTS, dtype=np.int64),
                normals=n / np.linalg.norm(n, axis=1, keepdims=True))


def test_textured_glb_round_trip(tmp_path):
    import cv2 as cv
    from avatarclip_b200 import export as X
    rng = np.random.default_rng(5)
    rig = _textured_rig(rng)
    F, T = rig["triangles"].shape[0], 64
    uv = B.uv(F, T).reshape(-1, 2).astype(np.float32)
    image = rng.integers(0, 256, (T, T, 3), dtype=np.uint8)
    path = X.write_glb(rig, str(tmp_path / "t.glb"), texture=(uv, image))
    glb = E.read_glb(path)
    j = glb["json"]
    assert glb["header"][2] == glb["size"] == os.path.getsize(path)
    assert all(v.get("byteOffset", 0) % 4 == 0 for v in j["bufferViews"])
    prim = j["meshes"][0]["primitives"][0]
    at = prim["attributes"]
    assert "COLOR_0" not in at and {"POSITION", "NORMAL", "TEXCOORD_0", "JOINTS_0", "WEIGHTS_0"} <= set(at)
    for name in at:
        assert j["accessors"][at[name]]["count"] == 3 * F, name
    corner = rig["triangles"].reshape(-1)
    assert np.array_equal(E.accessor(glb, prim["indices"]).reshape(-1), np.arange(3 * F))
    assert np.array_equal(E.accessor(glb, at["POSITION"]), rig["vertices"][corner])
    assert np.array_equal(E.accessor(glb, at["NORMAL"]), rig["normals"][corner])
    got_uv = E.accessor(glb, at["TEXCOORD_0"])
    assert j["accessors"][at["TEXCOORD_0"]]["type"] == "VEC2" and np.array_equal(got_uv, uv)
    assert got_uv.min() >= 0 and got_uv.max() <= 1
    # corner UVs sample only their own face's texels
    fp = B.footprint_owners(F, T, got_uv.astype(np.float64).reshape(F, 3, 2) * T)
    assert (fp == np.arange(F)[:, None, None]).all()
    # skin: the shared vertex's weights on every corner
    W = rig["lbs_weights"][rig["nearest"]][corner]
    got = np.zeros_like(W)
    Js = E.accessor(glb, at["JOINTS_0"]).astype(np.int64)
    np.add.at(got, (np.arange(W.shape[0])[:, None].repeat(4, 1), Js), E.accessor(glb, at["WEIGHTS_0"]))
    assert np.array_equal(got, W)
    assert np.abs(E.skin(glb) - rig["vertices"][corner]).max() <= 1e-6
    # material, texture, sampler and the PNG
    mat = j["materials"][prim["material"]]["pbrMetallicRoughness"]
    assert mat["baseColorTexture"] == {"index": 0} and mat.get("baseColorFactor", [1, 1, 1, 1]) == [1, 1, 1, 1]
    tex = j["textures"][0]
    assert j["samplers"][tex["sampler"]] == {"magFilter": 9729, "minFilter": 9729, "wrapS": 33071, "wrapT": 33071}
    img = j["images"][tex["source"]]
    assert img["mimeType"] == "image/png"
    bv = j["bufferViews"][img["bufferView"]]
    png = glb["bin"][bv["byteOffset"]:bv["byteOffset"] + bv["byteLength"]]
    assert png[:8] == b"\x89PNG\r\n\x1a\n"
    dec = cv.imdecode(np.frombuffer(png, np.uint8), cv.IMREAD_UNCHANGED)
    assert np.array_equal(dec[..., ::-1], image)                               # the exact bytes, RGB, row 0 on top


def test_textured_glb_needs_normals_and_matching_uv(tmp_path):
    from avatarclip_b200 import export as X
    rng = np.random.default_rng(6)
    rig = _textured_rig(rng)
    F = rig["triangles"].shape[0]
    tex = (B.uv(F, 64).reshape(-1, 2), np.zeros((64, 64, 3), np.uint8))
    with pytest.raises(ValueError, match="normals"):
        X.write_glb(dict(rig, normals=None), str(tmp_path / "a.glb"), texture=tex)
    with pytest.raises(ValueError, match="uv"):
        X.write_glb(rig, str(tmp_path / "b.glb"), texture=(tex[0][:-1], tex[1]))
    assert not (tmp_path / "a.glb").exists() and not (tmp_path / "b.glb").exists()


def test_untextured_glb_ignores_normals(tmp_path):
    from avatarclip_b200 import export as X
    rig = _textured_rig(np.random.default_rng(7))
    a = X.write_glb(rig, str(tmp_path / "a.glb"))
    b = X.write_glb(dict(rig, normals=None), str(tmp_path / "b.glb"))
    assert open(a, "rb").read() == open(b, "rb").read()
    assert "TEXCOORD_0" not in E.read_glb(a)["json"]["meshes"][0]["primitives"][0]["attributes"]


# ---------------------------------------------------------------- CLI
def test_cli_texture_flags_need_conf(tmp_path, capsys):
    from avatarclip_b200 import export as X
    base = ["--mesh", str(tmp_path / "nope.ply"), "--smpl", str(tmp_path / "nope.npz"), "--stand_pose",
            str(tmp_path / "nope.npy"), "--out", str(tmp_path / "o.glb")]
    for extra in (["--case", "smpl"], ["--checkpoint", "ckpt_000100.pth"], ["--texture_size", "1024"]):
        with pytest.raises(SystemExit) as e:
            X.main(base + extra)
        err = capsys.readouterr().err
        assert e.value.code == 2 and f"{extra[0]} needs --conf" in err and "no such file" not in err, extra
    for size in ("0", "16385"):
        with pytest.raises(SystemExit) as e:
            X.main(base + ["--conf", str(tmp_path / "nope.conf"), "--texture_size", size])
        assert e.value.code == 2 and "--texture_size must be in [1, 16384]" in capsys.readouterr().err
    with pytest.raises(SystemExit) as e:
        X.main(base + ["--conf", str(tmp_path / "nope.conf")])
    assert e.value.code == 2 and "no such file" in capsys.readouterr().err
    a = X.build_parser().parse_args(base + ["--conf", "c.conf", "--case", "hulk", "--checkpoint", "ckpt_000100.pth",
                                            "--texture_size", "1024"])
    assert (a.conf, a.case, a.checkpoint, a.texture_size) == ("c.conf", "hulk", "ckpt_000100.pth", 1024)
    assert not (tmp_path / "o.glb").exists()


def test_export_avatar_refuses_texture_arguments_without_conf(tmp_path):
    from avatarclip_b200 import export as X
    for kw in (dict(checkpoint="ckpt_000100.pth"), dict(texture_size=1024)):
        with pytest.raises(ValueError, match="need conf"):
            X.export_avatar(str(tmp_path / "nope.ply"), str(tmp_path / "o.glb"), {}, str(tmp_path / "p.npy"), **kw)
