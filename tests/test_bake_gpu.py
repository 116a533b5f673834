"""Texture baking on the GPU (avc_bake.cu, avatarclip_b200.bake, export's textured .glb): the texel map against the
fp64 oracle (oracle/bake.py), smooth normals, Runner.surface_colors' independence of the ray chunk, and the textured
export end to end on the small stand-pose checkpoint of tests/golden/ref_tree_checkpoint.tar."""
import io
import os

import numpy as np
import pytest
import torch

import util_neus as U
from oracle import bake as B
from oracle import drive as D
from oracle import export as E

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_avatar2fbx_small.pt")


@pytest.fixture(scope="module")
def g():
    return torch.load(GOLDEN, map_location="cpu", weights_only=False)


@pytest.fixture(scope="module")
def smpl(g):
    return D.golden_smpl(g["smpl_seed"])


def _stand(g):
    return np.load(io.BytesIO(g["stand_pose_npy"].numpy().tobytes()))


def _template():
    v, f = D.template_obj()
    return v.astype(np.float32), f.astype(np.int32)


# ---------------------------------------------------------------- kernels
def _check_texel_points(v, f, T):
    from avatarclip_b200 import bake
    owner, pts, uv = bake.texel_points(torch.from_numpy(v).cuda(), torch.from_numpy(f).cuda(), T)
    want_own, want_pts = B.texel_points(v, f, T)
    assert np.array_equal(owner.cpu().numpy(), want_own)
    extent = float((v.max(0) - v.min(0)).max())
    err = float(np.abs(pts.cpu().numpy().astype(np.float64) - want_pts).max()) / extent
    assert err <= 1e-6, err
    assert np.abs(uv.cpu().numpy().astype(np.float64) - B.uv(f.shape[0], T).reshape(-1, 2)).max() <= 1e-7
    return err


@pytest.mark.parametrize("F,T", [(1, 8), (2, 9), (5, 31), (99, 100), (1000, 256), (13776, 1024)])
def test_texel_points_equal_oracle(F, T):
    v, f = _template()
    f = f[:F]
    err = _check_texel_points(v, f, T)
    U.log_parity("bake_texel_points", {"F": F, "T": T, "point_err_rel_extent": err})


def test_texel_points_on_clustered_avatar(g, smpl):
    """The stand-pose template subdivided once (55 104 faces), clustered at resolution 128, on a 2048 texture."""
    from avatarclip_b200 import export as X
    from avatarclip_b200.drive import Mesh
    v, f = D.bench_mesh(smpl, _stand(g), levels=1)
    m = X.simplify_mesh(Mesh(torch.from_numpy(v).cuda(), torch.from_numpy(f.astype(np.int32)).cuda(), None), 128)
    err = _check_texel_points(m.vertices.cpu().numpy(), m.triangles.cpu().numpy(), 2048)
    U.log_parity("bake_texel_points_avatar", {"F": int(m.triangles.shape[0]), "point_err_rel_extent": err})


def test_texel_points_abi_rejects_bad_arguments():
    import ctypes as C
    from avatarclip_b200 import bake
    L = bake._L()
    t = torch.zeros(64, device="cuda")
    p = C.c_void_p(t.data_ptr())
    E_BADCFG, E_NULL, E_SIZE = -1, -2, -3
    assert L.avc_bake_texel_points(p, p, 3, 1, 7, p, p, None, None) == E_BADCFG      # c = 7 < 8
    assert L.avc_bake_texel_points(p, p, 3, 0, 64, p, p, None, None) == E_SIZE
    assert L.avc_bake_texel_points(p, p, 0, 1, 64, p, p, None, None) == E_SIZE
    assert L.avc_bake_texel_points(None, p, 3, 1, 64, p, p, None, None) == E_NULL
    assert L.avc_bake_texel_points(p, p, 3, 1, 64, None, p, None, None) == E_NULL
    assert L.avc_bake_vertex_normals(p, p, p, None, 3, 1, p, None) == E_NULL
    assert L.avc_bake_vertex_normals(p, p, p, p, 3, 0, p, None) == E_SIZE
    torch.cuda.synchronize()


def test_vertex_normals_reproducible_and_equal_numpy(g, smpl):
    from avatarclip_b200 import bake
    v, f = D.bench_mesh(smpl, _stand(g), levels=2)
    f = np.concatenate([f, np.array([[0, 0, 1]])]).astype(np.int32)        # a degenerate face adds nothing
    v = np.concatenate([v, np.zeros((1, 3), np.float32)])                   # an unreferenced vertex: (0, 1, 0)
    vt, ft = torch.from_numpy(v).cuda(), torch.from_numpy(f).cuda()
    a, b = bake.vertex_normals(vt, ft), bake.vertex_normals(vt, ft)
    assert torch.equal(a, b)
    want = B.vertex_normals(v, f)
    err = np.abs(a.cpu().numpy() - want).max(1)
    # the float32 sum loses about eps x (sum of |face normals|) / |their sum|: up to 500 at the creases of this mesh
    cr = np.cross(v[f[:, 1]] - v[f[:, 0]], v[f[:, 2]] - v[f[:, 0]]).astype(np.float64)
    mag, acc = np.zeros(v.shape[0]), np.zeros((v.shape[0], 3))
    for k in range(3):
        np.add.at(mag, f[:, k], np.linalg.norm(cr, axis=1))
        np.add.at(acc, f[:, k], cr)
    cond = np.maximum(1.0, mag / np.maximum(np.linalg.norm(acc, axis=1), 1e-300))
    U.log_parity("bake_vertex_normals", {"V": v.shape[0], "max_abs_err": float(err.max()),
                                         "max_err_over_cond": float((err / cond).max())})
    assert (err <= 1e-6 * cond).all() and a[-1].tolist() == [0.0, 1.0, 0.0]
    assert (err[cond < 2] <= 1e-6).all()


# ---------------------------------------------------------------- the NeuS run
def _conf(tmp_path):
    """confs/examples_small/example.conf with the small stand-pose checkpoint, without the extra colour head (the
    checkpoint has none), run directory under tmp_path."""
    ag = U.reference_tree(tmp_path / "ref")
    text = open(os.path.join(ag, "confs/examples_small/example.conf")).read()
    for old, new in (("./exp/", str(tmp_path / "exp") + "/"), ("./data/", ag + "/data/"),
                     ("./pretrained_models/", ag + "/pretrained_models/")):
        text = text.replace(old, new)
    text = text.replace("        extra_color = True\n", "")
    p = tmp_path / "example.conf"
    p.write_text(text)
    return str(p)


@pytest.fixture(scope="module")
def run(tmp_path_factory):
    from avatarclip_b200.runner import Runner
    tmp = tmp_path_factory.mktemp("bake_run")
    conf = _conf(tmp)
    r = Runner(conf, "validate_mesh", "smpl", device="cuda")
    assert not r.extra_color
    return conf, r


def test_surface_colors_do_not_depend_on_the_chunk(run):
    """With mid-bin samples the bytes are a function of the points alone: any ray chunk, any subset.  With the conf's
    jitter (perturb = 1) every render call draws new offsets, so the bytes move with the chunk: that spread is logged."""
    _, r = run
    gen = torch.Generator().manual_seed(0)
    d = torch.randn(5000, 3, generator=gen)
    pts = (d / d.norm(dim=1, keepdim=True) * torch.rand(5000, 1, generator=gen) * 0.6).cuda()
    base = r.surface_colors(pts, perturb=0)
    assert base.shape == (5000, 3) and base.dtype == np.uint8 and base.std() > 0
    for chunk in (333, 4096, 5000, 65536):
        assert np.array_equal(r.surface_colors(pts, chunk=chunk, perturb=0), base), chunk
    assert np.array_equal(r.surface_colors(pts[:40], chunk=1, perturb=0), base[:40])
    sub = np.sort(np.random.default_rng(1).choice(5000, 700, replace=False))
    assert np.array_equal(r.surface_colors(pts[torch.from_numpy(sub).cuda()], perturb=0), base[sub])
    torch.manual_seed(0)
    j512 = r.surface_colors(pts).astype(np.int64)
    torch.manual_seed(0)
    j4096 = r.surface_colors(pts, chunk=4096).astype(np.int64)
    diff = np.abs(j512 - j4096)
    U.log_parity("bake_surface_colors_jitter", {"frac_points_differ": float((diff.max(1) > 0).mean()),
                                                "max_byte_diff": int(diff.max()),
                                                "vs_midbin_max_byte_diff": int(np.abs(j512 - base).max())})
    print(f"[bake] perturb = 1: {100 * (diff.max(1) > 0).mean():.1f}% of points change with the chunk, by up to "
          f"{int(diff.max())}")


def test_textured_export_end_to_end(run, g, smpl, tmp_path):
    from avatarclip_b200 import bake
    from avatarclip_b200 import export as X
    from avatarclip_b200.runner import Runner
    import cv2 as cv
    conf, r = run
    r.iter_step = 100
    ply = r.validate_mesh(resolution=64)
    ckpt = r.save_checkpoint()
    stand = tmp_path / "stand_pose.npy"
    stand.write_bytes(g["stand_pose_npy"].numpy().tobytes())
    T = 1024
    out = X.export_avatar(ply, str(tmp_path / "avatar.glb"), smpl, str(stand), resolution=64, conf=conf,
                          checkpoint=os.path.basename(ckpt), texture_size=T)
    rig = X.rig_avatar(ply, smpl, str(stand), 64, ply_frame=True)
    plain = X.rig_avatar(ply, smpl, str(stand), 64)
    assert set(rig) == set(plain) | {"vertices_ply"}
    assert all(np.array_equal(rig[k], plain[k]) for k in plain if k not in ("name", "colors"))
    tri = rig["triangles"]
    F = tri.shape[0]
    glb = E.read_glb(out)
    j = glb["json"]
    prim = j["meshes"][0]["primitives"][0]
    at = prim["attributes"]
    assert "COLOR_0" not in at and all(j["accessors"][at[k]]["count"] == 3 * F for k in at)
    uv = E.accessor(glb, at["TEXCOORD_0"]).astype(np.float64)
    assert uv.min() >= 0 and uv.max() <= 1
    fp = B.footprint_owners(F, T, uv.reshape(F, 3, 2) * T)
    assert (fp == np.arange(F)[:, None, None]).all()                    # corner UVs sample their own face's texels
    nrm = E.accessor(glb, at["NORMAL"]).astype(np.float64)
    assert np.abs(np.linalg.norm(nrm, axis=1) - 1).max() <= 1e-6
    img = j["images"][j["textures"][j["materials"][prim["material"]]["pbrMetallicRoughness"]["baseColorTexture"]
                                    ["index"]]["source"]]
    bv = j["bufferViews"][img["bufferView"]]
    png = glb["bin"][bv["byteOffset"]:bv["byteOffset"] + bv["byteLength"]]
    tex = cv.imdecode(np.frombuffer(png, np.uint8), cv.IMREAD_UNCHANGED)[..., ::-1].reshape(-1, 3)
    own = B.texel_owner(F, T).reshape(-1)
    assert (tex[own < 0] == 0).all() and tex[own >= 0].std() > 0
    # a seeded sample of used texels: validate_mesh's colour recipe on the kernel's own texel points, called on those
    # points alone, in a Runner built as the export builds it
    r2 = Runner(conf, "validate_mesh", "smpl", device="cuda")
    r2.load_checkpoint(os.path.basename(ckpt))
    owner, pts, _ = bake.texel_points(torch.from_numpy(rig["vertices_ply"]).cuda(), torch.from_numpy(tri).cuda(), T,
                                      with_uv=False)
    assert np.array_equal(owner.cpu().numpy(), own)
    used = np.flatnonzero(own >= 0)
    sample = np.sort(np.random.default_rng(2).choice(used, 3000, replace=False))
    want = r2.surface_colors(pts[torch.from_numpy(sample).cuda()], perturb=0)
    assert np.array_equal(tex[sample], want)
    U.log_parity("bake_end_to_end", {"faces": F, "texture": T, "used_texels": int(used.size)})


def test_cli_refuses_a_texture_too_small(run, g, smpl, tmp_path, capsys):
    from avatarclip_b200 import export as X
    conf, r = run
    r.iter_step = 200
    ply = r.validate_mesh(resolution=64)
    stand = tmp_path / "stand_pose.npy"
    stand.write_bytes(g["stand_pose_npy"].numpy().tobytes())
    np.savez(tmp_path / "smpl.npz", **{k: np.asarray(v) for k, v in smpl.items()})
    with pytest.raises(SystemExit) as e:
        X.main(["--mesh", ply, "--smpl", str(tmp_path / "smpl.npz"), "--stand_pose", str(stand), "--out",
                str(tmp_path / "o.glb"), "--conf", conf, "--texture_size", "16"])
    err = capsys.readouterr().err
    assert e.value.code == 2 and "smallest texture size that fits is" in err and "--resolution" in err
    assert not (tmp_path / "o.glb").exists()
