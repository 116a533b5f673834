"""avc_mesh_decimate against its fp64 restatement (oracle/decimate.py): faces, float32 positions and colours bit for
bit; run-to-run and workspace independence; the no-op below the target; the ABI's refusals; the distance bar against
vertex clustering on an avatar-sized mesh; and the export with --target_faces end to end."""
import ctypes as C
import io
import os

import numpy as np
import pytest
import torch

import util_neus as U
from oracle import decimate as O
from oracle import drive as D

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


def _mesh(v, f, c=None):
    from avatarclip_b200.drive import Mesh
    return Mesh(torch.from_numpy(np.ascontiguousarray(v, np.float32)).cuda(),
                torch.from_numpy(np.ascontiguousarray(f, np.int32)).cuda(), c)


def _inputs(g, smpl):
    tv, tf = D.template_obj()
    sv, sf = O.sphere()
    fv, ff, _ = O.fan(12)
    return {"template_subdivided": (*D.bench_mesh(smpl, _stand(g), levels=1), 3000),
            "template": (tv, tf, 2000), "sphere": (sv, sf, 400), "fan_boundary": (fv, ff, 40)}


@pytest.mark.parametrize("name", ["template_subdivided", "template", "sphere", "fan_boundary"])
def test_decimate_equals_oracle(g, smpl, name):
    from avatarclip_b200 import export as X
    v, f, target = _inputs(g, smpl)[name]
    c = np.random.default_rng(5).random(v.shape).astype(np.float32)
    m, rounds = X._decimate(_mesh(v, f, c), target)
    want = O.decimate(v, f, target, colors=c)
    got_v, got_f = m.vertices.cpu().numpy(), m.triangles.cpu().numpy()
    assert rounds == want["rounds"]
    assert np.array_equal(got_f, want["faces"])
    assert got_v.tobytes() == want["vertices"].tobytes()
    assert m.vertex_colors.tobytes() == want["colors"].tobytes()
    U.log_parity("decimate_equals_oracle", {"mesh": name, "faces_in": int(f.shape[0]), "faces_out": int(got_f.shape[0]),
                                            "rounds": rounds})


def _raw(v, f, target, ws_fill=None, colors=None):
    from avatarclip_b200 import _lib
    from avatarclip_b200 import export as X
    L = X._L()
    V, F = v.shape[0], f.shape[0]
    need = C.c_size_t()
    assert L.avc_mesh_decimate_workspace_bytes(V, F, C.byref(need)) == 0
    ws = torch.empty(need.value, dtype=torch.uint8, device="cuda")
    if ws_fill is not None:
        ws.random_(0, 256, generator=torch.Generator("cuda").manual_seed(ws_fill))
    vo, fo = torch.zeros(V, 3, device="cuda"), torch.zeros(F, 3, dtype=torch.int32, device="cuda")
    co = None if colors is None else torch.zeros(V, 3, device="cuda")
    counts = torch.zeros(3, dtype=torch.int32, device="cuda")
    _lib.check(L.avc_mesh_decimate(_lib.ptr(v), _lib.ptr(colors), V, _lib.ptr(f), F, target, _lib.ptr(vo),
                                   _lib.ptr(co), _lib.ptr(fo), _lib.ptr(counts), _lib.ptr(ws), ws.numel(),
                                   _lib.stream_ptr()), "avc_mesh_decimate")
    K, T, _ = counts.tolist()
    return vo[:K].cpu().numpy().tobytes() + fo[:T].cpu().numpy().tobytes() + \
        (b"" if co is None else co[:K].cpu().numpy().tobytes()), counts.tolist()


def test_deterministic_whatever_the_workspace_held(g, smpl):
    v, f = D.bench_mesh(smpl, _stand(g), levels=2)
    vt, ft = torch.from_numpy(v).cuda(), torch.from_numpy(f.astype(np.int32)).cuda()
    ct = torch.rand(v.shape, generator=torch.Generator().manual_seed(1)).cuda()
    a, ca = _raw(vt, ft, 5000, None, ct)
    b, cb = _raw(vt, ft, 5000, 7, ct)
    assert ca == cb and a == b and ca[1] in (4999, 5000)


@pytest.mark.parametrize("extra", [0, 10])
def test_at_or_above_the_face_count_is_a_no_op(extra):
    v, f = O.sphere(16)
    vt, ft = torch.from_numpy(v).cuda(), torch.from_numpy(f.astype(np.int32)).cuda()
    ct = torch.rand(v.shape).cuda()
    out, counts = _raw(vt, ft, f.shape[0] + extra, 3, ct)
    assert counts == [v.shape[0], f.shape[0], 0]
    assert out == v.tobytes() + f.astype(np.int32).tobytes() + ct.cpu().numpy().tobytes()


def test_abi_rejects_bad_arguments():
    from avatarclip_b200 import export as X
    L = X._L()
    t = torch.zeros(1 << 16, device="cuda")
    p = C.c_void_p(t.data_ptr())
    E_BADCFG, E_NULL, E_SIZE = -1, -2, -3
    sz = C.c_size_t()
    assert L.avc_mesh_decimate_workspace_bytes(4, 4, None) == E_NULL
    assert L.avc_mesh_decimate_workspace_bytes(0, 4, C.byref(sz)) == E_SIZE
    assert L.avc_mesh_decimate_workspace_bytes(4, 0, C.byref(sz)) == E_SIZE
    assert L.avc_mesh_decimate_workspace_bytes(4, (1 << 29) + 1, C.byref(sz)) == E_SIZE
    assert L.avc_mesh_decimate_workspace_bytes(4, 4, C.byref(sz)) == 0
    n = t.numel() * 4
    assert L.avc_mesh_decimate(p, None, 4, p, 4, 0, p, None, p, p, p, n, None) == E_BADCFG
    assert L.avc_mesh_decimate(p, None, 4, p, 4, 2, p, None, p, p, p, sz.value - 1, None) == E_SIZE
    assert L.avc_mesh_decimate(None, None, 4, p, 4, 2, p, None, p, p, p, n, None) == E_NULL
    assert L.avc_mesh_decimate(p, None, 4, None, 4, 2, p, None, p, p, p, n, None) == E_NULL
    assert L.avc_mesh_decimate(p, p, 4, p, 4, 2, p, None, p, p, p, n, None) == E_NULL     # colours need colors_out
    assert L.avc_mesh_decimate(p, None, 4, p, 4, 2, p, None, p, None, p, n, None) == E_NULL
    assert L.avc_mesh_decimate(p, None, 4, p, 4, 2, p, None, p, p, None, n, None) == E_NULL
    torch.cuda.synchronize()


# ---------------------------------------------------------------- quality against vertex clustering
def test_quality_beats_vertex_clustering_on_avatar_sized_mesh(g, smpl):
    """test_export_gpu.py's ``big`` mesh (the template subdivided three times, 881 664 faces) reduced to 13 776 faces
    (``reduce_mesh`` at resolution 256) against vertex clustering at the smallest resolution that keeps at least as
    many faces, both measured against the input by the two-sided sampled distance (2 000 000 samples on the input)."""
    from avatarclip_b200 import export as X
    v, f = D.bench_mesh(smpl, _stand(g), levels=3)
    target = 13776
    red = X.reduce_mesh(_mesh(v, f), 256, target)
    F = red.triangles.shape[0]
    assert 0.95 * target <= F <= target, F
    lo, hi = 8, 256
    while lo < hi:                                   # the smallest resolution keeping >= target faces
        mid = (lo + hi) // 2
        if X.simplify_mesh(_mesh(v, f), mid).triangles.shape[0] >= target:
            hi = mid
        else:
            lo = mid + 1
    cl = X.simplify_mesh(_mesh(v, f), lo)
    assert cl.triangles.shape[0] >= target
    spacing = O.spacing_for(v, f)
    dr = O.surface_distance(v, f, red.vertices.cpu().numpy(), red.triangles.cpu().numpy(), spacing)
    dc = O.surface_distance(v, f, cl.vertices.cpu().numpy(), cl.triangles.cpu().numpy(), spacing)
    top = O.topology(red.vertices.cpu().numpy(), red.triangles.cpu().numpy())
    U.log_parity("decimate_quality", {"faces": int(F), "cluster_resolution": lo,
                                      "cluster_faces": int(cl.triangles.shape[0]), "decimated": dr, "clustered": dc,
                                      "topology": top, "spacing": spacing})
    print(f"[decimate] quality: reduced ({F} faces) {dr}; clustered at {lo} ({cl.triangles.shape[0]} faces) {dc}; "
          f"topology {top}")
    assert dr["mean"] < dc["mean"] and dr["p99"] < dc["p99"]


# ---------------------------------------------------------------- end to end
def _conf(tmp_path):
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
    tmp = tmp_path_factory.mktemp("decimate_run")
    conf = _conf(tmp)
    return conf, Runner(conf, "validate_mesh", "smpl", device="cuda")


def test_textured_export_with_target_faces(run, g, smpl, tmp_path, capsys):
    """A texture size the clustered mesh is refused at is baked with --target_faces: at most the target's faces, the
    skin equal to drive.lbs of the reduced bind pose at every frame, every texel footprint on its own face."""
    from oracle import bake as B
    from oracle import export as E
    from avatarclip_b200 import drive as XD
    from avatarclip_b200 import export as X
    conf, r = run
    r.iter_step = 300
    ply = r.validate_mesh(resolution=128)
    ckpt = os.path.basename(r.save_checkpoint())
    stand = tmp_path / "stand_pose.npy"
    stand.write_bytes(g["stand_pose_npy"].numpy().tobytes())
    np.savez(tmp_path / "smpl.npz", **{k: np.asarray(x) for k, x in smpl.items()})
    F0 = X.rig_avatar(ply, smpl, str(stand), 128)["triangles"].shape[0]
    T = 512
    while 8 * B.grid(F0, T)[0] <= T:                  # a size the clustered mesh does not fit
        T //= 2
    target = 2 * (T // 8) ** 2                         # the most faces a T x T atlas holds
    assert target < F0
    base = ["--mesh", ply, "--smpl", str(tmp_path / "smpl.npz"), "--stand_pose", str(stand), "--resolution", "128",
            "--conf", conf, "--checkpoint", ckpt, "--texture_size", str(T)]
    with pytest.raises(SystemExit) as e:
        X.main(base + ["--out", str(tmp_path / "refused.glb")])
    assert e.value.code == 2 and "smallest texture size that fits is" in capsys.readouterr().err
    np.save(tmp_path / "a.npy", np.random.default_rng(4).normal(0, 0.3, (5, 72)).astype(np.float32))
    out = str(tmp_path / "dec.glb")
    assert X.main(base + ["--out", out, "--target_faces", str(target), "--motion", str(tmp_path / "a.npy")]) == 0
    assert "decimation stopped" not in capsys.readouterr().err
    rig = X.rig_avatar(ply, smpl, str(stand), 128, target_faces=target)
    F = rig["triangles"].shape[0]
    assert 0.9 * target <= F <= target, (F, target)
    glb = E.read_glb(out)
    j = glb["json"]
    at = j["meshes"][0]["primitives"][0]["attributes"]
    assert j["accessors"][at["POSITION"]]["count"] == 3 * F
    uv = E.accessor(glb, at["TEXCOORD_0"]).astype(np.float64)
    fp = B.footprint_owners(F, T, uv.reshape(F, 3, 2) * T)
    assert (fp == np.arange(F)[:, None, None]).all()
    # the skin: glTF skinning at every frame equals drive.lbs of the reduced T-pose vertices, as the export tests check
    sg = {k: x.cuda() for k, x in smpl.items()}
    w = sg["lbs_weights"][torch.from_numpy(rig["nearest"]).cuda()]
    tp = torch.from_numpy(rig["vertices"]).cuda()
    J0 = rig["joints"][0].astype(np.float64)
    Rx = np.array([[1, 0, 0], [0, 0, -1], [0, 1, 0]], dtype=np.float64)
    poses = XD.read_pose_my(str(tmp_path / "a.npy"))
    corner = rig["triangles"].reshape(-1)
    assert np.abs(E.skin(glb) - rig["vertices"][corner]).max() <= 1e-5
    err = 0.0
    for k in range(len(poses)):
        p_drive = XD.lbs(sg, tp, w, poses[k].cuda()).cpu().numpy().astype(np.float64)[corner]
        err = max(err, np.abs((E.skin(glb, k) - J0) @ Rx.T + J0 - p_drive).max())
    assert err <= 1e-5, err
    U.log_parity("decimate_end_to_end", {"clustered_faces": F0, "texture": T, "target": target, "faces": F,
                                         "skin_err": err})


def test_target_at_or_above_the_clustered_count_writes_the_same_bytes(run, g, smpl, tmp_path):
    from avatarclip_b200 import export as X
    conf, r = run
    r.iter_step = 400
    ply = r.validate_mesh(resolution=64)
    stand = tmp_path / "stand_pose.npy"
    stand.write_bytes(g["stand_pose_npy"].numpy().tobytes())
    F0 = X.rig_avatar(ply, smpl, str(stand), 64)["triangles"].shape[0]
    a = X.export_avatar(ply, str(tmp_path / "a.glb"), smpl, str(stand), resolution=64)
    for t in (F0, F0 + 1000):
        b = X.export_avatar(ply, str(tmp_path / f"b{t}.glb"), smpl, str(stand), resolution=64, target_faces=t)
        assert open(a, "rb").read() == open(b, "rb").read()


def test_export_reports_a_stop_above_the_target(g, smpl, tmp_path, capsys):
    from avatarclip_b200 import export as X
    from avatarclip_b200 import handoff
    v, f = O.tetrahedron()
    ply = handoff.write_ply(str(tmp_path / "tet.ply"), v * 0.3, f, np.full(v.shape, 200, np.uint8))
    stand = tmp_path / "stand_pose.npy"
    stand.write_bytes(g["stand_pose_npy"].numpy().tobytes())
    X.export_avatar(ply, str(tmp_path / "tet.glb"), smpl, str(stand), target_faces=1)
    err = capsys.readouterr().err
    assert "decimation stopped at 4 faces, above --target_faces 1" in err
    assert _glb_faces(str(tmp_path / "tet.glb")) == 4


def _glb_faces(path):
    from oracle import export as E
    glb = E.read_glb(path)
    prim = glb["json"]["meshes"][0]["primitives"][0]
    return glb["json"]["accessors"][prim["indices"]]["count"] // 3
