"""Avatar export kernels (avc_cluster.cu, avc_nearest_vertex_f32) and avatarclip_b200.export against the CPU oracle, what
the reference's export_fbx.py computed (tests/golden/ref_avatar2fbx_small.pt) and drive's skinning."""
import ctypes as C
import io
import os

import numpy as np
import pytest
import torch

import util_neus as U
from oracle import drive as D
from oracle import export as E

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_avatar2fbx_small.pt")


@pytest.fixture(scope="module")
def g():
    return torch.load(GOLDEN, map_location="cpu", weights_only=False)


@pytest.fixture(scope="module")
def smpl(g):
    s = D.golden_smpl(g["smpl_seed"])
    assert {k: float(v.double().sum()) for k, v in s.items()} == g["smpl_sums"]
    return s


def _stand(g):
    return np.load(io.BytesIO(g["stand_pose_npy"].numpy().tobytes()))


@pytest.fixture(scope="module")
def big(g, smpl):
    """The mesh tools/bench_export.py times: the template subdivided three times (440 834 vertices), PLY frame."""
    v, f = D.bench_mesh(smpl, _stand(g), levels=3)
    c = np.random.default_rng(2).integers(0, 256, v.shape, dtype=np.uint8)
    return v, f, c


def _simplify(v, f, c, resolution=256):
    from avatarclip_b200 import export as X
    from avatarclip_b200.drive import Mesh
    m = X.simplify_mesh(Mesh(torch.from_numpy(np.ascontiguousarray(v)).cuda(),
                             torch.from_numpy(np.ascontiguousarray(f, dtype=np.int32)).cuda(), c), resolution)
    return m.vertices.cpu().numpy(), m.triangles.cpu().numpy(), m.vertex_colors


def _check_cluster(v, f, c, resolution=256):
    want_v, want_f, want_c = E.simplify(v, f, c, resolution)
    got_v, got_f, got_c = _simplify(v, f, None, resolution)
    assert got_c is None
    assert np.array_equal(got_v, want_v) and np.array_equal(got_f, want_f)
    got_v, got_f, got_c = _simplify(v, f, c, resolution)
    assert np.array_equal(got_v, want_v) and np.array_equal(got_f, want_f)
    ulp = np.abs(got_c.view(np.int32).astype(np.int64) - want_c.view(np.int32).astype(np.int64)).max()
    assert ulp <= 1
    return len(want_v), len(want_f), int(ulp)


# ---------------------------------------------------------------- clustering
def test_cluster_equals_oracle_on_golden(g):
    m = g["mesh"]
    K, T, ulp = _check_cluster(m["v"].numpy(), m["f"].numpy(), m["c"].numpy())
    assert K < len(m["v"]) and T == len(g["ref"]["triangles"])


def test_cluster_equals_oracle_on_hand_built_cases():
    from test_export_cpu import hand_mesh
    v, f = hand_mesh()
    c = np.arange(24, dtype=np.uint8).reshape(8, 3) * 7
    _check_cluster(v, f, c, resolution=4)
    _check_cluster(v, np.concatenate([f[[1]], f]), c, resolution=4)
    got_v, got_f, _ = _simplify(v, f, None, resolution=4)
    assert got_f.tolist() == [[0, 1, 2], [0, 2, 1], [1, 3, 4], [4, 3, 1]] and len(got_v) == 6
    got_v, got_f, _ = _simplify(np.ones((3, 3), np.float32), np.array([[0, 1, 2]]), None)      # one point
    assert got_v.tolist() == [[1.0, 1.0, 1.0]] and got_f.shape == (0, 3)
    got_v, got_f, _ = _simplify(v, np.zeros((0, 3), np.int32), None, resolution=4)             # no triangles
    assert len(got_v) == 6 and got_f.shape == (0, 3)


def test_cluster_equals_oracle_on_avatar_sized_mesh(big):
    v, f, c = big
    K, T, ulp = _check_cluster(v, f, c)
    U.log_parity("export_cluster_bench_mesh", {"vertices": K, "triangles": T, "colour_ulp": ulp})
    assert K < len(v)


def test_cluster_fan_and_crowded_voxel():
    """A fan of 200 000 triangles around one vertex: about 125 rim vertices per voxel, so most triangles collapse and
    the rest repeat one another many times over.  The rim lies on a 2^-20 grid, as the coordinates of a mesh a metre
    across do in float32, so the float64 sums are exact (a 1e-16 next to a 1e-2 in one voxel would not be)."""
    n = 200_000
    ang = np.linspace(0, 2 * np.pi, n, endpoint=False)
    rim = (np.round(np.stack([np.cos(ang), np.sin(ang), np.zeros(n)], 1) * 2.0 ** 20) / 2.0 ** 20).astype(np.float32)
    v = np.concatenate([np.zeros((1, 3), np.float32), rim])
    f = np.stack([np.zeros(n, np.int64), 1 + np.arange(n), 1 + (np.arange(n) + 1) % n], 1).astype(np.int32)
    _check_cluster(v, f, np.zeros((n + 1, 3), np.uint8))


def test_cluster_abi_rejects_bad_arguments():
    from avatarclip_b200 import export as X
    L = X._L()
    t = torch.zeros(64, 32, device="cuda")
    p = C.c_void_p(t.data_ptr())
    sz = C.c_size_t()
    E_BADCFG, E_NULL, E_SIZE = -1, -2, -3
    assert L.avc_mesh_cluster_workspace_bytes(0, 4, C.byref(sz)) == E_SIZE
    assert L.avc_mesh_cluster_workspace_bytes(4, -1, C.byref(sz)) == E_SIZE
    assert L.avc_mesh_cluster_workspace_bytes(4, 4, None) == E_NULL
    assert L.avc_mesh_cluster_workspace_bytes(4, 4, C.byref(sz)) == 0 and sz.value > 0
    assert L.avc_mesh_cluster(p, None, 4, p, 4, 0, p, None, p, p, p, sz.value, None) == E_BADCFG
    assert L.avc_mesh_cluster(p, None, 4, p, 4, (1 << 21) - 1, p, None, p, p, p, sz.value, None) == E_BADCFG
    assert L.avc_mesh_cluster(p, None, 4, p, 4, 256, p, None, p, p, p, sz.value - 1, None) == E_SIZE
    assert L.avc_mesh_cluster(p, p, 4, p, 4, 256, p, None, p, p, p, sz.value, None) == E_NULL     # colours, no output
    assert L.avc_mesh_cluster(p, None, 4, None, 4, 256, p, None, p, p, p, sz.value, None) == E_NULL
    assert L.avc_mesh_cluster(p, None, 4, p, 4, 256, p, None, p, None, p, sz.value, None) == E_NULL
    assert L.avc_nearest_vertex_f32(None, 4, p, 4, p, None) == E_NULL
    assert L.avc_nearest_vertex_f32(p, 0, p, 4, p, None) == E_SIZE
    assert L.avc_nearest_vertex_f32(p, 4, p, 0, p, None) == E_SIZE
    torch.cuda.synchronize()


# ---------------------------------------------------------------- float32 nearest vertex
def test_nearest_f32_equals_reference(g, smpl):
    from avatarclip_b200 import export as X
    m = g["mesh"]
    rot = np.matmul(E.simplify(m["v"].numpy(), m["f"].numpy(), None)[0], D.ROT)
    tmpl = D.load_template(smpl, _stand(g))[0]
    got = X.find_nearest_ind(torch.from_numpy(rot).cuda(), {"vertices": tmpl[None].cuda()}).cpu().numpy()
    assert np.array_equal(got, g["ref"]["nearest"].numpy())


def test_nearest_f32_on_avatar_sized_mesh(g, smpl, big):
    from avatarclip_b200 import export as X
    v = D.rotate(big[0]).astype(np.float32)
    tmpl = D.load_template(smpl, _stand(g))[0]
    got = X.find_nearest_ind(torch.from_numpy(v).cuda(), {"vertices": tmpl[None].cuda()}).cpu().numpy()
    sub = np.sort(np.random.default_rng(1).choice(v.shape[0], 16384, replace=False))
    assert np.array_equal(got[sub], E.find_nearest_ind(v[sub], tmpl.numpy()))


def test_nearest_f32_and_f64_differ_where_float32_ties():
    """1 + 1e-8 rounds to 1 in float32: the float32 search sees a tie and keeps the first reference point, the float64
    one finds the second truly nearer."""
    from avatarclip_b200 import drive
    from avatarclip_b200 import export as X
    q = np.array([[0.0, 0.0, 0.0], [0.0, 2.0, 0.0]], np.float32)
    ref = np.array([[1.0, 1e-4, 0.0], [1.0, 0.0, 0.0], [0.0, 2.0, 0.5]], np.float32)
    qt, rt = torch.from_numpy(q).cuda(), {"vertices": torch.from_numpy(ref).cuda()[None]}
    assert X.find_nearest_ind(qt, rt).tolist() == [0, 2] == E.find_nearest_ind(q, ref).tolist()
    assert drive.find_nearest_ind(qt, rt).tolist() == [1, 2] == D.find_nearest_ind(q, ref).tolist()


# ---------------------------------------------------------------- rig and file
def _write_inputs(g, smpl, tmp_path):
    from avatarclip_b200 import handoff
    m = g["mesh"]
    ply = handoff.write_ply(str(tmp_path / "avatar.ply"), m["v"].numpy(), m["f"].numpy(), m["c"].numpy())
    stand = tmp_path / "stand_pose.npy"
    stand.write_bytes(g["stand_pose_npy"].numpy().tobytes())
    return ply, str(stand)


@pytest.mark.parametrize("variant", ["ref", "ref_wide"])
def test_rig_avatar_equals_reference(g, smpl, tmp_path, variant):
    from avatarclip_b200 import export as X
    s = smpl if variant == "ref" else E.wide_smpl(smpl)
    r = g[variant]
    ply, stand = _write_inputs(g, smpl, tmp_path)
    rig = X.rig_avatar(ply, s, stand)
    assert np.array_equal(rig["triangles"], g["ref"]["triangles"].numpy())
    assert np.array_equal(rig["colors"], g["ref"]["colors"].numpy())
    n_diff = int((rig["nearest"] != r["nearest"].numpy()).sum())
    e_v = np.abs(rig["vertices"] - r["vertices"].numpy() / 100).max()
    e_j = np.abs(rig["joints"] - r["joints"].numpy() / 100).max()
    U.log_parity(f"export_rig_{variant}", {"nearest_differ": n_diff, "tpose": float(e_v), "joints": float(e_j)})
    assert n_diff == 0 and e_v <= 1e-5 and e_j <= 1e-5


def test_export_avatar_end_to_end(g, smpl, tmp_path):
    from avatarclip_b200 import drive
    from avatarclip_b200 import export as X
    s = E.wide_smpl(smpl)
    ply, stand = _write_inputs(g, smpl, tmp_path)
    motion = np.random.default_rng(3).normal(0, 0.3, (37, 72)).astype(np.float32)
    np.save(tmp_path / "walk.npy", motion)
    out = X.export_avatar(ply, str(tmp_path / "out" / "avatar.glb"), s, stand, str(tmp_path / "walk.npy"), fps=30)
    glb = E.read_glb(out)
    rig = X.rig_avatar(ply, s, stand)
    prim = glb["json"]["meshes"][0]["primitives"][0]
    assert "JOINTS_1" in prim["attributes"]                               # six influences on some vertices
    assert np.abs(E.skin(glb) - rig["vertices"]).max() <= 1e-5            # the bind pose is the T-pose
    sg = {k: v.cuda() for k, v in s.items()}
    w = sg["lbs_weights"][torch.from_numpy(rig["nearest"]).cuda()]
    tp = torch.from_numpy(rig["vertices"]).cuda()
    J0 = rig["joints"][0].astype(np.float64)
    Rx = np.array([[1, 0, 0], [0, 0, -1], [0, 1, 0]], dtype=np.float64)   # R_x(pi / 2)
    poses = drive.read_pose_my(str(tmp_path / "walk.npy"))
    assert len(glb["json"]["animations"][0]["channels"]) == 23 and len(poses) == 37
    err = 0.0
    for k in range(37):
        p_drive = drive.lbs(sg, tp, w, poses[k].cuda()).cpu().numpy().astype(np.float64)
        p_glb = E.skin(glb, k)
        err = max(err, np.abs((p_glb - J0) @ Rx.T + J0 - p_drive).max())
    U.log_parity("export_glb_vs_drive", {"frames": 37, "max_abs_err": float(err)})
    print(f"[export] 37 frames: skinned .glb vs drive.lbs max abs err {err:.2e} m")
    assert err <= 1e-5


def test_cli_end_to_end(g, smpl, tmp_path):
    from avatarclip_b200 import export as X
    ply, stand = _write_inputs(g, smpl, tmp_path)
    np.savez(tmp_path / "smpl.npz", **{k: np.asarray(v) for k, v in smpl.items()})
    np.save(tmp_path / "a.npy", np.random.default_rng(4).normal(0, 0.3, (5, 72)).astype(np.float32))
    assert X.main(["--mesh", ply, "--smpl", str(tmp_path / "smpl.npz"), "--stand_pose", stand, "--motion",
                   str(tmp_path / "a.npy"), "--out", str(tmp_path / "cli.glb")]) == 0
    glb = E.read_glb(str(tmp_path / "cli.glb"))
    assert glb["json"]["animations"][0]["name"] == "a" and glb["json"]["nodes"][0]["name"] == "avatar"


def test_cpu_tensors_raise(g):
    from avatarclip_b200 import AvcError
    from avatarclip_b200 import export as X
    with pytest.raises(AvcError):
        X.find_nearest_ind(g["mesh"]["v"].cuda(), {"vertices": torch.zeros(1, 10, 3)})
