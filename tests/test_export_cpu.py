"""Avatar export (Avatar2FBX) without a GPU: the CPU oracle against what the reference's own export_fbx.py computed
(tests/golden/ref_avatar2fbx_small.pt, recorded by oracle/pin_avatar2fbx.py), the restated vertex clustering on
hand-built meshes, the glTF writer read back by the oracle's reader, the CLI's rejections and the refusal of CPU
tensors."""
import io
import os

import numpy as np
import pytest
import torch

from oracle import drive as D
from oracle import export as E

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


# ---------------------------------------------------------------- the oracle against the reference
@pytest.mark.parametrize("variant", ["ref", "ref_wide"])
def test_oracle_reproduces_reference(g, smpl, variant):
    s = smpl if variant == "ref" else E.wide_smpl(smpl)
    if variant == "ref_wide":
        assert float(s["lbs_weights"].double().sum()) == g["wide_sum"]
    m, r = g["mesh"], g[variant]
    o = E.smpl_object(m["v"].numpy(), m["f"].numpy(), m["c"].numpy(), s, _stand(g))
    assert np.array_equal(o["nearest"], r["nearest"].numpy())
    assert np.array_equal(o["triangles"], g["ref"]["triangles"].numpy())
    assert np.array_equal(o["colors"], g["ref"]["colors"].numpy())
    assert (o["vertices"] / 100 - r["vertices"] / 100).abs().max().item() <= 1e-5
    assert (o["joints"] / 100 - r["joints"] / 100).abs().max().item() <= 1e-5
    assert len(o["vertices"]) < len(m["v"]) and len(o["triangles"]) < len(m["f"])     # clustering merged vertices


def test_golden_mesh_edge_cases(g):
    m = g["mesh"]
    v, f = m["v"].numpy(), m["f"].numpy()
    vox = E.voxel_size(v)
    lo = v.astype(np.float64).min(0) - vox * 0.5
    q = (np.float64(v[m["boundary_vertex"], 0]) - lo[0]) / vox
    assert q == np.floor(q)                                   # exactly on a voxel boundary
    cl = E.cluster(v, f)[3]
    assert m["isolated_vertex"] not in set(f.reshape(-1).tolist())
    assert (cl == cl[m["isolated_vertex"]]).sum() == 1
    assert g["ref_wide"]["max_influences"] > 4 >= g["ref"]["max_influences"]


# ---------------------------------------------------------------- the restated clustering on hand-built meshes
def hand_mesh():
    """Extent 4 on x with resolution 4: voxel 1, voxel_min_bound = min - 0.5 = 0, so a vertex's voxel is floor(x)."""
    v = np.array([[0.5, 0.5, 0.5],     # 0: voxel (0,0,0)
                  [2.5, 0.5, 0.5],     # 1: (2,0,0)
                  [0.7, 0.6, 0.5],     # 2: (0,0,0) with 0
                  [1.5, 1.5, 0.5],     # 3: (1,1,0)
                  [3.0, 0.5, 0.5],     # 4: x = 3.0 exactly on a boundary -> (3,0,0)
                  [2.9, 0.5, 0.5],     # 5: (2,0,0) with 1
                  [4.5, 2.5, 0.5],     # 6: (4,2,0): the max bound
                  [1.2, 2.2, 0.5]],    # 7: (1,2,0): in no triangle
                 dtype=np.float32)
    f = np.array([[0, 1, 3],      # -> (0,1,2) kept
                  [1, 3, 0],      # rotation of it: dropped
                  [3, 0, 1],      # rotation: dropped
                  [0, 3, 1],      # reversed: kept
                  [0, 2, 3],      # 0 and 2 share a voxel: dropped
                  [5, 4, 6],      # -> (1,3,4) kept
                  [2, 5, 3],      # -> (0,1,2) again through other vertices: dropped
                  [6, 4, 5]],     # -> (4,3,1), a reversal of (1,3,4): kept
                 dtype=np.int32)
    return v, f


def test_cluster_hand_built():
    v, f = hand_mesh()
    c = np.arange(24, dtype=np.float64).reshape(8, 3) / 255.0
    ov, t, oc, cl = E.cluster(v, f, c, resolution=4)
    # output order = first appearance: vertex 0 -> 0, 1 -> 1, 3 -> 2, 4 -> 3, 6 -> 4, 7 -> 5
    assert cl.tolist() == [0, 1, 0, 2, 3, 1, 4, 5]
    assert np.allclose(ov, [[0.6, 0.55, 0.5], [2.7, 0.5, 0.5], [1.5, 1.5, 0.5], [3.0, 0.5, 0.5], [4.5, 2.5, 0.5],
                            [1.2, 2.2, 0.5]], atol=1e-7, rtol=0)
    assert np.array_equal(ov[0], (v[0].astype(np.float64) + v[2]) / 2)       # the float64 mean
    assert np.array_equal(oc[1], (c[1] + c[5]) / 2)
    assert t.tolist() == [[0, 1, 2], [0, 2, 1], [1, 3, 4], [4, 3, 1]]


def test_cluster_keeps_first_rotation_and_isolated_vertex():
    v, f = hand_mesh()
    f2 = np.concatenate([f[[1]], f])             # now (1,3,0) comes first: its rotation (1,2,0) is the one kept
    _, t, _, cl = E.cluster(v, f2, resolution=4)
    assert t[0].tolist() == [1, 2, 0] and [0, 1, 2] not in t.tolist()
    sv, st, sc = E.simplify(v, f, None, resolution=4)
    assert sv.shape == (6, 3) and sc is None and st.dtype == np.int32
    assert np.array_equal(sv[5], v[7])                                       # the isolated vertex survives alone
    assert (cl == cl[7]).sum() == 1
    one = E.cluster(np.ones((3, 3), np.float32), np.array([[0, 1, 2]]))       # a single point: one voxel
    assert one[0].shape == (1, 3) and one[1].shape == (0, 3)


# ---------------------------------------------------------------- write_glb read back by the oracle
def _rig(rng, N=50, wide_rows=(3,)):
    W = np.zeros((30, 24), np.float32)
    for r in range(30):
        idx = rng.choice(24, 6 if r in wide_rows else 3, replace=False)
        W[r, idx] = rng.random(len(idx)) + 0.1
    W /= W.sum(1, keepdims=True)
    nearest = rng.integers(0, 30, N)
    nearest[0] = wide_rows[0]
    J = rng.normal(0, 0.3, (24, 3)).astype(np.float32)
    return dict(name="toy", vertices=rng.normal(0, 0.5, (N, 3)).astype(np.float32),
                triangles=rng.integers(0, N, (40, 3)).astype(np.int32), joints=J, nearest=nearest,
                colors=rng.random((N, 3)).astype(np.float32), lbs_weights=W,
                parents=np.asarray(D.olbs.SMPL_PARENTS, dtype=np.int64))


def test_write_glb_round_trip(tmp_path):
    from avatarclip_b200 import export as X
    rng = np.random.default_rng(0)
    rig = _rig(rng)
    motion = rng.normal(0, 0.8, (9, 75)).astype(np.float32)
    np.save(tmp_path / "m.npy", motion)
    path = X.write_glb(rig, str(tmp_path / "a.glb"), str(tmp_path / "m.npy"), fps=24)
    glb = E.read_glb(path)
    magic, version, length = glb["header"]
    assert magic == b"glTF" and version == 2 and length == glb["size"] == os.path.getsize(path)
    assert [c[0] for c in glb["chunks"]] == [0x4E4F534A, 0x004E4942]
    assert all(c[2] % 4 == 0 and c[1] % 4 == 0 for c in glb["chunks"])
    j = glb["json"]
    assert all(v.get("byteOffset", 0) % 4 == 0 for v in j["bufferViews"])
    prim = j["meshes"][0]["primitives"][0]
    pa = j["accessors"][prim["attributes"]["POSITION"]]
    assert pa["min"] == rig["vertices"].min(0).astype(np.float64).tolist()
    assert pa["max"] == rig["vertices"].max(0).astype(np.float64).tolist()
    assert np.array_equal(E.accessor(glb, prim["attributes"]["POSITION"]), rig["vertices"])
    assert np.array_equal(E.accessor(glb, prim["indices"]).reshape(-1, 3), rig["triangles"])
    sk = j["skins"][0]
    assert len(sk["joints"]) == 24 == j["accessors"][sk["inverseBindMatrices"]]["count"]
    assert [j["nodes"][n]["name"] for n in sk["joints"]][:2] == ["mixamorig:Hips", "mixamorig:LeftUpLeg"]
    # every non-zero weight, in two sets because vertex 0 has six influences
    assert "JOINTS_1" in prim["attributes"] and "JOINTS_2" not in prim["attributes"]
    W = rig["lbs_weights"][rig["nearest"]]
    got = np.zeros_like(W)
    for s in range(2):
        Js = E.accessor(glb, prim["attributes"][f"JOINTS_{s}"]).astype(np.int64)
        Ws = E.accessor(glb, prim["attributes"][f"WEIGHTS_{s}"])
        np.add.at(got, (np.arange(W.shape[0])[:, None].repeat(4, 1), Js), Ws)
    assert np.array_equal(got, W)
    assert np.abs(got.sum(1) - 1).max() <= 1e-6
    col = E.accessor(glb, prim["attributes"]["COLOR_0"])
    c = rig["colors"].astype(np.float64)
    assert np.allclose(col, np.where(c <= 0.04045, c / 12.92, ((c + 0.055) / 1.055) ** 2.4), atol=1e-7, rtol=0)
    # animation: 23 rotation channels, times k / fps strictly increasing, unit and sign-aligned quaternions
    an = j["animations"][0]
    assert len(an["channels"]) == 23 and all(ch["target"]["path"] == "rotation" for ch in an["channels"])
    assert sorted(ch["target"]["node"] - 1 for ch in an["channels"]) == list(range(1, 24))   # no root channel
    t = E.accessor(glb, an["samplers"][0]["input"])[:, 0]
    assert np.all(np.diff(t) > 0) and np.allclose(t, np.arange(9) / 24)
    for smp in an["samplers"]:
        assert smp["interpolation"] == "LINEAR"
        q = E.accessor(glb, smp["output"]).astype(np.float64)
        assert np.abs(np.linalg.norm(q, axis=1) - 1).max() <= 1e-6
        assert np.all((q[1:] * q[:-1]).sum(1) >= 0)
    # the keyed rotation is the motion's axis-angle
    q = E.accessor(glb, an["samplers"][4]["output"]).astype(np.float64)
    joint = an["channels"][4]["target"]["node"] - 1
    R = D.olbs.batch_rodrigues(torch.from_numpy(motion[:, 3 * joint:3 * joint + 3].astype(np.float64)))
    assert max(np.abs(E.quat_to_mat(q[k]) - R[k].numpy()).max() for k in range(9)) <= 1e-6


def test_write_glb_bind_pose_and_no_motion(tmp_path):
    from avatarclip_b200 import export as X
    rig = _rig(np.random.default_rng(1), wide_rows=(2,))
    rig["colors"] = None
    rig["lbs_weights"][2] = 0
    rig["lbs_weights"][2, :4] = 0.25                       # at most four influences: one weight set
    rig["nearest"][0] = 2
    path = X.write_glb(rig, str(tmp_path / "b.glb"))
    glb = E.read_glb(path)
    prim = glb["json"]["meshes"][0]["primitives"][0]
    assert "animations" not in glb["json"] and "COLOR_0" not in prim["attributes"]
    assert "JOINTS_1" not in prim["attributes"]
    assert np.abs(E.skin(glb) - rig["vertices"]).max() <= 1e-6          # G_j . IBM_j = I in the bind pose
    with pytest.raises(ValueError):
        X.write_glb(dict(rig, joints=rig["joints"][:23]), str(tmp_path / "c.glb"))


# ---------------------------------------------------------------- CLI and CPU tensors
def _npz(path, smpl, **override):
    arrs = {k: np.asarray(v) for k, v in smpl.items()}
    arrs.update(override)
    np.savez(path, **{k: v for k, v in arrs.items() if v is not None})
    return str(path)


def test_cli_rejections(smpl, tmp_path, capsys):
    from avatarclip_b200 import export as X
    a = X.build_parser().parse_args(["--mesh", "m.ply", "--smpl", "s.npz", "--stand_pose", "p.npy", "--out", "o.glb",
                                     "--motion", "a.npy", "--fps", "24"])
    assert (a.mesh, a.smpl, a.stand_pose, a.out, a.motion, a.fps, a.resolution) == \
        ("m.ply", "s.npz", "p.npy", "o.glb", "a.npy", 24.0, 256)
    (tmp_path / "m.ply").write_bytes(b"")
    (tmp_path / "p.npy").write_bytes(b"")
    ok = _npz(tmp_path / "ok.npz", smpl)
    np.save(tmp_path / "bad_motion.npy", np.zeros((4, 60), np.float32))
    base = ["--mesh", str(tmp_path / "m.ply"), "--stand_pose", str(tmp_path / "p.npy"), "--out", str(tmp_path / "o.glb")]
    cases = [
        (["--smpl", str(tmp_path / "nope.npz")], "--smpl: no such file"),
        (["--smpl", ok, "--motion", str(tmp_path / "nope.npy")], "--motion: no such file"),
        (["--smpl", _npz(tmp_path / "m.npz", smpl, J_regressor=None)], "missing"),
        (["--smpl", _npz(tmp_path / "w.npz", smpl, lbs_weights=np.zeros((6890, 23), np.float32))], "lbs_weights"),
        (["--smpl", ok, "--motion", str(tmp_path / "bad_motion.npy")], "--motion: "),
        (["--smpl", ok, "--fps", "0"], "--fps"),
        (["--smpl", ok, "--resolution", "0"], "--resolution"),
    ]
    for extra, msg in cases:
        with pytest.raises(SystemExit) as e:
            X.main(base + extra)
        assert e.value.code == 2 and msg in capsys.readouterr().err, extra
    with pytest.raises(SystemExit) as e:
        X.main(["--mesh", "m.ply"])
    assert e.value.code == 2
    assert not (tmp_path / "o.glb").exists()


def test_cpu_tensors_raise(g, smpl):
    from avatarclip_b200 import AvcError
    from avatarclip_b200 import drive
    from avatarclip_b200 import export as X
    m = g["mesh"]
    with pytest.raises(AvcError):
        X.simplify_mesh(drive.Mesh(m["v"], m["f"], None))
    with pytest.raises(AvcError):
        X.find_nearest_ind(m["v"], {"vertices": torch.zeros(1, 10, 3)})
    with pytest.raises(AvcError):
        X.rig_avatar("unused.ply", smpl, "unused.npy", device="cpu")
