"""Quadric-error decimation without a GPU: the fp64 oracle (oracle/decimate.py) keeps a closed manifold closed, keeps a
flat square's corners and boundary, stops a tetrahedron, never moves a non-manifold fan, and hits the target; the
export CLI refuses a bad --target_faces before any device work."""
import io
import os

import numpy as np
import pytest
import torch

from oracle import decimate as O
from oracle import drive as D

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_avatar2fbx_small.pt")


@pytest.fixture(scope="module")
def g():
    return torch.load(GOLDEN, map_location="cpu", weights_only=False)


def _closed_inputs(g):
    smpl = D.golden_smpl(g["smpl_seed"])
    stand = np.load(io.BytesIO(g["stand_pose_npy"].numpy().tobytes()))
    v, f = D.bench_mesh(smpl, stand, levels=1)
    return {"avatar": (v, f, 4000), "sphere": (*O.sphere(), 500)}


@pytest.mark.parametrize("name", ["avatar", "sphere"])
def test_closed_manifold_stays_closed(g, name):
    v, f, target = _closed_inputs(g)[name]
    before = O.topology(v, f)
    assert before["boundary_edges"] == 0 and before["nonmanifold_edges"] == 0 and before["misoriented_edges"] == 0
    r = O.decimate(v, f, target)
    after = O.topology(r["vertices"], r["faces"])
    assert r["faces"].shape[0] in (target - 1, target), r["faces"].shape
    assert after == before, (before, after)
    assert r["vertices"].shape[0] == np.unique(r["faces"]).size                 # no vertex left without a face
    print(f"[decimate] {name}: {f.shape[0]} -> {r['faces'].shape[0]} faces in {r['rounds']} rounds")


@pytest.mark.parametrize("target", [2, 7, 40, 101])
def test_flat_grid_keeps_its_square(target):
    n = 16
    v, f = O.grid(n)
    r = O.decimate(v, f, target)
    rv, rf = r["vertices"], r["faces"]
    assert rf.shape[0] in (target - 1, target)
    for c in ([0, 0, 0], [1, 0, 0], [0, 1, 0], [1, 1, 0]):
        assert (rv == np.array(c, np.float32)).all(1).any(), c
    assert (rv[:, 2] == 0).all() and (rv[:, :2] >= 0).all() and (rv[:, :2] <= 1).all()
    e = np.sort(np.concatenate([rf[:, [0, 1]], rf[:, [1, 2]], rf[:, [2, 0]]]), 1)
    u, cnt = np.unique(e, axis=0, return_counts=True)
    b = u[cnt == 1]
    length = np.linalg.norm(rv[b[:, 0]].astype(np.float64) - rv[b[:, 1]], axis=1).sum()
    assert abs(length - 4.0) <= 1e-6, length
    assert O.topology(rv, rf)["euler"] == 1


def test_tetrahedron_stops_at_four_faces():
    v, f = O.tetrahedron()
    r = O.decimate(v, f, 1)
    assert r["faces"].shape[0] == 4 and r["rounds"] == 0
    assert np.array_equal(r["faces"], f) and np.array_equal(r["vertices"], v)


def test_non_manifold_fan_never_moves():
    v, f, fan = O.fan(8)
    r = O.decimate(v, f, 12)
    rv, rf = r["vertices"], r["faces"]
    assert rf.shape[0] < f.shape[0] // 4 and r["rounds"] > 0
    # vertices keep their input order: the fan's 0 and 1 come first, its two page tips last, and none of them moves
    out = {0: 0, 1: 1, fan[2]: rv.shape[0] - 2, fan[3]: rv.shape[0] - 1}
    for x, k in out.items():
        assert rv[k].tobytes() == v[x].tobytes(), x
    rows = {tuple(t) for t in rf.tolist()}
    assert (0, 1, out[fan[2]]) in rows and (1, 0, out[fan[3]]) in rows        # the pages, still on edge (0, 1)
    assert O.topology(rv, rf)["nonmanifold_edges"] == 1


def test_at_or_below_target_is_the_input():
    v, f = O.sphere(12)
    r = O.decimate(v, f, f.shape[0])
    assert r["rounds"] == 0 and np.array_equal(r["faces"], f) and np.array_equal(r["vertices"], v)


def test_colours_interpolate_along_the_edge():
    v, f = O.sphere(16)
    c = np.random.default_rng(0).random(v.shape).astype(np.float32)
    r = O.decimate(v, f, 200, colors=c)
    assert r["colors"].shape == r["vertices"].shape
    assert r["colors"].min() >= c.min() and r["colors"].max() <= c.max()


def test_surface_distance_of_a_mesh_to_itself_is_the_sampling_error():
    v, f = O.sphere(20)
    d = O.surface_distance(v, f, v, f, spacing=0.02)
    assert d["mean"] < 0.02 and d["samples"] > 1000


def test_cli_refuses_a_bad_target_before_device_work(g, tmp_path, capsys):
    from avatarclip_b200 import export as X
    smpl = D.golden_smpl(g["smpl_seed"])
    np.savez(tmp_path / "smpl.npz", **{k: np.asarray(x) for k, x in smpl.items()})
    stand = tmp_path / "stand_pose.npy"
    stand.write_bytes(g["stand_pose_npy"].numpy().tobytes())
    (tmp_path / "m.ply").write_bytes(b"ply\n")
    base = ["--smpl", str(tmp_path / "smpl.npz"), "--stand_pose", str(stand), "--out", str(tmp_path / "o.glb"),
            "--device", "cpu"]
    for argv, msg in ((["--mesh", str(tmp_path / "m.ply"), "--target_faces", "0"], "--target_faces must be >= 1"),
                      (["--mesh", str(tmp_path / "m.ply"), "--target_faces", "-3"], "--target_faces must be >= 1"),
                      (["--mesh", str(tmp_path / "none.ply"), "--target_faces", "100"], "no such file")):
        with pytest.raises(SystemExit) as e:
            X.main(argv + base)
        assert e.value.code == 2 and msg in capsys.readouterr().err
    assert not (tmp_path / "o.glb").exists()
    with pytest.raises(ValueError, match="target_faces"):
        X.export_avatar(str(tmp_path / "m.ply"), str(tmp_path / "o.glb"), smpl, str(stand), target_faces=0)


def test_decimate_mesh_refuses_cpu_tensors():
    from avatarclip_b200 import _lib
    from avatarclip_b200 import export as X
    from avatarclip_b200.drive import Mesh
    v, f = O.tetrahedron()
    with pytest.raises(_lib.AvcError, match="no CPU path"):
        X.decimate_mesh(Mesh(torch.from_numpy(v), torch.from_numpy(f.astype(np.int32))), 2)
