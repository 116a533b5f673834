"""Mesh animation (drive.py) without a GPU: the CPU oracle against what the reference's own drive.py computed
(tests/golden/ref_drive_small.pt, recorded by oracle/pin_drive.py), the product's host-side pieces (PC2 writer, motion
decoding, SMPL .npz loader, CLI) and its refusal of CPU tensors."""
import io
import os

import numpy as np
import pytest
import torch

from oracle import drive as D

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_drive_small.pt")


@pytest.fixture(scope="module")
def g():
    return torch.load(GOLDEN, map_location="cpu", weights_only=False)


@pytest.fixture(scope="module")
def smpl(g):
    s = D.golden_smpl(g["smpl_seed"])
    # the golden stores the generator seed, not the 17 MB of tensors: make sure they are re-created bit for bit
    assert {k: float(v.double().sum()) for k, v in s.items()} == g["smpl_sums"]
    return s


def _stand(g):
    return np.load(io.BytesIO(g["stand_pose_npy"].numpy().tobytes()))


def _frames(pc2: bytes, V: int):
    return np.frombuffer(pc2[32:], dtype="<f4").reshape(-1, V, 3)


def test_oracle_reproduces_reference(g, smpl):
    m, r = g["mesh"], g["ref"]
    o = D.generate(m["v"].numpy(), m["f"].numpy(), m["c"].numpy(), smpl, _stand(g), g["motion"].numpy())
    assert np.array_equal(o["nearest"], r["nearest"].numpy())
    assert np.array_equal(o["cleaned_v"], r["cleaned_v"].numpy())
    assert np.array_equal(o["cleaned_f"], r["cleaned_f"].numpy())
    assert np.array_equal(o["cleaned_c"], r["cleaned_c"].numpy())
    assert len(o["keep_idx"]) == len(r["cleaned_v"]) < len(m["v"])         # the singletons and the small piece went
    assert (o["template"] - r["template"]).abs().max().item() <= 1e-6
    assert (o["tpose"] - r["tpose"]).abs().max().item() <= 1e-6
    V = len(r["cleaned_v"])
    pc2 = r["pc2"].numpy().tobytes()
    assert o["pc2"][:32] == pc2[:32]
    assert np.abs(_frames(o["pc2"], V) - _frames(pc2, V)).max() <= 1e-6


def test_oracle_cleanup_tie_keeps_smaller_minimum_index(g):
    t = g["tie"]
    idx, v, f, c = D.cleanup_mesh(t["v"].numpy(), t["f"].numpy(), t["c"].numpy())
    assert np.array_equal(v, t["cleaned_v"].numpy()) and np.array_equal(f, t["cleaned_f"].numpy())
    assert np.array_equal(c, t["cleaned_c"].numpy())
    lab = D.components(len(t["v"]), t["f"].numpy())
    roots, sizes = np.unique(lab, return_counts=True)
    tied = roots[sizes == sizes.max()]
    assert len(tied) == 2 and idx[0] == tied.min()


def test_write_pc2_bytes_equal_reference(g, tmp_path):
    from avatarclip_b200.drive import write_pc2
    pc2 = g["ref"]["pc2"].numpy().tobytes()
    frames = _frames(pc2, len(g["ref"]["cleaned_v"]))
    write_pc2(str(tmp_path / "a.pc2"), [torch.from_numpy(f.copy()) for f in frames])
    assert (tmp_path / "a.pc2").read_bytes() == pc2


def test_read_pose_my_matches_reference(g, tmp_path):
    from avatarclip_b200.drive import read_pose_my
    np.save(tmp_path / "action.npy", g["motion"].numpy())
    got = read_pose_my(str(tmp_path / "action.npy"))
    assert len(got) == 5 and tuple(got[0].shape) == (1, 24, 3, 3)
    assert (torch.cat(got) - g["ref"]["pose_list"]).abs().max().item() <= 1e-6
    with pytest.raises(ValueError):
        np.save(tmp_path / "bad.npy", np.zeros((4, 60), np.float32))
        read_pose_my(str(tmp_path / "bad.npy"))


def _npz(path, smpl, **override):
    arrs = {k: np.asarray(v) for k, v in smpl.items()}
    arrs.update(override)
    np.savez(path, **{k: v for k, v in arrs.items() if v is not None})
    return str(path)


def test_smpl_npz_loader(smpl, tmp_path):
    from avatarclip_b200.drive import SMPL_KEYS, load_smpl_npz
    d = load_smpl_npz(_npz(tmp_path / "ok.npz", smpl))
    assert set(SMPL_KEYS) <= set(d) and d["posedirs"].shape == (207, 6890 * 3)
    with pytest.raises(ValueError, match="missing"):
        load_smpl_npz(_npz(tmp_path / "m.npz", smpl, J_regressor=None))
    with pytest.raises(ValueError, match="posedirs"):
        load_smpl_npz(_npz(tmp_path / "p.npz", smpl, posedirs=np.zeros((207, 30), np.float32)))
    with pytest.raises(ValueError, match="lbs_weights"):
        load_smpl_npz(_npz(tmp_path / "w.npz", smpl, lbs_weights=np.zeros((6890, 23), np.float32)))
    with pytest.raises(ValueError, match="v_template"):
        load_smpl_npz(_npz(tmp_path / "v.npz", smpl, v_template=np.zeros((6890, 4), np.float32)))
    with pytest.raises(ValueError, match="J_regressor"):
        load_smpl_npz(_npz(tmp_path / "j.npz", smpl, J_regressor=np.zeros((40, 6890), np.float32)))
    bad_par = np.asarray(smpl["parents"]).copy()
    bad_par[5] = 7
    with pytest.raises(ValueError, match="parents"):
        load_smpl_npz(_npz(tmp_path / "t.npz", smpl, parents=bad_par))


def test_cli_parses_and_fails_cleanly_on_missing_files(tmp_path, capsys):
    from avatarclip_b200 import drive
    a = drive.build_parser().parse_args(["--mesh", "m.ply", "--motion", "a.npy", "--smpl", "s.npz", "--stand_pose",
                                         "p.npy", "--out_dir", "o", "--frames_per_chunk", "8"])
    assert (a.mesh, a.motion, a.smpl, a.stand_pose, a.out_dir, a.frames_per_chunk) == \
        ("m.ply", "a.npy", "s.npz", "p.npy", "o", 8)
    assert "smplx.build_layer" in drive.build_parser().format_help()
    (tmp_path / "m.ply").write_bytes(b"")
    with pytest.raises(SystemExit) as e:
        drive.main(["--mesh", str(tmp_path / "m.ply"), "--motion", str(tmp_path / "nope.npy"), "--smpl", "s.npz",
                    "--stand_pose", "p.npy", "--out_dir", str(tmp_path / "o")])
    assert e.value.code == 2 and "--motion: no such file" in capsys.readouterr().err
    with pytest.raises(SystemExit) as e:
        drive.main(["--mesh", "m.ply"])
    assert e.value.code == 2
    assert not (tmp_path / "o").exists()


def test_cpu_tensors_raise(g, smpl):
    from avatarclip_b200 import AvcError
    from avatarclip_b200 import drive
    m = drive.Mesh(g["mesh"]["v"], g["mesh"]["f"], None)
    with pytest.raises(AvcError):
        drive.cleanup_mesh(m)
    with pytest.raises(AvcError):
        drive.find_nearest_ind(g["ref"]["cleaned_v"], {"vertices": g["ref"]["template"][None]})
    w = smpl["lbs_weights"][g["ref"]["nearest"].long()]
    with pytest.raises(AvcError):
        drive.inv_lbs(smpl, g["ref"]["cleaned_v"], w, g["ref"]["pose_rot"], torch.zeros(1, 10))
    with pytest.raises(AvcError):
        drive.lbs(smpl, g["ref"]["tpose"], w, g["ref"]["pose_rot"], torch.zeros(1, 10))
    with pytest.raises(AvcError):
        drive.smpl_tensors(smpl, "cpu")
