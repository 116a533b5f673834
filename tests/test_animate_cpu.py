"""AvatarAnimate's pose stage on the CPU: the fp64 oracle (oracle/animate.py) against what the reference computed
(tests/golden/ref_animate_small.pt), matrot2aa's edge cases against an independent route, the 85 shipped AvatarAnimate
confs, and the command line's argument handling up to the point where the device is needed."""
import glob
import math
import os
import tarfile

import numpy as np
import pytest
import torch
from scipy.spatial.transform import Rotation

from oracle import animate as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")


@pytest.fixture(scope="module")
def golden():
    return torch.load(os.path.join(GOLDEN, "ref_animate_small.pt"), map_location="cpu", weights_only=False)


@pytest.fixture(scope="module")
def confs(tmp_path_factory):
    d = tmp_path_factory.mktemp("animate_confs")
    with tarfile.open(os.path.join(GOLDEN, "ref_animate_confs.tar.gz")) as tf:
        tf.extractall(str(d), filter="data")
    return sorted(glob.glob(str(d / "confs" / "**" / "*.conf"), recursive=True))


def test_codebook_oracle_vs_golden(golden):
    cb = golden["codebook"]
    book = O.make_codebook(golden["text_feature"])
    cos = O.cosine(book["codebook_embedding"], golden["text_feature"])
    assert np.abs(cos - cb["cos"].numpy()).max() <= 1e-12
    top = np.argsort(-cos, kind="stable")[:40]
    assert top.tolist() == cb["topk"].tolist()
    srt = np.sort(cos)[::-1]
    assert np.min(srt[:40] - srt[1:41]) > 1e-3              # no ties for the top-40
    poses, _ = O.vposer_decode(book["codebook"][top], O.vposer_state())
    keep = O.suppress(poses.reshape(40, -1), 0.07)
    assert keep[:5] == cb["keep"].tolist() and len(keep) < 40
    assert np.abs(poses.reshape(40, -1)[keep[:5]] - cb["poses"].numpy()).max() <= 1e-5


def test_realnvp_oracle_vs_golden(golden):
    """Each candidate the reference kept is one of the oracle's decodes of that candidate's prior draws."""
    nv = golden["realnvp"]
    sd = O.realnvp_state()
    decoded = []
    for z in nv["z"]:
        x = O.realnvp_decode(z, golden["text_feature"], sd)
        decoded.append(O.vposer_decode(x, O.vposer_state())[0].reshape(len(x), -1))
    for p in nv["poses"].numpy():
        assert min(np.abs(d - p).max(axis=1).min() for d in decoded) <= 1e-5
    c = golden["realnvp_conf"]
    assert nv["z"].shape == (c["topk"], c["num_batch"] * c["num_sample"], 32)
    assert nv["eyes"].shape == (5 * (c["topk"] * c["num_batch"] + c["topk"]), 3)
    # the numpy elevation stream: one randn per camera per scoring call, in the reference's order
    np.random.seed(golden["np_seed"])
    for k, e in enumerate(nv["eyes"].numpy()):
        ref = O.eye(np.random.randn() * 0.3, O.ANGLES[k % 5])
        assert np.abs(np.asarray(ref) - e).max() <= 1e-6      # stored as float32


def _aa_route(R):
    return Rotation.from_matrix(R).as_rotvec()


@pytest.mark.parametrize("case", ["identity", "tiny", "near_pi_x", "near_pi_y", "near_pi_z", "pi_xy", "general"])
def test_matrot2aa_edge_cases(case):
    vecs = {"identity": [0.0, 0.0, 0.0], "tiny": [1e-7, -2e-7, 3e-8], "near_pi_x": [math.pi - 1e-4, 0.0, 0.0],
            "near_pi_y": [0.0, math.pi - 1e-5, 0.0], "near_pi_z": [0.0, 0.0, math.pi - 1e-3],
            "pi_xy": list(np.array([1.0, 1.0, 0.0]) / math.sqrt(2) * (math.pi - 1e-6)), "general": [0.3, -1.2, 0.7]}
    R = Rotation.from_rotvec(vecs[case]).as_matrix()
    aa = O.matrot2aa(R[None])[0]
    # the same rotation (angle-axis is unique up to the antipodal pair at pi)
    assert np.abs(Rotation.from_rotvec(aa).as_matrix() - R).max() <= 1e-9
    if np.linalg.norm(vecs[case]) < math.pi - 1e-3:
        assert np.abs(aa - _aa_route(R)).max() <= 1e-9


def test_matrot2aa_covers_every_quaternion_branch():
    """Rotations chosen so that rotation_matrix_to_quaternion takes each of its four branches."""
    cases = {0: [math.pi * 0.9, 0.1, 0.0], 1: [0.1, math.pi * 0.9, 0.0], 2: [0.0, 0.3, math.pi * 0.9], 3: [0.2, 0.1, 0.3]}
    for branch, v in cases.items():
        R = Rotation.from_rotvec(v).as_matrix()
        m = R.T
        got = (0 if m[0, 0] > m[1, 1] else 1) if m[2, 2] < 1e-6 else (2 if m[0, 0] < -m[1, 1] else 3)
        assert got == branch
        assert np.abs(O.matrot2aa(R[None])[0] - np.asarray(v)).max() <= 1e-9


def test_rot6d_gram_schmidt():
    x = np.random.default_rng(0).normal(size=(50, 6))
    R = O.rot6d_to_matrix(x)
    assert np.abs(R @ np.transpose(R, (0, 2, 1)) - np.eye(3)).max() <= 1e-12
    assert np.abs(np.linalg.det(R) - 1).max() <= 1e-12
    a = x.reshape(-1, 3, 2)[:, :, 0]
    assert np.abs(R[:, :, 0] - a / np.linalg.norm(a, axis=1, keepdims=True)).max() <= 1e-12


def test_all_shipped_confs_parse_and_are_classified(confs):
    from avatarclip_b200 import animate as A
    from avatarclip_b200 import conf
    assert len(confs) == 85
    ok, refused = [], []
    for p in confs:
        c = conf.parse_file(p)
        why = A.refusal(c)
        (ok if why is None else refused).append((p, c, why))
    assert len(ok) == 24 and len(refused) == 61
    assert all(c["pose_generator"]["type"] in A.IN_SCOPE and "/pose_ablation/" in p for p, c, _ in ok)
    motion = [w for p, c, w in refused if c.get_string("general.mode") == "motion"]
    assert len(motion) == 37 and all("motion stage" in w for w in motion)
    opt = [w for p, c, w in refused if c.get_string("general.mode") == "pose"]
    assert len(opt) == 24 and all("gradient" in w for w in opt)


def test_in_scope_confs_build(confs, monkeypatch):
    """The 24 in-scope confs reach their generator's constructor with the reference's kwargs."""
    from avatarclip_b200 import animate as A
    from avatarclip_b200 import conf
    seen = []
    monkeypatch.setattr(A.VPoserCodebook, "__init__", lambda self, **kw: seen.append(("C", kw)))
    monkeypatch.setattr(A.VPoserRealNVP, "__init__", lambda self, **kw: seen.append(("R", kw)))
    for p in confs:
        c = conf.parse_file(p)
        if A.refusal(c) is None:
            A.build_pose_generator(dict(c["pose_generator"]), assets=None)
    assert len(seen) == 24 and {k for k, _ in seen} == {"C", "R"}
    assert all(set(kw) == {"name", "assets"} for _, kw in seen)
    with pytest.raises(NotImplementedError):
        A.build_pose_generator({"type": "PoseOptimizer"}, None)
    with pytest.raises(KeyError):
        A.build_pose_generator({"type": "Nope"}, None)


def test_cli_refuses_before_reading_files(confs, capsys):
    from avatarclip_b200 import animate as A
    motion = [p for p in confs if "motion_ablation" in p][0]
    optim = [p for p in confs if "pose_optimizer" in p][0]
    for p, msg in ((motion, "motion stage"), (optim, "PoseOptimizer")):
        with pytest.raises(SystemExit) as e:
            A.parse_args(["--conf", p, "--smpl", "/nonexistent.npz"])
        assert e.value.code != 0 and msg in capsys.readouterr().err
    with pytest.raises(SystemExit):
        A.parse_args(["--conf", "/nonexistent.conf", "--smpl", "x"])


def test_cli_paths(confs, tmp_path, capsys):
    from avatarclip_b200 import animate as A
    cb = [p for p in confs if "vposer_codebook" in p][0]
    nvp = [p for p in confs if "vposer_realnvp" in p][0]
    files = {n: tmp_path / n for n in ("smpl.npz", "uv.obj", "clip.pt", "bpe.gz", "cb.pth", "nvp.pth")}
    for f in files.values():
        f.write_bytes(b"x")
    (tmp_path / "vp").mkdir()
    common = ["--smpl", str(files["smpl.npz"]), "--uv_obj", str(files["uv.obj"]), "--clip_model",
              str(files["clip.pt"]), "--bpe", str(files["bpe.gz"]), "--vposer", str(tmp_path / "vp")]
    a, c, pg = A.parse_args(["--conf", cb, "--codebook", str(files["cb.pth"])] + common)
    assert pg == {"type": "VPoserCodebook", "codebook_path": str(files["cb.pth"])}
    a, c, pg = A.parse_args(["--conf", nvp, "--realnvp", str(files["nvp.pth"])] + common)
    assert pg == {"type": "VPoserRealNVP", "ckpt_path": str(files["nvp.pth"])}
    with pytest.raises(SystemExit):
        A.parse_args(["--conf", nvp, "--realnvp", str(tmp_path / "missing.pth")] + common)
    assert "ckpt_path: no such file" in capsys.readouterr().err
    assert "pose_realnvp.pth" in A.build_parser().format_help()


def test_vposer_loader_layouts(tmp_path):
    from avatarclip_b200 import animate as A
    sd = O.vposer_state()
    os.makedirs(tmp_path / "vp" / "snapshots")
    torch.save({"state_dict": {"vp_model." + k: v for k, v in sd.items()}},
               tmp_path / "vp" / "snapshots" / "V02_05_epoch=08_val_loss=0.03.ckpt")
    got = A.load_vposer(str(tmp_path / "vp"))
    assert set(got) == set(sd) and all(torch.equal(got[k], sd[k]) for k in sd)
    with pytest.raises(FileNotFoundError):
        A.load_vposer(str(tmp_path))
    with pytest.raises(ValueError):
        A.load_vposer({"decoder_net.0.weight": sd["decoder_net.0.weight"]})


def test_write_candidates(tmp_path):
    from avatarclip_b200 import animate as A
    poses = torch.randn(3, 63)
    imgs = np.zeros((3, 512, 512, 3), np.uint8)
    files = A.write_candidates(str(tmp_path / "out"), poses, imgs)
    assert len(files) == 6
    p = np.load(tmp_path / "out" / "candidate_2.npy")
    assert p.dtype == np.float32 and p.shape == (63,) and np.array_equal(p, poses[2].numpy())


def test_device_ops_refuse_cpu_tensors():
    from avatarclip_b200 import _lib
    from avatarclip_b200 import animate as A
    with pytest.raises(_lib.AvcError):
        A.cosine_topk(torch.zeros(4, 8), torch.ones(8), 2)
    with pytest.raises(_lib.AvcError):
        A.pose_suppress(torch.zeros(4, 63), 0.07)


def test_cli_path_precedence(tmp_path):
    """An explicit flag wins over a path in the conf, which wins over the reference's default."""
    from avatarclip_b200 import animate as A
    for n in ("smpl.npz", "uv.obj", "clip.pt", "bpe.gz", "conf_cb.pth", "flag_cb.pth"):
        (tmp_path / n).write_bytes(b"x")
    (tmp_path / "vp_conf").mkdir()
    (tmp_path / "vp_flag").mkdir()
    conf = tmp_path / "cb.conf"
    conf.write_text("general {\n    base_exp_dir = ./exp\n    mode = pose\n    text = a man\n}\n\npose_generator {\n"
                    f"    type = VPoserCodebook\n    codebook_path = {tmp_path / 'conf_cb.pth'}\n"
                    f"    vposer_path = {tmp_path / 'vp_conf'}\n}}\n")
    common = ["--conf", str(conf), "--smpl", str(tmp_path / "smpl.npz"), "--uv_obj", str(tmp_path / "uv.obj"),
              "--clip_model", str(tmp_path / "clip.pt"), "--bpe", str(tmp_path / "bpe.gz")]
    a, _, pg = A.parse_args(common)
    assert pg["codebook_path"] == str(tmp_path / "conf_cb.pth") and a.vposer == str(tmp_path / "vp_conf")
    assert "vposer_path" not in pg
    a, _, pg = A.parse_args(common + ["--codebook", str(tmp_path / "flag_cb.pth"), "--vposer", str(tmp_path / "vp_flag")])
    assert pg["codebook_path"] == str(tmp_path / "flag_cb.pth") and a.vposer == str(tmp_path / "vp_flag")
