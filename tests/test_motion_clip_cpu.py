"""MotionOptimizer with its CLIP term on the CPU: the 85 shipped AvatarAnimate confs as the motion_clip command
classifies them, its refusals before any file is read, and the host side of the loop against what the reference
computed (tests/golden/ref_motion_clip_small.pt): the draw order and Adam on the recorded gradients."""
import glob
import os
import re
import tarfile
import types

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")
MOTION_CMD = re.compile(r"avatarclip_b200\.motion(?![_\w])")


@pytest.fixture(scope="module")
def golden():
    return torch.load(os.path.join(GOLDEN, "ref_motion_clip_small.pt"), map_location="cpu", weights_only=False)


@pytest.fixture(scope="module")
def confs(tmp_path_factory):
    d = tmp_path_factory.mktemp("motion_clip_confs")
    with tarfile.open(os.path.join(GOLDEN, "ref_animate_confs.tar.gz")) as tf:
        tf.extractall(str(d), filter="data")
    return sorted(glob.glob(str(d / "confs" / "**" / "*.conf"), recursive=True))


def test_conf_classification(confs):
    """Of the 85 shipped confs the command runs base.conf and the 12 motion_optimizer ones; every other conf is refused
    with the command that runs it."""
    from avatarclip_b200 import conf
    from avatarclip_b200 import motion as M
    from avatarclip_b200 import motion_clip as MC
    assert len(confs) == 85
    ok, refused = [], []
    for p in confs:
        c = conf.parse_file(p)
        why = MC.refusal(c)
        (ok if why is None else refused).append((p, c, why))
        if why is None:         # exactly the confs the motion command refuses for their CLIP term
            assert "clip_coef" in M.refusal(c) and "avatarclip_b200.motion_clip" in M.refusal(c)
    assert len(ok) == 13
    assert sorted(os.path.basename(p) for p, _, _ in ok if "/motion_optimizer/" not in p) == ["base.conf"]
    pose = [w for p, c, w in refused if c.get_string("general.mode") == "pose"]
    assert len(pose) == 48 and all("avatarclip_b200.animate" in w and "avatarclip_b200.pose_optimizer" in w
                                   for w in pose)
    motion = [(p, w) for p, c, w in refused if c.get_string("general.mode") == "motion"]
    assert len(motion) == 24 and all(("/baseline/" in p or "/interpolation/" in p) and MOTION_CMD.search(w)
                                     for p, w in motion)
    assert all(M.refusal(conf.parse_file(p)) is None for p, _ in motion)


@pytest.mark.parametrize("block, msg", [
    ("type = MotionOptimizer\n    clip_coef = 0.0", "avatarclip_b200.motion "),
    ("type = MotionInterpolation", "avatarclip_b200.motion"),
    ("type = MotionOptimizer\n    optim_name = SGD", "only Adam"),
    ("type = MotionOptimizer\n    optim_cfg {\n        lr = 0.1\n        momentum = 0.9\n    }", "not Adam's"),
    ("type = MotionOptimizer\n    clip_num_part = 61", "empty batch"),
    ("type = MotionOptimizer\n    num_frame = 20\n    clip_num_part = 30", "empty batch"),
    ("type = Nope", "unknown")])
def test_cli_refuses_before_reading_files(tmp_path, capsys, block, msg):
    from avatarclip_b200 import motion_clip as MC
    conf = tmp_path / "m.conf"
    conf.write_text("general {\n    base_exp_dir = ./exp\n    mode = motion\n    text = a man\n}\n\npose_generator {\n"
                    f"    type = VPoserCodebook\n}}\n\nmotion_generator {{\n    {block}\n}}\n")
    with pytest.raises(SystemExit) as e:
        MC.parse_args(["--conf", str(conf), "--smpl", "/nonexistent.npz"])
    err = capsys.readouterr().err
    assert e.value.code != 0 and msg in err and "--smpl" not in err.split("error:")[-1]


def test_cli_refuses_pose_confs_and_reads_files_last(confs, tmp_path, capsys):
    from avatarclip_b200 import motion_clip as MC
    for pose in ([p for p in confs if "vposer_codebook" in p][0], [p for p in confs if "/pose_optimizer/" in p][0]):
        with pytest.raises(SystemExit) as e:
            MC.parse_args(["--conf", pose, "--smpl", "/nonexistent.npz"])
        err = capsys.readouterr().err
        assert e.value.code != 0 and "avatarclip_b200.animate" in err and "no such file" not in err
    base = [p for p in confs if p.endswith("/base.conf")][0]
    with pytest.raises(SystemExit):                # a runnable conf: now the files are checked
        MC.parse_args(["--conf", base, "--smpl", "/nonexistent.npz"])
    assert "codebook_path: no such file" in capsys.readouterr().err


def test_cli_paths(confs, tmp_path):
    from avatarclip_b200 import motion_clip as MC
    base = [p for p in confs if "/motion_ablation/motion_optimizer/" in p][0]
    for n in ("smpl.npz", "uv.obj", "clip.pt", "bpe.gz", "cb.pth", "vae.pth"):
        (tmp_path / n).write_bytes(b"x")
    (tmp_path / "vp").mkdir()
    a, c, pg, mg = MC.parse_args(["--conf", base, "--motion_vae", str(tmp_path / "vae.pth"), "--smpl",
                                  str(tmp_path / "smpl.npz"), "--uv_obj", str(tmp_path / "uv.obj"), "--clip_model",
                                  str(tmp_path / "clip.pt"), "--bpe", str(tmp_path / "bpe.gz"), "--vposer",
                                  str(tmp_path / "vp"), "--codebook", str(tmp_path / "cb.pth")])
    assert pg == {"type": "VPoserCodebook", "codebook_path": str(tmp_path / "cb.pth")}
    assert mg == {"type": "MotionOptimizer", "ckpt_path": str(tmp_path / "vae.pth")}
    assert "motion_clip" in MC.build_parser().format_help()


def test_generators_build_with_the_reference_defaults(confs, monkeypatch):
    from avatarclip_b200 import conf
    from avatarclip_b200 import motion as M
    from avatarclip_b200 import motion_clip as MC
    seen = []
    monkeypatch.setattr(M, "load_motion_vae", lambda *a, **k: seen.append(a))
    assets = types.SimpleNamespace(device="cuda")
    for p in confs:
        c = conf.parse_file(p)
        if MC.refusal(c) is None:
            g = MC.build_motion_generator(dict(c["motion_generator"]), assets)
            assert isinstance(g, MC.MotionOptimizer) and g.cfg == M.OPTIMIZER_DEFAULTS
    assert len(seen) == 13
    with pytest.raises(NotImplementedError, match="avatarclip_b200.motion "):
        MC.build_motion_generator({"type": "MotionOptimizer", "clip_coef": 0.0}, assets)
    with pytest.raises(KeyError):
        MC.build_motion_generator({"type": "MotionInterpolation"}, assets)
    with pytest.raises(NotImplementedError, match="rasteriser's gradient"):     # the motion command still refuses
        M.build_motion_generator({"type": "MotionOptimizer"}, {})


def test_clip_rows():
    from avatarclip_b200 import motion_clip as MC
    for T in range(1, 65):
        for P in range(1, T + 1):
            assert MC.clip_rows(T, P) == max(len(range(st, T, P)) for st in range(P))


@pytest.mark.parametrize("run", ["shipped", "clip_only"])
def test_draw_order_vs_golden(golden, run):
    """Seeding numpy as the reference run was seeded, the host's up-front draws are its st_idx and elevations."""
    from avatarclip_b200 import motion_clip as MC
    r, c = golden["runs"][run], golden["conf"][run]
    np.random.seed(golden["np_seed"])
    st, el = MC.draw_iterations(golden["num_iter"], c["clip_num_part"])
    assert np.array_equal(st, r["st_idx"].numpy()) and np.array_equal(el, r["elevation"].numpy())
    assert r["rows"].tolist() == [MC.clip_rows(60, c["clip_num_part"])] * golden["num_iter"]


@pytest.mark.parametrize("run", ["shipped", "clip_only"])
def test_adam_on_recorded_gradients_vs_golden(golden, run):
    r = golden["runs"][run]
    assert r["optim_cfg"] == {"lr": golden["conf"][run]["lr"]}
    z = torch.nn.Parameter(r["latent_init"].clone())
    opt = torch.optim.Adam([z], **r["optim_cfg"])
    for i, g in enumerate(r["grads"]):
        assert torch.equal(z.detach(), r["params"][i])
        z.grad = g.clone()
        opt.step()
    assert torch.equal(z.detach(), r["latent"])
    assert r["motion"].shape == (60, 69) and r["motion"][:, 63:].abs().max() == 0
