"""AvatarAnimate's motion stage on the CPU: the oracle (oracle/motion.py) against what the reference computed
(tests/golden/ref_motion_small.pt), the 85 shipped AvatarAnimate confs as the motion command classifies them, and the
command line's argument handling, refusals and loader checks up to the point where the device is needed."""
import glob
import os
import tarfile

import numpy as np
import pytest
import torch

from oracle import animate as OA
from oracle import motion as OM

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden")


@pytest.fixture(scope="module")
def golden():
    return torch.load(os.path.join(GOLDEN, "ref_motion_small.pt"), map_location="cpu", weights_only=False)


@pytest.fixture(scope="module")
def confs(tmp_path_factory):
    d = tmp_path_factory.mktemp("motion_confs")
    with tarfile.open(os.path.join(GOLDEN, "ref_animate_confs.tar.gz")) as tf:
        tf.extractall(str(d), filter="data")
    return sorted(glob.glob(str(d / "confs" / "**" / "*.conf"), recursive=True))


def _rel(a, b):
    a, b = torch.as_tensor(a, dtype=torch.float64), torch.as_tensor(b, dtype=torch.float64)
    return float((a - b).abs().max() / b.abs().max())


def test_interpolation_oracle_vs_golden(golden):
    m = OM.interpolation_motion(golden["poses"], OM.vposer_encoder_state(), OA.vposer_state())
    assert golden["interpolation"].shape == (60, 69) and golden["interpolation"][:, 63:].abs().max() == 0
    assert _rel(m, golden["interpolation"][:, :63]) <= 1e-5


@pytest.mark.parametrize("run", ["delta0", "delta"])
def test_optimizer_oracle_vs_golden(golden, run):
    """The fp64 restatement follows the reference's losses, latent and motion over the pinned iterations."""
    r, c = golden["optimizer"][run], golden["optimizer_conf"][run]
    losses, z, motion = OM.optimize(OM.motion_vae_state(), golden["poses"], r["latent_init"], golden["num_iter"],
                                    c["recon_coef"], c["delta_coef"], lr=c["lr"])
    assert _rel(r["loss"], losses) <= 1e-5 and _rel(r["latent"], z) <= 1e-5
    assert _rel(r["motion"][:, :63], motion) <= 1e-4
    assert r["loss"][-1] < 0.5 * r["loss"][0]


def test_interpolate_is_sequential_fp32():
    from avatarclip_b200 import motion as M
    lat = np.random.default_rng(0).normal(size=(5, 32)).astype(np.float32)
    out = M.interpolate_latents(lat, (0, 14, 29, 44, 59), 60)
    ref = OM.interpolate(torch.from_numpy(lat), (0, 14, 29, 44, 59), 60, dtype=torch.float32).numpy()
    assert out.dtype == np.float32 and np.array_equal(out, ref)
    for i, a in enumerate((0, 14, 29, 44, 59)):
        assert np.abs(out[a] - lat[i]).max() <= 1e-5


def test_conf_classification(confs):
    """Of the 85 shipped confs the motion command runs the 24 motion_ablation interpolation / baseline ones."""
    from avatarclip_b200 import animate as A
    from avatarclip_b200 import conf
    from avatarclip_b200 import motion as M
    assert len(confs) == 85
    ok, refused = [], []
    for p in confs:
        c = conf.parse_file(p)
        why = M.refusal(c)
        (ok if why is None else refused).append((p, c, why))
        assert (A.refusal(c) is None) == (c.get_string("general.mode") == "pose" and
                                         A.pose_generator_refusal(c) is None)
    assert len(ok) == 24 and len(refused) == 61
    assert all("/motion_ablation/interpolation/" in p or "/motion_ablation/baseline/" in p for p, _, _ in ok)
    pose = [w for p, c, w in refused if c.get_string("general.mode") == "pose"]
    assert len(pose) == 48 and all("avatarclip_b200.animate" in w for w in pose)
    clip = [w for p, c, w in refused if c.get_string("general.mode") == "motion"]
    assert len(clip) == 13 and all("clip_coef" in w and "rasteriser's gradient" in w for w in clip)


def test_animate_refusal_names_the_motion_command(confs):
    from avatarclip_b200 import animate as A
    from avatarclip_b200 import conf
    motion = [conf.parse_file(p) for p in confs if "motion" in os.path.basename(os.path.dirname(p)) or "base.conf" in p]
    whys = [A.refusal(c) for c in motion if c.get_string("general.mode") == "motion"]
    assert whys and all("motion stage" in w and "avatarclip_b200.motion" in w for w in whys)


def test_in_scope_confs_build(confs, monkeypatch):
    from avatarclip_b200 import conf
    from avatarclip_b200 import motion as M
    seen = []
    monkeypatch.setattr(M, "load_motion_vae", lambda *a, **k: seen.append(("vae", a)))
    for p in confs:
        c = conf.parse_file(p)
        if M.refusal(c) is None:
            g = M.build_motion_generator(dict(c["motion_generator"]), vposer={}, device="cuda")
            assert type(g).__name__ == c["motion_generator"]["type"]
            if isinstance(g, M.MotionOptimizer):
                assert g.cfg["clip_coef"] == 0 and g.cfg["delta_coef"] == 0 and list(g.cfg["recon_coef"]) == [1.0] * 5
    assert len(seen) == 12
    with pytest.raises(NotImplementedError, match="rasteriser's gradient"):
        M.build_motion_generator({"type": "MotionOptimizer"}, {})
    with pytest.raises(KeyError):
        M.build_motion_generator({"type": "Nope"}, {})


@pytest.mark.parametrize("block, msg", [
    ("type = MotionOptimizer", "rasteriser's gradient"),
    ("type = MotionOptimizer\n    clip_coef = 0\n    optim_name = SGD", "only Adam"),
    ("type = MotionOptimizer\n    clip_coef = 0\n    optim_cfg {\n        lr = 0.1\n        momentum = 0.9\n    }",
     "not Adam's"),
    ("type = MotionInterpolation\n    anchor_position = [0, 30, 58]", "num_frame - 1"),
    ("type = MotionInterpolation\n    anchor_position = [1, 30, 59]", "start at 0")])
def test_cli_refuses_before_reading_files(tmp_path, capsys, block, msg):
    from avatarclip_b200 import motion as M
    conf = tmp_path / "m.conf"
    conf.write_text("general {\n    base_exp_dir = ./exp\n    mode = motion\n    text = a man\n}\n\npose_generator {\n"
                    f"    type = VPoserCodebook\n}}\n\nmotion_generator {{\n    {block}\n}}\n")
    with pytest.raises(SystemExit) as e:
        M.parse_args(["--conf", str(conf), "--smpl", "/nonexistent.npz"])
    assert e.value.code != 0 and msg in capsys.readouterr().err


def test_cli_refuses_other_modes_and_pose_generators(confs, capsys):
    from avatarclip_b200 import motion as M
    pose = [p for p in confs if "vposer_codebook" in p][0]
    with pytest.raises(SystemExit) as e:
        M.parse_args(["--conf", pose, "--smpl", "/nonexistent.npz"])
    assert e.value.code != 0 and "avatarclip_b200.animate" in capsys.readouterr().err


def test_cli_paths(confs, tmp_path, capsys):
    """An explicit flag wins over the conf's path, which wins over the reference's default."""
    from avatarclip_b200 import motion as M
    base = [p for p in confs if "/motion_ablation/baseline/" in p][0]
    interp = [p for p in confs if "/motion_ablation/interpolation/" in p][0]
    for n in ("smpl.npz", "uv.obj", "clip.pt", "bpe.gz", "cb.pth", "vae.pth", "conf_vae.pth"):
        (tmp_path / n).write_bytes(b"x")
    (tmp_path / "vp").mkdir()
    common = ["--smpl", str(tmp_path / "smpl.npz"), "--uv_obj", str(tmp_path / "uv.obj"), "--clip_model",
              str(tmp_path / "clip.pt"), "--bpe", str(tmp_path / "bpe.gz"), "--vposer", str(tmp_path / "vp"),
              "--codebook", str(tmp_path / "cb.pth")]
    a, c, pg, mg = M.parse_args(["--conf", base, "--motion_vae", str(tmp_path / "vae.pth")] + common)
    assert pg == {"type": "VPoserCodebook", "codebook_path": str(tmp_path / "cb.pth")}
    assert mg["type"] == "MotionOptimizer" and mg["ckpt_path"] == str(tmp_path / "vae.pth")
    a, c, pg, mg = M.parse_args(["--conf", interp] + common)
    assert mg == {"type": "MotionInterpolation"}
    with pytest.raises(SystemExit):
        M.parse_args(["--conf", base] + common)
    assert "ckpt_path: no such file: data/motion_vae.pth" in capsys.readouterr().err
    conf = tmp_path / "own.conf"
    conf.write_text(open(base).read().replace("clip_coef = 0.0", f"clip_coef = 0.0\n    ckpt_path = {tmp_path}/conf_vae.pth"))
    a, c, pg, mg = M.parse_args(["--conf", str(conf)] + common)
    assert mg["ckpt_path"] == str(tmp_path / "conf_vae.pth")
    a, c, pg, mg = M.parse_args(["--conf", str(conf), "--motion_vae", str(tmp_path / "vae.pth")] + common)
    assert mg["ckpt_path"] == str(tmp_path / "vae.pth")
    assert "motion_vae.pth" in M.build_parser().format_help()


def test_loader_refuses_a_missing_key():
    from avatarclip_b200 import motion as M
    sd = OM.motion_vae_state(latent=32, num_layers=2, n_out=132)
    del sd["decoder.seqTransDecoder.layers.1.norm2.bias"]
    with pytest.raises(ValueError, match=r"missing decoder\.seqTransDecoder\.layers\.1\.norm2\.bias"):
        M.load_motion_vae({"state_dict": sd}, latent_dim=32, num_layers=2, num_heads=2)
    sd = OM.motion_vae_state(latent=32, num_layers=2, n_out=132)
    with pytest.raises(ValueError, match="expected"):
        M.load_motion_vae(sd, latent_dim=64, num_layers=2, num_heads=2)


def test_vposer_loader_encoder_keys(tmp_path):
    from avatarclip_b200 import animate as A
    dec, enc = OA.vposer_state(), OM.vposer_encoder_state()
    sd = {"vp_model." + k: v for k, v in {**dec, **enc}.items()}
    assert set(A.load_vposer(sd)) == set(dec)
    got = A.load_vposer(sd, encoder=True)
    assert set(got) == set(dec) | set(A.VPOSER_ENCODER_KEYS) and set(A.VPOSER_ENCODER_KEYS) <= set(enc)
    with pytest.raises(ValueError, match="encoder_net"):
        A.load_vposer({"vp_model." + k: v for k, v in dec.items()}, encoder=True)


def test_positional_table_matches_oracle():
    from avatarclip_b200 import motion as M
    assert (M.positional_table(60, 256).double() - OM.positional_table(60, 256)).abs().max() <= 1e-5


def test_device_ops_refuse_cpu_tensors():
    from avatarclip_b200 import _lib
    from avatarclip_b200 import motion as M
    with pytest.raises(_lib.AvcError):
        M.vposer_encode(torch.zeros(2, 63), OM.vposer_encoder_state())
