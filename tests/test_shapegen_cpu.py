"""ShapeGen without a GPU: the fp64 oracle against what the reference's own shape_gen computed
(tests/golden/ref_shapegen_small.pt, recorded by oracle/pin_shapegen.py), the OBJ format, parse_prompt, analytic cases
of the textured rasteriser, the SMPL .npz loader and the command line."""
import math
import os

import numpy as np
import pytest
import torch

from oracle import drive as D
from oracle import shapegen as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "ref_shapegen_small.pt")


@pytest.fixture(scope="module")
def golden():
    return torch.load(GOLDEN, map_location="cpu", weights_only=False)


def test_golden_is_small_and_records_a_robust_choice(golden):
    assert os.path.getsize(GOLDEN) < 1 << 20
    cos = golden["cos"].numpy()
    top = np.sort(cos)[::-1]
    assert golden["best"] == int(np.argmax(cos)) == O.CODEBOOK_WINNER
    assert top[0] - top[1] >= 0.05


def test_oracle_matches_the_reference_shape_gen(golden):
    tv, tf = D.template_obj()
    vae = O.vae_state(tv)
    dec = lambda z: O.vae_decode(z, vae["dec1.weight"], vae["dec1.bias"], vae["dec2.weight"], vae["dec2.bias"], tv)
    assert np.abs(dec(torch.zeros(1, 16)).reshape(-1, 3) - golden["zero_beta_v"].numpy()).max() < 1e-5
    best = golden["best"]
    assert np.abs(dec(golden["codebook_latents"][best]).reshape(-1, 3) - golden["v"].numpy()).max() < 1e-5
    cos = O.codebook_cos(golden["codebook_emb"], golden["image_embed"], golden["delta_embed"])
    assert np.abs(cos - golden["cos"].numpy()).max() < 1e-6


def test_oracle_render_matches_the_reference(golden, tmp_path):
    tv, tf = D.template_obj()
    vae = O.vae_state(tv)
    v0 = O.vae_decode(torch.zeros(1, 16), vae["dec1.weight"], vae["dec1.bias"], vae["dec2.weight"], vae["dec2.bias"], tv)
    tex = O.load_obj_textures(O.write_uv_obj(str(tmp_path), tv, tf))
    eye = (2 * math.sin(math.radians(150)), 0.0, -2 * math.cos(math.radians(150)))
    img = O.raster_textured(v0.reshape(-1, 3), tf, tex, eye)
    ref = golden["neutral_image"].float().permute(1, 2, 0).numpy()       # stored as fp16
    assert np.abs(img - ref).max() < 1e-3
    assert (img.sum(-1) > 0).mean() > 0.05                               # the body covers part of the image
    assert len(np.unique(np.round(img[img.sum(-1) > 0], 2), axis=0)) > 100   # ... and it is textured


def test_write_obj_is_byte_identical_and_reads_back(golden, tmp_path):
    from avatarclip_b200 import shapegen as S
    small = golden["small_obj"]
    path = tmp_path / "small.obj"
    S.writeOBJ(str(path), small["v"].numpy(), small["f"].numpy())
    assert path.read_text() == small["text"]
    V, F, Vt, Ft = S.readOBJ(str(path))
    assert np.array_equal(V, small["v"].numpy()) and F == small["f"].tolist() and Vt is None and Ft is None
    S.writeOBJ(str(path), V, F, Vt=np.array([[0.25, 0.5]] * 3, np.float32), Ft=[[0, 1, 2]] * 3)
    V2, F2, Vt2, Ft2 = S.readOBJ(str(path))
    assert np.array_equal(V2, V) and F2 == F and Ft2 == [[0, 1, 2]] * 3 and Vt2.shape == (3, 2)
    assert "f 1/1 2/2 3/3\n" in path.read_text()


def test_parse_prompt_matches_the_reference(golden):
    from avatarclip_b200 import shapegen as S
    assert len(golden["parse_prompt"]) >= 5
    for prompt, want in golden["parse_prompt"].items():
        got = S.parse_prompt(prompt)
        assert got[0] == want[0] and got[1:] == want[1:], prompt
    assert S.parse_prompt("plain")[1:] == (1.0, -math.inf)
    with pytest.raises(ValueError):
        S.parse_prompt("a:b:c:d")                    # the reference raises on a non-numeric weight too


def _constant_cubes(F, colour, R=8):
    return np.broadcast_to(np.asarray(colour, dtype=np.float64), (F, R, R, R, 3)).copy()


def test_raster_constant_texture_is_colour_times_light():
    """A constant-colour texture renders colour * (0.5 + 0.5 cos(normal, +y)): a triangle facing +y is fully lit, one
    tilted by 60 degrees gets 0.75, a vertical one 0.5."""
    colour = (0.8, 0.4, 0.2)
    for tilt, light in ((0.0, 1.0), (60.0, 0.75), (90.0, 0.5)):
        t = math.radians(tilt)
        # a triangle around the origin whose normal is (sin t, cos t, 0)
        ex, ey = np.array([math.cos(t), -math.sin(t), 0.0]), np.array([0.0, 0.0, 1.0])
        v = np.stack([-0.6 * ex - 0.6 * ey, 0.6 * ex - 0.6 * ey, 0.6 * ey])
        img = O.raster_textured(v, [[0, 1, 2]], _constant_cubes(1, colour), eye=(1.0, 1.2, 1.6), n=64)
        covered = img.sum(-1) > 0
        assert covered.mean() > 0.02
        full = img[covered]
        want = np.asarray(colour) * light
        # pixels whose four supersamples all hit the triangle carry exactly colour * light
        inner = np.isclose(full, want, atol=1e-12).all(1)
        assert inner.mean() > 0.6
        assert (full <= want + 1e-12).all()


def test_raster_empty_view_and_behind_camera():
    v, f = D.template_obj()
    cubes = _constant_cubes(len(f), (1.0, 1.0, 1.0))
    away = O.raster_textured(v, f, cubes, eye=(0.0, 0.0, 2.0), at=(0.0, 0.0, 4.0), n=32)
    assert not away.any()


def test_texture_cube_samples_the_flipped_image_at_normalised_barycentrics():
    img = np.random.default_rng(0).uniform(0, 1, (5, 7, 3)).astype(np.float32)
    tri = np.array([[0.0, 0.0], [0.75, 0.0], [0.0, 0.5]], np.float32)
    uv = np.stack([tri, tri + [1.0, -2.0], tri])                # face 1: the same triangle one / two periods away
    tex = O.load_textures(img, uv, np.array([1, 1, 0]), np.ones((3, 8, 8, 8, 3)))
    assert (tex[2] == 1.0).all()                                 # not this material: untouched
    assert np.allclose(tex[1], tex[0], atol=1e-12)               # REPEAT
    f = img[::-1].astype(np.float64)
    assert np.allclose(tex[0, 0, 0, 0], f[0, 0])                 # (0, 0, 0): the first corner, uv (0, 0)
    assert np.allclose(tex[0, 7, 0, 0], f[0, 0])                 # barycentric (1, 0, 0)
    assert np.allclose(tex[0, 0, 7, 0], 0.5 * (f[0, 4] + f[0, 5]))   # (0, 1, 0): uv (0.75, 0) -> x = 4.5
    assert np.allclose(tex[0, 0, 0, 7], f[2, 0])                 # (0, 0, 1): uv (0, 0.5) -> y = 2 of the flipped image
    assert np.allclose(tex[0, 0, 7, 7], 0.75 * f[1, 2] + 0.25 * f[1, 3])   # uv (0.375, 0.25) -> (2.25, 1)
    assert np.allclose(tex[0, 2, 2, 2], tex[0, 7, 7, 7])         # (i, j, k) / (i + j + k)


def test_uv_obj_reader_agrees_with_the_oracle(tmp_path):
    from avatarclip_b200 import shapegen as S
    tv, tf = D.template_obj()
    obj = O.write_uv_obj(str(tmp_path), tv[:50], tf[:40])
    uv, mats, images = S.read_uv_obj(obj)
    ouv, omats, oimages = O.read_uv_obj(obj)
    assert np.array_equal(uv, ouv) and mats == omats and images == oimages
    assert set(images) == {"skin", "cloth"} and set(mats) == {"skin", "cloth", "bare"}


def _write_smpl_npz(path, with_faces=True, V=60):
    from oracle import lbs as olbs
    d = {k: v.numpy() for k, v in olbs.synthetic_smpl(V=V, seed=2).items() if k in D.SMPL_KEYS}
    d["v_template"] = olbs.synthetic_smpl(V=V, seed=2)["v_shaped"].reshape(V, 3).numpy()
    if with_faces:
        d["faces"] = np.random.default_rng(0).integers(0, V, (30, 3)).astype(np.int64)
    np.savez(path, **d)
    return d


def test_smpl_npz_loader_needs_faces(tmp_path):
    from avatarclip_b200 import drive, shapegen as S
    d = _write_smpl_npz(tmp_path / "smpl.npz")
    s = S.load_smpl_npz(str(tmp_path / "smpl.npz"))
    assert s["faces"].dtype == np.int32 and np.array_equal(s["faces"], d["faces"])
    assert set(drive.load_smpl_npz(str(tmp_path / "smpl.npz"))) == set(drive.SMPL_KEYS)
    _write_smpl_npz(tmp_path / "nofaces.npz", with_faces=False)
    assert set(drive.load_smpl_npz(str(tmp_path / "nofaces.npz"))) == set(drive.SMPL_KEYS)   # unchanged for drive
    with pytest.raises(ValueError, match="faces"):
        S.load_smpl_npz(str(tmp_path / "nofaces.npz"))
    bad = dict(np.load(tmp_path / "smpl.npz"))
    bad["faces"] = bad["faces"] + 1000
    np.savez(tmp_path / "bad.npz", **bad)
    with pytest.raises(ValueError, match="faces"):
        S.load_smpl_npz(str(tmp_path / "bad.npz"))


def test_cli_defaults_and_argument_checks(tmp_path):
    from avatarclip_b200 import shapegen as S
    p = S.build_parser()
    a = p.parse_args(["--smpl", "x.npz"])
    assert a.AE_path_fname == "./data/model_VAE_16.pth" and a.codebook_fname == "./data/codebook.pth"
    assert a.neutral_txt == "a 3d rendering of a person in unreal engine"
    assert a.target_txt == "a 3d rendering of a strong man in unreal engine"
    assert a.output_folder == "./output/coarse_shape" and a.render_folder is None and a.pose_type == "stand_pose"
    assert "faces" in p.epilog
    files = {k: tmp_path / k for k in ("ae.pth", "cb.pth", "smpl.npz", "uv.obj", "clip.pt", "bpe.gz", "pose.npy")}
    for f in files.values():
        f.write_bytes(b"x")
    argv = ["--AE_path_fname", str(files["ae.pth"]), "--codebook_fname", str(files["cb.pth"]), "--smpl",
            str(files["smpl.npz"]), "--uv_obj", str(files["uv.obj"]), "--clip_model", str(files["clip.pt"]), "--bpe",
            str(files["bpe.gz"])]
    a = S.parse_args(argv + ["--render_folder", str(tmp_path / "r"), "--stand_pose", str(files["pose.npy"])])
    assert a.render_folder == str(tmp_path / "r")
    a = S.parse_args(argv + ["--render_folder", "r", "--pose_type", "t_pose", "--stand_pose", "missing.npy"])
    assert a.pose_type == "t_pose"
    with pytest.raises(SystemExit):
        S.parse_args(argv + ["--render_folder", "r", "--stand_pose", "missing.npy"])
    with pytest.raises(SystemExit):
        S.parse_args(argv[:-1] + [str(tmp_path / "missing.gz")])
    with pytest.raises(SystemExit):
        S.parse_args(argv + ["--pose_type", "a_pose"])
    assert S.output_fname("out", "a strong  man") == os.path.join("out", "a_strong__man.obj")


def test_coarse_shape_poses(tmp_path):
    from avatarclip_b200 import shapegen as S
    t = S.coarse_shape_pose("t_pose")
    assert t.shape == (1, 24, 3) and t[0, 0, 0] == np.float32(np.pi / 2) and np.count_nonzero(t) == 1
    np.save(tmp_path / "stand.npy", np.arange(72, dtype=np.float64).reshape(1, 72))
    s = S.coarse_shape_pose("stand_pose", str(tmp_path / "stand.npy"))
    assert s.dtype == np.float32 and s.shape == (1, 72)


def test_no_cpu_path():
    from avatarclip_b200 import _lib, shapegen as S
    with pytest.raises(_lib.AvcError):
        S.codebook_argmax(torch.zeros(4, 8), torch.zeros(8), torch.ones(8))
    with pytest.raises(_lib.AvcError):
        S.clip_prep_nearest(torch.zeros(1, 8, 8, 3))
