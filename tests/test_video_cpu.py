"""Video rendering (avatarclip_b200.video) without a GPU: the fp64 oracle on hand-built cases, the cameras' framing
and the CLI's argument checks."""
import numpy as np
import pytest

from oracle import video as OV


def _pixels_not(rgb, bg=(255, 255, 255)):
    return int((rgb != np.array(bg, dtype=np.uint8)).any(-1).sum())


@pytest.mark.parametrize("ss", [1, 2])
def test_oracle_quad_covers_its_pixels(ss):
    verts, faces, colors, cam, n, covered = OV.case_quad()
    o = OV.render_frame(verts, faces, colors, cam, n, ss)
    assert int((o["face"] >= 0).sum()) == covered * ss * ss
    assert _pixels_not(o["rgb"]) == covered
    assert not o["ambiguous"].any()
    assert (o["rgb"][20:44, 10:51] == 90).all()                  # facing the camera: ambient + diffuse = 1


def test_oracle_nearer_triangle_wins():
    verts, faces, colors, cam, n, (y, x) = OV.case_overlap()
    for order in (faces, faces[::-1]):
        o = OV.render_frame(verts, order, colors, cam, n, 2)
        assert o["rgb"][y, x].tolist() == [255, 0, 0]
        red = int(np.nonzero((order == [0, 1, 2]).all(1))[0][0])
        assert (o["face"][2 * y:2 * y + 2, 2 * x:2 * x + 2] == red).all()


@pytest.mark.parametrize("colors", [True, False])
def test_oracle_known_normal_gives_exact_shade(colors):
    verts, faces, col, cam, n, want, (y, x) = OV.case_tilted(colors)
    o = OV.render_frame(verts, faces, col, cam, n, 2)
    assert o["rgb"][y, x].tolist() == list(want)
    inside = o["face"].reshape(n, 2, n, 2).min((1, 3)) >= 0
    assert inside.sum() > 100 and (o["rgb"][inside] == np.array(want, np.uint8)).all()
    assert np.abs(o["value"][inside] - np.array(want)).max() < 1e-3       # the float32 corners tilt it by ~1e-7


def test_oracle_adjacency_lists_faces_in_order():
    faces = np.array([[2, 0, 1], [0, 1, 3], [3, 2, 0], [1, 1, 2], [0, 7, 1]])
    off, vf = OV.adjacency(faces, 4)
    lists = [vf[off[v]:off[v + 1]].tolist() for v in range(4)]
    assert lists == [[0, 1, 2, 4], [0, 1, 3, 3, 4], [0, 2, 3], [1, 2]]


def _inside(points, cams, n):
    for cam in cams:
        p = OV.project(points, cam, n, 1)
        assert (p[:, 2] > 0).all()
        assert (p[:, :2] > 0).all() and (p[:, :2] < n).all()


def test_turntable_cameras_keep_the_sphere_in_frame():
    from avatarclip_b200 import video
    rng = np.random.default_rng(0)
    d = rng.normal(size=(4000, 3))
    center, radius = np.array([0.3, -0.2, 1.1]), 0.9
    sphere = center + radius * d / np.linalg.norm(d, axis=1, keepdims=True)
    cams = video.orbit_cameras(center, radius, 24, 96)
    _inside(sphere, cams, 96)
    # frame 0 sits on the -y side looking along +y with +z up (image row 0 at the top)
    p = OV.project(np.array([center + [0, 0, radius], center + [radius, 0, 0]]), cams[0], 96, 1)
    assert p[0, 1] < 48 and abs(p[0, 0] - 48) < 1e-3 and p[1, 0] > 48
    assert np.allclose(cams[0, 8:11], [0, 1, 0], atol=1e-7)
    # one full turn: frame 6 of 24 has turned 90 degrees about +z
    assert np.allclose(cams[6, 8:11], [-1, 0, 0], atol=1e-6)


def test_motion_cameras_keep_every_frame_in_frame():
    import torch
    from avatarclip_b200 import video
    rng = np.random.default_rng(1)
    frames = [rng.normal(size=(500, 3)) * [0.3, 0.2, 0.8] + [0.1 * k, 0.05 * k, 0] for k in range(10)]
    allv = np.concatenate(frames)
    center, radius = video._bounding_sphere(torch.from_numpy(allv.min(0)), torch.from_numpy(allv.max(0)))
    assert (np.linalg.norm(allv - center, axis=1) <= radius + 1e-9).all()
    cams = video.orbit_cameras(center, radius, len(frames), 128, degrees=90.0)
    for fr, cam in zip(frames, cams):
        _inside(fr, [cam], 128)


def test_cli_reports_argument_errors(tmp_path, capsys):
    from avatarclip_b200 import video
    mesh = tmp_path / "m.ply"
    mesh.write_bytes(b"")
    base = ["--mesh", str(mesh), "--out", str(tmp_path / "o.mp4")]
    cases = [
        (["--mesh", str(tmp_path / "nope.ply"), "--out", "o.mp4"], "--mesh: no such file"),
        (base + ["--image_size", "0"], "--image_size"),
        (base + ["--supersample", "5"], "--supersample"),
        (base + ["--fps", "0"], "--fps"),
        (base + ["--frames", "0"], "--frames must be >= 1"),
        (base + ["--smpl", "s.npz"], "--smpl is only used with --motion"),
        (base + ["--orbit_degrees", "90"], "--orbit_degrees is only used with --motion"),
        (base + ["--motion", "a.npy", "--stand_pose", "p.npy"], "--motion needs --smpl"),
        (base + ["--motion", "a.npy", "--smpl", "s.npz", "--stand_pose", "p.npy", "--frames", "5"], "--frames sets"),
        (base + ["--motion", str(tmp_path / "a.npy"), "--smpl", "s.npz", "--stand_pose", "p.npy"],
         "--motion: no such file"),
    ]
    for argv, msg in cases:
        with pytest.raises(SystemExit) as e:
            video.main(argv)
        assert e.value.code == 2 and msg in capsys.readouterr().err, argv
    with pytest.raises(SystemExit) as e:
        video.main(["--mesh", str(mesh)])
    assert e.value.code == 2
    assert not (tmp_path / "o.mp4").exists()
    a = video.build_parser().parse_args(base)
    assert (a.image_size, a.supersample, a.fps, a.frames, a.orbit_degrees) == (512, 2, 60, None, 0.0)


def test_write_video_round_trips_frame_count_and_size(tmp_path):
    import cv2
    from avatarclip_b200 import video
    rng = np.random.default_rng(2)
    frames = [rng.integers(0, 256, (48, 48, 3), dtype=np.uint8) for _ in range(7)]
    path = str(tmp_path / "v.mp4")
    assert video.write_video(iter(frames), path, 30) == 7
    cap = cv2.VideoCapture(path)
    try:
        assert cap.isOpened()
        assert int(cap.get(cv2.CAP_PROP_FRAME_COUNT)) == 7
        assert (int(cap.get(cv2.CAP_PROP_FRAME_WIDTH)), int(cap.get(cv2.CAP_PROP_FRAME_HEIGHT))) == (48, 48)
    finally:
        cap.release()
    with pytest.raises(ValueError):
        video.write_video(iter(frames), path, 0)


def test_cpu_device_raises(tmp_path):
    from avatarclip_b200 import AvcError, handoff, video
    verts, faces, colors, *_ = OV.case_quad()
    ply = handoff.write_ply(str(tmp_path / "q.ply"), verts, faces, colors)
    with pytest.raises(AvcError):
        video.iter_turntable_frames(ply, n_frames=2, image_size=16, device="cpu")
    with pytest.raises(ValueError):
        video.iter_turntable_frames(ply, n_frames=2, image_size=0, device="cpu")
