"""Video rendering kernels (avc_video.cu) and avatarclip_b200.video on the device: against the fp64 oracle
(oracle/video.py) on the SMPL template and hand-built cases, determinism, chunking, the rig shared with drive, the
orientation of the frames, an avatar-sized mesh, the CLI and the argument checks."""
import ctypes as C
import io
import os

import numpy as np
import pytest
import torch

import util_neus as U
from oracle import drive as D
from oracle import video as OV

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_drive_small.pt")


@pytest.fixture(scope="module")
def g():
    return torch.load(GOLDEN, map_location="cpu", weights_only=False)


@pytest.fixture(scope="module")
def smpl(g):
    s = D.golden_smpl(g["smpl_seed"])
    assert {k: float(v.double().sum()) for k, v in s.items()} == g["smpl_sums"]
    return s


@pytest.fixture(scope="module")
def files(g, smpl, tmp_path_factory):
    """The template in the stand pose as a validate_mesh PLY with seeded colours, the stand pose, a seeded 3-frame
    motion and one whose body pose is all zeros; plus the same PLY with the head red on grey."""
    from avatarclip_b200 import handoff
    d = tmp_path_factory.mktemp("video")
    stand_bytes = g["stand_pose_npy"].numpy().tobytes()
    v, f = D.bench_mesh(smpl, np.load(io.BytesIO(stand_bytes)), levels=0)
    colors = np.random.default_rng(5).integers(0, 256, v.shape, dtype=np.uint8)
    head = smpl["v_template"][:, 1].numpy() > 0.35                    # SMPL's template is y-up
    red = np.where(head[:, None], np.array([[220, 30, 30]], np.uint8), np.array([[160, 160, 160]], np.uint8))
    stand = d / "stand_pose.npy"
    stand.write_bytes(stand_bytes)
    np.save(d / "motion.npy", np.random.default_rng(6).normal(0, 0.3, (3, 72)).astype(np.float32))
    np.save(d / "zero.npy", np.zeros((2, 72), np.float32))
    return dict(ply=handoff.write_ply(str(d / "avatar.ply"), v, f, colors),
                red=handoff.write_ply(str(d / "red.ply"), v, f, red),
                stand=str(stand), motion=str(d / "motion.npy"), zero=str(d / "zero.npy"), head=head, dir=d)


def _motion_inputs(files, smpl, image_size):
    from avatarclip_b200 import video
    m = video.motion_rig(files["ply"], files["motion"], smpl, files["stand"])
    V = m.rig.tpose.shape[0]
    verts = video.skin(m, 0, m.A.shape[0], torch.empty(m.A.shape[0], V, 3, device="cuda"))
    flat = verts.reshape(-1, 3)
    cams = video.orbit_cameras(*video._bounding_sphere(flat.amin(0), flat.amax(0)), m.A.shape[0], image_size, 0.0)
    return m, verts, cams


# ---------------------------------------------------------------- kernels against the oracle
def test_adjacency_matches_oracle(files):
    """The template mesh, and a triangle strip over more than 2 x 1024 x 1024 vertices (its last vertex in no face):
    more 2048-element scan tiles than one pass of the tile-sum scan covers, so its running carry is used."""
    from avatarclip_b200 import drive, video
    mesh = drive.read_ply(files["ply"])
    Vs = 3 * 2 ** 20 + 7
    i = torch.arange(Vs - 3, dtype=torch.int32, device="cuda")
    strip = torch.stack([i, i + 1 + i % 2, i + 2 - i % 2], 1)
    for faces, V in ((mesh.triangles, mesh.vertices.shape[0]), (strip, Vs)):
        adj = video.adjacency(faces, V)
        off, vf = OV.adjacency(faces.cpu().numpy(), V)
        assert np.array_equal(adj.offsets.cpu().numpy(), off)
        assert np.array_equal(adj.vf.cpu().numpy(), vf)


def test_template_motion_matches_oracle(files, smpl):
    from avatarclip_b200 import video
    n, ss = 128, 2
    m, verts, cams = _motion_inputs(files, smpl, n)
    mesh = m.rig.mesh
    adj = video.adjacency(mesh.triangles, mesh.vertices.shape[0])
    colors = torch.from_numpy(mesh.vertex_colors).cuda()
    face = torch.empty(3, n * ss, n * ss, dtype=torch.int32, device="cuda")
    rgb = video.render(verts, mesh.triangles, adj, colors, cams, n, ss, face_out=face).cpu().numpy()
    face = face.cpu().numpy()
    # the whole motion path renders the same frames
    got = list(video.iter_motion_frames(files["ply"], files["motion"], smpl, files["stand"], image_size=n,
                                        supersample=ss))
    assert len(got) == 3 and all(np.array_equal(a, b) for a, b in zip(got, rgb))
    tris = mesh.triangles.cpu().numpy()
    worst_amb, worst_lsb = 0.0, 0
    for i in range(3):
        o = OV.render_frame(verts[i].cpu().numpy(), tris, mesh.vertex_colors, cams[i], n, ss)
        amb = o["ambiguous"]
        assert np.array_equal(face[i][~amb], o["face"][~amb])
        covered = (face[i] >= 0) | (o["face"] >= 0)
        assert covered.sum() > 2000
        worst_amb = max(worst_amb, amb[covered].mean())
        ok = ~o["pixel_ambiguous"]
        lsb = np.abs(rgb[i].astype(int) - o["rgb"].astype(int))[ok].max()
        worst_lsb = max(worst_lsb, int(lsb))
    U.log_parity("video_template_motion", {"ambiguous_frac": float(worst_amb), "max_lsb": worst_lsb})
    assert worst_amb <= 0.005 and worst_lsb <= 1


def _one(verts, faces, colors, cam, n, ss, face=None):
    from avatarclip_b200 import video
    v = torch.from_numpy(verts).cuda()
    f = torch.from_numpy(faces).cuda()
    adj = video.adjacency(f, v.shape[0])
    c = None if colors is None else torch.from_numpy(colors).cuda()
    return video.render(v, f, adj, c, cam[None], n, ss, face_out=face)[0].cpu().numpy()


@pytest.mark.parametrize("ss", [1, 2])
def test_hand_built_cases_exact(ss):
    verts, faces, colors, cam, n, covered = OV.case_quad()
    face = torch.empty(1, n * ss, n * ss, dtype=torch.int32, device="cuda")
    rgb = _one(verts, faces, colors, cam, n, ss, face)
    o = OV.render_frame(verts, faces, colors, cam, n, ss)
    assert np.array_equal(rgb, o["rgb"]) and np.array_equal(face[0].cpu().numpy(), o["face"])
    assert int((face >= 0).sum()) == covered * ss * ss
    verts, faces, colors, cam, n, (y, x) = OV.case_overlap()
    for order in (faces, faces[::-1].copy()):
        rgb = _one(verts, order, colors, cam, n, ss)
        assert rgb[y, x].tolist() == [255, 0, 0]
        assert np.array_equal(rgb, OV.render_frame(verts, order, colors, cam, n, ss)["rgb"])
    for with_colors in (True, False):
        verts, faces, colors, cam, n, want, (y, x) = OV.case_tilted(with_colors)
        face = torch.empty(1, n * ss, n * ss, dtype=torch.int32, device="cuda")
        rgb = _one(verts, faces, colors, cam, n, ss, face)
        o = OV.render_frame(verts, faces, colors, cam, n, ss)
        amb = o["ambiguous"]
        assert np.array_equal(face[0].cpu().numpy()[~amb], o["face"][~amb])
        inside = o["face"].reshape(n, ss, n, ss).min((1, 3)) >= 0
        assert rgb[y, x].tolist() == list(want) and (rgb[inside] == np.array(want, np.uint8)).all()
        # partly covered pixels may hold a mean that ends in .5 exactly: the fp32 sum rounds it either way
        assert np.abs(rgb.astype(int) - o["rgb"].astype(int)).max() <= 1


# ---------------------------------------------------------------- determinism, chunking, the shared rig
def test_renders_are_bitwise_reproducible(files, smpl):
    from avatarclip_b200 import video
    m, verts, cams = _motion_inputs(files, smpl, 96)
    mesh = m.rig.mesh
    colors = torch.from_numpy(mesh.vertex_colors).cuda()
    a = video.render(verts, mesh.triangles, video.adjacency(mesh.triangles, verts.shape[1]), colors, cams, 96, 3)
    b = video.render(verts, mesh.triangles, video.adjacency(mesh.triangles, verts.shape[1]), colors, cams, 96, 3)
    assert torch.equal(a, b)


def test_chunking_does_not_change_frames(files, smpl):
    from avatarclip_b200 import video
    kw = dict(image_size=64, supersample=2, orbit_degrees=45.0)
    one = list(video.iter_motion_frames(files["ply"], files["motion"], smpl, files["stand"], frames_per_chunk=1, **kw))
    default = list(video.iter_motion_frames(files["ply"], files["motion"], smpl, files["stand"], **kw))
    assert len(one) == len(default) == 3 and all(np.array_equal(a, b) for a, b in zip(one, default))
    t1 = list(video.iter_turntable_frames(files["ply"], n_frames=5, image_size=64, frames_per_chunk=2))
    t2 = list(video.iter_turntable_frames(files["ply"], n_frames=5, image_size=64))
    assert len(t1) == 5 and all(np.array_equal(a, b) for a, b in zip(t1, t2))
    assert not np.array_equal(t1[0], t1[1])                            # the camera turns


def test_motion_vertices_are_the_pc2_payload(files, smpl, tmp_path):
    from avatarclip_b200 import drive, video
    _, pc2 = drive.generate_animation(files["ply"], files["motion"], str(tmp_path), smpl, files["stand"])
    m = video.motion_rig(files["ply"], files["motion"], smpl, files["stand"])
    V = m.rig.tpose.shape[0]
    verts = video.skin(m, 0, 3, torch.empty(3, V, 3, device="cuda"))
    assert open(pc2, "rb").read()[32:] == verts.cpu().numpy().astype("<f4").tobytes()


# ---------------------------------------------------------------- orientation
def _red_centroid(rgb):
    r, gch, b = (rgb[..., k].astype(int) for k in range(3))
    red = (r > gch + 60) & (r > b + 60)
    ys, xs = np.nonzero(red)
    return red.sum(), ys.mean() / rgb.shape[0], xs.mean() / rgb.shape[1]


def test_head_is_up_and_in_the_middle(files, smpl):
    from avatarclip_b200 import video
    motion = next(video.iter_motion_frames(files["red"], files["zero"], smpl, files["stand"], image_size=256))
    turn = next(video.iter_turntable_frames(files["red"], n_frames=4, image_size=256))
    for rgb in (motion, turn):
        count, y, x = _red_centroid(rgb)
        assert count > 100, count
        assert y < 0.4 and 0.4 < x < 0.6, (y, x)


# ---------------------------------------------------------------- avatar-sized mesh
def test_avatar_sized_mesh(g, smpl, tmp_path):
    """440 834 vertices: every covered sample lies inside its face, and the colours match the fp64 resolve of the
    device's faces within 1 LSB (the full oracle z-buffer is too slow at this size)."""
    from avatarclip_b200 import handoff, video
    stand = tmp_path / "stand_pose.npy"
    stand.write_bytes(g["stand_pose_npy"].numpy().tobytes())
    v, f = D.bench_mesh(smpl, np.load(str(stand)), levels=3)
    assert v.shape[0] == 440834
    colors = np.random.default_rng(7).integers(0, 256, v.shape, dtype=np.uint8)
    ply = handoff.write_ply(str(tmp_path / "big.ply"), v, f, colors)
    np.save(tmp_path / "m.npy", np.random.default_rng(8).normal(0, 0.3, (2, 72)).astype(np.float32))
    n, ss = 96, 2
    m = video.motion_rig(ply, str(tmp_path / "m.npy"), smpl, str(stand))
    mesh = m.rig.mesh
    verts = video.skin(m, 0, 2, torch.empty(2, mesh.vertices.shape[0], 3, device="cuda"))
    flat = verts.reshape(-1, 3)
    cams = video.orbit_cameras(*video._bounding_sphere(flat.amin(0), flat.amax(0)), 2, n, 0.0)
    face = torch.empty(2, n * ss, n * ss, dtype=torch.int32, device="cuda")
    rgb = video.render(verts, mesh.triangles, video.adjacency(mesh.triangles, verts.shape[1]),
                       torch.from_numpy(mesh.vertex_colors).cuda(), cams, n, ss, face_out=face).cpu().numpy()
    got = list(video.iter_motion_frames(ply, str(tmp_path / "m.npy"), smpl, str(stand), image_size=n, supersample=ss))
    assert all(np.array_equal(a, b) for a, b in zip(got, rgb))
    tris = mesh.triangles.cpu().numpy()
    for i in range(2):
        fc = face[i].cpu().numpy()
        assert 0.1 < (fc >= 0).mean() < 0.9
        vi = verts[i].cpu().numpy()
        proj = OV.project(vi, cams[i], n, ss)
        _, value, w = OV.shade(proj, OV.vertex_normals(vi, tris), tris, mesh.vertex_colors, cams[i], fc, n, ss)
        assert w.min() > -1e-3                                          # inside its face up to fp32 rounding
        assert np.abs(rgb[i].astype(float) - value).max() <= 1.0 + 1e-6


# ---------------------------------------------------------------- CLI, errors
def test_cli_writes_playable_mp4(files, smpl, tmp_path):
    import cv2
    from avatarclip_b200 import video
    npz = tmp_path / "smpl.npz"
    np.savez(npz, **{k: np.asarray(v) for k, v in smpl.items()})
    runs = [(["--mesh", files["ply"], "--out", str(tmp_path / "t.mp4"), "--frames", "6", "--image_size", "64"], 6),
            (["--mesh", files["ply"], "--out", str(tmp_path / "m.mp4"), "--motion", files["motion"], "--smpl", str(npz),
              "--stand_pose", files["stand"], "--image_size", "80", "--orbit_degrees", "30"], 3)]
    for argv, frames in runs:
        assert video.main(argv) == 0
        cap = cv2.VideoCapture(argv[3])
        try:
            size = int(argv[argv.index("--image_size") + 1])
            assert cap.isOpened() and int(cap.get(cv2.CAP_PROP_FRAME_COUNT)) == frames
            assert (int(cap.get(cv2.CAP_PROP_FRAME_WIDTH)), int(cap.get(cv2.CAP_PROP_FRAME_HEIGHT))) == (size, size)
            ok, img = cap.read()
            assert ok and img.shape == (size, size, 3)
        finally:
            cap.release()


def test_meshless_ply_and_bad_motion_raise(files, smpl, tmp_path):
    from avatarclip_b200 import handoff, video
    empty = handoff.write_ply(str(tmp_path / "e.ply"), np.zeros((3, 3), np.float32), np.zeros((0, 3), np.int32))
    with pytest.raises(ValueError):
        video.iter_turntable_frames(empty, n_frames=2, image_size=16)
    with pytest.raises(ValueError):
        video.iter_motion_frames(empty, files["motion"], smpl, files["stand"], image_size=16)
    np.save(tmp_path / "bad.npy", np.zeros((4, 60), np.float32))
    with pytest.raises(ValueError):
        video.iter_motion_frames(files["ply"], str(tmp_path / "bad.npy"), smpl, files["stand"], image_size=16)


def test_abi_rejects_bad_arguments():
    from avatarclip_b200 import video
    L = video._L()
    t = torch.zeros(1 << 16, device="cuda")
    p = C.c_void_p(t.data_ptr())
    sz = C.c_size_t()
    E_BADCFG, E_NULL, E_SIZE = -1, -2, -3
    bg = (C.c_uint8 * 3)(0, 0, 0)
    cam = np.array(OV.axis_camera(10.0), np.float32)
    bad_cam = cam.copy()
    bad_cam[12] = 0.0
    cp, bcp = cam.ctypes.data_as(C.c_void_p), bad_cam.ctypes.data_as(C.c_void_p)
    assert L.avc_video_adjacency_workspace_bytes(0, C.byref(sz)) == E_SIZE
    assert L.avc_video_adjacency_workspace_bytes(4, None) == E_NULL
    assert L.avc_video_adjacency(None, 4, 1, p, p, p, 4096, None) == E_NULL
    assert L.avc_video_adjacency(p, 4, 0, p, p, p, 4096, None) == E_SIZE
    assert L.avc_video_adjacency(p, 4, 1, p, p, p, 1, None) == E_SIZE
    for args in ((4, 1, 1, 0, 1), (4, 1, 1, 4097, 1), (4, 1, 1, 8, 0), (4, 1, 1, 8, 5), (4, 1, 0, 8, 1),
                 (4, 1, 65536, 8, 1), (0, 1, 1, 8, 1), (4, 0, 1, 8, 1)):
        assert L.avc_video_render_workspace_bytes(*args, C.byref(sz)) == E_BADCFG, args
    assert L.avc_video_render_workspace_bytes(4, 1, 1, 8, 1, C.byref(sz)) == 0
    need = sz.value
    ws = torch.empty(need, dtype=torch.uint8, device="cuda")
    w = C.c_void_p(ws.data_ptr())

    def call(cams=cp, stride=0, ws_bytes=need, n=8, ss=1, verts=p, out=p):
        return L.avc_video_render(verts, stride, p, p, p, None, 4, 1, cams, 1, n, ss, bg, out, None, w, ws_bytes, None)
    assert call(cams=bcp) == E_BADCFG
    assert call(stride=-1) == E_BADCFG
    assert call(n=0) == E_BADCFG and call(ss=5) == E_BADCFG
    assert call(ws_bytes=need - 1) == E_SIZE
    assert call(verts=None) == E_NULL and call(out=None) == E_NULL and call(cams=None) == E_NULL
    torch.cuda.synchronize()


def test_cpu_tensors_raise():
    from avatarclip_b200 import AvcError, video
    verts, faces, colors, cam, n, _ = OV.case_quad()
    with pytest.raises(AvcError):
        video.adjacency(torch.from_numpy(faces), 4)
    adj = video.adjacency(torch.from_numpy(faces).cuda(), 4)
    with pytest.raises(AvcError):
        video.render(torch.from_numpy(verts), torch.from_numpy(faces).cuda(), adj, None, cam[None], n, 1)
    with pytest.raises(AvcError):
        video.render(torch.from_numpy(verts).cuda(), torch.from_numpy(faces).cuda(), adj, torch.from_numpy(colors),
                     cam[None], n, 1)
