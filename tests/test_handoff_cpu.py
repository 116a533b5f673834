"""On-disk hand-off formats (avatarclip_b200/handoff.py), host side: the vertex-coloured binary PLY of Runner.validate_mesh
(main.py:913-916) and the camera matrices of the ShapeGen -> AppearanceGen directory (AvatarGen/ShapeGen/render.py:16-58)."""
import os

import numpy as np
import pytest

from avatarclip_b200 import handoff

REF_RENDER = os.path.join(os.environ.get("AVC_REFERENCE", ""), "AvatarGen/ShapeGen/render.py")


def test_ply_round_trip_and_header(tmp_path):
    rng = np.random.RandomState(0)
    v = rng.randn(50, 3).astype(np.float32)
    f = rng.randint(0, 50, size=(80, 3)).astype(np.int64)
    c = rng.randint(0, 256, size=(50, 3)).astype(np.uint8)
    p = handoff.write_ply(str(tmp_path / "m.ply"), v, f, c)
    raw = open(p, "rb").read()
    head = raw[:raw.index(b"end_header\n")].decode("ascii").split("\n")
    assert head[:2] == ["ply", "format binary_little_endian 1.0"]
    assert "element vertex 50" in head and "element face 80" in head
    assert head.index("property uchar alpha") == head.index("property uchar red") + 3          # r g b a, like trimesh's export
    assert "property list uchar int vertex_indices" in head
    assert len(raw) == raw.index(b"end_header\n") + len(b"end_header\n") + 50 * (12 + 4) + 80 * (1 + 12)
    vv, ff, cc = handoff.read_ply(p)
    assert np.array_equal(vv, v) and np.array_equal(ff, f.astype(np.int32)) and np.array_equal(cc, c)
    p2 = handoff.write_ply(str(tmp_path / "plain.ply"), v, f)                                    # no colours
    vv, ff, cc = handoff.read_ply(p2)
    assert np.array_equal(vv, v) and np.array_equal(ff, f.astype(np.int32)) and cc is None
    p3 = handoff.write_ply(str(tmp_path / "empty.ply"), np.zeros((0, 3)), np.zeros((0, 3)), np.zeros((0, 3), dtype=np.uint8))
    vv, ff, cc = handoff.read_ply(p3)                                                            # an empty iso-surface
    assert vv.shape == (0, 3) and ff.shape == (0, 3) and cc.shape == (0, 3)


def test_hand_off_cameras():
    d = 2.2
    assert np.allclose(handoff.get_points_from_angles(d, 0, 0), [0, 0, -d])
    assert np.allclose(handoff.get_points_from_angles(d, 0, 90), [d, 0, 0], atol=1e-12)
    assert np.allclose(handoff.get_points_from_angles(d, 90, 0), [0, d, 0], atol=1e-12)
    eyes = [handoff.get_points_from_angles(d, e, a) for a in range(0, 360, 20) for e in range(-60, 60, 20)]
    assert len(eyes) == 108 and np.allclose([np.linalg.norm(e) for e in eyes], d)               # render.py:47-48
    for eye in eyes[::7]:
        m = handoff.lookat_inverse_view(eye, np.zeros(3), np.array([0.0, 1.0, 0.0]))
        R = m[:3, :3]
        assert np.allclose(R.T @ R, np.eye(3), atol=1e-12) and abs(np.linalg.det(R) - 1.0) < 1e-12
        assert np.allclose(m[:3, 3], eye) and np.allclose(m[3], [0, 0, 0, 1])
        assert np.allclose(R[:, 2], eye / np.linalg.norm(eye))                                    # camera looks down -z at the origin


def test_camera_matrix_equals_the_reference_lines():
    """ShapeGen/render.py:16-30 (norm_np_arr + lookat) against handoff.lookat_inverse_view (the reference's matrices are
    stored under tests/golden/)."""
    import textwrap
    from util_neus import reference_golden
    eyes = [handoff.get_points_from_angles(2.2, e, a) for a in range(0, 360, 40) for e in (-60, -20, 0, 40)]

    def reference():
        lines = open(REF_RENDER).read().split("\n")[15:30]
        assert lines[0].startswith("def norm_np_arr") and "return viewMatrix" in lines[-1]
        ns = {"np": np}
        exec(textwrap.dedent("\n".join(lines)), ns)
        return [ns["lookat"](eye, np.array([0, 0, 0]), np.array([0, 1, 0]))[0] for eye in eyes]
    for eye, ref in zip(eyes, reference_golden("camera_matrices", reference), strict=True):
        assert np.array_equal(ref, handoff.lookat_inverse_view(eye, np.array([0, 0, 0]), np.array([0, 1, 0])))


def test_read_obj_triangulates_and_strips_texture_indices(tmp_path):
    from avatarclip_b200.views import read_obj
    p = tmp_path / "t.obj"
    p.write_text("# comment\nv 0 0 0\nv 1 0 0\nv 1 1 0\nv 0 1 0\nvt 0 0\nvn 0 0 1\nf 1/1/1 2/1/1 3/1/1 4/1/1\nf 1 2 3\n")
    v, f = read_obj(str(p))
    assert v.shape == (4, 3) and v.dtype == np.float32
    assert f.tolist() == [[0, 1, 2], [0, 2, 3], [0, 1, 2]] and f.dtype == np.int32          # quad -> fan of two triangles


def test_read_obj_on_the_shipped_template(tmp_path):
    """dataset.template_obj of the shipped confs (main.py:292,316): the SMPL topology, 6890 vertices / 13 776 triangles."""
    from avatarclip_b200.views import read_obj
    from util_neus import reference_tree
    v, f = read_obj(os.path.join(reference_tree(tmp_path), "data/zero_beta_smpl.obj"))
    assert v.shape == (6890, 3) and f.shape == (13776, 3) and f.min() == 0 and f.max() == 6889
    assert np.abs(v).max() < 1.5
