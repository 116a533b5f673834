"""PoseOptimizer without a GPU: the fp64 oracle's edge sweep (oracle/pose_optimizer.py) on hand-built scenes, its
light, SMPL, resize and loss backward against finite differences, and how the pose_optimizer command classifies the
85 shipped AvatarAnimate confs."""
import glob
import os
import tarfile

import numpy as np
import pytest
import torch

from oracle import pose_optimizer as OP

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")


def _ndc(p, is_):
    return (2.0 * np.asarray(p, dtype=np.float64) + 1 - is_) / is_


def _inside(tri, is_):
    """fidx of one triangle (pixel coordinates, any winding) drawn with index 0 at pixel centres; row 0 at the top."""
    fidx = np.full((is_, is_), -1)
    (x0, y0), (x1, y1), (x2, y2) = tri
    det = (y1 - y2) * (x0 - x2) + (x2 - x1) * (y0 - y2)
    for yi in range(is_):
        for xi in range(is_):
            w0 = ((y1 - y2) * (xi - x2) + (x2 - x1) * (yi - y2)) / det
            w1 = ((y2 - y0) * (xi - x2) + (x0 - x2) * (yi - y2)) / det
            if min(w0, w1, 1 - w0 - w1) >= 0:
                fidx[is_ - 1 - yi, xi] = 0
    return fidx


def _scene(tri, is_):
    fidx = _inside(tri, is_)
    rgb = np.where(fidx[..., None] == 0, 1.0, 0.0) * np.ones(3)
    return fidx, rgb


TRI = [(2.2, 4.3), (12.6, 4.7), (7.1, 13.4)]     # counter-clockwise in the pixel frame (y up)


def test_single_triangle_out_pixel():
    """g only at the pixel just below the bottom edge in column 7: the gradient of each end point's y is -diff / dist,
    and moving P0 by its dist flips exactly that pixel of the column."""
    is_ = 16
    fidx, rgb = _scene(TRI, is_)
    d0, d1 = 7, 4
    assert fidx[is_ - 1 - 5, d0] == 0 and fidx[is_ - 1 - d1, d0] == -1
    g = np.zeros((is_, is_, 3))
    g[is_ - 1 - d1, d0] = -1.0
    out = OP.edge_sweep(_ndc(TRI, is_), 0, fidx, rgb, g)
    f32 = np.float32
    pp = f32(0.5) * ((_ndc(TRI, is_).astype(f32) * f32(is_) + f32(is_)) - f32(1))    # the sweep's pixel frame
    p0, p1 = pp[0], pp[1]
    cross = np.float32(np.float32(np.float32(p1[1] - p0[1]) / np.float32(p1[0] - p0[0])) * np.float32(d0 - p0[0])) + p0[1]
    diff = 3.0
    base = (d1 - float(cross)) * 2.0 / is_
    dist0 = float(p1[0] - p0[0]) / float(p1[0] - d0) * base
    dist1 = float(p1[0] - p0[0]) / (d0 - float(p0[0])) * base
    assert out[0, 1] == pytest.approx(-diff / (dist0 - OP.EPS), rel=1e-12)
    assert out[1, 1] == pytest.approx(-diff / (dist1 - OP.EPS), rel=1e-12)
    assert out[2, 1] == 0 and (out[:, 0] == 0).all()
    moved = [list(p) for p in TRI]
    moved[0][1] += dist0 * is_ / 2 * 1.001
    flipped = (_inside(moved, is_)[:, d0] == 0) != (fidx[:, d0] == 0)
    assert np.nonzero(flipped)[0].tolist() == [is_ - 1 - d1]


def test_no_contribution_when_diff_not_positive():
    is_ = 16
    fidx, rgb = _scene(TRI, is_)
    g = np.zeros((is_, is_, 3))
    g[fidx == -1] = 1.0             # every out pixel would get darker-than-in: diff < 0
    g[fidx == 0] = -1.0             # every in pixel: diff (rgb - rgb_out) . g < 0
    assert (OP.edge_sweep(_ndc(TRI, is_), 0, fidx, rgb, g) == 0).all()


def test_drawn_copy_winding():
    """The face given clockwise is swept as fill_back's reversed copy: the same gradient as the face given
    counter-clockwise, and not what the clockwise winding's own sweep gives."""
    is_ = 16
    fidx, rgb = _scene(TRI, is_)
    rng = np.random.default_rng(0)
    g = rng.standard_normal((is_ // 2, is_ // 2, 3))
    ndc = _ndc(TRI, is_)
    proj = np.concatenate([ndc, np.ones((3, 1))], 1)
    verts = np.concatenate([ndc, np.full((3, 1), 5.0)], 1)
    eye, rot = np.zeros(3), np.eye(3)
    ccw = OP.raster_backward_image(verts, [[0, 1, 2]], proj, eye, rot, fidx, rgb, g, 2)
    cw = OP.raster_backward_image(verts, [[2, 1, 0]], proj, eye, rot, fidx, rgb, g, 2)
    assert np.abs(ccw).max() > 0
    np.testing.assert_allclose(cw, ccw, rtol=1e-12, atol=1e-12)
    g_ss = np.repeat(np.repeat(g, 2, 0), 2, 1) / 4
    own = OP.edge_sweep(ndc[[2, 1, 0]], 0, fidx, rgb, g_ss)
    drawn = OP.edge_sweep(ndc, 0, fidx, rgb, g_ss)
    assert not np.allclose(own[[2, 1, 0]], drawn)


def test_border_columns_skipped():
    """The bottom edge crosses each column in (-1, 0]: its out pixel is off the image, so the only pixels that could
    move it (row 0 outside the face) give no y gradient, while the row sweeps still see them (x gradient)."""
    is_ = 8
    tri = [(1.2, -0.3), (6.6, -0.2), (3.9, 5.5)]
    fidx, rgb = _scene(tri, is_)
    g = np.zeros((is_, is_, 3))
    g[is_ - 1, :][fidx[is_ - 1, :] == -1] = -1.0
    out = OP.edge_sweep(_ndc(tri, is_), 0, fidx, rgb, g)
    assert (out[:, 1] == 0).all() and np.abs(out[:, 0]).max() > 0


def test_edge_with_equal_coordinates_contributes_nothing():
    """A vertical edge on an exact pixel column (corners 2 -> 0, edge 2): neural_renderer divides 0 by 0 in its column
    sweep; here that part adds nothing, and the sweep equals the one that leaves the part out, while leaving out any
    other part changes it."""
    is_ = 16
    tri = [(3.0, 2.5), (12.5, 8.5), (3.0, 13.5)]
    fidx, rgb = _scene(tri, is_)
    g = np.random.default_rng(1).standard_normal((is_, is_, 3))
    ndc = _ndc(tri, is_)
    out = OP.edge_sweep(ndc, 0, fidx, rgb, g)
    assert np.isfinite(out).all() and np.abs(out).max() > 0
    np.testing.assert_array_equal(out, OP.edge_sweep(ndc, 0, fidx, rgb, g, skip={(2, 0)}))
    for part in ((2, 1), (0, 0), (1, 0)):
        assert not np.array_equal(out, OP.edge_sweep(ndc, 0, fidx, rgb, g, skip={part}))


def test_light_backward_matches_finite_differences():
    rng = np.random.default_rng(2)
    v = rng.standard_normal((3, 3))
    eye = np.array([0.3, 1.5, 2.0])
    if OP.face_light(*v, eye)[0] <= 0.5 + 1e-3:
        v[:, 1] *= -1
    g = OP.light_backward(*v, eye, 1.0)
    h = 1e-6
    for i in range(3):
        for k in range(3):
            vp, vm = v.copy(), v.copy()
            vp[i, k] += h
            vm[i, k] -= h
            fd = (OP.face_light(*vp, eye)[0] - OP.face_light(*vm, eye)[0]) / (2 * h)
            assert g[i, k] == pytest.approx(fd, abs=1e-6)


def test_prep_backward_and_loss():
    from oracle import shapegen as OS
    rng = np.random.default_rng(3)
    for n, S in ((10, 7), (7, 10), (256, 224)):
        g = rng.standard_normal((2, 3, S, S))
        x = torch.tensor(rng.random((2, n, n, 3)), dtype=torch.float64, requires_grad=True)
        idx = torch.clamp(torch.floor(torch.arange(S, dtype=torch.float32) * (np.float32(n) / np.float32(S))).long(),
                          max=n - 1)
        y = (x.permute(0, 3, 1, 2)[:, :, idx][:, :, :, idx] - torch.tensor(OS.CLIP_MEAN).view(1, 3, 1, 1)) / \
            torch.tensor(OS.CLIP_STD, dtype=torch.float64).view(1, 3, 1, 1)
        (y * torch.as_tensor(g)).sum().backward()
        np.testing.assert_allclose(OP.clip_prep_nearest_bwd(g, n), x.grad.numpy(), rtol=1e-12, atol=1e-12)
    emb, text = rng.standard_normal((5, 3, 16)), rng.standard_normal(16)
    loss, g = OP.pose_clip_loss(emb, text)
    f = emb.mean(0)
    np.testing.assert_allclose(loss, 1 - f @ text / np.linalg.norm(f, axis=1) / np.linalg.norm(text), rtol=1e-12)
    h = 1e-6
    e2 = emb.copy()
    e2[2, 1, 5] += h
    assert g[2, 1, 5] == pytest.approx((OP.pose_clip_loss(e2, text)[0][1] - loss[1]) / h, abs=1e-5)


def test_smpl_pose_grad_matches_finite_differences():
    from oracle import lbs as olbs
    sm = olbs.synthetic_smpl(V=40, seed=4, dtype=torch.float64)
    s = dict(v_template=sm["v_shaped"][0], posedirs=sm["posedirs"], J_regressor=sm["J_regressor"],
             parents=sm["parents"], lbs_weights=sm["lbs_weights"])
    rng = np.random.default_rng(4)
    pose = rng.standard_normal((2, 63)) * 0.6
    g = rng.standard_normal((2, 40, 3))

    def f(p):
        dt = torch.float64
        full = torch.cat([torch.tensor(OP.GLOBAL_ORIENT, dtype=dt).expand(2, 3), torch.as_tensor(p), torch.zeros(2, 6,
                                                                                                               dtype=dt)], 1)
        v, _ = olbs.my_lbs(s["v_template"][None].expand(2, -1, -1), full, s["posedirs"], s["J_regressor"],
                           s["parents"], s["lbs_weights"])
        return float(((v.numpy() @ OP.ROT) * g).sum())
    grad = OP.smpl_pose_grad(s, pose, g)
    h = 1e-6
    for b, k in ((0, 0), (1, 31), (1, 62)):
        pp, pm = pose.copy(), pose.copy()
        pp[b, k] += h
        pm[b, k] -= h
        assert grad[b, k] == pytest.approx((f(pp) - f(pm)) / (2 * h), rel=1e-5, abs=1e-7)


# ---------------------------------------------------------------- the command
@pytest.fixture(scope="module")
def confs(tmp_path_factory):
    d = tmp_path_factory.mktemp("pose_optimizer_confs")
    with tarfile.open(os.path.join(GOLDEN, "ref_animate_confs.tar.gz")) as tf:
        tf.extractall(d, filter="data")
    return sorted(glob.glob(str(d / "confs" / "**" / "*.conf"), recursive=True))


def test_conf_classification(confs):
    """Of the 85 shipped confs the command runs exactly the 12 pose_optimizer ones."""
    from avatarclip_b200 import conf
    from avatarclip_b200 import pose_optimizer as PO
    assert len(confs) == 85
    runs, refused = [], []
    modes = {}
    for p in confs:
        c = conf.parse_file(p)
        modes[p] = c.get_string("general.mode", "pose")
        why = PO.refusal(c)
        (runs if why is None else refused).append((p, why))
    assert len(runs) == 12 and all("/pose_ablation/pose_optimizer/" in p for p, _ in runs)
    vp = [w for p, w in refused if "/pose_ablation/vposer_optimizer/" in p]
    assert len(vp) == 12 and all("decoder's backward" in w for w in vp)
    gen = [w for p, w in refused if "/pose_ablation/vposer_" in p and "vposer_optimizer" not in p]
    assert len(gen) == 24 and all("avatarclip_b200.animate" in w for w in gen)
    mot = [w for p, w in refused if modes[p] == "motion"]
    assert len(mot) == 37 and all("avatarclip_b200.motion" in w for w in mot)


def test_cli_refuses_before_reading_files(confs, capsys):
    """Every refusal exits non-zero with its reason, although --smpl names no file; a runnable conf reaches the file
    checks."""
    from avatarclip_b200 import conf
    from avatarclip_b200 import pose_optimizer as PO
    for p in confs:
        why = PO.refusal(conf.parse_file(p))
        with pytest.raises(SystemExit) as e:
            PO.parse_args(["--conf", p, "--smpl", "/nonexistent.npz"])
        err = capsys.readouterr().err
        assert e.value.code != 0
        assert (why.split(":")[0] in err) if why else ("--smpl: no such file" in err)


def test_adam_refusals(tmp_path, capsys):
    from avatarclip_b200 import pose_optimizer as PO
    for block, msg in (("optim_name = SGD", "only Adam"),
                       ("optim_cfg {\n        lr = 0.1\n        momentum = 0.9\n    }", "not Adam's"),
                       ("optim_cfg {\n        lr = 0.1\n        amsgrad = true\n    }", "plain Adam")):
        c = tmp_path / "c.conf"
        c.write_text("general {\n    base_exp_dir = ./x\n    mode = pose\n    text = a man\n}\n"
                     f"pose_generator {{\n    type = PoseOptimizer\n    {block}\n}}\n")
        with pytest.raises(SystemExit) as e:
            PO.parse_args(["--conf", str(c), "--smpl", "/nonexistent.npz"])
        assert e.value.code != 0 and msg in capsys.readouterr().err
    with pytest.raises(NotImplementedError, match="only Adam"):
        PO.PoseOptimizer(optim_name="SGD", name="PoseOptimizer", assets=None)


def test_animate_and_motion_name_the_command(confs):
    from avatarclip_b200 import animate as A
    from avatarclip_b200 import conf
    from avatarclip_b200 import motion as M
    c = conf.parse_file([p for p in confs if "/pose_ablation/pose_optimizer/" in p][0])
    assert "avatarclip_b200.pose_optimizer" in A.refusal(c)
    assert "avatarclip_b200.pose_optimizer" in M.refusal(c)


# ---------------------------------------------------------------- the reference's loop (oracle/pin_pose_optimizer.py)
@pytest.fixture(scope="module")
def golden():
    return torch.load(os.path.join(GOLDEN, "ref_pose_optimizer_small.pt"), map_location="cpu", weights_only=False)


def test_loop_against_the_reference(golden):
    """What the reference's own PoseOptimizer did: the torch.randn(63) draws in order, the numpy elevations (pose k's
    num_iteration x 5 before pose k + 1's, then the sort's), torch Adam at lr 0.01 on the recorded gradients,
    pose_padding and the stable descending sort of the written candidates."""
    from avatarclip_b200 import animate as A
    from avatarclip_b200 import motion as M
    K, T = golden["conf"]["topk"], golden["conf"]["num_iteration"]
    torch.manual_seed(golden["torch_seed"])
    assert torch.equal(torch.stack([torch.randn(63) for _ in range(K)]), golden["init"])
    np.random.seed(golden["np_seed"])
    eyes = A.PoseScorer(None).draw_eyes(K * T + K)
    np.testing.assert_allclose(eyes, golden["eyes"].double().numpy(), rtol=0, atol=1e-6)
    final = []
    for k in range(K):
        p = torch.nn.Parameter(golden["init"][k].clone())
        opt = torch.optim.Adam([p], lr=0.01)
        for t in range(T):
            assert torch.equal(p.data, golden["params"][k, t])
            p.grad = golden["grads"][k, t].clone()
            opt.step()
        final.append(M.pose_padding(p.data))
    sc = golden["sort_scores"].tolist()
    order = sorted(range(K), key=lambda i: sc[i], reverse=True)
    np.testing.assert_array_equal(golden["files"].numpy(), torch.stack([final[i] for i in order]).numpy())
    assert golden["files"].shape == (K, 69) and (golden["files"][:, 63:] == 0).all()
    assert (golden["loss"] > 0).all() and float(golden["grads"].abs().max()) > 0
