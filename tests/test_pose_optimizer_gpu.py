"""PoseOptimizer on the device: the textured rasteriser's backward against the fp64 oracle (oracle/pose_optimizer.py)
on the device's own face-index and colour maps, the SMPL posing backward against fp64 autograd, the resize backward
and the loss kernel against fp64, one whole iteration's pose gradient, the CUDA-graph loop against the same calls
launched one by one, and the command line on synthetic files.  Reads only tests/golden and synthetic data."""
import math
import os

import numpy as np
import pytest
import torch

from oracle import animate as O
from oracle import drive as D
from oracle import pose_optimizer as OP
from oracle import shapegen as OS
from avatarclip_b200.handoff import get_points_from_angles

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _rel(out, ref):
    ref = np.asarray(ref, dtype=np.float64)
    return float(np.abs(np.asarray(torch.as_tensor(out).detach().cpu(), dtype=np.float64) - ref).max() /
                 np.abs(ref).max())


def _align(x):
    return (x + 255) // 256 * 256


def _device_maps(ws_f, ws_b, V, A, B, ncams, is_, cam_bytes):
    """(fidx [AB, is, is], proj [AB, V, 3], rgb_ss [AB, is, is, 3]) read back from the two workspaces."""
    o_proj = _align(ncams * cam_bytes)
    o_z = o_proj + _align(A * B * V * 16)
    proj = ws_f[o_proj:o_proj + A * B * V * 16].view(torch.float32).reshape(A * B, V, 4)[..., :3].cpu().numpy()
    z = ws_f[o_z:o_z + A * B * is_ * is_ * 8].view(torch.int64).reshape(A * B, is_, is_).cpu().numpy()
    fidx = (z & 0xffffffff).astype(np.int64)
    fidx[fidx == 0xffffffff] = -1
    rgb = ws_b[:A * B * is_ * is_ * 12].view(torch.float32).reshape(A * B, is_, is_, 3).cpu().numpy()
    return fidx, proj, rgb


def _sphere(n_lat=10, n_lon=14, r=0.7, c=(0.45, 0.0, 0.0)):
    """A UV sphere offset to one side (so that it crosses the image border from the cameras below) with every other
    face's winding reversed (both drawn copies occur)."""
    vs = [(0.0, r, 0.0), (0.0, -r, 0.0)]
    for i in range(1, n_lat):
        th = math.pi * i / n_lat
        for j in range(n_lon):
            ph = 2 * math.pi * j / n_lon
            vs.append((r * math.sin(th) * math.cos(ph), r * math.cos(th), r * math.sin(th) * math.sin(ph)))
    v = np.asarray(vs) + np.asarray(c)
    ring = lambda i, j: 2 + (i - 1) * n_lon + j % n_lon
    fs = []
    for j in range(n_lon):
        fs.append((0, ring(1, j + 1), ring(1, j)))
        fs.append((1, ring(n_lat - 1, j), ring(n_lat - 1, j + 1)))
    for i in range(1, n_lat - 1):
        for j in range(n_lon):
            fs += [(ring(i, j), ring(i, j + 1), ring(i + 1, j)), (ring(i, j + 1), ring(i + 1, j + 1), ring(i + 1, j))]
    f = np.asarray(fs, dtype=np.int32)
    f[1::2] = f[1::2, ::-1]
    return v.astype(np.float32), f


EYES = [get_points_from_angles(2.0, el, az) for az, el in zip(O.ANGLES, (0.4, -0.3, 25.0, 0.1, -20.0))]


@pytest.mark.parametrize("B", [1, 5])
def test_raster_backward_vs_oracle(B):
    from avatarclip_b200 import pose_optimizer as PO
    from avatarclip_b200 import video
    n, ss, A = 48, 2, 5
    is_ = n * ss
    v0, faces = _sphere()
    rng = np.random.default_rng(B)
    verts = np.stack([v0 + rng.normal(0, 0.03, v0.shape).astype(np.float32) for _ in range(B)])
    V, F = v0.shape[0], faces.shape[0]
    tex = rng.random((F, 3, 3, 3, 3)).astype(np.float32)
    eyes = np.stack([np.roll(np.asarray(EYES), b, 0) for b in range(B)])        # [B, A, 3]
    dev = "cuda"
    vt, ft, tt = torch.tensor(verts, device=dev), torch.tensor(faces, device=dev), torch.tensor(tex, device=dev)
    cams = PO.look_at_cams(eyes, n, ss, device=dev)
    ws_f = PO.raster_fwd_workspace(V, A, B, 1, n, ss, dev)
    rgb = torch.empty(A, B, n, n, 3, device=dev)
    PO.raster_textured_batch_dev(vt, ft, tt, cams, A, 1, rgb, ws_f, n, ss)
    from avatarclip_b200 import animate as AN
    np.testing.assert_array_equal(rgb.cpu().numpy(), AN.raster_textured_batch(vt, ft, tt, eyes, 1, n, ss).cpu().numpy())
    g_rgb = torch.tensor(rng.standard_normal((A, B, n, n, 3)).astype(np.float32), device=dev)
    adj = video.adjacency(ft, V)
    ws_b = PO.raster_bwd_workspace(F, A, B, n, ss, dev)
    g = torch.empty(B, V, 3, device=dev)
    PO.raster_textured_batch_bwd(vt, ft, tt, adj, A, 1, g_rgb, ws_f, g, ws_b, n, ss)
    ws_b2 = torch.full_like(ws_b, 0x7f)            # another workspace holding garbage: the same bits
    g2 = torch.full_like(g, float("nan"))
    PO.raster_textured_batch_bwd(vt, ft, tt, adj, A, 1, g_rgb, ws_f, g2, ws_b2, n, ss)
    assert torch.equal(g, g2)
    cam_bytes = cams.shape[1]
    fidx, proj, rgb_ss = _device_maps(ws_f, ws_b, V, A, B, B * A, is_, cam_bytes)
    ref = np.zeros((B, V, 3))
    n_back, n_border, n_dark = 0, 0, 0
    for a in range(A):
        for b in range(B):
            i = a * B + b
            eye, rot = OS.look_at_camera(eyes[b, a])
            ref[b] += OP.raster_backward_image(verts[b], faces, proj[i], eye, rot, fidx[i], rgb_ss[i],
                                               g_rgb[a, b].cpu().numpy(), ss)
            drawn = np.unique(fidx[i][fidx[i] >= 0])
            q = proj[i][faces[drawn]]
            n_back += int(((q[:, 2, 1] - q[:, 0, 1]) * (q[:, 1, 0] - q[:, 0, 0]) <
                           (q[:, 1, 1] - q[:, 0, 1]) * (q[:, 2, 0] - q[:, 0, 0])).sum())
            n_border += int(np.isin(drawn, np.concatenate([fidx[i][0], fidx[i][-1], fidx[i][:, 0], fidx[i][:, -1]])).sum())
            n_dark += sum(OP.face_light(*verts[b][faces[f]].astype(np.float64), eye)[0] == 0.5 for f in drawn)
    err = _rel(g, ref)
    print(f"B={B}: raster backward err {err:.2e} (reversed copies {n_back}, border faces {n_border}, unlit {n_dark})")
    assert n_back > 0 and n_border > 0 and n_dark > 0
    assert err <= 1e-5


def _smpl_dev():
    from avatarclip_b200 import drive
    s = D.golden_smpl()
    return s, drive.smpl_tensors(s, "cuda")


def test_smpl_pose_backward_vs_fp64():
    from avatarclip_b200 import pose_optimizer as PO
    s, sd = _smpl_dev()
    rng = np.random.default_rng(5)
    B = 4
    pose = (rng.standard_normal((B, 63)) * 0.8).astype(np.float32)
    pose[0, :9] = 0.0                              # zero-angle joints
    pose[1, 3:6] = [3.6, -0.4, 0.2]                # angles above pi
    pose[2, 30:33] = [-2.9, 2.7, 1.1]
    g = rng.standard_normal((B, s["v_template"].shape[0], 3)).astype(np.float32)
    pt, gt = torch.tensor(pose, device="cuda"), torch.tensor(g, device="cuda")
    out = PO.smpl_pose_batch_bwd(sd, pt, gt)
    ref = OP.smpl_pose_grad({k: np.asarray(v) for k, v in s.items()}, pose, g)
    err = _rel(out, ref)
    print(f"SMPL backward err {err:.2e}")
    assert err <= 1e-5
    assert torch.equal(out, PO.smpl_pose_batch_bwd(sd, pt, gt))
    out45 = PO.smpl_pose_batch_bwd(sd, pt[:, :45].contiguous(), gt)          # a shorter pose: its own joints only
    assert _rel(out45, OP.smpl_pose_grad({k: np.asarray(v) for k, v in s.items()}, pose[:, :45], g)) <= 1e-5


@pytest.mark.parametrize("n,S", [(256, 224), (48, 224), (300, 224), (7, 10)])
def test_prep_backward_vs_fp64(n, S):
    from avatarclip_b200 import pose_optimizer as PO
    g = torch.randn(3, 3, S, S, generator=torch.Generator().manual_seed(n))
    out = PO.clip_prep_nearest_bwd(g.cuda(), n)
    assert _rel(out, OP.clip_prep_nearest_bwd(g.numpy(), n)) <= 1e-6


def test_loss_vs_fp64():
    from avatarclip_b200 import pose_optimizer as PO
    gen = torch.Generator().manual_seed(6)
    emb, text = torch.randn(5, 4, 512, generator=gen), torch.randn(512, generator=gen)
    loss, g = PO.pose_clip_loss(emb.cuda(), text.cuda())
    rl, rg = OP.pose_clip_loss(emb.numpy(), text.numpy())
    assert _rel(loss, rl) <= 1e-6 and _rel(g, rg) <= 1e-5


@pytest.fixture(scope="module")
def assets(tmp_path_factory):
    from avatarclip_b200 import animate as A
    from avatarclip_b200 import shapegen as S
    tv, tf = D.template_obj()
    s = {k: np.asarray(v) for k, v in D.golden_smpl().items()}
    s["faces"] = tf
    d = tmp_path_factory.mktemp("pose_optimizer")
    uv = OS.write_uv_obj(str(d / "uv"), s["v_template"], s["faces"])
    clip = S.load_clip(OS.clip_states(), OS.write_bpe(d / "bpe.txt.gz"))
    return A.Assets(s, clip, None, uv), s


def test_one_iteration_gradient_vs_oracle_chain(assets):
    """PoseStep's pose gradient against the fp64 chain from the tower's input gradient on: the resize, raster and SMPL
    backward on the device's own maps.  The tower itself is checked by test_clip_gpu.py (fp16 input-gradient floor
    3.5e-3); with its output taken as given the remaining chain holds 1e-4."""
    from avatarclip_b200 import pose_optimizer as PO
    a, s = assets
    n, ss, A, B = 32, 2, 5, 2
    step = PO.PoseStep(a, B, A, n, ss)
    gen = torch.Generator().manual_seed(7)
    step.pose.copy_(torch.randn(B, 63, generator=gen) * 0.3)
    step.set_text(torch.randn(512, generator=gen).cuda())
    eyes = np.stack([np.asarray(EYES[:A]) for _ in range(B)])
    step.cams.copy_(PO.look_at_cams(eyes, n, ss, device="cuda"))
    step.run()
    torch.cuda.synchronize()
    V, F = s["v_template"].shape[0], s["faces"].shape[0]
    fidx, proj, rgb_ss = _device_maps(step.ws_rf, step.ws_rb, V, A, B, B * A, n * ss, step.cams.shape[1])
    g_rgb = OP.clip_prep_nearest_bwd(step.g_prep.cpu().numpy(), n).reshape(A, B, n, n, 3)
    assert _rel(step.g_rgb, g_rgb) <= 1e-6
    verts = step.verts.cpu().numpy()
    gv = np.zeros((B, V, 3))
    for ai in range(A):
        for b in range(B):
            eye, rot = OS.look_at_camera(eyes[b, ai])
            gv[b] += OP.raster_backward_image(verts[b], s["faces"], proj[ai * B + b], eye, rot, fidx[ai * B + b],
                                              rgb_ss[ai * B + b], g_rgb[ai, b], ss)
    ref = OP.smpl_pose_grad(s, step.pose.cpu().numpy(), gv)
    err = _rel(step.grad, ref)
    print(f"one iteration: pose gradient err {err:.2e} against the fp64 chain from the tower's input gradient")
    assert err <= 1e-4


def test_graph_loop_matches_launches(assets):
    """optimise() (one captured graph, replayed) against the same calls launched one by one: the first iteration's
    loss and pose gradient to the CLIP tower's rounding (it sums with atomics, so runs are not bitwise equal), and
    every iteration's loss loosely (Adam's first step is lr times the gradient's sign, so entries near 0 may step
    either way)."""
    from avatarclip_b200 import _lib
    from avatarclip_b200 import pose_optimizer as PO
    a, _ = assets
    opt = PO.PoseOptimizer(name="PoseOptimizer", assets=a, num_iteration=3, topk=2)
    gen = torch.Generator().manual_seed(8)
    init, tf = torch.randn(2, 63, generator=gen), torch.randn(512, generator=gen).cuda()
    rs = np.random.RandomState(9)
    eyes = np.stack([[[get_points_from_angles(2.0, rs.randn() * 0.3, az) for az in O.ANGLES]
                      for _ in range(3)] for _ in range(2)])
    out = opt.optimise(init, tf, eyes, record_grad=True)
    step = PO.PoseStep(a, 2, 5)
    step.set_text(tf)
    step.pose.copy_(init.cuda())
    m, v = torch.zeros_like(step.pose), torch.zeros_like(step.pose)
    state = torch.tensor([0.0, 0.01, 0.0, 0.0], device="cuda")
    cams = PO.look_at_cams(np.ascontiguousarray(eyes.transpose(1, 0, 2, 3)), device="cuda").view(3, 10, -1)
    for it in range(3):
        step.cams.copy_(cams[it])
        step.run()
        assert (step.loss - opt.last["loss"][it]).abs().max() <= (1e-5 if it == 0 else 1e-2)
        if it == 0:
            assert _rel(opt.last["grad"][0], step.grad.cpu().numpy()) <= 1e-3
        _lib.check(_lib.lib().avc_adam_step_dev(_lib.ptr(step.pose), _lib.ptr(step.grad), _lib.ptr(m), _lib.ptr(v),
                                                step.pose.numel(), _lib.ptr(state), 0.9, 0.999, 1e-8, 1.0,
                                                _lib.stream_ptr()), "avc_adam_step_dev")
    assert (step.pose - out).abs().max() <= 3 * 2 * 0.01 + 1e-5       # 3 steps of at most ~lr each
    assert (out.cpu() - init).abs().max() > 0


def test_cli_writes_candidates(assets, tmp_path):
    from avatarclip_b200 import pose_optimizer as PO
    _, s = assets
    smpl = tmp_path / "smpl.npz"
    np.savez(smpl, **{k: np.asarray(v) for k, v in s.items()})
    uv = OS.write_uv_obj(str(tmp_path / "uv"), s["v_template"], s["faces"])
    visual, text = OS.clip_states()
    clip_model = tmp_path / "clip.pt"
    torch.save({**{k: v.half() for k, v in visual.items()}, **{k: v.half() for k, v in text.items()}}, clip_model)
    bpe = OS.write_bpe(tmp_path / "bpe.txt.gz")
    out = tmp_path / "exp"
    conf = tmp_path / "po.conf"
    conf.write_text(f"general {{\n    base_exp_dir = {out}\n    mode = pose\n    text = a rendered 3d man is crying\n}}\n"
                    "pose_generator {\n    type = PoseOptimizer\n    num_iteration = 3\n    topk = 2\n}\n")
    assert PO.main(["--conf", str(conf), "--smpl", str(smpl), "--uv_obj", uv, "--clip_model", str(clip_model),
                    "--bpe", str(bpe), "--seed", "0"]) == 0
    for i in range(2):
        p = np.load(out / f"candidate_{i}.npy")
        assert p.shape == (69,) and p.dtype == np.float32 and (p[63:] == 0).all() and np.isfinite(p).all()
        assert (out / f"candidate_{i}.jpg").stat().st_size > 0


def test_vertical_edge_on_a_pixel_column():
    """Faces with an edge exactly on a pixel column (x = 0 seen from (0, 0, -2) on an odd image: column 23 of 47): the
    sweep that divides 0 by 0 in neural_renderer adds nothing; the gradient is finite and matches the oracle."""
    from avatarclip_b200 import pose_optimizer as PO
    from avatarclip_b200 import video
    n, ss, A, B = 47, 1, 1, 1
    xs, ys = (-0.3, 0.0, 0.3), (-0.3, 0.0, 0.3)
    v = np.array([(x, y, 0.1 * x * x + 0.05 * y) for y in ys for x in xs], dtype=np.float32)
    f = []
    for j in range(2):
        for i in range(2):
            a = j * 3 + i
            f += [(a, a + 1, a + 4), (a, a + 4, a + 3)]
    faces = np.array(f, dtype=np.int32)
    tex = np.random.default_rng(9).random((faces.shape[0], 2, 2, 2, 3)).astype(np.float32)
    eyes = np.array([[[0.0, 0.0, -2.0]]])
    dev = "cuda"
    vt, ft, tt = (torch.tensor(x, device=dev) for x in (v[None], faces, tex))
    cams = PO.look_at_cams(eyes, n, ss, device=dev)
    ws_f = PO.raster_fwd_workspace(v.shape[0], A, B, 1, n, ss, dev)
    rgb = torch.empty(A, B, n, n, 3, device=dev)
    PO.raster_textured_batch_dev(vt, ft, tt, cams, A, 1, rgb, ws_f, n, ss)
    g_rgb = torch.tensor(np.random.default_rng(10).standard_normal((A, B, n, n, 3)).astype(np.float32), device=dev)
    ws_b = PO.raster_bwd_workspace(faces.shape[0], A, B, n, ss, dev)
    g = torch.empty(B, v.shape[0], 3, device=dev)
    PO.raster_textured_batch_bwd(vt, ft, tt, video.adjacency(ft, v.shape[0]), A, 1, g_rgb, ws_f, g, ws_b, n, ss)
    fidx, proj, rgb_ss = _device_maps(ws_f, ws_b, v.shape[0], A, B, 1, n, cams.shape[1])
    px = 0.5 * (proj[0][:, 0].astype(np.float32) * np.float32(n) + np.float32(n) - np.float32(1))
    assert (px[1::3] == 23.0).all()
    eye, rot = OS.look_at_camera(eyes[0, 0])
    ref = OP.raster_backward_image(v, faces, proj[0], eye, rot, fidx[0], rgb_ss[0], g_rgb[0, 0].cpu().numpy(), ss)
    assert torch.isfinite(g).all() and _rel(g[0], ref) <= 1e-5


def test_end_to_end_against_the_reference(assets):
    """PoseOptimizer on the inputs of tests/golden/ref_pose_optimizer_small.pt (the reference's own loop, oracle stand-
    ins, topk 2 x 3 iterations): the same initial poses and elevations, each iteration's loss within the fp16 tower's
    bar, the returned poses within a measured bar and the same sort order where the scores' gap exceeds its bar.
    Measured on an H100: loss 6.3e-4, first pose gradient 1.4e-2 of its largest entry (the fp16 tower's input
    gradient), returned poses 3.0e-2 (Adam's sign-like steps on near-zero entries), sort scores 2.0e-3."""
    from avatarclip_b200 import pose_optimizer as PO
    a, _ = assets
    gd = torch.load(os.path.join(ROOT, "tests", "golden", "ref_pose_optimizer_small.pt"), map_location="cpu",
                    weights_only=False)
    K, T = gd["conf"]["topk"], gd["conf"]["num_iteration"]
    np.random.seed(gd["np_seed"])
    torch.manual_seed(gd["torch_seed"])
    opt = PO.PoseOptimizer(name="PoseOptimizer", assets=a, **gd["conf"])
    poses = opt.get_topk_poses(gd["text"], text_feature=gd["text_feature"], record_grad=True).cpu()
    last = opt.last
    assert torch.equal(last["init"], gd["init"])
    np.testing.assert_allclose(last["eyes"].reshape(-1, 5, 3), gd["eyes"][:K * T].double().numpy(), rtol=0, atol=1e-6)
    e_loss = float((last["loss"].cpu().T - gd["loss"]).abs().max())
    e_grad0 = _rel(last["grad"][0].cpu(), gd["grads"][:, 0])
    sc = torch.tensor(last["sort_scores"])
    order = sorted(range(K), key=lambda i: float(sc[i]), reverse=True)
    ref_order = sorted(range(K), key=lambda i: float(gd["sort_scores"][i]), reverse=True)
    final = torch.stack([gd["files"][ref_order.index(k)] for k in range(K)])      # candidate k's returned pose
    mine = torch.stack([poses[order.index(k)] for k in range(K)])
    e_pose = float((mine - final).abs().max())
    e_score = float((sc - gd["sort_scores"]).abs().max())
    print(f"end to end: loss err {e_loss:.2e}, first gradient err {e_grad0:.2e}, pose err {e_pose:.2e}, "
          f"score err {e_score:.2e}")
    assert e_loss <= 3.5e-3 and e_score <= 3.5e-3 and e_grad0 <= 3e-2
    assert e_pose <= 2 * T * 0.01                  # Adam moves each entry by at most about lr per step
    gaps = [abs(float(gd["sort_scores"][i] - gd["sort_scores"][j])) for i in range(K) for j in range(i)]
    if min(gaps) > 2 * 3.5e-3:
        assert order == ref_order
