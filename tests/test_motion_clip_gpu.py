"""MotionOptimizer with its CLIP term on the device: the frame selection and the CLIP-gradient kernel against
restatements in fp64, one iteration's latent gradient against the fp64 chain from the CLIP tower's input gradient, the
new entry points with clip_coef = 0 against avc_motion_optimize bit for bit, the captured loop against the same calls
launched one by one, the whole loop against what the reference computed (tests/golden/ref_motion_clip_small.pt), and
the command line on synthetic files.  Reads only tests/golden and synthetic data."""
import math
import os

import numpy as np
import pytest
import torch

from oracle import animate as OA
from oracle import drive as D
from oracle import motion as OM
from oracle import pose_optimizer as OP
from oracle import shapegen as OS

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "ref_motion_clip_small.pt")


def _rel(out, ref):
    ref = torch.as_tensor(np.asarray(ref), dtype=torch.float64)
    return float((torch.as_tensor(out).detach().cpu().double() - ref).abs().max() / ref.abs().max())


@pytest.fixture(scope="module")
def golden():
    return torch.load(GOLDEN, map_location="cpu", weights_only=False)


@pytest.fixture(scope="module")
def assets(tmp_path_factory):
    from avatarclip_b200 import animate as A
    from avatarclip_b200 import shapegen as S
    tv, tf = D.template_obj()
    s = {k: np.asarray(v) for k, v in D.golden_smpl().items()}
    s["faces"] = tf
    d = tmp_path_factory.mktemp("motion_clip")
    uv = OS.write_uv_obj(str(d / "uv"), s["v_template"], s["faces"])
    clip = S.load_clip(OS.clip_states(), OS.write_bpe(d / "bpe.txt.gz"))
    return A.Assets(s, clip, None, uv), s


def _st(v):
    return torch.tensor([v], dtype=torch.int32, device="cuda")


@pytest.mark.parametrize("T,P", [(60, 30), (60, 7), (13, 5), (64, 64), (2, 1), (60, 1)])
def test_select_vs_restatement(T, P):
    """Every st of a (num_frame, clip_num_part) pair: the rows' poses, frames and weights; where R varies with st the
    rows past the motion have weight 0 and a valid frame."""
    from avatarclip_b200 import motion_clip as MC
    m = torch.randn(T, 63, generator=torch.Generator().manual_seed(T * 100 + P)).cuda()
    R = MC.clip_rows(T, P)
    coef = np.float32(0.001)
    past = 0
    for st in range(P):
        pose, frame, weight = MC.select(m, P, float(coef), _st(st), R)
        want_f = [st + r * P if st + r * P < T else st for r in range(R)]
        want_w = np.array([coef * (np.float32(st + r * P) / np.float32(T)) if st + r * P < T else 0.0
                           for r in range(R)], dtype=np.float32)
        assert frame.tolist() == want_f and np.array_equal(weight.cpu().numpy(), want_w)
        assert torch.equal(pose, m[want_f])
        past += sum(st + r * P >= T for r in range(R))
    assert (past > 0) == (T % P != 0)


# rotations whose 6D forms take matrix_to_quaternion's four argmax branches, one near pi and the identity
BRANCH_ROTVECS = [[0.3, -0.2, 0.1], [math.pi * 0.9, 0.1, 0.0], [0.1, math.pi * 0.9, 0.0], [0.0, 0.2, math.pi * 0.9],
                  [math.pi - 0.01, 0.0, 0.0], [0.0, 0.0, 0.0], [1.2, -0.6, 0.4], [-0.5, 1.1, -0.9]]


def _branch_state():
    """A small decoder whose outputs sit on every branch of the rotation chain (the final bias is the branch rotations'
    6D forms, the weight small; decoder joint 5 is the identity exactly)."""
    from scipy.spatial.transform import Rotation
    sd = OM.motion_vae_state(seed=5, latent=64, num_layers=2, n_out=132)
    six = np.stack([Rotation.from_rotvec(v).as_matrix()[:2].reshape(6) for v in BRANCH_ROTVECS])
    W = sd["decoder.final.weight"] * 0.05
    W[5 * 6:6 * 6] = 0
    sd["decoder.final.weight"], sd["decoder.final.bias"] = W, torch.from_numpy(np.tile(six, (3, 1))[:22].reshape(-1)).float()
    return sd


def test_clip_gradient_every_branch_vs_fp64():
    """The CLIP rows' gradient through the rotation chain and the decoder, with the rest of the loss off: the latent
    gradient of sum_r w_r (loss_r + <g_r, motion[frame_r]>) against fp64 autograd of oracle/motion.py, at
    clip_num_part 7 (9 rows, the last past the motion for st = 5), and the loss sum_r w_r loss_r."""
    from avatarclip_b200 import motion as M
    from avatarclip_b200 import motion_clip as MC
    sd = _branch_state()
    w = M.load_motion_vae(sd, latent_dim=64, num_layers=2, num_heads=2)
    gen = torch.Generator().manual_seed(3)
    z = torch.randn(64, generator=gen)
    out = OM.decoder(z.double(), sd, num_layers=2, num_heads=2).reshape(60, 22, 6)[:, 1:]
    m = OM.rotation_6d_to_matrix(out)
    e = [m[..., i, j] for i in range(3) for j in range(3)]
    qa = torch.stack([1 + e[0] + e[4] + e[8], 1 + e[0] - e[4] - e[8], 1 - e[0] + e[4] - e[8], 1 - e[0] - e[4] + e[8]], -1)
    P, st, R = 7, 5, MC.clip_rows(60, 7)
    frames = [st + r * P for r in range(R) if st + r * P < 60]
    assert set(qa[frames].argmax(-1).flatten().tolist()) == {0, 1, 2, 3}
    g = torch.randn(R, 63, generator=gen)
    lr = torch.rand(R, generator=gen)
    ms = MC.ClipMotionStep(w, torch.zeros(1, 63).cuda(), [0.0], 0.0, 1, record_grad=True)
    ms.init(z.cuda(), 0.01)
    ms.forward()
    pose, frame, weight = MC.select(ms.motion, P, 0.5, _st(st), R)
    assert frame.tolist()[-1] == st and float(weight[-1]) == 0.0 and len(frames) == R - 1
    ms.backward(frame, weight, g.cuda(), lr.cuda())
    zz = z.double().requires_grad_()
    mot = OM.decode(zz, sd, num_layers=2, num_heads=2)
    wt = weight.cpu().double()
    (wt[:, None] * g.double() * mot[frame.cpu().long()]).sum().backward()
    err = _rel(ms.grad, zz.grad)
    ref_loss = float((wt * lr.double()).sum())
    print(f"CLIP gradient through the branch decoder: err {err:.2e}, loss {float(ms.loss[0]):.7f} vs {ref_loss:.7f}")
    assert err <= 1e-4 and abs(float(ms.loss[0]) - ref_loss) <= 1e-5 * ref_loss


def test_clip_coef_zero_is_avc_motion_optimize(golden):
    """Through the new entry points with clip_coef = 0 (so every row's weight is 0), whatever the rows' loss and
    gradient, the losses, latent, gradient and motion are bitwise avc_motion_optimize's."""
    from avatarclip_b200 import motion as M
    from avatarclip_b200 import motion_clip as MC
    vae = M.load_motion_vae(OM.motion_vae_state())
    poses, z0 = golden["poses"].cuda(), golden["runs"]["shipped"]["latent_init"].cuda()
    coef, n = [1, 0.8, 0.6, 0.4, 0.2], 6
    z, motion, loss, grad = M.motion_optimize(vae, poses, coef, 0.01, z0, n, lr=0.01, record_loss=True,
                                              return_grad=True)
    ms = MC.ClipMotionStep(vae, poses, coef, 0.01, n, record_grad=True)
    ms.init(z0, 0.01)
    g, lo = torch.randn(2, 63, device="cuda"), torch.rand(2, device="cuda")
    for it in range(n):
        ms.forward()
        _, frame, weight = MC.select(ms.motion, 30, 0.0, _st(it % 30), 2)
        ms.backward(frame, weight, g, lo)
    assert torch.equal(ms.loss, loss) and torch.equal(ms.latent(), z) and torch.equal(ms.motion, motion)
    assert torch.equal(ms.grad, grad)


def _device_maps(ws_f, ws_b, V, N, is_, cam_bytes):
    """(fidx [N, is, is], proj [N, V, 3], rgb_ss [N, is, is, 3]) read back from the raster workspaces (the layout
    test_pose_optimizer_gpu.py reads)."""
    al = lambda x: (x + 255) // 256 * 256
    o_proj = al(N * cam_bytes)
    o_z = o_proj + al(N * V * 16)
    proj = ws_f[o_proj:o_proj + N * V * 16].view(torch.float32).reshape(N, V, 4)[..., :3].cpu().numpy()
    zb = ws_f[o_z:o_z + N * is_ * is_ * 8].view(torch.int64).reshape(N, is_, is_).cpu().numpy()
    fidx = (zb & 0xffffffff).astype(np.int64)
    fidx[fidx == 0xffffffff] = -1
    rgb = ws_b[:N * is_ * is_ * 12].view(torch.float32).reshape(N, is_, is_, 3).cpu().numpy()
    return fidx, proj, rgb


def test_one_iteration_gradient_vs_oracle_chain(assets, golden):
    """One iteration with the CLIP term alone (recon_coef 0, delta_coef 0, clip_coef 1) at clip_num_part 20 (3 rows):
    the latent gradient against the fp64 chain from the tower's input gradient -- the device's g_prep taken as given,
    then oracle/pose_optimizer.py's resize, raster and SMPL backward on the device's own maps, the weighted scatter
    and fp64 autograd through oracle/motion.py's decoder and rotation chain.  The tower itself is checked by
    test_clip_gpu.py.  Measured on an H100 80GB HBM3 (700 W): 1.3e-6 of the largest entry."""
    from avatarclip_b200 import motion as M
    from avatarclip_b200 import motion_clip as MC
    from avatarclip_b200 import pose_optimizer as PO
    from avatarclip_b200.handoff import get_points_from_angles
    a, s = assets
    sd = OM.motion_vae_state()
    vae = M.load_motion_vae(sd)
    z0 = golden["runs"]["clip_only"]["latent_init"]
    n, ss, P, st = 32, 2, 20, 7
    R = MC.clip_rows(60, P)
    step = PO.PoseStep(a, R, 1, n, ss)
    step.set_text(golden["text_feature"].cuda())
    eye = get_points_from_angles(2.0, 0.13, MC.CLIP_AZIMUTH)
    step.cams.copy_(PO.look_at_cams(np.repeat(eye[None, None], R, 0), n, ss, device="cuda").view(R, -1))
    ms = MC.ClipMotionStep(vae, golden["poses"].cuda(), [0.0] * 5, 0.0, 1, record_grad=True)
    ms.init(z0.cuda(), 0.01)
    ms.forward()
    _, frame, weight = MC.select(ms.motion, P, 1.0, _st(st), R, step.pose)
    step.run()
    ms.backward(frame, weight, step.grad, step.loss)
    torch.cuda.synchronize()
    V = s["v_template"].shape[0]
    fidx, proj, rgb_ss = _device_maps(step.ws_rf, step.ws_rb, V, R, n * ss, step.cams.shape[1])
    g_rgb = OP.clip_prep_nearest_bwd(step.g_prep.cpu().numpy(), n)
    verts = step.verts.cpu().numpy()
    e, rot = OS.look_at_camera(eye)
    gv = np.stack([OP.raster_backward_image(verts[r], s["faces"], proj[r], e, rot, fidx[r], rgb_ss[r], g_rgb[r], ss)
                   for r in range(R)])
    gpose = OP.smpl_pose_grad(s, step.pose.cpu().numpy(), gv)
    zz = z0.double().requires_grad_()
    mot = OM.decode(zz, sd)
    wt = weight.cpu().double()
    (wt[:, None] * torch.from_numpy(gpose) * mot[frame.cpu().long()]).sum().backward()
    err = _rel(ms.grad, zz.grad)
    loss = float((wt * step.loss.cpu().double()).sum())
    print(f"one iteration, CLIP term alone: latent gradient err {err:.2e} against the fp64 chain from the tower's "
          f"input gradient; loss {float(ms.loss[0]):.6f} vs {loss:.6f}")
    assert err <= 1e-4 and abs(float(ms.loss[0]) - loss) <= 1e-5


def _optimizer(assets, golden, run, **kw):
    from avatarclip_b200 import motion_clip as MC
    c = {**golden["conf"][run], "num_iteration": golden["num_iter"], **kw}
    c.pop("lr")
    return MC.MotionOptimizer(assets, ckpt_path=OM.motion_vae_state(), **c)


def test_graph_loop_matches_launches(assets, golden):
    """optimise() (one captured graph, replayed) against the same calls launched one by one: the first iteration's
    loss and latent gradient to the CLIP tower's rounding (it sums with atomics, so runs are not bitwise equal), the
    later losses loosely and the latent within Adam's steps."""
    from avatarclip_b200 import motion_clip as MC
    from avatarclip_b200 import pose_optimizer as PO
    from avatarclip_b200.handoff import get_points_from_angles
    a, _ = assets
    opt = _optimizer(a, golden, "clip_only", num_iteration=3)
    r = golden["runs"]["clip_only"]
    st, el = np.array([4, 29, 0], dtype=np.int32), np.array([0.2, -0.4, 0.05])
    poses, tf = golden["poses"].cuda(), golden["text_feature"].cuda()
    z, motion = opt.optimise(poses, r["latent_init"], tf, st, el, record_grad=True)
    R = MC.clip_rows(60, 30)
    step = PO.PoseStep(a, R, 1)
    step.set_text(tf)
    ms = MC.ClipMotionStep(opt.vae, poses, [0.0] * 5, 0.0, 3, record_grad=True)
    ms.init(r["latent_init"].cuda(), 0.01)
    for it in range(3):
        eye = get_points_from_angles(2.0, el[it], MC.CLIP_AZIMUTH)
        step.cams.copy_(PO.look_at_cams(np.repeat(eye[None, None], R, 0), device="cuda").view(R, -1))
        ms.forward()
        _, frame, weight = MC.select(ms.motion, 30, 1.0, _st(int(st[it])), R, step.pose)
        step.run()
        ms.backward(frame, weight, step.grad, step.loss)
        torch.cuda.synchronize()
        assert abs(float(ms.loss[it] - opt.last["loss"][it])) <= (1e-5 if it == 0 else 1e-2)
        if it == 0:
            assert _rel(opt.last["grad"][0], ms.grad.cpu()) <= 1e-3
    assert (ms.latent() - z).abs().max() <= 3 * 2 * 0.01
    assert torch.isfinite(motion).all() and (z.cpu() - r["latent_init"]).abs().max() > 0


@pytest.mark.parametrize("run", ["shipped", "clip_only"])
def test_end_to_end_against_the_reference(assets, golden, run):
    """MotionOptimizer on the inputs of tests/golden/ref_motion_clip_small.pt (the reference's own loop, oracle
    stand-ins): the same draws, each iteration's loss within the fp16 tower's bar, the first latent gradient within a
    bar measured on the H100 and the final latent within Adam's steps.  Measured on an H100 80GB HBM3 (700 W): shipped
    coefficients, loss 7.5e-7 to 3.1e-6, first latent gradient 1.5e-4 of its largest entry, final latent 3.2e-3 to
    4.8e-3; the CLIP term alone, loss 4.2e-4 to 1.7e-3, first latent gradient 1.1e-2 to 1.2e-2 (the fp16 tower's
    input gradient, as PoseOptimizer's 1.4e-2), final latent 1.1e-2 to 1.3e-2.  The tower sums with atomics, so runs
    differ in the last bits and Adam's sign-like steps carry that into the later losses."""
    a, _ = assets
    r = golden["runs"][run]
    opt = _optimizer(a, golden, run)
    np.random.seed(golden["np_seed"])
    m = opt.get_motion(golden["text"], golden["poses"].cuda(), latent=r["latent_init"],
                       text_feature=golden["text_feature"], record_grad=True)
    last = opt.last
    assert np.array_equal(last["st_idx"], r["st_idx"].numpy()) and np.array_equal(last["elevation"],
                                                                                   r["elevation"].numpy())
    e_loss = float((last["loss"].cpu().double() - r["loss"].double()).abs().max())
    e_grad0 = _rel(last["grad"][0], r["grads"][0])
    e_lat = float((last["latent"].cpu() - r["latent"]).abs().max())
    n = golden["num_iter"]
    print(f"{run}: loss err {e_loss:.2e}, first latent gradient err {e_grad0:.2e}, final latent {e_lat:.2e}")
    assert m.shape == (60, 69) and torch.isfinite(m).all() and not m[:, 63:].any()
    assert e_loss <= 3.5e-3 and e_grad0 <= 3e-2
    assert e_lat <= 2 * n * 0.01


def test_cli_writes_motion(tmp_path, monkeypatch):
    from avatarclip_b200 import motion_clip as MC
    tv, tf = D.template_obj()
    smpl = {k: np.asarray(v) for k, v in D.golden_smpl().items()}
    smpl["faces"] = tf
    np.savez(tmp_path / "smpl.npz", **smpl)
    os.makedirs(tmp_path / "vposer" / "snapshots")
    torch.save({"state_dict": {"vp_model." + k: v for k, v in OA.vposer_state().items()}},
               tmp_path / "vposer" / "snapshots" / "V02_05_epoch=13_val_loss=0.03.ckpt")
    visual, text = OS.clip_states()
    torch.save({**{k: v.half() for k, v in visual.items()}, **{k: v.half() for k, v in text.items()}},
               tmp_path / "clip.pt")
    uv = OS.write_uv_obj(str(tmp_path / "data"), smpl["v_template"], smpl["faces"])
    torch.save(OA.make_codebook(torch.randn(512, generator=torch.Generator().manual_seed(0))),
               tmp_path / "data" / "codebook.pth")
    torch.save({"state_dict": OM.motion_vae_state()}, tmp_path / "data" / "motion_vae.pth")
    (tmp_path / "m.conf").write_text("general {\n    base_exp_dir = ./exp/m\n    mode = motion\n    text = a rendered 3d "
                                     "man is walking\n}\n\npose_generator {\n    type = VPoserCodebook\n}\n\n"
                                     "motion_generator {\n    type = MotionOptimizer\n    num_iteration = 5\n}\n")
    monkeypatch.chdir(tmp_path)
    rc = MC.main(["--conf", "m.conf", "--smpl", "smpl.npz", "--vposer", "vposer", "--uv_obj", uv, "--clip_model",
                  "clip.pt", "--bpe", OS.write_bpe(tmp_path / "bpe.txt.gz"), "--seed", "0"])
    assert rc == 0
    out = tmp_path / "exp" / "m"
    for i in range(5):
        assert np.load(out / f"candidate_{i}.npy").shape == (63,) and (out / f"candidate_{i}.jpg").exists()
    m = np.load(out / "motion.npy")
    assert m.shape == (60, 69) and m.dtype == np.float32 and np.isfinite(m).all() and not m[:, 63:].any()
    assert (out / "motion.mp4").stat().st_size > 0
