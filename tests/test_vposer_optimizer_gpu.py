"""VPoserOptimizer on the device: the VPoser decoder's backward (avc_vposer_decode_bwd) against fp64 autograd of the
restatement in oracle/vposer_optimizer.py on every branch of matrot2aa, one iteration's latent gradient against the fp64
chain, the CUDA-graph loop against the same calls launched one by one, the reference's own loop
(tests/golden/ref_vposer_optimizer_small.pt) and the command line on synthetic files.  Reads only tests/golden and
synthetic data."""
import os

import numpy as np
import pytest
import torch

from oracle import animate as O
from oracle import drive as D
from oracle import pose_optimizer as OP
from oracle import shapegen as OS
from oracle import vposer_optimizer as OV
from avatarclip_b200.handoff import get_points_from_angles
from test_pose_optimizer_gpu import EYES, _device_maps, _rel

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("B", [1, 5, 8, 13])
def test_decoder_backward_vs_fp64(B):
    """g_z against autograd of the fp64 restatement with the device's weights, the joints steered onto all four
    quaternion branches and both atan2 branches; pose_out bit for bit avc_vposer_decode's.  B covers part of a tile of
    8 rows, a full one and more than one.  Measured on an H100: at most 7.3e-7 of the largest entry."""
    from avatarclip_b200 import animate as A
    from avatarclip_b200 import vposer_optimizer as VO
    sd = OV.steered_state()
    dec = {k: v.cuda() for k, v in sd.items()}
    gen = torch.Generator().manual_seed(B)
    z = torch.randn(B, 32, generator=gen)
    g = torch.randn(B, 21, 3, generator=gen)
    R = OV.decoder_rotations(z.double(), sd)
    assert set(OV.branches(R).tolist()) == {0, 1, 2, 3} and set(OV.atan2_negative(R).tolist()) == {False, True}
    pose = torch.full((B, 21, 3), float("nan"), device="cuda")
    g_z = VO.vposer_decode_bwd(z.cuda(), dec, g.cuda(), pose_out=pose)
    assert torch.equal(pose, A.vposer_decode(z.cuda(), dec))
    zz = z.double().requires_grad_(True)
    (OV.decode(zz, {k: v.double() for k, v in sd.items()}) * g.double()).sum().backward()
    err = _rel(g_z, zz.grad)
    print(f"decoder backward B={B}: err {err:.2e} of the largest entry")
    assert err <= 1e-5


@pytest.fixture(scope="module")
def assets(tmp_path_factory):
    from avatarclip_b200 import animate as A
    from avatarclip_b200 import shapegen as S
    tv, tf = D.template_obj()
    s = {k: np.asarray(v) for k, v in D.golden_smpl().items()}
    s["faces"] = tf
    d = tmp_path_factory.mktemp("vposer_optimizer")
    uv = OS.write_uv_obj(str(d / "uv"), s["v_template"], s["faces"])
    clip = S.load_clip(OS.clip_states(), OS.write_bpe(d / "bpe.txt.gz"))
    return A.Assets(s, clip, O.vposer_state(), uv), s


def test_one_iteration_gradient_vs_oracle_chain(assets):
    """One iteration's latent gradient (decode, PoseStep, decoder backward) against the fp64 chain from the tower's
    input gradient on: the resize, raster and SMPL backward on the device's own maps, then autograd of the fp64
    decoder.  As for PoseOptimizer the tower itself is checked by test_clip_gpu.py.  Measured on an H100: 8.7e-7 to
    1.6e-6 over three runs (the tower's atomics)."""
    from avatarclip_b200 import pose_optimizer as PO
    from avatarclip_b200 import vposer_optimizer as VO
    a, s = assets
    n, ss, A, B = 32, 2, 5, 2
    step = PO.PoseStep(a, B, A, n, ss)
    gen = torch.Generator().manual_seed(17)
    z = torch.randn(B, 32, generator=gen).cuda()
    step.set_text(torch.randn(512, generator=gen).cuda())
    eyes = np.stack([np.asarray(EYES[:A]) for _ in range(B)])
    step.cams.copy_(PO.look_at_cams(eyes, n, ss, device="cuda"))
    ws = VO.vposer_workspace(a.vposer)
    VO.vposer_decode_into(z, a.vposer, step.pose, ws)
    step.run()
    g_z = VO.vposer_decode_bwd(z, a.vposer, step.grad, ws=ws)
    torch.cuda.synchronize()
    V = s["v_template"].shape[0]
    fidx, proj, rgb_ss = _device_maps(step.ws_rf, step.ws_rb, V, A, B, B * A, n * ss, step.cams.shape[1])
    g_rgb = OP.clip_prep_nearest_bwd(step.g_prep.cpu().numpy(), n).reshape(A, B, n, n, 3)
    verts = step.verts.cpu().numpy()
    gv = np.zeros((B, V, 3))
    for ai in range(A):
        for b in range(B):
            eye, rot = OS.look_at_camera(eyes[b, ai])
            gv[b] += OP.raster_backward_image(verts[b], s["faces"], proj[ai * B + b], eye, rot, fidx[ai * B + b],
                                              rgb_ss[ai * B + b], g_rgb[ai, b], ss)
    g_pose = OP.smpl_pose_grad(s, step.pose.cpu().numpy(), gv)
    zz = z.cpu().double().requires_grad_(True)
    (OV.decode(zz, O.vposer_state()).reshape(B, 63) * torch.as_tensor(g_pose)).sum().backward()
    err = _rel(g_z, zz.grad)
    print(f"one iteration: latent gradient err {err:.2e} against the fp64 chain from the tower's input gradient")
    assert err <= 1e-5


def test_graph_loop_matches_launches(assets):
    """optimise() (one captured graph, replayed) against the same calls launched one by one: the first iteration's
    loss and latent gradient to the CLIP tower's rounding (it sums with atomics), every iteration's loss loosely, and the
    returned poses the decode of the latents before the last step."""
    from avatarclip_b200 import pose_optimizer as PO
    from avatarclip_b200 import vposer_optimizer as VO
    a, _ = assets
    opt = VO.VPoserOptimizer(name="VPoserOptimizer", assets=a, num_iteration=3, topk=2)
    gen = torch.Generator().manual_seed(18)
    init, tf = torch.randn(2, 32, generator=gen), torch.randn(512, generator=gen).cuda()
    rs = np.random.RandomState(19)
    eyes = np.stack([[[get_points_from_angles(2.0, rs.randn() * 0.3, az) for az in O.ANGLES]
                      for _ in range(3)] for _ in range(2)])
    out = opt.optimise(init, tf, eyes, record_grad=True)
    step = PO.PoseStep(a, 2, 5)
    step.set_text(tf)
    z = init.cuda()
    ws = VO.vposer_workspace(a.vposer)
    m, v = torch.zeros_like(z), torch.zeros_like(z)
    state = torch.tensor([0.0, 0.01, 0.0, 0.0], device="cuda")
    cams = PO.look_at_cams(np.ascontiguousarray(eyes.transpose(1, 0, 2, 3)), device="cuda").view(3, 10, -1)
    for it in range(3):
        step.cams.copy_(cams[it])
        VO.vposer_decode_into(z, a.vposer, step.pose, ws)
        before = z.clone()
        step.run()
        g_z = VO.vposer_decode_bwd(z, a.vposer, step.grad, ws=ws)
        assert (step.loss - opt.last["loss"][it]).abs().max() <= (1e-5 if it == 0 else 1e-2)
        if it == 0:
            assert _rel(opt.last["grad"][0], g_z.cpu().numpy()) <= 1e-3
        PO.adam_step(z, g_z, m, v, state, (0.9, 0.999), 1e-8)
    assert (z - opt.last["latent"]).abs().max() <= 3 * 2 * 0.01 + 1e-5       # 3 steps of at most ~lr each
    assert (opt.last["latent"].cpu() - init).abs().max() > 0
    # the returned poses decode the graph's own pre-step latents: one step of at most ~lr away from its final ones
    from avatarclip_b200 import animate as A
    assert _rel(out, A.vposer_decode(before, a.vposer).reshape(2, 63).cpu()) <= 0.1
    assert not torch.equal(out, A.vposer_decode(opt.last["latent"], a.vposer).reshape(2, 63))


def test_cli_writes_candidates(assets, tmp_path):
    """--vposer names a written VPoser checkpoint (a Lightning state_dict with vp_model. prefixes)."""
    from avatarclip_b200 import vposer_optimizer as VO
    _, s = assets
    smpl = tmp_path / "smpl.npz"
    np.savez(smpl, **{k: np.asarray(v) for k, v in s.items()})
    uv = OS.write_uv_obj(str(tmp_path / "uv"), s["v_template"], s["faces"])
    visual, text = OS.clip_states()
    clip_model = tmp_path / "clip.pt"
    torch.save({**{k: v.half() for k, v in visual.items()}, **{k: v.half() for k, v in text.items()}}, clip_model)
    bpe = OS.write_bpe(tmp_path / "bpe.txt.gz")
    vposer = tmp_path / "vposer.ckpt"
    torch.save({"state_dict": {"vp_model." + k: v for k, v in O.vposer_state().items()}}, vposer)
    out = tmp_path / "exp"
    conf = tmp_path / "vo.conf"
    conf.write_text(f"general {{\n    base_exp_dir = {out}\n    mode = pose\n    text = a rendered 3d man is crying\n}}\n"
                    "pose_generator {\n    type = VPoserOptimizer\n    num_iteration = 3\n    topk = 2\n}\n")
    assert VO.main(["--conf", str(conf), "--smpl", str(smpl), "--vposer", str(vposer), "--uv_obj", uv,
                    "--clip_model", str(clip_model), "--bpe", str(bpe), "--seed", "0"]) == 0
    for i in range(2):
        p = np.load(out / f"candidate_{i}.npy")
        assert p.shape == (69,) and p.dtype == np.float32 and (p[63:] == 0).all() and np.isfinite(p).all()
        assert (out / f"candidate_{i}.jpg").stat().st_size > 0


def test_end_to_end_against_the_reference(assets):
    """VPoserOptimizer on the inputs of tests/golden/ref_vposer_optimizer_small.pt (the reference's own loop, oracle
    stand-ins, topk 2 x 3 iterations): the same initial latents and elevations, each iteration's loss within the fp16
    tower's bar, the final latents and the returned poses within measured bars, and the same sort order where the
    scores' gap exceeds its bar.  Measured on an H100: loss 4.4e-4, first latent gradient 3.9e-2 of its largest entry
    (the fp16 tower's input gradient summed through the decoder's 63 pose entries), final latents 2.4e-2 (Adam's
    sign-like first steps), returned poses 1.3e-3, sort scores 2.0e-5."""
    from avatarclip_b200 import vposer_optimizer as VO
    a, _ = assets
    gd = torch.load(os.path.join(ROOT, "tests", "golden", "ref_vposer_optimizer_small.pt"), map_location="cpu",
                    weights_only=False)
    K, T = gd["conf"]["topk"], gd["conf"]["num_iteration"]
    np.random.seed(gd["np_seed"])
    torch.manual_seed(gd["torch_seed"])
    opt = VO.VPoserOptimizer(name="VPoserOptimizer", assets=a, **gd["conf"])
    poses = opt.get_topk_poses(gd["text"], text_feature=gd["text_feature"], record_grad=True).cpu()
    last = opt.last
    assert torch.equal(last["init"], gd["init"])
    np.testing.assert_allclose(last["eyes"].reshape(-1, 5, 3), gd["eyes"][:K * T].double().numpy(), rtol=0, atol=1e-6)
    e_loss = float((last["loss"].cpu().T - gd["loss"]).abs().max())
    e_grad0 = _rel(last["grad"][0].cpu(), gd["grads"][:, 0])
    sc = torch.tensor(last["sort_scores"])
    order = sorted(range(K), key=lambda i: float(sc[i]), reverse=True)
    ref_order = sorted(range(K), key=lambda i: float(gd["sort_scores"][i]), reverse=True)
    mine = torch.stack([poses[order.index(k)] for k in range(K)])[:, :63]       # candidate k's returned pose
    e_pose = float((mine - gd["poses"]).abs().max())
    e_score = float((sc - gd["sort_scores"]).abs().max())
    final = []                              # the reference's latents after its last step: torch Adam on its gradients
    for k in range(K):
        p = torch.nn.Parameter(gd["init"][k].clone())
        adam = torch.optim.Adam([p], lr=0.01)
        for t in range(T):
            p.grad = gd["grads"][k, t].clone()
            adam.step()
        final.append(p.data)
    e_lat = float((last["latent"].cpu() - torch.stack(final)).abs().max())
    print(f"end to end: loss err {e_loss:.2e}, first gradient err {e_grad0:.2e}, latent err {e_lat:.2e}, "
          f"pose err {e_pose:.2e}, score err {e_score:.2e}")
    assert e_loss <= 3.5e-3 and e_score <= 3.5e-3 and e_grad0 <= 8e-2
    assert e_lat <= 2 * T * 0.01                   # Adam moves each entry by at most about lr per step
    assert e_pose <= 1e-2
    gaps = [abs(float(gd["sort_scores"][i] - gd["sort_scores"][j])) for i in range(K) for j in range(i)]
    if min(gaps) > 2 * 3.5e-3:
        assert order == ref_order
