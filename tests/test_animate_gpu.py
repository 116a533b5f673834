"""AvatarAnimate's pose stage on the device: every kernel of avc_pose.cu against fp64 (oracle/animate.py) or the kernel
it batches, both generators end to end on the seeded inputs of tests/golden/ref_animate_small.pt, and the command line
on synthetic files.  Reads only tests/golden and synthetic data."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import animate as O
from oracle import drive as D
from oracle import shapegen as OS

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "ref_animate_small.pt")
CODEBOOK_CONF = """general {
    base_exp_dir = ./exp/pose_ablation/vposer_codebook/cry
    mode = pose
    text = a rendered 3d man is crying
}

pose_generator {
    type = VPoserCodebook
}
"""


def _rel(out, ref):
    ref = np.asarray(ref, dtype=np.float64)
    return float(np.abs(np.asarray(out.detach().cpu(), dtype=np.float64) - ref).max() / np.abs(ref).max())


@pytest.fixture(scope="module")
def golden():
    return torch.load(GOLDEN, map_location="cpu", weights_only=False)


@pytest.fixture(scope="module")
def smpl():
    tv, tf = D.template_obj()
    s = {k: np.asarray(v) for k, v in D.golden_smpl().items()}
    s["faces"] = tf
    return s


@pytest.fixture(scope="module")
def assets(smpl, tmp_path_factory):
    from avatarclip_b200 import animate as A
    from avatarclip_b200 import shapegen as S
    d = tmp_path_factory.mktemp("animate")
    uv = OS.write_uv_obj(str(d / "uv"), smpl["v_template"], smpl["faces"])
    clip = S.load_clip(OS.clip_states(), OS.write_bpe(d / "bpe.txt.gz"))
    return A.Assets(smpl, clip, O.vposer_state(), uv)


@pytest.mark.parametrize("B", [1, 37, 2560])
def test_vposer_decode_vs_fp64(B):
    from avatarclip_b200 import animate as A
    sd = O.vposer_state()
    z = torch.randn(B, 32, generator=torch.Generator().manual_seed(B))
    pose, rot = A.vposer_decode(z.cuda(), {k: v.cuda() for k, v in sd.items()}, return_matrot=True)
    ref_pose, ref_rot = O.vposer_decode(z, sd)
    assert pose.shape == (B, 21, 3)
    assert _rel(rot, ref_rot) <= 1e-5 and _rel(pose, ref_pose) <= 1e-5


BRANCH_ROTVECS = [
    [0.0, 0.0, 0.0], [2e-3, -1e-3, 1e-3],                                          # identity, near identity
    [np.pi - 0.02, 0.0, 0.0], [0.0, np.pi - 0.02, 0.0], [0.0, 0.0, np.pi - 0.02],   # near pi: branches 0, 1, 2
    [0.9 * np.pi, 0.1, 0.0], [0.1, 0.9 * np.pi, 0.0], [0.0, 0.3, 0.9 * np.pi],     # branches 0, 1, 2
    [2.2, 0.0, 0.0], [0.0, 1.8, 0.0], [0.0, 0.0, 2.0], [-2.4, 0.3, 0.2], [0.2, -2.1, 0.4], [0.3, 0.1, -2.6],
    [0.2, 0.1, 0.3], [1.5, 0.0, 0.0], [0.7, -0.6, 0.5], [-1.2, 0.4, 0.9], [0.0, 1.2, -0.8], [1.0, 1.0, 0.0],
    [-0.5, -0.5, -0.5]]


def _branch_vposer_state():
    """vposer_state with the last layer's bias set to the 6D form of BRANCH_ROTVECS and its weights scaled down: each
    joint decodes to a rotation within ~0.01 rad of its target, so the set spans every quaternion branch."""
    from scipy.spatial.transform import Rotation
    sd = O.vposer_state()
    R = Rotation.from_rotvec(np.asarray(BRANCH_ROTVECS)).as_matrix()         # [21, 3, 3]
    sd["decoder_net.5.bias"] = torch.from_numpy(R[:, :, :2].reshape(-1)).float()   # [3][2] per joint: columns 0, 1
    sd["decoder_net.5.weight"] = sd["decoder_net.5.weight"] * 0.05
    return sd


def _quaternion_branch(R):
    m = np.transpose(R, (0, 2, 1))
    return np.where(m[:, 2, 2] < 1e-6, np.where(m[:, 0, 0] > m[:, 1, 1], 0, 1),
                    np.where(m[:, 0, 0] < -m[:, 1, 1], 2, 3))


def test_vposer_decode_every_quaternion_branch():
    from avatarclip_b200 import animate as A
    sd = _branch_vposer_state()
    z = torch.randn(64, 32, generator=torch.Generator().manual_seed(7))
    pose, rot = A.vposer_decode(z.cuda(), {k: v.cuda() for k, v in sd.items()}, return_matrot=True)
    ref_pose, ref_rot = O.vposer_decode(z, sd)
    br = _quaternion_branch(ref_rot.reshape(-1, 3, 3))
    assert all((br == k).sum() >= 64 for k in range(4)), np.bincount(br)
    ang = np.linalg.norm(ref_pose.reshape(-1, 3), axis=1)
    assert (ang < 0.02).sum() >= 64 and (ang > np.pi - 0.05).sum() >= 3 * 64
    assert _rel(rot, ref_rot) <= 1e-5 and _rel(pose, ref_pose) <= 1e-5


def test_realnvp_decode_vs_fp64():
    from avatarclip_b200 import animate as A
    sd = O.realnvp_state()
    g = torch.Generator().manual_seed(0)
    z, f = torch.randn(500, 32, generator=g), torch.randn(512, generator=g) * 0.05
    nvp_w = A.pack_realnvp(sd, 8, "cuda")
    x = A.realnvp_decode(z.cuda(), f.cuda(), nvp_w)
    assert _rel(x, O.realnvp_decode(z, f, sd)) <= 1e-5
    # torch's own fp32 expression of decode (:233-240) agrees too
    m = sd["mask"]
    xt, ft = z.clone(), f[None].expand(500, -1)
    net = lambda p, i, h: (lambda a: a @ sd[f"{p}.{i}.4.weight"].T + sd[f"{p}.{i}.4.bias"])(F.leaky_relu(F.leaky_relu(
        h @ sd[f"{p}.{i}.0.weight"].T + sd[f"{p}.{i}.0.bias"]) @ sd[f"{p}.{i}.2.weight"].T + sd[f"{p}.{i}.2.bias"]))
    for i in range(8):
        x_ = xt * m[i]
        tr = torch.cat((x_, ft), -1)
        s, t = torch.tanh(net("s", i, tr)) * (1 - m[i]), net("t", i, tr) * (1 - m[i])
        xt = x_ + (1 - m[i]) * (xt * torch.exp(s) + t)
    assert (x.cpu() - xt).abs().max().item() <= 1e-4


def test_smpl_pose_batch_equals_lbs_fwd_per_row(smpl):
    from avatarclip_b200 import animate as A
    from avatarclip_b200 import drive as Dr
    from avatarclip_b200.lbs import my_lbs
    s = Dr.smpl_tensors(smpl)
    g = torch.Generator().manual_seed(1)
    for P in (63, 69):
        bp = torch.randn(19, P, generator=g) * 0.4
        v = A.smpl_pose_batch(s, bp.cuda(), A.SCORE_ORIENT)
        for b in range(bp.shape[0]):
            full = torch.zeros(1, 72)
            full[0, :3] = torch.tensor(A.SCORE_ORIENT)
            full[0, 3:3 + P] = bp[b]
            ref, _ = my_lbs(s["v_template"][None], full.cuda(), None, None, s["posedirs"], s["J_regressor"],
                            s["parents"], s["lbs_weights"])
            assert torch.equal(v[b], ref[0]), (P, b, (v[b] - ref[0]).abs().max().item())
        assert _rel(v, O.smpl_vertices(smpl, bp)) <= 1e-5
    rot = A.smpl_pose_batch(s, bp.cuda(), A.SCORE_ORIENT, A.RENDER_ROT)
    assert torch.equal(rot, v @ torch.from_numpy(A.RENDER_ROT).cuda())


def test_raster_batch_equals_single_renders(assets, smpl):
    from avatarclip_b200 import animate as A
    from avatarclip_b200 import shapegen as S
    bp = torch.randn(5, 63, generator=torch.Generator().manual_seed(2)) * 0.3
    v = A.smpl_pose_batch(assets.smpl, bp.cuda(), A.SCORE_ORIENT, A.RENDER_ROT)
    eyes = np.array([[O.eye(el, az) for az in (120, 180, 240)] for el in (0.1, -0.4)])    # 2 groups x 3 angles
    imgs = A.raster_textured_batch(v, assets.faces, assets.textures, eyes, group=3)
    assert imgs.shape == (3, 5, 256, 256, 3)
    for a in range(3):
        for b in range(5):
            one = S.raster_textured(v[b], assets.faces, assets.textures, eyes[b // 3, a])
            assert torch.equal(imgs[a, b], one), (a, b)
    assert (imgs.sum(-1) > 0).float().mean().item() > 0.02


def test_cosine_topk_vs_fp64_and_torch():
    from avatarclip_b200 import animate as A
    g = torch.Generator(device="cuda").manual_seed(3)
    for N in (4096, 65536):
        rows = torch.randn(N, 512, generator=g, device="cuda")
        vec = torch.randn(512, generator=g, device="cuda")
        cos, idx = A.cosine_topk(rows, vec, 40)
        ref = O.cosine(rows.cpu(), vec.cpu())
        assert np.abs(cos.cpu().numpy() - ref).max() <= 1e-6
        assert idx.cpu().tolist() == np.argsort(-ref, kind="stable")[:40].tolist()
        assert idx.cpu().tolist() == torch.topk(F.cosine_similarity(rows, vec[None]), 40).indices.cpu().tolist()
    rows[7] = rows[3] = vec * 2                            # a tie: the smaller index first
    _, idx = A.cosine_topk(rows, vec, 2)
    assert idx.cpu().tolist() == [3, 7]


def test_pose_suppress_vs_reference_loop():
    from avatarclip_b200 import animate as A
    g = torch.Generator().manual_seed(4)
    base = torch.randn(40, 63, generator=g) * 0.5
    for k in range(1, 40, 3):
        base[k] = base[k - 1] + torch.randn(63, generator=g) * 0.05
    keep = A.pose_suppress(base.cuda(), 0.07).cpu().tolist()
    assert keep == O.suppress(base.numpy(), 0.07) and len(keep) < 40
    # the reference's own loop (:304-317) on the same tensor
    new = []
    for i, p in enumerate(base):
        if not new:
            new.append(i)
            continue
        md = 10
        for j in new:
            md = min(torch.abs(p - base[j]).mean(), md)
        if md > 0.07:
            new.append(i)
    assert keep == new


def test_pose_score_vs_fp64():
    from avatarclip_b200 import animate as A
    g = torch.Generator().manual_seed(5)
    emb, text = torch.randn(5, 30, 512, generator=g), torch.randn(512, generator=g)
    score, best = A.pose_score(emb.cuda(), text.cuda(), 10)
    ref = O.cosine(emb.double().mean(0), text)
    assert np.abs(score.cpu().numpy() - ref).max() <= 1e-6
    assert best.cpu().tolist() == [int(np.argmax(ref[g0:g0 + 10])) for g0 in (0, 10, 20)]


def test_codebook_end_to_end_vs_golden(golden, assets, tmp_path):
    from avatarclip_b200 import animate as A
    cb = golden["codebook"]
    torch.save(O.make_codebook(golden["text_feature"]), tmp_path / "codebook.pth")
    gen = A.build_pose_generator({"type": "VPoserCodebook", "codebook_path": str(tmp_path / "codebook.pth")}, assets)
    poses = gen.get_topk_poses(golden["text"])
    assert gen.last["topk"].cpu().tolist() == cb["topk"].tolist()
    assert gen.last["keep"].cpu().tolist()[:5] == cb["keep"].tolist()
    assert poses.shape == (5, 63) and np.abs(poses.cpu().numpy() - cb["poses"].numpy()).max() <= 1e-5
    assert np.abs(gen.last["cos"].cpu().numpy() - cb["cos"].numpy()).max() < 0.02     # fp16 text tower vs fp32 oracle


def test_realnvp_end_to_end_vs_golden(golden, assets, tmp_path):
    from avatarclip_b200 import animate as A
    nv = golden["realnvp"]
    tf = golden["text_feature"]
    # the text tower alone: fp16 on the device against the fp32 oracle tower the golden used
    t_dev = assets.clip.text.encode_text(assets.clip.tokenizer.tokenize(golden["text"],
                                                                        context_length=assets.clip.text.context))
    assert ((t_dev.float().cpu()[0] - tf).norm() / tf.norm()).item() < 0.02
    torch.save({"state_dict": O.realnvp_state()}, tmp_path / "realnvp.pth")
    gen = A.build_pose_generator({"type": "VPoserRealNVP", "ckpt_path": str(tmp_path / "realnvp.pth"),
                                  **golden["realnvp_conf"]}, assets)
    # the rest of the pipeline conditioned on the reference's own text feature
    np.random.seed(golden["np_seed"])
    poses = gen.get_topk_poses(golden["text"], z=nv["z"].cuda(), text_feature=tf)
    assert poses.shape == nv["poses"].shape
    # fp32 throughout against the reference's fp32 CPU decode fed to the fp64 VPoser: torch's own fp32 route on the CPU
    # lands 6e-6 of the largest angle away, the device's sums (other orders, fp32 matrot2aa) 1.9e-5; a wrong
    # conditioning or selection moves the poses by 1e-3 and more
    err = np.abs(poses.cpu().numpy() - nv["poses"].numpy()).max() / np.abs(nv["poses"].numpy()).max()
    assert err <= 3e-5, err
    # the scores of every draw, the best kept per candidate and the sort's, against the reference's cosines
    # (fp16 image tower against the fp32 oracle tower: test_shapegen_gpu's tolerance)
    got = np.stack(gen.last["scores"])
    assert got.shape == tuple(nv["scores"].shape)
    assert np.abs(got - nv["scores"].numpy()).max() < 0.02
    assert np.abs(np.asarray(gen.last["best_scores"]) - nv["best_scores"].numpy()).max() < 0.02
    assert np.abs(np.asarray(gen.last["sort_scores"]) - nv["sort_scores"].numpy()).max() < 0.02
    # the numpy stream: 5 elevations per scoring call, batches then the sort, as the reference drew them
    np.random.seed(golden["np_seed"])
    eyes = gen.scorer.draw_eyes(len(nv["eyes"]) // 5).reshape(-1, 3)
    assert np.abs(eyes - nv["eyes"].numpy()).max() <= 1e-6      # stored as float32


def test_realnvp_without_a_positive_score_raises(assets, tmp_path):
    from avatarclip_b200 import animate as A
    torch.save({"state_dict": O.realnvp_state()}, tmp_path / "realnvp.pth")
    gen = A.build_pose_generator({"type": "VPoserRealNVP", "ckpt_path": str(tmp_path / "realnvp.pth"), "topk": 1,
                                  "num_batch": 1, "num_sample": 2}, assets)
    with pytest.raises(RuntimeError, match="above 0"):
        gen.get_pose(torch.zeros(512, device="cuda"), torch.randn(2, 32, device="cuda"))


def test_cli_writes_candidates(smpl, tmp_path, monkeypatch):
    from avatarclip_b200 import animate as A
    np.savez(tmp_path / "smpl.npz", **{k: np.asarray(v) for k, v in smpl.items()})
    os.makedirs(tmp_path / "vposer" / "snapshots")
    torch.save({"state_dict": {"vp_model." + k: v for k, v in O.vposer_state().items()}},
               tmp_path / "vposer" / "snapshots" / "V02_05_epoch=13_val_loss=0.03.ckpt")
    visual, text = OS.clip_states()
    torch.save({**{k: v.half() for k, v in visual.items()}, **{k: v.half() for k, v in text.items()}},
               tmp_path / "clip.pt")
    uv = OS.write_uv_obj(str(tmp_path / "data"), smpl["v_template"], smpl["faces"])
    torch.save(O.make_codebook(torch.randn(512, generator=torch.Generator().manual_seed(0))),
               tmp_path / "data" / "codebook.pth")
    (tmp_path / "cry.conf").write_text(CODEBOOK_CONF)
    monkeypatch.chdir(tmp_path)
    rc = A.main(["--conf", "cry.conf", "--smpl", "smpl.npz", "--vposer", "vposer", "--uv_obj", uv, "--clip_model",
                 "clip.pt", "--bpe", OS.write_bpe(tmp_path / "bpe.txt.gz")])
    assert rc == 0
    out = tmp_path / "exp" / "pose_ablation" / "vposer_codebook" / "cry"
    import cv2
    for i in range(5):
        p = np.load(out / f"candidate_{i}.npy")
        assert p.shape == (63,) and p.dtype == np.float32
        img = cv2.imread(str(out / f"candidate_{i}.jpg"))
        assert img.shape == (512, 512, 3)
        assert (img < 200).any(axis=-1).mean() > 0.005 and (img > 250).all(axis=-1).mean() > 0.5
